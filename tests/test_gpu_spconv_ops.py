"""The three sparse-convolution kernels one operator at a time (ABI wrappers of sessd_b200.ops, no runner) on crafted rulebooks, against
fp64 references, with element-wise tolerances derived from each kernel's numerics.

Notation: u = 2^-24 (fp32 unit roundoff); a row's P valid (row, offset) pairs; x the fp32 input features, w [kvol, Cin, Cout] the
weights, bn / sh the folded BatchNorm scale / shift; mag = sum over the row's pairs and input channels of |x| |w| (fp64).

fp32 kernels (spconv_forward_rows, spconv_forward SIMT) vs the exact fp64 result of their fp32 inputs:
    |got - ref| <= (P Cin + 2) u (|bn| mag + |sh|)
  The accumulator is a chain of P Cin fmaf (one rounding each: the classic gamma_n <= n u / (1 - n u) bound on mag, the 1 / (1 - n u)
  is below the +2 slack here), then fmaf(acc, bn, sh) adds one rounding of |bn| |acc| + |sh| and carries |bn| times the chain's error;
  ReLU is 1-Lipschitz.  Missing neighbours of the SIMT kernel are fmaf(0, w, acc) == acc: exact.
rows vs SIMT: value-equal (==, +-0 alike).  Both run acc = fmaf(x[c], w[k][c][n], acc) over the row's offsets in ascending k and the
  channels in ascending c, from +0, then fmaf(acc, bn, sh); the SIMT kernel's extra fmaf(0, w, acc) for offsets the row lacks return acc
  unchanged (acc never becomes -0: it starts at +0 and an exact-zero RN sum is +0).
pair-gather tensor-core kernel (spconv_forward_cg) vs an fp64 emulation of what it multiplies: the input planes a = (a_hi, a_lo) with
  x S_in = a_hi + a_lo + d, the pack_weight_sp_h2 tiles b = (b_hi, b_lo) with w 2^e = b_hi + b_lo + d', and
  emul = (sum a_hi b_hi + a_hi b_lo + a_lo b_hi) (1 / S_in) sc + sh with sc = bn 2^-e (ReLU after).  The products are exact on the tensor
  cores (fp16 x fp16 fits fp32), so what remains is the fp32 accumulation.  Model of one k=16 wgmma step D = C + sum_16 p_i: the addends
  are aligned to the largest exponent and the sum is normalised to fp32, each of the two steps losing at most 1 ulp of a magnitude
  <= |C| + sum |p_i|, i.e. <= 2 * 2^-23 (|C| + sum |p_i|); |C| <= the sum of the |p| before it, so over G steps the accumulator is off by
  <= 2 * 2^-23 G sum |p|.  Steps whose products are all zero for the row (offsets the row lacks) add an exact zero and are not counted:
  G = 2 P Cp / 16 (the cross accumulator sees two k=16 products per 16 channels and offset, the main one half as many; both use G).  The
  epilogue's acc_m + acc_c and fmaf(., sc, sh) add two roundings (the +2 and the 2^-23 |sh| term):
    |got - emul| <= c 2^-23 (G + 2) |sc| magA / S_in + 2^-23 |sh|,   c = 2,   magA = sum |a_hi||b_hi| + |a_hi||b_lo| + |a_lo||b_hi|
cg vs fp64: the bound above plus the split's own error.  S_in maps max|x| into [2^14, 2^15), so |d| <= 2^-9 (half an ulp of a_lo <= 8)
  <= 2^-23 amax_in S_in; max_c |w 2^e| lies in [2^10, 2^11), so |d'| <= 2^-13 <= 2^-23 wmax_n 2^e; the dropped a_lo b_lo is
  <= 2^-22 |x| wmax_n / (S_in 2^e).  Per product that is <= 2^-21.4 (amax_in |w| + |x| wmax_n); with a 2.6x margin:
    + 2^-20 |bn| sum over pairs and channels (amax_in |w| + |x| wmax_n)
planes outputs (fp16 (hi, lo) [rows][2][cpo] at the scale S = pow2_scale_for_bound(amax_in gain + shift_max) that maps the bound into
  [2^14, 2^15)): o S is exact (power of two), |o S - hi| <= 8 and lo = fp16(o S - hi) is off by <= 2^-9, so
  |(hi + lo) / S - o| <= 2^-9 / S <= 2^-23 bound; checked at 2^-22 bound.

Each tolerance is shown to catch a subtly wrong kernel on the CPU (negative controls): the emulation without the cross products, with one
(row, offset) pair dropped, with a row's product taken from the previous offset of its stage within a tile (a missed dirty-row clear),
with two offsets' weights swapped, and the fp64 result with one pair dropped.  The staging faults that carry stale rows from tile to
tile (dirty masks reset at each tile, a two-warp group's second warp never clearing, a two-stage warp not rotating its masks) are
replayed by cg_ring_model on the tables of test_gpu_spconv_cg_grid, which is where they are flagged.  Smallest ratio of error to bound
of each control over the control cases (cg vs emulation bound / cg vs fp64 bound): no cross products 9.1 / 4.1, missed dirty-row clear
71 / 36, one pair dropped 1190 / 740, two offsets' weights swapped 9230 / 5000; fp64 with one pair dropped vs the fp32 bound 540.
Largest ratios measured on one H100 80GB HBM3 (400 W power limit), the same at deep 0 and deep 1: cg vs emulation 0.46 (single-pair
rows: the wgmma accumulation is not round-to-nearest, ~1 ulp per step), cg vs fp64 0.03, rows and SIMT vs fp64 0.55, planes 0.1.
With (64,32) added and `single` sized against the device grid, the largest cg ratios measured on an H100 (132 SMs) over all eight
instantiations were 0.49 vs the emulation, 0.05 vs fp64 and 0.051 for the planes.
"""
import numpy as np
import pytest
import torch

from cg_ring_model import NACTS, CgLayout, cg_grid, replay, tile_ring
from oracle.spconv_ref import conv_from_nbr

U = 2.0 ** -24
CG_C = 2.0                                     # wgmma accumulation: ulps per k=16 step (module docstring)
BIG = 3 * 132 * 128 + 77                       # `single` for the fp32 kernels: 397 tiles (the cg cases size it against the device grid)
SWEEP = 8 * 132 * 128 + 50                     # nact_sweep: 1057 tiles, >= 4 per CTA at 264 CTAs, >= 8 at 132 (ring_positions)
NACT_SCHEDULE_SEED = 2
# grids of spconv_cg (cg_ring_model.cg_grid: min(tiles, blocks_per_sm x SMs)) with the ring lengths that run at them: the default
# pipeline (2 CTAs per SM; 2 stages at Cp 64, 4 at Cp 32) and the deep one (1 CTA per SM; 4 and 8 stages), on 132- and 114-SM parts.
# The deep grids are checked at 2 stages too.
GRID_RINGS = ((264, (2, 4)), (228, (2, 4)), (132, (2, 4, 8)), (114, (2, 4, 8)))
SLACK = 3                                      # sentinel rows past max_out in every output buffer
PATTERNS = ("full", "single", "flip", "nact_sweep", "empty_tiles", "duplicates", "high_rows")
F32_SENTINEL = -1234.5
F16_SENTINEL = 0x5A5A                          # an fp16 bit pattern no kernel output here produces in padding


def cg_stages(cp, deep):
    """kStages of CgCfg<cp, *, deep> (spconv_cg.cu)"""
    return (2 if cp == 64 else 4) * (2 if deep else 1)


# ------------------------------------------------------------------------------------------------------------------ crafted rulebooks
def crafted_nbr(pattern, n, kvol, n_in, seed):
    """nbr int64 [n, kvol], -1 = no neighbour, input rows in [0, n_in)."""
    rng = np.random.default_rng(seed)
    r = np.arange(n)
    nbr = np.full((n, kvol), -1, np.int64)
    rand = rng.integers(0, n_in, (n, kvol))
    if pattern == "full":
        nbr[:] = rand
    elif pattern == "single":              # one offset per row, rotating: a stage's consecutive fills (k, k + kStages) hit disjoint rows
        k = (r + r // 128) % kvol
        nbr[r, k] = rand[r, k]
    elif pattern == "flip":                # valid iff (r + k) even: every row's validity flips between consecutive offsets.  A stage's
        # fills k and k + kStages share their parity at every (even) ring length, so within a tile no dirty row is ever cleared; the
        # clears across tiles are test_gpu_spconv_cg_grid's
        ok = (r[:, None] + np.arange(kvol)[None, :]) % 2 == 0
        nbr[ok] = rand[ok]
    elif pattern == "nact_sweep":          # tiles with exactly nact active offsets, nact from NACTS (<= kvol)
        choices = np.array([a for a in NACTS if a <= kvol])
        # the counts follow one fixed schedule (whatever the seed), checked to meet every ring position at SWEEP rows
        sched = choices[np.random.default_rng(NACT_SCHEDULE_SEED).integers(0, len(choices), -(-n // 128))]
        for t in range(-(-n // 128)):
            rows = np.arange(t * 128, min(n, (t + 1) * 128))
            ks = np.sort(rng.choice(kvol, int(sched[t]), replace=False))
            ok = rng.random((len(rows), len(ks))) < 0.5
            ok[np.arange(len(ks)) % len(rows), np.arange(len(ks))] = True      # every chosen offset keeps >= 1 pair
            sub = nbr[rows[0]:rows[-1] + 1]
            sub[:, ks] = np.where(ok, rand[rows[0]:rows[-1] + 1][:, ks], -1)
    elif pattern == "empty_tiles":         # every third tile (from the second) without any pair, between busy tiles
        ok = (rng.random((n, kvol)) < 0.7) & ((r // 128) % 3 != 1)[:, None]
        nbr[ok] = rand[ok]
    elif pattern == "duplicates":          # inputs from a pool of 3 rows: shared by many outputs and by several offsets of one output
        ok = rng.random((n, kvol)) < 0.6
        pool = rng.integers(0, n_in, 3)
        nbr[ok] = pool[(r[:, None] + (np.arange(kvol)[None, :] // 4)) % 3][ok]
    elif pattern == "high_rows":           # input rows at the top of the input buffer, the last one included
        ok = rng.random((n, kvol)) < 0.5
        hi = rng.integers(max(0, n_in - 4096), n_in, (n, kvol))
        hi[::5, 0] = n_in - 1
        ok[::5, 0] = True
        nbr[ok] = hi[ok]
    else:
        raise ValueError(pattern)
    return nbr


class Case:
    """One crafted layer: nbr [max_out, kvol] (rows >= n_eff hold valid-looking entries the kernels must ignore), device row count n_dev,
    the input rows actually used (in_rows) with their fp32 features x, weights, folded BN.  live: the first n_eff rows of the table
    (default: crafted_nbr(pattern, ...))."""

    def __init__(self, pattern, n, kvol, cin, cout, seed, n_in=None, max_out=None, n_dev=None, relu=True, shift=True, live=None):
        rng = np.random.default_rng(seed + 1000)
        self.pattern, self.kvol, self.cin, self.cout, self.relu = pattern, kvol, cin, cout, relu
        self.max_out = n + 40 if max_out is None else max_out
        self.n_dev = n if n_dev is None else n_dev
        self.n_eff = min(self.n_dev, self.max_out)
        self.n_in = n_in if n_in is not None else max(64, n // 2)
        if live is None:
            live = crafted_nbr(pattern, self.n_eff, kvol, self.n_in, seed)
        assert live.shape == (self.n_eff, kvol)
        self.nbr = rng.integers(0, self.n_in, (self.max_out, kvol))
        self.nbr[:self.n_eff] = live
        self.in_rows = np.unique(live[live >= 0])
        self.nbr_c = np.where(live >= 0, np.searchsorted(self.in_rows, live), -1)   # compact input indices (references)
        m = len(self.in_rows)
        # per-row magnitudes spread over 2^-8 .. 1: a wrong product on a small row cannot hide under the layer maximum
        self.x = (rng.standard_normal((m, cin)) * np.exp2(rng.uniform(-8, 0, (m, 1)))).astype(np.float32)
        self.w = (rng.standard_normal((kvol, cin, cout)) * np.exp2(rng.uniform(-3, 1, (1, 1, cout))) / np.sqrt(cin * kvol)).astype(np.float32)
        self.bn = ((rng.random(cout) + 0.5) * np.where(rng.random(cout) < 0.2, -1, 1)).astype(np.float32)
        self.sh = (0.2 * rng.standard_normal(cout)).astype(np.float32) if shift else None
        self.P = (self.nbr_c >= 0).sum(1)

    @property
    def shv(self):
        return np.zeros(self.cout) if self.sh is None else self.sh.astype(np.float64)

    def conv(self, x, w):
        return conv_from_nbr(x, self.nbr_c, w, np.float64)

    def finish(self, acc, scale):
        y = acc * scale.astype(np.float64) + self.shv
        return np.maximum(y, 0) if self.relu else y

    def ref64(self):
        return self.finish(self.conv(self.x, self.w), self.bn)

    def tol_fp32(self):
        mag = self.conv(np.abs(self.x), np.abs(self.w))
        return (self.P[:, None] * self.cin + 2) * U * (np.abs(self.bn) * mag + np.abs(self.shv))

    def ref64_dropped_pair(self):
        """the fp64 result with one (row, offset) pair dropped (negative control)"""
        r, k = self._pick_pair()
        y = self.conv(self.x, self.w)
        y[r] -= self.x[self.nbr_c[r, k]].astype(np.float64) @ self.w[k].astype(np.float64)
        return self.finish(y, self.bn)

    def _pick_pair(self):
        rows, ks = np.nonzero(self.nbr_c >= 0)
        i = len(rows) // 2
        return rows[i], ks[i]


# ------------------------------------------------------------------------------------------------------------------ fp16 split (cg)
def pow2_scale_for_bound(bound):
    """numpy restatement of common.cuh pow2_scale_for_bound: the power of two that maps an fp32 bound into [2^14, 2^15)"""
    e = int((np.array(bound, np.float32).view(np.uint32) >> 23) & 0xFF)
    if e in (0, 255):
        return 1.0
    return float(np.array(min(max(268 - e, 2), 252) << 23, np.uint32).view(np.float32))


def device_bound_scale(amax, gain, shift_max):
    """the kernels' pow2_scale_for_bound(amax * gain + shift_max) in fp32; the product may be fused or not, the scale must not care"""
    fused = np.float32(np.float64(np.float32(amax)) * np.float64(np.float32(gain)) + np.float64(np.float32(shift_max)))
    unfused = np.float32(np.float32(amax) * np.float32(gain)) + np.float32(shift_max)
    s = pow2_scale_for_bound(fused)
    assert s == pow2_scale_for_bound(unfused)
    return s, float(fused)


def split16(v, s):
    """fp32 values -> fp16 (hi, lo) at the exact scale s (the operand format of the tensor-core layers)"""
    xs = v.astype(np.float32) * np.float32(s)
    hi = xs.astype(np.float16)
    return hi, (xs - hi.astype(np.float32)).astype(np.float16)


class CgEmu:
    """What spconv_forward_cg multiplies for a Case at plane width cp, in fp64, plus the tolerances of the module docstring."""

    def __init__(self, case, cp):
        from sessd_b200 import ops
        assert case.cin == cp
        self.case, self.cp = case, cp
        self.amax_in = float(np.abs(case.x).max())
        self.s_in = pow2_scale_for_bound(self.amax_in)
        self.a_hi, self.a_lo = split16(case.x, self.s_in)
        tiles, inv = ops.pack_weight_sp_h2(torch.from_numpy(case.w), cp)
        self.tiles, self.inv = tiles, inv
        t = tiles.numpy().astype(np.float64)                                         # [kvol, 2, cout, cp]
        self.b_hi, self.b_lo = t[:, 0].transpose(0, 2, 1), t[:, 1].transpose(0, 2, 1)  # [kvol, cp, cout]
        self.sc = (torch.from_numpy(case.bn) * inv).numpy()                          # kernel scale bn * 2^-e (exact)
        self.A = np.concatenate([self.a_hi, self.a_lo], 1).astype(np.float64)
        self.gain = float(self.gain_of(case))
        self.shift_max = 0.0 if case.sh is None else float(np.abs(case.sh).max())

    @staticmethod
    def gain_of(case):
        from sessd_b200 import ops
        return ops.conv_gain(torch.from_numpy(case.w), torch.from_numpy(case.bn))

    def acc(self, perm=None, cross=True):
        """sum over pairs of a_hi (b_hi + b_lo) + a_lo b_hi (cross=False: a_hi b_hi only); perm: the offsets' weights permuted"""
        bh, bl = (self.b_hi, self.b_lo) if perm is None else (self.b_hi[perm], self.b_lo[perm])
        return self.case.conv(self.A, np.concatenate([bh + bl, bh], 1) if cross else np.concatenate([bh, 0 * bh], 1))

    def emul(self, acc=None):
        return self.case.finish((self.acc() if acc is None else acc) / self.s_in, self.sc)

    def tol_emul(self):
        c = self.case
        magA = c.conv(np.abs(self.A), np.concatenate([np.abs(self.b_hi) + np.abs(self.b_lo), np.abs(self.b_hi)], 1))
        g = 2 * c.P[:, None] * self.cp / 16
        return CG_C * 2.0 ** -23 * (g + 2) * np.abs(self.sc) * magA / self.s_in + 2.0 ** -23 * np.abs(c.shv)

    def tol_fp64(self):
        c = self.case
        aw = np.abs(c.w).astype(np.float64)
        valid = (c.nbr_c >= 0).astype(np.float64)
        sum_w = valid @ aw.sum(1)                                                    # [n, cout]: sum over pairs, channels of |w|
        rowsum_x = np.abs(c.x).astype(np.float64).sum(1)
        sum_x = np.where(c.nbr_c >= 0, rowsum_x[np.maximum(c.nbr_c, 0)], 0).sum(1)   # [n]: sum over pairs, channels of |x|
        split = self.amax_in * sum_w + sum_x[:, None] * aw.max(axis=(0, 1))[None, :]
        return self.tol_emul() + 2.0 ** -20 * np.abs(c.bn) * split

    # ---- negative controls: outputs of subtly wrong kernels
    def wrong_no_cross(self):
        return self.emul(self.acc(cross=False))

    def wrong_dropped_pair(self):
        r, k = self.case._pick_pair()
        a = self.acc()
        a[r] -= self.A[self.case.nbr_c[r, k]] @ np.concatenate([self.b_hi[k] + self.b_lo[k], self.b_hi[k]], 0)
        return self.emul(a)

    def wrong_stale_row(self, stages):
        """a row that lacks offset klist[j] of its tile but had klist[j - stages] (same stage, previous fill) multiplies that stale
        input row by W[klist[j]]: what a missed dirty-row clear computes"""
        c = self.case
        for t in range(-(-c.n_eff // 128)):
            rows = c.nbr_c[t * 128:(t + 1) * 128]
            klist = np.nonzero((rows >= 0).any(0))[0]
            for j in range(stages, len(klist)):
                hit = np.nonzero((rows[:, klist[j]] < 0) & (rows[:, klist[j - stages]] >= 0))[0]
                if len(hit):
                    r = t * 128 + hit[0]
                    a = self.acc()
                    k = klist[j]
                    a[r] += self.A[c.nbr_c[r, klist[j - stages]]] @ np.concatenate([self.b_hi[k] + self.b_lo[k], self.b_hi[k]], 0)
                    return self.emul(a)
        raise AssertionError("no row changes validity within a stage in this case")

    def wrong_swapped_weights(self):
        ks = np.nonzero((self.case.nbr_c >= 0).any(0))[0]
        k1, k2 = ks[0], ks[-1]
        assert k1 != k2
        perm = np.arange(self.case.kvol)
        perm[[k1, k2]] = perm[[k2, k1]]
        return self.emul(self.acc(perm=perm))


def ratio(got, ref, tol):
    """max |got - ref| / tol; an element whose tolerance is 0 must match exactly"""
    d = np.abs(np.asarray(got, np.float64) - ref)
    r = np.divide(d, tol, out=np.where(d > 0, np.inf, 0.0), where=tol > 0)
    return float(r.max()) if r.size else 0.0


def check_planes(hi, lo, cout, s, bound, f32):
    """planes rows [n][2 cpo] fp16 vs the fp32 output rows: per element |(hi + lo) / S - o| <= 2^-22 bound; returns the ratio"""
    back = (hi[:, :cout].astype(np.float64) + lo[:, :cout].astype(np.float64)) / s
    return ratio(back, f32.astype(np.float64), np.full(f32.shape, 2.0 ** -22 * bound))


def ring_positions(nbr, n, stages, grid):
    """(nact, st0, ph0) of every tile of a persistent cg launch of `grid` CTAs: tile t runs on CTA t % grid after that CTA's earlier
    tiles (cg_ring_model.tile_ring)"""
    _cta, _round, p, nact = tile_ring(nbr, n, grid)
    return set(zip(nact.tolist(), (p % stages).tolist(), ((p // stages) & 1).tolist()))


# ================================================================================================================== CPU section
def test_nact_sweep_reaches_every_ring_position():
    """The nact_sweep rulebook of the GPU tests meets every active-offset count of NACTS at every ring position (st0, phase) a persistent
    CTA can carry in, for the ring lengths that run at each grid (GRID_RINGS: 264 and 132 CTAs on 132 SMs, 228 and 114 on 114)."""
    nbr = crafted_nbr("nact_sweep", SWEEP, 27, 4000, 11)
    for grid, rings in GRID_RINGS:
        for stages in rings:
            seen = ring_positions(nbr, SWEEP, stages, grid)
            want = {(a, s, p) for a in NACTS for s in range(stages) for p in (0, 1)}
            assert want <= seen, (grid, stages, sorted(want - seen)[:5])


@pytest.mark.parametrize("pattern", PATTERNS)
def test_crafted_rulebooks_have_their_shape(pattern):
    n, kvol, n_in = 5 * 128 + 9, 27, 3000
    nbr = crafted_nbr(pattern, n, kvol, n_in, 5)
    valid = nbr >= 0
    assert nbr.min() >= -1 and nbr.max() < n_in
    if pattern == "full":
        assert valid.all()
    if pattern == "single":
        assert (valid.sum(1) == 1).all()
        assert all(valid[t * 128:(t + 1) * 128].any(0).all() for t in range(n // 128))      # full tiles fill every offset
    if pattern == "flip":
        assert (valid[:, 1:] != valid[:, :-1]).all()
        for cp, deep in ((32, 0), (64, 0), (32, 1)):                # ring lengths 4, 2, 8, one tile per CTA: no clear
            assert not replay(nbr, n, n, -(-n // 128), CgLayout(cp, 32, deep)).clears
    if pattern == "nact_sweep":
        nact = [int(valid[t * 128:(t + 1) * 128].any(0).sum()) for t in range(-(-n // 128))]
        assert set(nact) <= set(NACTS)
    if pattern == "empty_tiles":
        t = np.arange(n) // 128
        assert not valid[t % 3 == 1].any() and valid[t % 3 != 1].any(1).mean() > 0.9
    if pattern == "duplicates":
        assert len(np.unique(nbr[valid])) <= 3
        assert any(len(set(row[row >= 0])) < (row >= 0).sum() for row in nbr)
    if pattern == "high_rows":
        assert (nbr[valid] >= n_in - 4096).all() and (nbr == n_in - 1).any()


def test_pow2_scale_restatement():
    for b, want in ((1.0, 2.0 ** 14), (1.5, 2.0 ** 14), (2.0 ** 14, 1.0), (3e-5, 2.0 ** 30), (0.0, 1.0), (np.inf, 1.0), (1e38, 2.0 ** -112), (2.0 ** -120, 2.0 ** 125), (1e-40, 1.0)):
        assert pow2_scale_for_bound(b) == want, b
    for b in np.exp2(np.random.default_rng(0).uniform(-40, 40, 200)).astype(np.float32):
        assert 2.0 ** 14 <= float(b) * pow2_scale_for_bound(b) < 2.0 ** 15


def _control_cases():
    """CPU-sized crafted cases for the negative controls: ReLU off so that no error can hide below zero"""
    return [Case(p, n, 27, 32, 64, seed, relu=False) for p, n, seed in
            (("single", 3 * 128 + 5, 1), ("nact_sweep", 12 * 128, 2), ("empty_tiles", 6 * 128 + 3, 3), ("duplicates", 200, 4))]


def test_split_bounds_hold_for_the_exact_emulation():
    """Positive controls of the derivations: the fp64 emulation of the split (a kernel without accumulation error) is within the
    split's own error of the fp64 result, and the fp16 (hi, lo) epilogue restated in numpy meets the planes bound."""
    for case in _control_cases():
        emu = CgEmu(case, 32)
        ref = case.ref64()
        split_only = emu.tol_fp64() - emu.tol_emul()
        assert ratio(emu.emul(), ref, split_only) <= 0.5, case.pattern
        o = emu.emul().astype(np.float32)
        s, bound = device_bound_scale(emu.amax_in, emu.gain, emu.shift_max)
        hi, lo = split16(o, s)
        assert check_planes(hi, lo, 64, s, bound, o) <= 0.5


def test_negative_controls_are_flagged():
    """Each check flags each subtly wrong kernel on every control case (ratio of error to bound > 1).  The smallest ratios are printed."""
    least = {}
    for case in _control_cases():
        emu = CgEmu(case, 32)
        ref, em = case.ref64(), emu.emul()
        te, t64, t32 = emu.tol_emul(), emu.tol_fp64(), case.tol_fp32()
        assert ratio(em, em, te) == 0
        wrongs = {"no_cross": emu.wrong_no_cross(), "dropped_pair": emu.wrong_dropped_pair(),
                  "stale_row": emu.wrong_stale_row(cg_stages(32, 0)), "swapped_weights": emu.wrong_swapped_weights()}
        for name, wrong in wrongs.items():
            for check, r in (("cg_vs_emul", ratio(wrong, em, te)), ("cg_vs_fp64", ratio(wrong, ref, t64))):
                assert r > 1, (case.pattern, name, check, r)
                least[(name, check)] = min(least.get((name, check), np.inf), r)
        r = ratio(case.ref64_dropped_pair(), ref, t32)
        assert r > 1, (case.pattern, r)
        least[("fp64_dropped_pair", "fp32_vs_fp64")] = min(least.get(("fp64_dropped_pair", "fp32_vs_fp64"), np.inf), r)
    for key, r in sorted(least.items()):
        print("[control] %s / %s: smallest ratio %.3g" % (key[0], key[1], r))


# ================================================================================================================== GPU section
gpu = pytest.mark.gpu


@pytest.fixture
def sp_cg_deep():
    """set_sp_cg_deep is process-wide: whatever a test selects, 0 (the default) is restored afterwards"""
    from sessd_b200 import ops
    try:
        yield ops.set_sp_cg_deep
    finally:
        ops.set_sp_cg_deep(0)


def _dev(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).cuda()


def _f32_buffer(rows, cols):
    return torch.full((rows + SLACK, cols), F32_SENTINEL, dtype=torch.float32, device="cuda")


def _planes_buffer(case, cpo):
    """rows < n_eff zero (the padding channels must stay so), rows >= n_eff sentinel (must stay so)"""
    p = torch.zeros((case.max_out + SLACK, 2 * cpo), dtype=torch.float16, device="cuda")
    p[case.n_eff:] = torch.tensor(F16_SENTINEL, dtype=torch.int16).view(torch.float16)
    return p


def _untouched(buf, case):
    """rows [n_eff, max_out + slack) still hold the sentinel"""
    tail = buf[case.n_eff:]
    if buf.dtype == torch.float16:
        return bool((tail.view(torch.int16) == F16_SENTINEL).all())
    return bool((tail == F32_SENTINEL).all())


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.float16 else torch.int32)


def _n_dev(case):
    return torch.tensor([case.n_dev], dtype=torch.int32, device="cuda")


def _report(kernel, check, r):
    print("[ratio] %s %s: %.3g" % (kernel, check, r))
    assert r <= 1.0, (kernel, check, r)


def _rows_specs():
    """(pattern, n_dev, max_out, n_in) for the fp32 kernels: row counts 1, 127, 128, 129, BIG; n_dev < max_out, == and > (once)"""
    return [("full", 129, 169, None), ("single", BIG, BIG + 40, None), ("flip", 127, 128, None), ("nact_sweep", 3 * 128 + 5, 3 * 128 + 5, None),
            ("empty_tiles", 10 * 128 + 37, 10 * 128 + 77, None), ("duplicates", 1, 3, None), ("high_rows", 128, 137, 70001),
            ("full", 300, 200, None)]


def _fp32_case(spec, kvol, cin, cout, seed):
    pattern, n_dev, max_out, n_in = spec
    return Case(pattern, min(n_dev, max_out), kvol, cin, cout, seed, n_in=n_in, max_out=max_out, n_dev=n_dev,
                relu=seed % 2 == 0, shift=seed % 3 != 0)


def _input_rows(case):
    feat = torch.zeros((case.n_in, case.cin), dtype=torch.float32, device="cuda")
    feat[torch.from_numpy(case.in_rows).cuda()] = _dev(case.x)
    return feat


@gpu
@pytest.mark.parametrize("cin,cout", [(4, 16), (16, 16), (16, 32), (32, 32)])
@pytest.mark.parametrize("kvol", [27, 3])
def test_rows_kernels_match_fp64_and_simt(cin, cout, kvol):
    """spconv_forward_rows (+ abs-max) and spconv_forward_rows_planes (Cp 32 and 64: planes only / both) on every crafted pattern: fp32 rows
    within the fp32 bound of fp64, value-equal to the SIMT kernel, planes within 2^-22 bound of the fp32 rows, the scale restated bit for
    bit, the abs-max exact, padding channels [cout, cpo) still zero, rows past the device count untouched."""
    from sessd_b200 import ops
    worst = {}
    for i, spec in enumerate(_rows_specs()):
        case = _fp32_case(spec, kvol, cin, cout, 31 * i + cin + kvol)
        feat, nbr, n = _input_rows(case), _dev(case.nbr, torch.int32), _n_dev(case)
        w, bn = _dev(case.w), _dev(case.bn)
        sh = None if case.sh is None else _dev(case.sh)
        ne = case.n_eff
        out, amax = _f32_buffer(case.max_out, cout), torch.zeros(1, device="cuda")
        ops.spconv_forward_rows(feat, nbr, n, case.max_out, w, bn, sh, case.relu, out, amax)
        simt = ops.spconv_forward(feat, nbr, n, case.max_out, w, bn, sh, case.relu, _f32_buffer(case.max_out, cout))
        amax_in = torch.tensor([float(np.abs(case.x).max())], device="cuda")
        gain = CgEmu.gain_of(case)
        shift_max = 0.0 if case.sh is None else float(np.abs(case.sh).max())
        planes = {}
        for cpo in (32, 64):
            pl, info = _planes_buffer(case, cpo), torch.zeros(2, device="cuda")
            both = _f32_buffer(case.max_out, cout) if cpo == 32 else None
            ops.spconv_forward_rows_planes(feat, nbr, n, case.max_out, w, bn, sh, case.relu, amax_in, gain, shift_max, both, pl, info)
            planes[cpo] = (pl, info, both)
        torch.cuda.synchronize()
        got = out[:ne].cpu().numpy()
        worst["rows_vs_fp64"] = max(worst.get("rows_vs_fp64", 0), ratio(got, case.ref64(), case.tol_fp32()))
        assert worst["rows_vs_fp64"] <= 1, (spec, worst)
        assert np.array_equal(got, simt[:ne].cpu().numpy()), spec
        assert _untouched(out, case) and _untouched(simt, case), spec
        assert float(amax[0]) == float(np.abs(got).max()), spec
        s, bound = device_bound_scale(float(amax_in[0]), gain, shift_max)
        for cpo, (pl, info, both) in planes.items():
            p = pl[:ne].cpu().numpy()
            assert float(info[1]) == s and float(info[0]) == float(np.abs(got).max()), (spec, cpo)
            worst["planes"] = max(worst.get("planes", 0), check_planes(p[:, :cpo], p[:, cpo:], cout, s, bound, got))
            assert worst["planes"] <= 1, (spec, cpo, worst)
            assert not p[:, cout:cpo].any() and not p[:, cpo + cout:].any(), (spec, cpo)
            assert _untouched(pl, case), (spec, cpo)
            if both is not None:
                assert torch.equal(both[:ne], out[:ne]) and _untouched(both, case), spec
    for k, r in worst.items():
        _report("rows(%d,%d) kvol %d" % (cin, cout, kvol), k, r)


@gpu
@pytest.mark.parametrize("cin,cout", [(4, 16), (16, 16), (16, 32), (32, 32), (32, 64), (64, 64)])
def test_simt_kernel_matches_fp64(cin, cout):
    from sessd_b200 import ops
    worst = 0.0
    for kvol in (27, 8, 1):
        for i, spec in enumerate(_rows_specs() if kvol == 27 else _rows_specs()[2:5]):
            case = _fp32_case(spec, kvol, cin, cout, 17 * i + cin + kvol)
            out = _f32_buffer(case.max_out, cout)
            ops.spconv_forward(_input_rows(case), _dev(case.nbr, torch.int32), _n_dev(case), case.max_out, _dev(case.w), _dev(case.bn),
                               None if case.sh is None else _dev(case.sh), case.relu, out)
            torch.cuda.synchronize()
            worst = max(worst, ratio(out[:case.n_eff].cpu().numpy(), case.ref64(), case.tol_fp32()))
            assert worst <= 1, (spec, kvol, worst)
            assert _untouched(out, case), (spec, kvol)
    _report("simt(%d,%d)" % (cin, cout), "vs_fp64", worst)


@gpu
@pytest.mark.parametrize("kvol", [1, 3, 8, 27])
def test_tile_lists_regroup_crafted_tables_exactly(kvol):
    """rulebook_tile_lists on the crafted tables (empty tiles, partial last tiles, device count below / above the capacity) vs the numpy
    regrouping; records of tiles past the device count are left alone."""
    from cases import assert_tile_lists_match
    from sessd_b200 import ops
    for i, pattern in enumerate(PATTERNS):
        for n_dev, max_out in ((129, 300), (5 * 128 + 1, 5 * 128 + 1), (1, 1), (400, 260)):
            case_nbr = crafted_nbr(pattern, max_out, kvol, 70001 if pattern == "high_rows" else 500, 7 * i + kvol)
            n_eff = min(n_dev, max_out)
            tl = ops.alloc_tile_lists(max_out, kvol, "cuda")
            tl = torch.cat([tl, tl[:1]], 0).fill_(0x2BADBEEF).contiguous()
            ops.rulebook_tile_lists(_dev(case_nbr, torch.int32), torch.tensor([n_dev], dtype=torch.int32, device="cuda"), max_out, tl)
            torch.cuda.synchronize()
            rec = tl.cpu().numpy().view(np.uint32)
            assert_tile_lists_match(rec, case_nbr, n_eff)
            assert (rec[-(-n_eff // 128):] == 0x2BADBEEF).all(), (pattern, n_dev, max_out)


def _cg_specs():
    """every pattern meets every instantiation (each spec runs at deep 0 and 1); ReLU, shift and the outputs rotate over the cases.
    `single` is sized at run time against the device grid (None here), the others are fixed."""
    specs = []
    sizes = {"full": (1, 128, 129, 127), "single": (None,) * 4, "flip": (127, 129, 128, 255), "nact_sweep": (SWEEP,) * 4,
             "empty_tiles": (10 * 128 + 37,) * 4, "duplicates": (300, 300, 300, 300), "high_rows": (200, 200, 200, 200)}
    for ii, (cp, cout) in enumerate(((32, 32), (32, 64), (64, 64), (64, 32))):
        for pi, pattern in enumerate(PATTERNS):
            i = 7 * ii + pi
            n = sizes[pattern][ii]
            max_out, n_dev = (None, None) if n is None else (n + (i % 3) * 40, n)
            if pattern == "duplicates" and cout == 64 and cp == 32:
                max_out, n_dev = 260, 300                        # device count above the capacity: the kernel clamps
            specs.append(dict(cp=cp, cout=cout, pattern=pattern, n=n, max_out=max_out, n_dev=n_dev, relu=(i // 2) % 2 == 0,
                              shift=(i // 3) % 2 == 0, outputs=i % 3, seed=100 + i, n_in=70001 if pattern == "high_rows" else None))
    return specs


def _cg_id(s):
    return "%s-%d-%d" % (s["pattern"], s["cp"], s["cout"])


OUTPUTS = ("f32", "planes", "both")


def _run_cg(case, emu, planes_in, info_in, tl, outputs, cout):
    from sessd_b200 import ops
    cpo = 32 if cout <= 32 else 64
    out = _f32_buffer(case.max_out, cout) if outputs in ("f32", "both") else None
    pl = _planes_buffer(case, cpo) if outputs in ("planes", "both") else None
    info = torch.zeros(2, device="cuda") if pl is not None else None
    ops.spconv_forward_cg(planes_in, info_in, tl, _n_dev(case), case.max_out, emu.tiles.cuda(), _dev(emu.sc), None if case.sh is None else
                          _dev(case.sh), case.relu, emu.gain, emu.shift_max, out, pl, info)
    return out, pl, info


def _check_cg(case, emu, plane_rows, label, sp_cg_deep, first_output=2):
    """the case at deep 0 and deep 1 (outputs rotating from OUTPUTS[first_output]): each run twice (bitwise equal), fp32 rows vs the
    emulation and fp64, planes and out_info, sentinels; the fp32 rows of the two pipelines must be bitwise equal too (same wgmma sequence
    per tile, only the staging differs)"""
    from sessd_b200 import ops
    cout, ne = case.cout, case.n_eff
    planes_in = torch.zeros((plane_rows, 2 * emu.cp), dtype=torch.float16, device="cuda")
    planes_in[torch.from_numpy(case.in_rows).cuda()] = torch.from_numpy(np.concatenate([emu.a_hi, emu.a_lo], 1)).cuda()
    info_in = torch.tensor([emu.amax_in, emu.s_in], dtype=torch.float32, device="cuda")
    tl = ops.rulebook_tile_lists(_dev(case.nbr, torch.int32), _n_dev(case), case.max_out, ops.alloc_tile_lists(case.max_out, case.kvol, "cuda"))
    emul, tol_emul, ref, tol_fp64 = emu.emul(), emu.tol_emul(), case.ref64(), emu.tol_fp64()
    s, bound = device_bound_scale(emu.amax_in, emu.gain, emu.shift_max)
    rows_by_deep = []
    for deep in (0, 1):
        outputs = OUTPUTS[(first_output + deep) % 3]
        sp_cg_deep(deep)
        runs = [_run_cg(case, emu, planes_in, info_in, tl, outputs, cout) for _ in range(2)]
        f32 = runs[0][0] if runs[0][0] is not None else _run_cg(case, emu, planes_in, info_in, tl, "f32", cout)[0]
        torch.cuda.synchronize()
        for a, b in zip(runs[0], runs[1]):                                   # run to run: bitwise
            assert (a is None and b is None) or torch.equal(_bits(a), _bits(b)), deep
        got = f32[:ne].cpu().numpy()
        assert _untouched(f32, case), deep
        rows_by_deep.append(got)
        worst = {"vs_emul": ratio(got, emul, tol_emul), "vs_fp64": ratio(got, ref, tol_fp64)}
        _, pl, info = runs[0]
        if pl is not None:
            cpo = pl.shape[1] // 2
            p = pl[:ne].cpu().numpy()
            assert float(info[1]) == s and float(info[0]) == float(np.abs(got).max()), deep
            worst["planes"] = check_planes(p[:, :cpo], p[:, cpo:], cout, s, bound, got)
            assert _untouched(pl, case), deep
        for k, r in worst.items():
            _report("cg %s deep%d %s" % (label, deep, outputs), k, r)
    assert np.array_equal(rows_by_deep[0].view(np.int32), rows_by_deep[1].view(np.int32))


@gpu
@pytest.mark.parametrize("spec", _cg_specs(), ids=_cg_id)
def test_cg_kernel_matches_emulation_and_fp64(spec, sp_cg_deep):
    """spconv_forward_cg, all eight instantiations ((32,32), (32,64), (64,64), (64,32) x deep 0 / 1) on every crafted pattern, ReLU, shift
    and the outputs rotating: fp32 rows within the accumulation bound of the fp64 emulation and within that plus the split's error of
    fp64, planes within 2^-22 bound, out_info exact, run to run and deep 0 vs deep 1 bitwise, rows past the device count untouched.
    nact_sweep meets every (active offsets, st0, phase) a CTA can carry into a tile at the ring lengths of both grids
    (test_nact_sweep_reaches_every_ring_position) and `single`, 3 grid + 1 tiles at the device's default grid, gives every CTA three
    tiles or more (six at deep 1).  Whether each dirty-row clear across tiles is reached is left to the cases of
    test_gpu_spconv_cg_grid, which are built against the grid and assert it."""
    s = spec
    if s["n"] is None:
        n = 3 * cg_grid(s["cp"], s["cout"], 0, 1 << 30) * 128 + 77
        s = dict(s, n=n, max_out=n + (s["seed"] - 100) % 3 * 40, n_dev=n)
    case = Case(s["pattern"], min(s["n_dev"], s["max_out"]), 27, s["cp"], s["cout"], s["seed"], n_in=s["n_in"], max_out=s["max_out"],
                n_dev=s["n_dev"], relu=s["relu"], shift=s["shift"])
    _check_cg(case, CgEmu(case, s["cp"]), case.n_in + 1, _cg_id(s), sp_cg_deep, s["outputs"])


@gpu
@pytest.mark.parametrize("kvol", [1, 3, 8])
def test_cg_kernel_other_kernel_volumes(kvol, sp_cg_deep):
    """kvol other than 27 (1, 3, 8) on the pair-gather kernel, partial last tile, deep 0 and 1"""
    case = Case("flip" if kvol > 1 else "full", 3 * 128 + 17, kvol, 32, 64, 300 + kvol, relu=False)
    _check_cg(case, CgEmu(case, 32), case.n_in + 1, "kvol%d" % kvol, sp_cg_deep)


@gpu
def test_cg_kernel_input_rows_above_2_24(sp_cg_deep):
    """input row indices in (2^24, plane_rows) with plane_rows = 2^24 + 2^20 (a 2.3 GB plane buffer): the packed tile-list entry
    (row << 7 | tile row) is above 2^31 and the byte offset of the gathered row (row * 128) above 2^31, deep 0 and 1"""
    rows = (1 << 24) + (1 << 20)
    case = Case("high_rows", 3 * 128 + 1, 27, 32, 32, 77, n_in=rows)
    assert case.in_rows.min() > (1 << 24) and case.in_rows.max() == rows - 1
    _check_cg(case, CgEmu(case, 32), rows, "rows>2^24", sp_cg_deep)
    torch.cuda.empty_cache()
