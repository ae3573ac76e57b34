"""The BEV neck kernels one operator at a time (ABI wrappers of sessd_b200.ops, no runner) on crafted maps, against fp64 references,
with element-wise tolerances derived from each kernel's numerics.

Notation: u = 2^-24 (fp32 unit roundoff); x the fp32 input map [B][H][W][Cin], w [taps][Cin][Cout] the weights, bn / sh the folded
BatchNorm scale / shift, r the residual (added after the ReLU).  For an output pixel, P = the taps whose input position lies inside the
map (taps outside read TMA's zero fill: their products are exact zeros).

bev_conv_p2 / bev_deconv_p2 (wgmma on fp16 (hi, lo) planes) vs an fp64 emulation of what they multiply: the input planes
  a = (a_hi, a_lo) read back from the device, x S_in = a_hi + a_lo + d, and the pack_weight_h2 planes b = (b_hi, b_lo) with
  w 2^e = b_hi + b_lo + d'; emul = (sum a_hi b_hi + a_hi b_lo + a_lo b_hi) (1 / S_in) sc + sh with sc = bn 2^-e, then ReLU, then + r.
  The products are exact (fp16 x fp16 fits fp32); one k=16 wgmma step D = C + sum_16 p_i aligns the addends to the largest exponent and
  normalises once, losing <= 2 ulp of |C| + sum |p_i| <= 2 * 2^-23 sum |p| (|C| is bounded by the products before it).  Steps whose
  products are all zero add an exact zero and are not counted: G = 2 P Cin / 16 steps (the cross accumulator sees two k=16 products per
  16 channels and tap, the main one half as many; both use G).  The epilogue's acc_m + acc_c and fmaf(., sc, sh) add two roundings,
  the residual add one more of |relu(.)| + |r|:
    |got - emul| <= c 2^-23 (G + 2) |sc| magA / S_in + 2^-23 |sh| + 2^-23 (|relu(emul)| + |r|),   c = 2,
    magA = sum |a_hi| (|b_hi| + |b_lo|) + |a_lo| |b_hi|
  Where magA = 0 (no product in the receptive field) the output is exactly relu(sh) (+ r): checked with ==.
vs plain fp64 (F.conv2d-style tap gather / F.conv_transpose2d of the fp32 inputs): the bound above plus the split's own error.  S_in
  maps max|x| into [2^14, 2^15), so |d| <= 2^-9 <= 2^-23 amax_in S_in; max |w 2^e| over the taps and channels of channel n lies in
  [2^10, 2^11), so |d'| <= 2^-13 <= 2^-23 wmax_n 2^e; the dropped a_lo b_lo <= 2^-22 |x| wmax_n / (S_in 2^e).  Per product that is
  <= 2^-21.4 (amax_in |w| + |x| wmax_n); with a 2.6x margin:
    + 2^-20 |bn| sum over the P taps and the channels of (amax_in |w| + |x| wmax_n)
planes outputs [2][B][H][W][C] at S_out = pow2_scale_for_bound(bound), bound = amax_in gain + shift_max (+ amax_resid), computed in fp32
  (the product may be contracted into an FMA: both roundings are restated and must give the same scale).  o S_out is exact, hi =
  fp16(o S_out) is off by <= 8 and lo = fp16(o S_out - hi) by <= 2^-9, so |(hi + lo) / S_out - o| <= 2^-9 / S_out <= 2^-23 bound;
  checked at 2^-22 bound.  |o| <= bound gives |o S_out| < 2^15, so |hi| <= 2^15: the fp16 rounding of a value within 8 of 2^15 IS
  2^15 (the spacing there is 16), so |hi| < 2^15 does not follow; 2^15 is far below fp16's 65504 and (hi, lo) stays exact.
bev_conv_h2 / bev_deconv_h2 (lab): the same bounds, with the input split inside the kernel at pow2_scale_for_bound(amax_in).

Plane producers: bev_split_planes, sparse_to_dense_planes and the planes of ssfa_fuse_planes are a power-of-two scaling and two fp16
roundings: restated bit for bit in numpy.  absmax is exact.  ssfa_fuse_planes' fp32 output vs fp64, per pixel with C channels:
  the dot products d_k = sum_c x_k w_k run through a chain of <= C / 128 + 4 roundings per lane and a 5-level butterfly:
  |dd_k| <= (C / 128 + 12) u sum |x_k| |w_k|; l_k = fmaf(d_k, s_k, t_k): |dl_k| <= |s_k| |dd_k| + u (|s_k d_k| + |t_k|).  The pair
  softmax a_0 = 1 / (1 + exp(l_1 - l_0)) has |da_0 / dl| <= 1/4; expf (<= 2 ulp), the sum, the division and the product add <= 12 u
  relative, and the rounded l_0 - max adds <= u |l_0 - l_1| a_0 <= 0.3 u: |da| <= (|dl_0| + |dl_1|) / 4 + 16 u.  The output
  x_0 a_0 + x_1 a_1 adds two roundings: |dout| <= (|x_0| + |x_1|) (|da| + 2 u).

Launch schedule (bev_conv_p2.cuh, restated in p2_plan / ring_starts and checked against the launcher's own plan, sessd_bev_p2_plan):
total = nclass nblocks tiles work items, classes ordered by descending tap count, on min(total, SMs) persistent CTAs; an item takes
nchunks ntaps steps of the weight ring.  nchunks is even (Cin is a multiple of 64, chunks are 32 channels), so an item starts after an
even number s of steps of its CTA, at (stage, phase) = (s mod B, (s div B) mod 2) of a B-stage ring: B of the 2 B positions (even
stages with both phases for even B, every stage with the phase of its parity for odd B).  The planes launches of the sweep build the
11- (3x3 convs and deconvs), 12- (1x1 and n_tile 32) and 7-stage (stride-2 convs) rings and are checked to start items at every one
of those positions, and to run both one and two patch buffers.

Each tolerance is shown to catch a subtly wrong kernel on the CPU (negative controls).  Smallest ratio of error to bound over the control
cases (vs the emulation bound / vs the fp64 bound): cross products dropped 10 / 4.5, one tap read from the neighbouring tile at a tile
edge 1.2e4 / 6.3e3, previous item's accumulator carried into one tile 4.8e4 / 1.2e4, deconv parity class offset by one pixel
3.9e6 / 4.3e4, two taps' weights swapped 2.1e4 / 9.9e3; lo output plane dropped vs the planes bound 16; the residual's share left out
of the output scale: max |hi| / 2^15 = 1.3.
Largest ratios measured on one H100 80GB HBM3 (400 W power limit): p2 vs emulation 0.50, p2 vs fp64 0.50, p2 planes 0.38; h2 vs
emulation 0.46, vs fp64 0.44; ssfa_fuse vs fp64 0.08.
"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

U = 2.0 ** -24
CG_C = 2.0                                     # wgmma accumulation: ulps per k step (module docstring)
NUM_SMS = 132                                  # H100 SXM; the GPU tests recompute the schedule with the device's count
GUARD = 64                                     # sentinel elements before and after every output (keeps 128-byte alignment)
F32_SENTINEL = -1234.5
F16_SENTINEL = 0x5A5A
HI_LIMIT = 2.0 ** 15

# launcher constants of bevconv_p2.cuh
TILE_U, TILE_V = 8, 16
MAX_COPIES, MAX_ROWS_V = 6, 18
BSTAGES, MAX_BSTAGES = 6, 12
MAX_SMEM = 227 * 1024
CHUNK = 32
TAPS3 = [(dy, dx) for dy in (-1, 0, 1) for dx in (-1, 0, 1)]
TAPS1 = [(0, 0)]


def cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------------------------------ schedule restated
def orientation(grid_h, grid_w):
    """u_is_x of launch_p2: u (the 8-pixel tile edge) along x when that needs no more tiles than along y"""
    return 1 if cdiv(grid_w, TILE_U) * cdiv(grid_h, TILE_V) <= cdiv(grid_h, TILE_U) * cdiv(grid_w, TILE_V) else 0


def deconv_classes():
    """the four output-parity classes of p2_deconv, c = 2 py + px: (dy, dx, weight tap ky * 3 + kx) with 2y + py = 2(y + dy) - 1 + ky"""
    out = []
    for py in (0, 1):
        for px in (0, 1):
            ys = [(0, 1)] if py == 0 else [(1, 0), (0, 2)]
            xs = [(0, 1)] if px == 0 else [(1, 0), (0, 2)]
            out.append([(dy, dx, ky * 3 + kx) for dy, ky in ys for dx, kx in xs])
    return out


def p2_plan(mode, cin, cout, cout_pad, classes, stride, grid_h, grid_w, batch, smem_a=False):
    """p2_plan of bevconv_p2.cuh for a mode ("p2": planes, "h2": fp16 split in the kernel): None where the launcher refuses the launch.
    Stride-1 planes launches read A from registers out of one patch copy (smem_a: the loads probe's descriptor plan instead)."""
    if cin < 64 or cin % 64 or cout < 8 or cout % 8:
        return None
    n_tile = 32 if cout <= 32 else 128
    if cout_pad % n_tile or cout_pad < cout:
        return None
    u_is_x = orientation(grid_h, grid_w)
    keys = {}
    for cls in classes:
        for dy, dx, _ in cls:
            tu, tv = (dx, dy) if u_is_x else (dy, dx)
            k = (tu, tv % stride)
            if k not in keys:
                if len(keys) == MAX_COPIES:
                    return None
                keys[k] = [tv, tv]
            keys[k] = [min(keys[k][0], tv), max(keys[k][1], tv)]
    rows_v = max(TILE_V + (hi - lo) // stride for lo, hi in keys.values())
    if rows_v > MAX_ROWS_V:
        return None
    ncopies, pitch_u = len(keys), TILE_U
    if mode == "p2" and stride == 1 and not smem_a:       # one copy: from the taps' least shift, wide and tall enough for their greatest
        us, vs = [u for u, _ in keys], [v for lohi in keys.values() for v in lohi]
        ncopies, pitch_u, rows_v = 1, TILE_U + max(us) - min(us), TILE_V + max(vs) - min(vs)
        if pitch_u > 256 or rows_v > 256:
            return None
    per_buf = ncopies * 2 * cdiv(rows_v * pitch_u * 64, 512) * 512                  # fp16 (hi, lo) copies in whole 512-byte periods
    if mode == "h2":
        per_buf += ncopies * rows_v * TILE_U * CHUNK * 4                              # fp32 staging
    bstage, tail = 2 * n_tile * 64, 1536 + 16 + 2 * 4 * cout                          # barriers, tap offsets, BN scale and shift
    npatch = 2 if BSTAGES * bstage + tail + 2 * per_buf <= MAX_SMEM else 1
    bstages = min((MAX_SMEM - tail - npatch * per_buf) // bstage, MAX_BSTAGES)
    if bstages < 2:
        return None
    grid_u, grid_v = (grid_w, grid_h) if u_is_x else (grid_h, grid_w)
    tiles = cdiv(grid_u, TILE_U) * cdiv(grid_v, TILE_V) * batch
    ntaps = [len(c) for c in classes]
    return dict(u_is_x=u_is_x, n_tile=n_tile, nblocks=cout_pad // n_tile, tiles=tiles, total=len(classes) * (cout_pad // n_tile) * tiles,
                ncopies=ncopies, rows_v=rows_v, pitch_u=pitch_u, npatch=npatch, bstages=bstages,
                smem=bstages * bstage + tail + npatch * per_buf, ntaps=ntaps, order=sorted(range(len(classes)), key=lambda c: -ntaps[c]),
                nchunks=cin // CHUNK)


def ring_starts(plan, num_sms=NUM_SMS):
    """(stage, phase) of the weight ring at the start of every work item: item g runs on CTA g % grid after that CTA's earlier items"""
    grid = min(plan["total"], num_sms)
    per_cls = plan["nblocks"] * plan["tiles"]
    seen = set()
    for b in range(grid):
        st = ph = 0
        for g in range(b, plan["total"], grid):
            seen.add((st, ph))
            adv = st + plan["nchunks"] * plan["ntaps"][plan["order"][g // per_cls]]
            ph ^= (adv // plan["bstages"]) & 1
            st = adv % plan["bstages"]
    return seen


def reachable_starts(bstages):
    """every item is a multiple of nchunks steps, an even number: an item starts after s steps of its CTA, s even, s mod 2 bstages"""
    return {(s % bstages, s // bstages) for s in range(0, 2 * bstages, 2)}


# ------------------------------------------------------------------------------------------------------------------ crafted maps
def crafted_map(pattern, b, h, w, c, seed):
    """fp32 NHWC map: dense (pixel magnitudes 2^-12 .. 1), sparse (~5 % of the pixels, in clusters, the rest exact zero), tile_edges
    (large values on the first / last rows and columns of every 8x16 tile, either orientation, and of the map; small elsewhere), zero"""
    rng = np.random.default_rng(seed)
    mag = np.exp2(rng.uniform(-12, 0, (b, h, w, 1)))
    x = rng.standard_normal((b, h, w, c)) * mag
    if pattern == "sparse":
        seeds = rng.random((b, h, w)) < 0.013
        seeds[:, rng.integers(0, h), rng.integers(0, w)] = True
        occ = seeds.copy()
        for dy, dx in ((0, 1), (1, 0), (1, 1)):                              # 2x2 clusters
            occ[:, dy:, dx:] |= seeds[:, :h - dy, :w - dx]
        x = x * occ[..., None]
    elif pattern == "tile_edges":
        yy, xx = np.arange(h)[:, None], np.arange(w)[None, :]
        edge = np.zeros((h, w), bool)
        for t in (TILE_U, TILE_V):
            edge |= (yy % t == 0) | (yy % t == t - 1) | (xx % t == 0) | (xx % t == t - 1)
        edge |= (yy == h - 1) | (xx == w - 1)
        x = np.where(edge[None, :, :, None], rng.standard_normal((b, h, w, c)), x * 2.0 ** -10)
    elif pattern == "zero":
        x = np.zeros((b, h, w, c))
    elif pattern != "dense":
        raise ValueError(pattern)
    return x.astype(np.float32)


class BevCase:
    """One crafted layer.  kind "conv": tap list, in_stride, grid (default ceil(in / stride)), output extent and out_stride / out_off
    (default: the grid); kind "deconv": ConvTranspose2d(k3, s2, p1, op1), taps ky * 3 + kx of W[Cin][Cout][ky][kx]."""

    def __init__(self, kind, pattern, batch, in_hw, cin, cout, seed, taps=TAPS3, stride=1, cout_pad=None, grid=None, out_hw=None,
                 out_stride=1, out_off=(0, 0), relu=True, shift=True, resid=False, amax=None, resid_scale=1.0):
        rng = np.random.default_rng(seed + 1000)
        self.kind, self.pattern, self.batch, self.in_hw, self.cin, self.cout = kind, pattern, batch, tuple(in_hw), cin, cout
        self.relu, self.stride, self.out_stride, self.out_off = relu, stride, out_stride, tuple(out_off)
        self.cout_pad = cout_pad or (32 if cout <= 32 else cdiv(cout, 128) * 128)
        if kind == "conv":
            self.taps = list(taps)
            self.grid = tuple(grid) if grid else (cdiv(in_hw[0], stride), cdiv(in_hw[1], stride))
            self.out_hw = tuple(out_hw) if out_hw else self.grid
            self.classes = [[(dy, dx, t) for t, (dy, dx) in enumerate(self.taps)]]
        else:
            self.taps = None
            self.grid = tuple(in_hw)
            self.out_hw = (2 * in_hw[0], 2 * in_hw[1])
            self.classes = deconv_classes()
        ntap = len(self.taps) if kind == "conv" else 9
        self.x = crafted_map(pattern, batch, in_hw[0], in_hw[1], cin, seed)
        if amax is not None and pattern != "zero":
            self.x = (self.x * np.float32(amax / np.abs(self.x).max())).astype(np.float32)
        self.w = (rng.standard_normal((ntap, cin, cout)) * np.exp2(rng.uniform(-3, 1, (1, 1, cout))) / np.sqrt(cin * ntap)).astype(np.float32)
        self.bn = ((rng.random(cout) + 0.5) * np.where(rng.random(cout) < 0.2, -1, 1)).astype(np.float32)
        self.sh = (0.2 * rng.standard_normal(cout)).astype(np.float32) if shift else None
        self.r = None
        if resid:
            oh, ow = self.out_hw
            self.r = (rng.standard_normal((batch, oh, ow, cout)) * np.exp2(rng.uniform(-6, 0, (batch, oh, ow, 1))) * resid_scale).astype(np.float32)

    def plan(self, mode="p2"):
        return p2_plan(mode, self.cin, self.cout, self.cout_pad, self.classes, self.stride, self.grid[0], self.grid[1], self.batch)

    @property
    def shv(self):
        return np.zeros(self.cout) if self.sh is None else self.sh.astype(np.float64)

    @property
    def gain(self):
        from sessd_b200 import ops
        return ops.conv_gain(torch.from_numpy(self.w), torch.from_numpy(self.bn))

    @property
    def shift_max(self):
        return 0.0 if self.sh is None else float(np.abs(self.sh).max())

    @property
    def amax_r(self):
        return 0.0 if self.r is None else float(np.abs(self.r).max())

    def owned(self):
        """[B, out_h, out_w] mask of the output pixels the launch writes, and the (oy, ox) index arrays of the grid positions"""
        oys = np.arange(self.grid[0]) * self.out_stride + self.out_off[0]
        oxs = np.arange(self.grid[1]) * self.out_stride + self.out_off[1]
        if self.kind == "deconv":
            oys, oxs = np.arange(self.out_hw[0]), np.arange(self.out_hw[1])
        m = np.zeros((self.batch,) + self.out_hw, bool)
        m[:, oys[:, None], oxs[None, :]] = True
        return m, oys, oxs

    def resid_on_grid(self):
        if self.r is None:
            return None
        _, oys, oxs = self.owned()
        return self.r[:, oys[:, None], oxs[None, :]].astype(np.float64)

    def desc(self):
        from sessd_b200 import ops
        return ops.conv_desc(self.batch, self.in_hw, self.cin, self.out_hw, self.cout, self.grid, self.taps, in_stride=self.stride,
                             out_stride=self.out_stride, out_off=self.out_off, relu=self.relu)

    def label(self):
        return "%s-%s-b%d-%dx%d-%d-%d%s" % (self.kind, self.pattern, self.batch, self.in_hw[0], self.in_hw[1], self.cin, self.cout,
                                            "-s2" if self.stride == 2 else "")


# ------------------------------------------------------------------------------------------------------------------ fp64 references
def tap_conv(case, x, w):
    """x [B][H][W][C], w [T][C][N] (fp64 tensors) -> [B][gh][gw][N]: conv: sum_t x[b, y s + dy_t, x s + dx_t] @ w[t] (zero outside);
    deconv: F.conv_transpose2d(k3, s2, p1, op1) of W = w.reshape(3, 3, C, N).permute(2, 3, 0, 1)"""
    if case.kind == "deconv":
        c, n = w.shape[1], w.shape[2]
        wt = w.reshape(3, 3, c, n).permute(2, 3, 0, 1)
        return F.conv_transpose2d(x.permute(0, 3, 1, 2), wt, None, 2, 1, output_padding=1).permute(0, 2, 3, 1)
    s, (gh, gw) = case.stride, case.grid
    h, wd = x.shape[1], x.shape[2]
    dys, dxs = [d for d, _ in case.taps], [d for _, d in case.taps]
    pt, pl = max(0, -min(dys)), max(0, -min(dxs))
    pb, pr = max(0, (gh - 1) * s + max(dys) - (h - 1)), max(0, (gw - 1) * s + max(dxs) - (wd - 1))
    xp = F.pad(x, (0, 0, pl, pr, pt, pb))
    out = torch.zeros((x.shape[0], gh, gw, w.shape[2]), dtype=x.dtype, device=x.device)
    for t, (dy, dx) in enumerate(case.taps):
        out += xp[:, pt + dy:pt + dy + (gh - 1) * s + 1:s, pl + dx:pl + dx + (gw - 1) * s + 1:s] @ w[t]
    return out


def split16(v, s):
    """fp32 values -> fp16 (hi, lo) at the exact scale s: hi = fp16_rn(v s), lo = fp16_rn(v s - hi)"""
    xs = np.asarray(v, np.float32) * np.float32(s)
    hi = xs.astype(np.float16)
    return hi, (xs - hi.astype(np.float32)).astype(np.float16)


def pow2_scale_for_bound(bound):
    """numpy restatement of common.cuh pow2_scale_for_bound: the power of two that maps an fp32 bound into [2^14, 2^15)"""
    e = int((np.array(bound, np.float32).view(np.uint32) >> 23) & 0xFF)
    if e in (0, 255):
        return 1.0
    return float(np.array(min(max(268 - e, 2), 252) << 23, np.uint32).view(np.float32))


def output_scale(amax, gain, shift_max, amax_r=None):
    """(S_out, bound) of the kernels: fp32 amax * gain + shift_max (fused or not: both must give the same scale) (+ amax_r)"""
    fused = np.float32(np.float64(np.float32(amax)) * np.float64(np.float32(gain)) + np.float64(np.float32(shift_max)))
    unfused = np.float32(np.float32(amax) * np.float32(gain)) + np.float32(shift_max)
    if amax_r is not None:
        fused, unfused = np.float32(fused + np.float32(amax_r)), np.float32(unfused + np.float32(amax_r))
    s = pow2_scale_for_bound(fused)
    assert s == pow2_scale_for_bound(unfused)
    return s, float(fused)


class Emu:
    """What a BEV kernel multiplies for a BevCase (fp16 planes: a_planes = the device's input planes, else the restated split), in fp64
    on `dev`, plus the tolerances of the module docstring."""

    def __init__(self, case, dev, a_planes=None):
        from sessd_b200 import ops
        self.case, self.dev = case, dev
        d64 = lambda a: torch.as_tensor(np.asarray(a, np.float64), device=dev)       # noqa: E731
        self.amax_in = float(np.abs(case.x).max())
        wp = torch.from_numpy(case.w)
        self.s_in = pow2_scale_for_bound(self.amax_in)
        a_hi, a_lo = split16(case.x, self.s_in) if a_planes is None else a_planes
        planes, inv = ops.pack_weight_h2(wp, case.cout_pad)
        self.w_h2, self.inv = planes, inv
        t = planes.numpy()[:, :, :case.cout].transpose(0, 1, 3, 2)                                # [2][T][Cin][Cout]
        b_hi, b_lo = t[0], t[1]
        self.sc32 = (torch.from_numpy(case.bn) * inv[:case.cout]).numpy()
        self.sc = self.sc32.astype(np.float64)
        self.A_hi, self.A_lo, self.B_hi, self.B_lo = d64(a_hi), d64(a_lo), d64(b_hi), d64(b_lo)
        self.acc0 = self.acc()
        mag = tap_conv(case, self.A_hi.abs(), self.B_hi.abs() + self.B_lo.abs()) + tap_conv(case, self.A_lo.abs(), self.B_hi.abs())
        ones = torch.ones((case.batch,) + case.in_hw + (1,), dtype=torch.float64, device=dev)
        self.P = tap_conv(case, ones, torch.ones((self.B_hi.shape[0], 1, 1), dtype=torch.float64, device=dev))
        g = 2 * self.P * case.cin / 16
        sc, shv = d64(self.sc), d64(case.shv)
        self.magA = mag
        self.emul0 = self.emul()
        r = self.r
        self.tol_e = CG_C * 2.0 ** -23 * (g + 2) * sc.abs() * mag / self.s_in + 2.0 ** -23 * shv.abs()
        if r is not None:
            self.tol_e = self.tol_e + 2.0 ** -23 * ((self.emul0 - r).abs() + r.abs())
        x64, w64 = d64(case.x), d64(case.w)
        aw = w64.abs()
        split = (self.amax_in * tap_conv(case, ones, aw.sum(1, keepdim=True))
                 + tap_conv(case, x64.abs().sum(3, keepdim=True), torch.ones_like(aw[:, :1, :1])) * aw.amax(dim=(0, 1)))
        self.tol_64 = self.tol_e + 2.0 ** -20 * d64(case.bn).abs() * split
        self.ref = self.finish(tap_conv(case, x64, w64), d64(case.bn), 1.0)

    @property
    def r(self):
        rr = self.case.resid_on_grid()
        return None if rr is None else torch.as_tensor(rr, device=self.dev)

    def acc(self, B_hi=None, B_lo=None, A_hi=None, A_lo=None, cross=True):
        A_hi = self.A_hi if A_hi is None else A_hi
        A_lo = self.A_lo if A_lo is None else A_lo
        bh = self.B_hi if B_hi is None else B_hi
        bl = self.B_lo if B_lo is None else B_lo
        if not cross:
            return tap_conv(self.case, A_hi, bh)
        return tap_conv(self.case, A_hi, bh + bl) + tap_conv(self.case, A_lo, bh)

    def finish(self, acc, sc, s_in):
        y = acc / s_in * sc + torch.as_tensor(self.case.shv, device=self.dev)
        if self.case.relu:
            y = torch.clamp_min(y, 0)
        r = self.r
        return y if r is None else y + r

    def emul(self, acc=None):
        return self.finish(self.acc0 if acc is None else acc, torch.as_tensor(self.sc, device=self.dev), self.s_in)

    def exact_zero_field(self):
        """(mask, value) where no product reaches the output: relu(sh) (+ r) in fp32"""
        c = self.case
        y = np.broadcast_to(c.shv.astype(np.float32), self.magA.shape)
        if c.relu:
            y = np.maximum(y, np.float32(0))
        rr = c.resid_on_grid()
        if rr is not None:
            y = (y + rr.astype(np.float32)).astype(np.float32)
        return (self.magA == 0).cpu().numpy(), y

    # ---- negative controls: outputs of subtly wrong kernels
    def wrong_no_cross(self):
        return self.emul(self.acc(cross=False))

    def wrong_swapped_taps(self):
        t = self.B_hi.shape[0]
        perm = list(range(t))
        perm[0], perm[-1] = perm[-1], perm[0]
        return self.emul(self.acc(self.B_hi[perm], self.B_lo[perm]))

    def wrong_neighbour_tile_tap(self):
        """one tap of one tile-edge output pixel reads its input from the same place in the neighbouring tile (u + 8 along u); the pixel
        and tap are those where the wrong read differs most from the right one (relative to the tolerance)"""
        c = self.case
        assert c.kind == "conv" and c.stride == 1
        ux = c.plan()["u_is_x"]
        best = None
        gh, gw = c.grid
        a = torch.cat([self.A_hi, self.A_lo], 3)
        bw = [torch.cat([self.B_hi[t] + self.B_lo[t], self.B_hi[t]], 0) for t in range(len(c.taps))]

        def read(b, yy, xx):
            if 0 <= yy < c.in_hw[0] and 0 <= xx < c.in_hw[1]:
                return a[b, yy, xx]
            return torch.zeros_like(a[0, 0, 0])
        for y in range(gh):
            for x in range(gw):
                uu = x if ux else y
                if uu % TILE_U != TILE_U - 1:
                    continue
                for t, (dy, dx) in enumerate(c.taps):
                    sy, sx = (0, TILE_U) if ux else (TILE_U, 0)
                    for b in range(c.batch):
                        delta = (read(b, y + dy + sy, x + dx + sx) - read(b, y + dy, x + dx)) @ bw[t]
                        score = float((delta.abs() / self.s_in * torch.as_tensor(np.abs(self.sc), device=self.dev)
                                       / self.tol_e[b, y, x].clamp_min(1e-300)).max())
                        if best is None or score > best[0]:
                            best = (score, b, y, x, delta)
        _, b, y, x, delta = best
        acc = self.acc0.clone()
        acc[b, y, x] += delta
        return self.emul(acc)

    def wrong_carried_accumulator(self):
        """one 8x16 tile starts from the accumulator of the tile before it instead of zero (the tile with the largest accumulator is
        carried into its successor along v)"""
        c = self.case
        ux = c.plan()["u_is_x"]
        acc = self.acc0.clone()
        gu, gv = (c.grid[1], c.grid[0]) if ux else c.grid
        assert gv > TILE_V, "needs two tiles along v"
        src = acc[:, :TILE_V] if ux else acc[:, :, :TILE_V]
        n = min(TILE_V, gv - TILE_V)
        if ux:
            acc[:, TILE_V:TILE_V + n, :TILE_U] += src[:, :n, :TILE_U]
        else:
            acc[:, :TILE_U, TILE_V:TILE_V + n] += src[:, :TILE_U, :n]
        return self.emul(acc)

    def wrong_deconv_class_offset(self):
        """the (py, px) = (1, 1) class reads its input one pixel further along x (zero past the map)"""
        assert self.case.kind == "deconv"
        acc = self.acc0.clone()
        sub = acc[:, 1::2, 1::2]
        shifted = torch.zeros_like(sub)
        shifted[:, :, :-1] = sub[:, :, 1:]
        acc[:, 1::2, 1::2] = shifted
        return self.emul(acc)


def ratio(got, ref, tol):
    """max |got - ref| / tol (fp64, on ref's device); an element whose tolerance is 0 must match exactly"""
    dev = ref.device if isinstance(ref, torch.Tensor) else "cpu"
    t = lambda v: (v if isinstance(v, torch.Tensor) else torch.as_tensor(np.asarray(v, np.float64))).to(dev, torch.float64)   # noqa: E731
    d = (t(got) - t(ref)).abs()
    tol = torch.broadcast_to(t(tol), d.shape)
    r = torch.where(tol > 0, d / torch.where(tol > 0, tol, torch.ones_like(tol)), torch.where(d > 0, torch.inf, 0.0))
    return float(r.max()) if r.numel() else 0.0


def planes_ratio(hi, lo, s, bound, f32):
    back = (hi.astype(np.float64) + lo.astype(np.float64)) / s
    return ratio(back, f32.astype(np.float64), np.full(f32.shape, 2.0 ** -22 * bound))


# ================================================================================================================== CPU section
def _p2_specs():
    """The planes-path sweep: map extents {1, 7, 8, 9, 15, 16, 17, 40, 200x176}, both orientations of conv, stride-2 conv (odd inputs)
    and deconv, batch 1-3, Cin 64-256, cout 8-256 (cout_pad > cout), 1-9 taps incl. asymmetric lists, out_stride 2 + out_off and grids
    smaller than the output.  ReLU, shift and residual rotate."""
    A5 = [(0, 0), (-1, 1), (1, 0), (0, -2), (2, 1)]
    A7 = [(-1, -1), (-1, 0), (-1, 1), (0, -1), (0, 0), (0, 1), (1, 1)]
    s = [dict(kind="conv", pattern="dense", batch=1, in_hw=(16, 16), cin=128, cout=128),
         dict(kind="conv", pattern="dense", batch=2, in_hw=(9, 40), cin=64, cout=40, resid=True),
         dict(kind="conv", pattern="sparse", batch=3, in_hw=(40, 9), cin=192, cout=136, resid=True, relu=False),
         dict(kind="conv", pattern="tile_edges", batch=1, in_hw=(17, 40), cin=256, cout=256, relu=False),
         dict(kind="conv", pattern="zero", batch=2, in_hw=(7, 9), cin=64, cout=8, shift=False),
         dict(kind="conv", pattern="zero", batch=1, in_hw=(15, 17), cin=64, cout=24, resid=True),
         dict(kind="conv", pattern="dense", batch=1, in_hw=(1, 1), cin=64, cout=24, cout_pad=64, taps=TAPS1),
         dict(kind="conv", pattern="sparse", batch=3, in_hw=(200, 176), cin=64, cout=24, cout_pad=64, taps=A5),
         dict(kind="conv", pattern="dense", batch=2, in_hw=(200, 176), cin=64, cout=256, taps=A7, shift=False),
         dict(kind="conv", pattern="dense", batch=1, in_hw=(7, 9), cin=128, cout=128, taps=[(0, 0), (0, 1)]),
         dict(kind="conv", pattern="tile_edges", batch=2, in_hw=(40, 40), cin=256, cout=32, taps=TAPS1, relu=False),
         dict(kind="conv", pattern="dense", batch=2, in_hw=(15, 17), cin=128, cout=128, stride=2, resid=True),
         dict(kind="conv", pattern="sparse", batch=1, in_hw=(17, 40), cin=64, cout=256, stride=2),
         dict(kind="conv", pattern="tile_edges", batch=3, in_hw=(9, 7), cin=192, cout=40, stride=2, relu=False),
         dict(kind="conv", pattern="dense", batch=1, in_hw=(200, 176), cin=128, cout=256, stride=2),
         dict(kind="conv", pattern="dense", batch=2, in_hw=(8, 9), cin=64, cout=128, grid=(8, 9), out_hw=(17, 19), out_stride=2,
              out_off=(1, 0), resid=True),
         dict(kind="conv", pattern="sparse", batch=1, in_hw=(16, 24), cin=128, cout=40, grid=(12, 20), out_hw=(16, 24)),
         dict(kind="conv", pattern="dense", batch=3, in_hw=(9, 8), cin=64, cout=32, taps=[(0, 0), (1, -1), (-1, 1)], grid=(9, 7),
              out_hw=(12, 9), out_off=(2, 1)),
         dict(kind="deconv", pattern="dense", batch=1, in_hw=(7, 9), cin=128, cout=128, resid=True),
         dict(kind="deconv", pattern="sparse", batch=2, in_hw=(13, 17), cin=256, cout=128),
         dict(kind="deconv", pattern="tile_edges", batch=3, in_hw=(9, 40), cin=64, cout=40, relu=False),
         dict(kind="deconv", pattern="zero", batch=1, in_hw=(8, 16), cin=192, cout=24, resid=True),
         dict(kind="deconv", pattern="dense", batch=1, in_hw=(17, 40), cin=128, cout=136, resid=True),
         dict(kind="deconv", pattern="dense", batch=1, in_hw=(100, 88), cin=256, cout=128, resid=True),
         dict(kind="deconv", pattern="sparse", batch=2, in_hw=(1, 15), cin=64, cout=8, relu=False),
         # ring coverage (module docstring): 3 items per CTA of 4 steps on the 11-stage ring, 7 items of 18 steps on the 7-stage ring
         dict(kind="conv", pattern="dense", batch=4, in_hw=(96, 96), cin=64, cout=128, taps=[(0, 0), (0, 1)], resid=True),
         dict(kind="conv", pattern="dense", batch=4, in_hw=(160, 160), cin=64, cout=256, cout_pad=512, stride=2)]
    for i, d in enumerate(s):
        d.setdefault("seed", 500 + i)
        d.setdefault("shift", i % 3 != 2)
    return s


def _case(spec, **kw):
    d = dict(spec)
    d.update(kw)
    return BevCase(d.pop("kind"), d.pop("pattern"), d.pop("batch"), d.pop("in_hw"), d.pop("cin"), d.pop("cout"), d.pop("seed"), **d)


def _lab_specs():
    """(mode, spec) subset for the lab's h2 mode, incl. its shrunk-ring / single-patch-buffer configurations"""
    sp = _p2_specs()
    return [("h2", sp[1]), ("h2", sp[3]), ("h2", dict(sp[13], cout=32)), ("h2", sp[18]), ("h2", sp[21])]


P2_RINGS = (7, 11, 12)          # the weight rings the planes launches build: stride-2 3x3 convs, 3x3 convs and deconvs, the rest


def _sweep_plans():
    """(mode, kind, stride, plan) of every launch of the sweep and the lab subset"""
    out = []
    for mode, s in [("p2", s) for s in _p2_specs()] + _lab_specs():
        c = _case(s)
        out.append((mode, c.kind, c.stride, c.plan(mode)))
        assert out[-1][3] is not None, c.label()
    return out


def _ring_coverage(plans, num_sms):
    """{bstages: (stage, phase) starts} of the planes launches among plans; asserts that every launch starts only at reachable positions"""
    seen = {}
    for mode, _, _, p in plans:
        starts = ring_starts(p, num_sms)
        assert starts <= reachable_starts(p["bstages"]), (mode, p)
        if mode == "p2":
            seen.setdefault(p["bstages"], set()).update(starts)
    assert sorted(seen) == list(P2_RINGS)
    return seen


def test_schedule_reaches_every_ring_position_and_both_patch_paths():
    """The sweep's planes launches (restated launcher arithmetic) start work items at every reachable position of each weight ring they
    build (7, 11 and 12 stages); the sweep runs one and two patch buffers and both tile orientations of conv, stride-2 conv and deconv."""
    plans = _sweep_plans()
    seen = _ring_coverage(plans, NUM_SMS)
    for bstages in P2_RINGS:
        assert seen[bstages] == reachable_starts(bstages), (bstages, sorted(reachable_starts(bstages) - seen[bstages]))
    assert {p["npatch"] for _, _, _, p in plans} == {1, 2}
    orient = {(kind, stride, p["u_is_x"]) for _, kind, stride, p in plans}
    assert {(k, s, u) for k in ("conv",) for s in (1, 2) for u in (0, 1)} | {("deconv", 1, 0), ("deconv", 1, 1)} <= orient


def test_orientation_rule_examples():
    """u_is_x of the maps in the sweep, restated by hand: the production 200x176 map runs u = y, 100x88 u = x"""
    for hw, want in (((200, 176), 0), ((100, 88), 1), ((13, 17), 1), ((40, 9), 0), ((17, 40), 0), ((40, 17), 1), ((1, 1), 1)):
        assert orientation(*hw) == want, hw


def test_launcher_limits_restated():
    """The refusals the GPU test expects, from the launcher's arithmetic: > 6 patch copies, > 18 patch rows, cin % 64, cout % 8, and a
    stride-2 3x3 h2 conv with n_tile 128 (6 copies x 17 rows: 104 KB of planes + 104 KB of fp32 staging leave one 16 KB weight stage)
    -- while n_tile 32 (4 KB stages) still fits five."""
    cls = lambda taps: [[(dy, dx, t) for t, (dy, dx) in enumerate(taps)]]      # noqa: E731
    assert p2_plan("p2", 64, 64, 128, cls([(0, dx) for dx in range(-3, 4)]), 1, 16, 16, 1) is None                  # 7 copies
    assert p2_plan("p2", 64, 64, 128, cls([(0, dx) for dx in range(-3, 3)]), 1, 16, 16, 1, smem_a=True)["ncopies"] == 6
    assert p2_plan("p2", 64, 64, 128, cls([(0, dx) for dx in range(-3, 3)]), 1, 16, 16, 1)["ncopies"] == 1
    assert p2_plan("p2", 64, 64, 128, cls([(dy, 0) for dy in (-2, 0, 1)]), 1, 16, 16, 1) is None                    # 19 rows
    assert p2_plan("p2", 64, 64, 128, cls([(dy, 0) for dy in (-1, 0, 1)]), 1, 16, 16, 1)["rows_v"] == 18
    assert p2_plan("p2", 96, 64, 128, cls(TAPS3), 1, 16, 16, 1) is None
    assert p2_plan("p2", 64, 44, 128, cls(TAPS3), 1, 16, 16, 1) is None
    assert p2_plan("h2", 128, 128, 128, cls(TAPS3), 2, 16, 16, 1) is None
    p = p2_plan("h2", 128, 32, 32, cls(TAPS3), 2, 16, 16, 1)
    assert (p["npatch"], p["bstages"], p["ncopies"], p["rows_v"]) == (1, 5, 6, 17)
    assert p2_plan("p2", 128, 128, 128, cls(TAPS3), 2, 16, 16, 1)["npatch"] == 1
    assert p2_plan("p2", 128, 128, 128, cls(TAPS3), 1, 16, 16, 1)["npatch"] == 2


PLAN_WORDS = ("u_is_x", "n_tile", "nblocks", "tiles", "total", "ncopies", "rows_v", "pitch_u", "npatch", "bstages", "smem")


def launcher_plan(case, mode, smem_a=False):
    """the launcher's own plan of a case (sessd_bev_p2_plan: lab library, no device call) in p2_plan's terms, or None where it refuses"""
    from sessd_b200 import _lib, ops
    d = case.desc() if case.kind == "conv" else ops.conv_desc(case.batch, case.in_hw, case.cin, case.out_hw, case.cout, case.grid, [])
    rec = (C.c_int * 19)()
    if _lib.lib.sessd_bev_p2_plan(C.byref(d), int(case.kind == "deconv"), case.cout_pad, int(mode == "h2"), int(smem_a), rec) != 0:
        return None
    n = len(case.classes)
    assert list(rec[11 + n:15]) == [0] * (4 - n) and list(rec[15 + n:]) == [0] * (4 - n)
    return dict(zip(PLAN_WORDS, rec[:11]), ntaps=list(rec[11:11 + n]), order=list(rec[15:15 + n]))


def test_plan_restatement_matches_the_launcher():
    """p2_plan field by field against the launcher's plan for every sweep and lab launch (the sweep's stride-1 convs also as the loads
    probe's descriptor plan), and for the refusals of test_launcher_limits_restated and the launches next to them"""
    sweep = [_case(s) for s in _p2_specs()]
    runs = [("p2", c, False) for c in sweep] + [(m, _case(s), False) for m, s in _lab_specs()]
    runs += [("p2", c, True) for c in sweep if c.kind == "conv" and c.stride == 1]
    for mode, cin, cout, cout_pad, taps, stride in (("p2", 64, 64, 128, [(0, dx) for dx in range(-3, 4)], 1),       # 7 copies
                                                    ("p2", 64, 64, 128, [(0, dx) for dx in range(-3, 3)], 1),
                                                    ("p2", 64, 64, 128, [(-2, 0), (0, 0), (1, 0)], 1),              # 19 rows
                                                    ("p2", 64, 64, 128, [(-1, 0), (0, 0), (1, 0)], 1),
                                                    ("p2", 96, 64, 128, TAPS3, 1), ("p2", 64, 44, 128, TAPS3, 1),
                                                    ("h2", 128, 128, 128, TAPS3, 2), ("h2", 128, 32, 32, TAPS3, 2),
                                                    ("p2", 128, 128, 128, TAPS3, 2), ("p2", 128, 128, 128, TAPS3, 1)):
        runs.append((mode, BevCase("conv", "zero", 1, (16 * stride, 16 * stride), cin, cout, 0, taps=taps, stride=stride, cout_pad=cout_pad),
                     False))
    refused = 0
    for mode, c, smem_a in runs:
        want = p2_plan(mode, c.cin, c.cout, c.cout_pad, c.classes, c.stride, c.grid[0], c.grid[1], c.batch, smem_a)
        got = launcher_plan(c, mode, smem_a)
        refused += got is None
        if want is not None:
            want = {k: want[k] for k in PLAN_WORDS + ("ntaps", "order")}
        assert got == want, (mode, c.label(), smem_a)
    assert refused == 5


def test_crafted_maps_have_their_shape():
    x = crafted_map("sparse", 2, 200, 176, 8, 1)
    occ = (x != 0).any(3)
    assert 0.02 < occ.mean() < 0.08
    assert (x[~occ] == 0).all()
    d = crafted_map("dense", 1, 40, 40, 16, 2)
    m = np.abs(d).max(3)
    assert m.min() < 2.0 ** -10 and m.max() > 0.5
    e = crafted_map("tile_edges", 1, 33, 40, 16, 3)
    assert np.abs(e[0, 1:7, 1:7]).max() < 2.0 ** -7 and np.abs(e[0, 7]).min() == 0 or np.abs(e[0, 7]).max() > 0.5
    assert not crafted_map("zero", 1, 3, 3, 4, 0).any()


def test_split_restatements():
    for b, want in ((1.0, 2.0 ** 14), (2.0 ** 14, 1.0), (0.0, 1.0), (np.inf, 1.0), (2.0 ** -126, 2.0 ** 125), (1e-40, 1.0), (1e30, 2.0 ** -85)):
        assert pow2_scale_for_bound(b) == want, b


def _control_cases():
    """CPU-sized crafted cases for the negative controls: ReLU off so that no error can hide below zero"""
    return [BevCase("conv", "dense", 1, (20, 24), 64, 40, 1, relu=False, resid=True),
            BevCase("conv", "sparse", 2, (40, 18), 64, 40, 2, relu=False),
            BevCase("conv", "tile_edges", 1, (18, 33), 64, 24, 3, relu=False),
            BevCase("deconv", "dense", 1, (9, 11), 64, 40, 4, relu=False, resid=True),
            BevCase("deconv", "tile_edges", 1, (17, 9), 64, 24, 5, relu=False)]


def test_split_bounds_hold_for_the_exact_emulation():
    """Positive controls of the derivations: the fp64 emulation (a kernel without accumulation error) is within the split's own error of
    fp64 for the planes split, and the fp16 (hi, lo) epilogue restated in numpy meets the planes bound."""
    for case in _control_cases():
        emu = Emu(case, "cpu")
        assert ratio(emu.emul0, emu.ref, emu.tol_64 - emu.tol_e) <= 0.5, case.label()
        o = emu.emul0.numpy().astype(np.float32)
        s, bound = output_scale(emu.amax_in, case.gain, case.shift_max, case.amax_r if case.r is not None else None)
        hi, lo = split16(o, s)
        assert planes_ratio(hi, lo, s, bound, o) <= 0.5
        assert np.abs(hi.astype(np.float64)).max() <= HI_LIMIT


def test_negative_controls_are_flagged():
    """Each check flags each subtly wrong kernel on every control case it applies to (ratio of error to bound > 1).  The smallest ratios
    are printed."""
    least = {}

    def note(key, r):
        assert r > 1, (key, r)
        least[key] = min(least.get(key, np.inf), r)
    for case in _control_cases():
        emu = Emu(case, "cpu")
        em, ref = emu.emul0, emu.ref
        assert ratio(em, em, emu.tol_e) == 0
        wrongs = {"no_cross": emu.wrong_no_cross(), "swapped_taps": emu.wrong_swapped_taps()}
        if case.kind == "conv":
            wrongs["neighbour_tile_tap"] = emu.wrong_neighbour_tile_tap()
            wrongs["carried_accumulator"] = emu.wrong_carried_accumulator()
        else:
            wrongs["deconv_class_offset"] = emu.wrong_deconv_class_offset()
        for name, wrong in wrongs.items():
            note((name, "vs_emul"), ratio(wrong, em, emu.tol_e))
            note((name, "vs_fp64"), ratio(wrong, ref, emu.tol_64))
        o = em.numpy().astype(np.float32)
        amax_r = case.amax_r if case.r is not None else None
        s, bound = output_scale(emu.amax_in, case.gain, case.shift_max, amax_r)
        hi, lo = split16(o, s)
        note(("lo_plane_dropped", "planes"), planes_ratio(hi, np.zeros_like(lo), s, bound, o))
    # the residual's share of the bound left out of the output scale: a residual 1.5x the conv's bound (hi stays finite)
    case = BevCase("conv", "dense", 1, (16, 16), 64, 32, 6, relu=True, resid=True)
    emu = Emu(case, "cpu")
    s0, b0 = output_scale(emu.amax_in, case.gain, case.shift_max)
    case.r = (case.r / np.abs(case.r).max() * 1.5 * b0).astype(np.float32)
    o = emu.emul().numpy().astype(np.float32)
    hi, _ = split16(o, s0)
    note(("resid_left_out_of_bound", "hi_limit"), float(np.abs(hi.astype(np.float64)).max()) / HI_LIMIT)
    for key, r in sorted(least.items()):
        print("[control] %s / %s: smallest ratio %.3g" % (key[0], key[1], r))


# ================================================================================================================== GPU section
gpu = pytest.mark.gpu


def _dev(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).cuda()


def _is_sentinel(t):
    return t.view(torch.int16) == F16_SENTINEL if t.dtype == torch.float16 else t == F32_SENTINEL


def _guarded(shape, dtype):
    """(buffer, view): the view of `shape` inside a buffer with GUARD sentinel elements before and after it (everything sentinel)"""
    n = int(np.prod(shape))
    buf = torch.empty(n + 2 * GUARD, dtype=dtype, device="cuda")
    if dtype == torch.float16:
        buf.view(torch.int16).fill_(F16_SENTINEL)
    else:
        buf.fill_(F32_SENTINEL)
    return buf, buf[GUARD:GUARD + n].view(shape)


def _guards_intact(buf):
    return bool(_is_sentinel(buf[:GUARD]).all() and _is_sentinel(buf[-GUARD:]).all())


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.float16 else torch.int32)


def _report(worst, label):
    for k, r in sorted(worst.items()):
        print("[ratio] %s %s: %.3g" % (label, k, r))
        assert r <= 1.0, (label, k, r)


def _on_grid(t, case):
    _, oys, oxs = case.owned()
    return t[:, torch.as_tensor(oys, device=t.device)][:, :, torch.as_tensor(oxs, device=t.device)]


def _check_common(case, emu, bufs, got, worst):
    """guards, pixels the launch does not own, element-wise bounds vs the emulation and fp64, exact outputs of empty receptive fields"""
    owned = torch.as_tensor(case.owned()[0], device="cuda")
    for buf, view in bufs:
        assert _guards_intact(buf), case.label()
        assert bool(_is_sentinel(view[..., ~owned, :]).all()), case.label()
    worst["vs_emul"] = max(worst.get("vs_emul", 0), ratio(got, emu.emul0, emu.tol_e))
    worst["vs_fp64"] = max(worst.get("vs_fp64", 0), ratio(got, emu.ref, emu.tol_64))
    assert worst["vs_emul"] <= 1 and worst["vs_fp64"] <= 1, (case.label(), worst)
    mask, val = emu.exact_zero_field()
    g = got.cpu().numpy()
    assert np.array_equal(g[mask], val[mask]), case.label()


def _check_p2(case, worst):
    """bev_conv_p2 / bev_deconv_p2 on one case: fp32-only (twice), planes-only and both-output launches; returns (fp32 on the grid,
    planes view of the both-output launch, out_info, S_out, bound)"""
    from sessd_b200 import ops
    xd = _dev(case.x)
    amax_in = float(np.abs(case.x).max())
    info_in = torch.tensor([amax_in, 0.0], device="cuda")
    planes_in = torch.empty((2,) + case.x.shape, dtype=torch.float16, device="cuda")
    ops.bev_split_planes(xd, info_in, planes_in)
    torch.cuda.synchronize()
    s_in = pow2_scale_for_bound(amax_in)
    a_hi, a_lo = planes_in[0].cpu().numpy(), planes_in[1].cpu().numpy()
    rh, rl = split16(case.x, s_in)
    assert float(info_in[1]) == s_in and np.array_equal(a_hi.view(np.int16), rh.view(np.int16)) and np.array_equal(a_lo.view(np.int16), rl.view(np.int16))
    emu = Emu(case, "cuda", (a_hi, a_lo))
    gain, shift_max = case.gain, case.shift_max
    w, sc = emu.w_h2.cuda(), _dev(emu.sc32)
    sh = None if case.sh is None else _dev(case.sh)
    rd = None if case.r is None else _dev(case.r)
    rinfo = None if case.r is None else torch.tensor([case.amax_r, 0.0], device="cuda")
    oshape = (case.batch,) + case.out_hw + (case.cout,)

    def launch(outputs):
        fb, fv = _guarded(oshape, torch.float32) if outputs != "planes" else (None, None)
        pb, pv = _guarded((2,) + oshape, torch.float16) if outputs != "f32" else (None, None)
        oinfo = torch.zeros(2, device="cuda")
        if case.kind == "conv":
            ops.bev_conv_p2(planes_in, info_in, w, sc, sh, rd, rinfo, gain, shift_max, fv, pv, oinfo, case.desc())
        else:
            ops.bev_deconv_p2(planes_in, info_in, w, sc, sh, rd, rinfo, gain, shift_max, fv, pv, oinfo, case.relu)
        return fb, fv, pb, pv, oinfo
    runs = [launch(o) for o in ("f32", "f32", "planes", "both")]
    torch.cuda.synchronize()
    (fb1, fv1, _, _, i1), (fb2, fv2, _, _, i2), (_, _, pb3, pv3, i3), (fb4, fv4, pb4, pv4, i4) = runs
    assert torch.equal(_bits(fv1), _bits(fv2)) and torch.equal(_bits(fv1), _bits(fv4)), case.label()
    assert torch.equal(_bits(pv3), _bits(pv4)), case.label()
    assert torch.equal(i1, i2) and torch.equal(i1, i3) and torch.equal(i1, i4), case.label()
    got = _on_grid(fv1, case)
    _check_common(case, emu, [(fb1, fv1), (fb2, fv2), (pb3, pv3[0]), (pb3, pv3[1]), (fb4, fv4), (pb4, pv4[0]), (pb4, pv4[1])], got, worst)
    s_out, bound = output_scale(amax_in, gain, shift_max, case.amax_r if case.r is not None else None)
    assert float(i1[1]) == s_out and float(i1[0]) == float(got.abs().max()), (case.label(), i1.tolist(), s_out)
    hi, lo = _on_grid(pv4[0], case).cpu().numpy(), _on_grid(pv4[1], case).cpu().numpy()
    worst["planes"] = max(worst.get("planes", 0), planes_ratio(hi, lo, s_out, bound, got.cpu().numpy()))
    assert worst["planes"] <= 1, (case.label(), worst)
    assert np.isfinite(hi).all() and np.abs(hi.astype(np.float64)).max() <= HI_LIMIT, case.label()
    return got, hi, i1, s_out, bound


_P2 = _p2_specs()


@gpu
@pytest.mark.parametrize("spec", _P2, ids=[_case(s).label() for s in _P2])
def test_p2_kernels_match_emulation_and_fp64(spec):
    """bev_conv_p2 / bev_deconv_p2 on the geometry sweep: fp32 within the accumulation bound of the fp64 emulation and within that plus
    the split's error of fp64, exact where no product reaches the output, planes within 2^-22 bound with |hi| <= 2^15, out_info
    restated bit for bit, launches bitwise equal run to run and across output kinds, guards and unowned pixels untouched"""
    case = _case(spec)
    worst = {}
    _check_p2(case, worst)
    _report(worst, case.label())


@gpu
def test_p2_sweep_schedule_on_this_device():
    """the ring-position coverage of the CPU schedule test, recomputed with this device's SM count (the launcher's grid size)"""
    num_sms = torch.cuda.get_device_properties(0).multi_processor_count
    seen = _ring_coverage(_sweep_plans(), num_sms)
    for bstages in P2_RINGS:
        assert seen[bstages] == reachable_starts(bstages), (num_sms, bstages, sorted(reachable_starts(bstages) - seen[bstages]))


@gpu
@pytest.mark.parametrize("kind,resid", [("conv", False), ("conv", True), ("deconv", True)])
def test_p2_output_reaches_the_bound(kind, resid):
    """an interior output pixel driven to the output bound: x = amax sign(w bn) over its receptive field for the max-gain channel n*, the
    largest shift on n*, and (resid) a residual of +amax_resid there; the conv output comes within 3 % of the bound, the planes stay
    finite with |hi| <= 2^15"""
    case = BevCase(kind, "dense", 1, (16, 16), 64, 128, 77, relu=True, resid=resid)
    amax = 1.0
    gains = (np.abs(case.w.astype(np.float64)).sum((0, 1)) * np.abs(case.bn))
    n = int(np.argmax(gains))
    case.sh[n] = np.float32(np.abs(case.sh).max() + 0.5)
    sgn = np.sign(case.w[:, :, n] * case.bn[n]).astype(np.float32)                # [taps][Cin]
    case.x *= np.float32(0.5 / np.abs(case.x).max())
    if kind == "conv":
        y, x = 8, 8
        for t, (dy, dx) in enumerate(case.taps):
            case.x[0, y + dy, x + dx] = amax * sgn[t]
        oy, ox = y, x
    else:
        # output (2y + 1, 2x + 1) is class (1, 1): taps (dy, ky) in {(1, 0), (0, 2)} x (dx, kx) in {(1, 0), (0, 2)}; the deconv's
        # bound counts all nine taps, so only the reachable maximum of those four is checked
        y, x = 7, 7
        for dy, ky in ((1, 0), (0, 2)):
            for dx, kx in ((1, 0), (0, 2)):
                case.x[0, y + dy, x + dx] = amax * sgn[ky * 3 + kx]
        oy, ox = 2 * y + 1, 2 * x + 1
        gains = np.abs(case.w[[0, 2, 6, 8]].astype(np.float64)).sum((0, 1)) * np.abs(case.bn)
        assert gains[n] < 0.7 * case.gain          # the deconv's bound counts all nine taps: only four reach one output
    if resid:
        case.r[0, oy, ox, n] = np.float32(8 * np.abs(case.r).max())
    worst = {}
    got, hi, _, s_out, bound = _check_p2(case, worst)
    v = abs(float(got[0, oy, ox, n]))
    if kind == "conv":
        assert v >= 0.97 * bound, (v, bound)
    else:
        reach = amax * gains[n] + case.sh[n] + (case.r[0, oy, ox, n] if resid else 0.0)
        assert v >= 0.97 * reach, (v, reach)
    _report(worst, "bound-%s%s" % (kind, "-resid" if resid else ""))


@gpu
@pytest.mark.parametrize("kind,amax,resid_scale", [("conv", 1e-7, None), ("conv", 1e7, None), ("conv", 1e-7, 1.0), ("conv", 1e7, 1e9),
                                                   ("deconv", 1e-7, 1.0), ("deconv", 1e7, None)])
def test_p2_extreme_scales(kind, amax, resid_scale):
    """planes inputs with abs-max 1e-7 and 1e7, and residuals that dominate the output bound"""
    case = BevCase(kind, "dense", 2, (9, 17), 128, 40, 31, amax=amax, resid=resid_scale is not None, resid_scale=resid_scale or 1.0,
                   relu=kind == "deconv")
    worst = {}
    _check_p2(case, worst)
    _report(worst, "extreme-%s-%g-%s" % (kind, amax, resid_scale))


@gpu
def test_p2_zero_map_is_exact():
    """an all-zero map (an empty frame): zero input planes at S_in = 1, the output exactly relu(sh) (0 without a shift), out_info
    {max |relu(sh)|, S of the bound shift_max} (S = 1 when the bound is 0)"""
    from sessd_b200 import ops
    for shift in (False, True):
        case = BevCase("conv", "zero", 1, (20, 24), 64, 40, 3, shift=shift)
        worst = {}
        got, hi, info, s_out, bound = _check_p2(case, worst)
        want = np.maximum(case.shv, 0).astype(np.float32)
        assert np.array_equal(got.cpu().numpy(), np.broadcast_to(want, got.shape))
        assert float(info[0]) == float(want.max()) and float(info[1]) == (1.0 if not shift else pow2_scale_for_bound(case.shift_max))
        if not shift:
            assert bound == 0.0 and s_out == 1.0 and not hi.any()
        planes, pinfo = torch.empty((2, 5, 8), dtype=torch.float16, device="cuda"), torch.zeros(2, device="cuda")
        ops.bev_split_planes(torch.zeros((5, 8), device="cuda"), pinfo, planes)
        torch.cuda.synchronize()
        assert float(pinfo[1]) == 1.0 and not _bits(planes).any()


@gpu
def test_p2_refuses_launches_beyond_its_limits():
    """descriptors the launcher cannot run return an error (ops.check raises) without a launch and leave the output alone; the expected
    refusals are those of p2_plan (test_launcher_limits_restated): > 6 patch copies, > 18 patch rows, > 9 taps, cin % 64, cout % 8, and
    the stride-2 3x3 h2 conv at n_tile 128 (its fp32 staging leaves room for one weight stage); and a skip-plan item list with weights
    wider than round_up(cout, n_tile), whose item numbers would decode to other classes / n-blocks (conv and deconv)"""
    from sessd_b200 import _lib, ops
    bad = [dict(taps=[(0, dx) for dx in range(-3, 4)]), dict(taps=[(-2, 0), (0, 0), (1, 0)]), dict(taps=TAPS3 + [(2, 2)]),
           dict(cin=96), dict(cout=44, cout_pad=128), dict(cout_pad=256, items=True)]
    for kw in bad:
        cin, cout = kw.get("cin", 64), kw.get("cout", 64)
        taps = kw.get("taps", TAPS3)
        case = BevCase("conv", "dense", 1, (16, 16), 64, 64, 9)
        planes = torch.zeros((2, 1, 16, 16, cin), dtype=torch.float16, device="cuda")
        info = torch.tensor([1.0, 2.0 ** 14], device="cuda")
        w = torch.zeros((2, len(taps), kw.get("cout_pad", 128), cin), dtype=torch.float16, device="cuda")
        sc = torch.ones(kw.get("cout_pad", 128), device="cuda")
        buf, out = _guarded((1, 16, 16, cout), torch.float32)
        items = torch.zeros(64, dtype=torch.int32, device="cuda") if kw.get("items") else None
        if len(taps) <= 9:      # beyond the geometry's limits, or (with items) a geometry that runs without the item list
            assert (p2_plan("p2", cin, cout, kw.get("cout_pad", 128), [[(dy, dx, t) for t, (dy, dx) in enumerate(taps)]], 1, 16, 16, 1)
                    is None) == (items is None)
        d = ops.conv_desc(1, (16, 16), cin, (16, 16), cout, (16, 16), taps)
        n0 = _lib.launch_count()
        with pytest.raises(_lib.SessdError):
            ops.bev_conv_p2(planes, info, w, sc, None, None, None, 1.0, 0.0, out, None, torch.zeros(2, device="cuda"), d, items=items)
        if items is not None:
            dbuf, dout = _guarded((1, 32, 32, cout), torch.float32)
            with pytest.raises(_lib.SessdError):
                ops.bev_deconv_p2(planes, info, w, sc, None, None, None, 1.0, 0.0, dout, None, torch.zeros(2, device="cuda"), items=items)
            assert bool(_is_sentinel(dbuf).all())
        torch.cuda.synchronize()
        assert _lib.launch_count() == n0 and bool(_is_sentinel(buf).all()), kw
        del case
    x = torch.zeros((1, 16, 16, 128), device="cuda")
    for cout, ok in ((128, False), (32, True)):
        w, inv = ops.pack_weight_h2(torch.zeros((9, 128, cout), device="cuda"), 128 if cout > 32 else 32)
        buf, out = _guarded((1, 8, 8, cout), torch.float32)
        d = ops.conv_desc(1, (16, 16), 128, (8, 8), cout, (8, 8), TAPS3, in_stride=2)
        assert (p2_plan("h2", 128, cout, w.shape[2], [[(dy, dx, t) for t, (dy, dx) in enumerate(TAPS3)]], 2, 8, 8, 1) is not None) == ok
        if ok:
            ops.bev_conv_h2(x, w, inv[:cout].contiguous(), None, None, out, d, torch.zeros(1, device="cuda"), None)
            torch.cuda.synchronize()
            assert not out.any() and _guards_intact(buf)
        else:
            with pytest.raises(_lib.SessdError):
                ops.bev_conv_h2(x, w, inv[:cout].contiguous(), None, None, out, d, torch.zeros(1, device="cuda"), None)
            torch.cuda.synchronize()
            assert bool(_is_sentinel(buf).all())


_LAB = _lab_specs()


@gpu
@pytest.mark.parametrize("mode,spec", _LAB, ids=["%s-%s" % (m, _case(s).label()) for m, s in _LAB])
def test_lab_modes_match_emulation_and_fp64(mode, spec):
    """bev_conv_h2 / _deconv_h2 (fp16 split in the kernel) on a subset of the sweep, incl. the single-patch-buffer and shrunk-ring
    configurations: fp32 within the bounds of the split, exact on empty receptive fields, run to run bitwise, the running abs-max exact,
    guards and unowned pixels untouched"""
    from sessd_b200 import ops
    case = _case(spec)
    assert case.plan(mode) is not None
    emu = Emu(case, "cuda")
    xd = _dev(case.x)
    sh = None if case.sh is None else _dev(case.sh)
    rd = None if case.r is None else _dev(case.r)
    oshape = (case.batch,) + case.out_hw + (case.cout,)
    outs = []
    for _ in range(2):
        buf, out = _guarded(oshape, torch.float32)
        amax_out = torch.zeros(1, device="cuda")
        amax_in = torch.tensor([emu.amax_in], device="cuda")
        w, sc = emu.w_h2.cuda(), _dev(emu.sc32)
        if case.kind == "conv":
            ops.bev_conv_h2(xd, w, sc, sh, rd, out, case.desc(), amax_in, amax_out)
        else:
            ops.bev_deconv_h2(xd, w, sc, sh, rd, out, case.relu, amax_in, amax_out)
        outs.append((buf, out, amax_out))
    torch.cuda.synchronize()
    assert torch.equal(_bits(outs[0][1]), _bits(outs[1][1]))
    got = _on_grid(outs[0][1], case)
    worst = {}
    _check_common(case, emu, [(b, o) for b, o, _ in outs], got, worst)
    assert float(outs[0][2][0]) == float(got.abs().max())
    _report(worst, "%s %s" % (mode, case.label()))


# ------------------------------------------------------------------------------------------------------------------ plane producers
@gpu
def test_split_planes_bit_exact():
    """bev_split_planes: hi = fp16_rn(x S), lo = fp16_rn(x S - hi) with S = pow2_scale_for_bound(info[0]), bit for bit, info[1] = S; amax 0,
    subnormal, 2^-126, 1e30, inf and the data's own; n % 4 != 0 and n < 4 refused"""
    from sessd_b200 import _lib, ops
    base = (np.random.default_rng(4).standard_normal(4 * 301) * np.exp2(np.random.default_rng(5).uniform(-20, 0, 4 * 301))).astype(np.float32)
    base[:3] = [0.0, -0.0, 1.0]
    for amax in (0.0, 1e-40, 2.0 ** -126, 1e30, np.inf, float(np.abs(base).max()), 3.0):
        x = base if amax in (0.0, 1e-40, np.inf) else (base / np.abs(base).max() * np.float32(amax)).astype(np.float32)
        buf, planes = _guarded((2, x.size), torch.float16)
        info = torch.tensor([amax, -1.0], dtype=torch.float32, device="cuda")
        ops.bev_split_planes(_dev(x), info, planes)
        torch.cuda.synchronize()
        s = pow2_scale_for_bound(np.float32(amax))
        hi, lo = split16(x, s)
        assert float(info[1]) == s and float(info[0]) == float(np.float32(amax)), amax
        p = planes.cpu().numpy()
        assert np.array_equal(p[0].view(np.int16), hi.view(np.int16)) and np.array_equal(p[1].view(np.int16), lo.view(np.int16)), amax
        assert _guards_intact(buf)
    for n in (10, 3):
        with pytest.raises(_lib.SessdError):
            ops.bev_split_planes(torch.ones(n, device="cuda"), torch.ones(2, device="cuda"), torch.zeros((2, n), dtype=torch.float16, device="cuda"))


@gpu
def test_absmax_exact():
    """absmax: lengths 1-9 and 4k+1 .. 4k+3 with the maximum in the tail, at index 0, negative, or -0 only; a larger prior value stays
    (running max); n = 0 is a no-op; a pointer that is not 16-byte aligned is refused"""
    from sessd_b200 import _lib, ops
    rng = np.random.default_rng(6)
    store = torch.zeros(4 * 4000 + 16, device="cuda")
    for n in list(range(1, 10)) + [4 * 3999 + 1, 4 * 3999 + 2, 4 * 3999 + 3]:
        for where in ("tail", "first", "negative", "negzero"):
            for prior in (0.0, 100.0):
                x = (rng.standard_normal(n) * 0.1).astype(np.float32)
                if where == "tail":
                    x[-1] = 7.25
                elif where == "first":
                    x[0] = 7.25
                elif where == "negative":
                    x[rng.integers(0, n)] = -7.25
                else:
                    x[:] = -0.0
                store[:n] = _dev(x)
                amax = torch.tensor([prior], device="cuda")
                ops.absmax(store[:n], amax)
                torch.cuda.synchronize()
                want = max(prior, float(np.abs(x).max()))
                assert float(amax[0]) == want and not np.signbit(amax.cpu().numpy()[0]), (n, where, prior)
    amax = torch.tensor([2.5], device="cuda")
    # n = 0 through the C ABI: an empty tensor has no data pointer, a real one must still be left alone
    _lib.check(_lib.lib.sessd_absmax(C.c_void_p(store.data_ptr()), 0, C.c_void_p(amax.data_ptr()),
                                     C.c_void_p(torch.cuda.current_stream().cuda_stream)), "sessd_absmax")
    torch.cuda.synchronize()
    assert float(amax[0]) == 2.5
    with pytest.raises(_lib.SessdError):
        ops.absmax(store[1:9], amax)


@gpu
def test_sparse_to_dense_planes_bit_exact():
    """sparse_to_dense_planes == sparse_to_dense_indexed followed by the restated split, bit for bit, info = {amax, S}; the dense map
    itself placed from the bitmap index's row order; feature rows >= max_rows (the feature buffer's length) read as zero.  The bitmap
    index comes from a 1x1x1 strided rulebook of the crafted coordinates, as the encoder's last level builds it."""
    from sessd_b200 import ops
    rng = np.random.default_rng(8)
    b, d, h, w, c = 2, 2, 9, 13, 6
    cells = rng.choice(b * d * h * w, 70, replace=False)
    bb, rem = np.divmod(cells, d * h * w)
    zz, rem = np.divmod(rem, h * w)
    yy, xx = np.divmod(rem, w)
    coors = np.stack([bb, zz, yy, xx], 1).astype(np.int32)
    n, cap = len(coors), len(coors) + 10
    grid = ops.make_grid(b, (d, h, w))
    cd = torch.zeros((cap, 4), dtype=torch.int32, device="cuda")
    cd[:n] = _dev(coors, torch.int32)
    nd = torch.tensor([n], dtype=torch.int32, device="cuda")
    table = ops.hash_build(cd, nd, cap, grid)
    bitmap, scratch = ops.bitmap_alloc(grid, "cuda")
    out_coors, n_out = torch.zeros((cap, 4), dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    nbr, status = torch.empty((cap, 1), dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    ops.strided_rulebook(cd, nd, cap, grid, 0, table, (1, 1, 1), (1, 1, 1), (0, 0, 0), grid, bitmap, scratch, out_coors, n_out, cap, nbr, status)
    torch.cuda.synchronize()
    assert int(n_out[0]) == n and int(status[0]) == 0
    oc = out_coors[:n].cpu().numpy()
    assert sorted(map(tuple, oc)) == sorted(map(tuple, coors))
    for max_rows, scale in ((n, 1.0), (n - 9, 3e-6), (n - 1, 1e9)):
        feat = (rng.standard_normal((max_rows, c)) * scale).astype(np.float32)
        ref = np.zeros((b, h, w, c * d), np.float32)
        for i in range(max_rows):
            ref[oc[i, 0], oc[i, 2], oc[i, 3], np.arange(c) * d + oc[i, 1]] = feat[i]
        dense = ops.sparse_to_dense_indexed(_dev(feat), bitmap, grid, torch.full((b, h, w, c * d), F32_SENTINEL, device="cuda"))
        amax = torch.tensor([float(np.abs(feat).max())], device="cuda")
        info = torch.tensor([-1.0, -1.0], device="cuda")
        buf, planes = _guarded((2, b, h, w, c * d), torch.float16)
        ops.sparse_to_dense_planes(_dev(feat), bitmap, grid, amax, info, planes)
        torch.cuda.synchronize()
        dn = dense.cpu().numpy()
        assert np.array_equal(dn, ref), max_rows
        s = pow2_scale_for_bound(float(amax[0]))
        hi, lo = split16(dn, s)
        p = planes.cpu().numpy()
        assert np.array_equal(p[0].view(np.int16), hi.view(np.int16)) and np.array_equal(p[1].view(np.int16), lo.view(np.int16)), max_rows
        assert info.tolist() == [float(amax[0]), s] and _guards_intact(buf), max_rows


@gpu
@pytest.mark.parametrize("c", [4, 128, 132, 256])
@pytest.mark.parametrize("npix", [37, 1001])
def test_ssfa_fuse_planes_matches_fp64(c, npix):
    """ssfa_fuse_planes: the fp32 output within the module docstring's bound of the fp64 pair-softmax fusion, the planes the restated
    split of that fp32 output (both-output and planes-only launches alike), out_info = {max(amax0, amax1), S} exactly"""
    from sessd_b200 import ops
    rng = np.random.default_rng(c + npix)
    x0 = crafted_map("dense", 1, 1, npix, c, c).reshape(npix, c) * np.float32(3.0)
    x1 = crafted_map("sparse", 1, 1, npix, c, npix).reshape(npix, c)
    x1[::5] = (rng.standard_normal((len(x1[::5]), c)) * 2.0).astype(np.float32)
    w0, w1 = [(rng.standard_normal(c) / np.sqrt(c)).astype(np.float32) for _ in range(2)]
    s0, t0, s1, t1 = [float(np.float32(v)) for v in (1.7, -0.3, -2.2, 0.4)]
    a0, a1 = float(np.abs(x0).max()), float(np.abs(x1).max()) * 1.5
    info0, info1 = torch.tensor([a0, 0.0], device="cuda"), torch.tensor([a1, 0.0], device="cuda")
    fb, out = _guarded((npix, c), torch.float32)
    pb, planes = _guarded((2, npix, c), torch.float16)
    pb2, planes2 = _guarded((2, npix, c), torch.float16)
    oinfo, oinfo2 = torch.zeros(2, device="cuda"), torch.zeros(2, device="cuda")
    args = (_dev(x0), _dev(x1), _dev(w0), _dev(w1), s0, t0, s1, t1)
    ops.ssfa_fuse_planes(*args, out, info0, info1, oinfo, planes)
    ops.ssfa_fuse_planes(*args, None, info0, info1, oinfo2, planes2)
    torch.cuda.synchronize()
    X0, X1 = x0.astype(np.float64), x1.astype(np.float64)
    d0, d1 = X0 @ w0.astype(np.float64), X1 @ w1.astype(np.float64)
    l0, l1 = d0 * s0 + t0, d1 * s1 + t1
    p0 = 1.0 / (1.0 + np.exp(l1 - l0))
    ref = X0 * p0[:, None] + X1 * (1.0 - p0)[:, None]
    dd0, dd1 = [(c / 128 + 12) * U * (np.abs(X) @ np.abs(wk.astype(np.float64))) for X, wk in ((X0, w0), (X1, w1))]
    dl0 = abs(s0) * dd0 + U * (np.abs(s0 * d0) + abs(t0))
    dl1 = abs(s1) * dd1 + U * (np.abs(s1 * d1) + abs(t1))
    da = (dl0 + dl1) / 4 + 16 * U
    tol = (np.abs(X0) + np.abs(X1)) * (da + 2 * U)[:, None]
    got = out.cpu().numpy()
    r = ratio(got, ref, tol)
    print("[ratio] ssfa_fuse(%d, %d) vs_fp64: %.3g" % (c, npix, r))
    assert r <= 1, r
    s = pow2_scale_for_bound(np.float32(max(a0, a1)))
    hi, lo = split16(got, s)
    for p in (planes, planes2):
        pn = p.cpu().numpy()
        assert np.array_equal(pn[0].view(np.int16), hi.view(np.int16)) and np.array_equal(pn[1].view(np.int16), lo.view(np.int16))
    assert oinfo.tolist() == [float(np.float32(max(a0, a1))), s] and torch.equal(oinfo, oinfo2)
    assert _guards_intact(fb) and _guards_intact(pb) and _guards_intact(pb2)
