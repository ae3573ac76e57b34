"""spconv_forward_cg at the grid it launches: min(ceil(max_out / 128), blocks_per_sm x SMs) persistent CTAs, which carry their stage
ring and the producers' dirty-row masks (cg_ring_model) from tile to tile.

The tables here are built against that grid (cg_ring_model.carry_table, gap_table, edge_specs): every CTA runs three tiles or more,
rows a stage held for one tile are cleared by the CTA's next tile in every (stage, 32-row word), the even CTAs run busy, empty, busy
tiles, and the tile counts sit at the grid's edges.  Before a launch, the replay of the producers' bookkeeping asserts that the case
reaches what it is built for.  The outputs are then held to the bounds of test_gpu_spconv_ops (fp64 emulation, fp64, planes; the
derivations are in its module docstring), and to exact invariances: a tile computes the same bits whichever CTA and ring position
runs it, so tables permuted by whole tiles and one-tile launches must reproduce every tile's rows and planes bit for bit.

Negative controls (CPU): each staging fault of cg_ring_model -- dirty masks reset at each tile, the second warp of a two-warp group
never clearing its rows, a warp's two stages sharing one mask -- adds stale products on the carry and gap tables at grids 264, 132,
228 and 114, and each is flagged by both bounds.  Smallest ratio of error to bound over those cases (cg vs emulation bound / cg vs
fp64 bound): reset at tile 6.1e7 / 3.1e5, second warp never clears 8.1e7 / 3.7e5, no rotation 8.4e7 / 3.9e5.  On the GPU, a kernel
without the dirty-row clear and one that zeroes its dirty masks at the head of each tile each fail every carry, gap and permutation
test here, at all eight instantiations.
Largest ratios measured on an H100 (132 SMs: grids of 264 CTAs at deep 0, 132 at deep 1), over all cases and both depths: cg vs
emulation 0.49, cg vs fp64 0.073, planes 0.0049.  The GPU tests of this file take about 95 s there, most of it the fp64 references.
"""
import copy

import numpy as np
import pytest
import torch

from cg_ring_model import (BM, CG_SHAPES, CgLayout, carry_table, cg_grid, edge_specs, gap_table, grid_table, permute_tiles,
                           predicted_blocks_per_sm, replay, tile_permutation, tile_ring)
from test_gpu_spconv_ops import (Case, CgEmu, _check_cg, _dev, _n_dev, _run_cg, _bits, ratio, sp_cg_deep)  # noqa: F401 (fixture)

GRIDS = (264, 132, 228, 114)       # blocks_per_sm x SMs: default and deep pipeline on 132 SMs, then on 114
N_IN = 20000                       # input rows the crafted tables draw from
LAYOUTS = [(cp, deep) for cp in (32, 64) for deep in (0, 1)]        # the ring depends on (cp, deep) only
gpu = pytest.mark.gpu


def _rows_of(case, rows):
    """the case restricted to some of its output rows (same inputs, weights, scales): the bounds of those rows are unchanged"""
    sub = copy.copy(case)
    sub.nbr_c, sub.P = case.nbr_c[rows], case.P[rows]
    return sub


def _stale_ratios(case, cp, stale):
    """(cg vs emulation, cg vs fp64) ratios of what a kernel adding the stale products [(out_row, in_row, k)] computes, on the rows it
    changes (the other rows are the kernel as written)"""
    rows = np.unique(stale[:, 0])
    emu = CgEmu(_rows_of(case, rows), cp)
    acc = emu.acc()
    out = np.searchsorted(rows, stale[:, 0])
    src = np.searchsorted(case.in_rows, stale[:, 1])
    assert (case.in_rows[src] == stale[:, 1]).all()
    for k in np.unique(stale[:, 2]):
        m = stale[:, 2] == k
        np.add.at(acc, out[m], emu.A[src[m]] @ np.concatenate([emu.b_hi[k] + emu.b_lo[k], emu.b_hi[k]], 0))
    wrong = emu.emul(acc)
    return ratio(wrong, emu.emul(), emu.tol_emul()), ratio(wrong, emu.case.ref64(), emu.tol_fp64())


# ================================================================================================================== CPU section
def test_layout_restatement():
    """CgCfg's three producer layouts: Cp 64 default = 2 groups of 2 warps (64 rows each), Cp 32 default and Cp 64 deep = 4 groups of
    one warp with one stage, Cp 32 deep = 4 warps with 2 stages each; the default pipeline fits two CTAs in 228 KB, the deep one not"""
    want = {(32, 0): (4, 4, 1, 1), (64, 0): (2, 2, 2, 1), (64, 1): (4, 4, 1, 1), (32, 1): (8, 4, 1, 2)}
    for cp, cout in CG_SHAPES:
        for deep in (0, 1):
            lay = CgLayout(cp, cout, deep)
            assert (lay.stages, lay.groups, lay.group_warps, lay.group_stages) == want[(cp, deep)], lay
            assert lay.groups * lay.group_stages == lay.stages and lay.groups * lay.group_warps == 4
            assert predicted_blocks_per_sm(lay, 228 * 1024) == (1 if deep else 2), (lay, lay.smem)
            assert deep or lay.smem <= 113 * 1024


@pytest.mark.parametrize("grid", GRIDS)
def test_grid_tables_reach_their_targets(grid):
    """carry: >= 3 tiles per CTA, 1 - 4 pairs per row, every (nact, st0, ph0) and every clear slot (stage, 32-row word) within a tile
    and across consecutive tiles of a CTA; gap: busy, empty, busy on the even CTAs and a clear across the empty tile in every slot;
    the kernel as written multiplies no stale row; the edge tables have their tile counts and partial last tiles."""
    carry, gap = carry_table(grid, N_IN, grid), gap_table(grid, N_IN, grid + 1)
    ncarry = -(-len(carry) // BM)
    assert ncarry >= 3 * grid and len(carry) % BM
    p = (carry >= 0).sum(1)
    assert p.min() >= 1 and p.max() <= 4
    cta, rnd, _p, nact = tile_ring(gap, len(gap), grid)
    assert (nact[(rnd == 1) & (cta % 2 == 0)] == 0).all() and (nact[(rnd != 1) | (cta % 2 == 1)] > 0).all()
    for cp, deep in LAYOUTS:
        lay = CgLayout(cp, 32, deep)
        rc = replay(carry, len(carry), len(carry), grid, lay)
        assert not rc.missing_positions(lay.stages), (lay, rc.missing_positions(lay.stages)[:5])
        assert not rc.missing_clears(lay.stages), (lay, rc.missing_clears(lay.stages)[:5])
        rg = replay(gap, len(gap), len(gap), grid, lay)
        assert not rg.missing_gap_clears(lay.stages), (lay, rg.missing_gap_clears(lay.stages)[:5])
        assert len(rc.stale) == 0 and len(rg.stale) == 0
    for name, ntiles, last, max_out in edge_specs(grid):
        t = grid_table(grid, ntiles, last, N_IN, 7)
        assert len(t) == (ntiles - 1) * BM + last and 0 < last < BM and max_out >= len(t), name
    assert -(-edge_specs(grid)[-1][3] // BM) > grid >= 2 * edge_specs(grid)[-1][1]


def test_tile_permutations_move_tiles():
    """shuffle moves every tile to another CTA and round; rotate and reverse are permutations too"""
    for grid in GRIDS:
        full = 3 * grid
        for kind in ("reverse", "rotate", "shuffle"):
            perm = tile_permutation(kind, full, grid)
            assert sorted(perm) == list(range(full))
        perm = tile_permutation("shuffle", full, grid)
        new = np.arange(full)
        assert (new % grid != perm % grid).all() and (new // grid != perm // grid).all()


@pytest.mark.parametrize("grid", GRIDS)
def test_staging_faults_are_flagged(grid):
    """Each staging fault of cg_ring_model, on every layout that can have it, adds stale products on the carry and gap tables built
    against `grid`, and both checks flag it (ratio of error to bound > 1; ReLU off so that no error hides below zero).  The smallest
    ratios are printed."""
    least = {}
    for name, table in (("carry", carry_table(grid, N_IN, grid)), ("gap", gap_table(grid, N_IN, grid + 1))):
        for cp, deep in LAYOUTS:
            lay = CgLayout(cp, 32, deep)
            case = Case(name, len(table), 27, cp, 32, grid + cp + deep, n_in=N_IN, max_out=len(table) + 40, relu=False, live=table)
            for fault in lay.faults():
                stale = replay(case.nbr, case.n_dev, case.max_out, grid, lay, fault).stale
                assert len(stale), (name, lay, fault)
                for check, r in zip(("cg_vs_emul", "cg_vs_fp64"), _stale_ratios(case, cp, stale)):
                    assert r > 1, (name, lay, fault, check, r)
                    least[(fault, check)] = min(least.get((fault, check), np.inf), r)
    for key, r in sorted(least.items()):
        print("[control] grid %d %s / %s: smallest ratio %.3g" % (grid, key[0], key[1], r))


# ================================================================================================================== GPU section
def _device_grid(cp, cout, deep):
    return cg_grid(cp, cout, deep, 1 << 30)


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


@gpu
def test_layout_restatement_predicts_the_device_occupancy():
    """the shared memory of the restated CgCfg gives the CTAs per SM that spconv_cg_blocks_per_sm reports, for all eight instantiations"""
    from sessd_b200 import ops
    props = torch.cuda.get_device_properties(torch.cuda.current_device())
    for cp, cout in CG_SHAPES:
        for deep in (0, 1):
            lay = CgLayout(cp, cout, deep)
            got = ops.spconv_cg_blocks_per_sm(cp, cout, deep)
            print("[occupancy] cp %d cout %d deep %d: %d B of shared memory, %d CTAs per SM x %d SMs = grid %d" % (
                cp, cout, deep, lay.smem, got, props.multi_processor_count, got * props.multi_processor_count))
            assert lay.smem <= props.shared_memory_per_block_optin, lay
            assert predicted_blocks_per_sm(lay, props.shared_memory_per_multiprocessor) == got, (lay, lay.smem, got)


CASES = ("carry", "gap", "grid-1", "grid", "grid+1", "2grid+1", "exit")


def _grid_case(name, grid):
    """(table, max_out) of the named case built against the device grid"""
    if name in ("carry", "gap"):
        table = carry_table(grid, N_IN, grid) if name == "carry" else gap_table(grid, N_IN, grid + 1)
        return table, len(table) + 40
    i, (_name, ntiles, last, max_out) = [(i, e) for i, e in enumerate(edge_specs(grid)) if e[0] == name][0]
    return grid_table(grid, ntiles, last, N_IN, 50 + i), max_out


@gpu
@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("deep", [0, 1])
@pytest.mark.parametrize("cp,cout", CG_SHAPES, ids=["%d-%d" % s for s in CG_SHAPES])
def test_cg_at_the_launch_grid_matches_emulation_and_fp64(cp, cout, deep, name, sp_cg_deep):
    """The carry, gap and edge tables built against the (cp, cout, deep) grid of the device; the replay at the launch's grid must reach
    every (nact, st0, ph0) of the ring and every clear slot within and across tiles (carry) and a clear across an empty tile in every
    slot (gap), with no stale product.  Then _check_cg: deep 0 and 1 each run twice, fp32 rows vs the emulation and fp64 bounds, planes
    and out_info, sentinels, run to run and deep 0 vs deep 1 bitwise."""
    lay = CgLayout(cp, cout, deep)
    grid = _device_grid(cp, cout, deep)
    i = CASES.index(name)
    table, max_out = _grid_case(name, grid)
    launch = cg_grid(cp, cout, deep, max_out)
    rep = replay(table, len(table), max_out, launch, lay)
    assert len(rep.stale) == 0
    if name == "carry":
        assert launch == grid and not rep.missing_positions(lay.stages) and not rep.missing_clears(lay.stages)
    if name == "gap":
        assert launch == grid and not rep.missing_gap_clears(lay.stages)
    print("[grid] cp %d cout %d deep %d: %d SMs x %d CTAs = %d; %d stages, %d groups x %d warps" % (
        cp, cout, deep, _sms(), grid // _sms(), grid, lay.stages, lay.groups, lay.group_warps))
    print("[cover] %s: %d rows, %d tiles on %d CTAs, %d ring positions, %d clear slots (%s), %d across an empty tile" % (
        name, len(table), -(-len(table) // BM), launch, len(rep.positions), len(rep.clears),
        "/".join(sorted({kd for kd, _s, _w in rep.clears})), len(rep.gap_clears)))
    case = Case(name, len(table), 27, cp, cout, 7 * i + cp + cout + deep, n_in=N_IN, max_out=max_out, relu=i % 2 == 1,
                shift=i % 3 != 2, live=table)
    _check_cg(case, CgEmu(case, cp), N_IN + 1, "%s-%d-%d@%d" % (name, cp, cout, grid), sp_cg_deep, i % 3)


def _run_both(case, emu, planes_in, info_in, nbr, n, max_out):
    """fp32 rows and planes of one launch over the table nbr (n rows on the device, capacity max_out)"""
    from sessd_b200 import ops
    c = copy.copy(case)
    c.nbr, c.n_dev, c.n_eff, c.max_out = nbr, n, n, max_out
    tl = ops.rulebook_tile_lists(_dev(nbr[:max_out], torch.int32), _n_dev(c), max_out, ops.alloc_tile_lists(max_out, case.kvol, "cuda"))
    out, pl, _info = _run_cg(c, emu, planes_in, info_in, tl, "both", case.cout)
    return _bits(out[:n]).cpu().numpy(), _bits(pl[:n]).cpu().numpy()


@gpu
@pytest.mark.parametrize("deep", [0, 1])
@pytest.mark.parametrize("cp,cout", CG_SHAPES, ids=["%d-%d" % s for s in CG_SHAPES])
def test_cg_tiles_do_not_depend_on_cta_or_ring_position(cp, cout, deep, sp_cg_deep):
    """A tile's products and their order depend on its rows only, so every tile's fp32 rows and planes must be bitwise those of the
    unpermuted launch after the carry and gap tables are permuted by whole tiles (the partial last tile stays last), and after a sample
    of tiles runs alone in one-tile launches.  Every permutation moves every tile to another CTA; reversal and the shuffle (another
    round too) also move most tiles to another (st0, ph0), while rotation by one keeps most at theirs behind other predecessors.  Stale
    state carried from another tile shows here exactly, however small."""
    sp_cg_deep(deep)
    grid = _device_grid(cp, cout, deep)
    lay = CgLayout(cp, cout, deep)
    for name, table in (("carry", carry_table(grid, N_IN, grid)), ("gap", gap_table(grid, N_IN, grid + 1))):
        n = len(table)
        case = Case(name, n, 27, cp, cout, grid + cp + cout, n_in=N_IN, max_out=n, live=table)
        emu = CgEmu(case, cp)
        planes_in = torch.zeros((N_IN + 1, 2 * cp), dtype=torch.float16, device="cuda")
        planes_in[torch.from_numpy(case.in_rows).cuda()] = torch.from_numpy(np.concatenate([emu.a_hi, emu.a_lo], 1)).cuda()
        info_in = torch.tensor([emu.amax_in, emu.s_in], dtype=torch.float32, device="cuda")
        f32, pl = _run_both(case, emu, planes_in, info_in, case.nbr, n, n)
        full = n // BM
        _cta, _rnd, p0, _nact = tile_ring(case.nbr, n, grid)
        for kind in ("reverse", "rotate", "shuffle"):
            perm = tile_permutation(kind, full, grid)
            nbr = permute_tiles(case.nbr, n, perm)
            cta, _rnd, p, _nact = tile_ring(nbr, n, grid)
            moved_ring = int(((p[:full] % (2 * lay.stages)) != (p0[perm] % (2 * lay.stages))).sum())
            moved_cta = int((cta[:full] != perm % grid).sum())
            g32, gpl = _run_both(case, emu, planes_in, info_in, nbr, n, n)
            for got, want in ((g32, f32), (gpl, pl)):
                w = want[:full * BM].reshape(full, BM, -1)[perm].reshape(full * BM, -1)
                bad = np.nonzero((got[:full * BM] != w).any(1))[0]
                assert len(bad) == 0, (name, kind, "tiles", np.unique(perm[bad // BM])[:8])
                assert np.array_equal(got[full * BM:], want[full * BM:]), (name, kind, "partial tile")
            print("[perm] %s %s: %d of %d tiles on another CTA, %d at another (st0, ph0)" % (name, kind, moved_cta, full, moved_ring))
        sample = [0, 1, grid - 1, grid, 2 * grid + 1, 3 * grid - 1, full]         # the last one is the partial tile
        for t in sample:
            rows = min(BM, n - t * BM)
            g32, gpl = _run_both(case, emu, planes_in, info_in, case.nbr[t * BM:t * BM + rows], rows, rows)
            assert np.array_equal(g32, f32[t * BM:t * BM + rows]) and np.array_equal(gpl, pl[t * BM:t * BM + rows]), (name, t)
        print("[alone] %s: tiles %s run alone, bitwise equal" % (name, sample))


@gpu
def test_dgrad_64_32_runs_every_cta_three_tiles():
    """the data gradient of the 32 -> 64 strided layer (spconv_cg <64, 32>) through SparseConvFunction on a transposed table of
    3 grid + 1 tiles, so every CTA of the device grid runs three tiles or more, vs conv_backward_from_nbr at test_dgrad_matches_fp64's
    bound"""
    from test_gpu_spconv_grad import check_dgrad
    grid = _device_grid(64, 32, 0)
    n_in = 3 * grid * BM + 77
    print("[grid] dgrad <64,32>: %d input rows, %d tiles on %d CTAs" % (n_in, -(-n_in // BM), grid))
    check_dgrad("cg", 32, 64, False, n_in=n_in, n_out=n_in // 2)
