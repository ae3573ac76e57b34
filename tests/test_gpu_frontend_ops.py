"""The voxeliser and the rulebook builders one operator at a time (through sessd_b200.ops, no runner) on the crafted inputs of
tests/frontend_model.py, bit-exact against the oracles (oracle.cpu.points_to_voxel, oracle.spconv_ref) and the restatements:
hash collisions and wrapped probe runs, grid faces, every device-scan path and its thresholds, the 64-bit enumeration, generic
kernel shapes, the max_voxels cut, NaN / Inf points, 300-frame batches, refusals, and a strided level that overflows its
capacity (op level, then through SpMiddleRunner)."""
import numpy as np
import pytest
import torch

import frontend_model as fm
from oracle import spconv_ref as S

pytestmark = pytest.mark.gpu

PC_RANGE = fm.RANGE_MIN + (70.4, 40.0, 1.0)
SHAPE = (7, 9, 11)


def _i32(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.int32)).cuda()


def _n(v):
    return torch.tensor([int(v)], dtype=torch.int32, device="cuda")


def _np(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


# ------------------------------------------------------------------------------------------------------------ voxeliser
def _voxelize(clouds, mp, mv, nf=4, cap=None):
    from sessd_b200 import ops
    cfg = ops.make_voxel_cfg(fm.VOXEL_SIZE, PC_RANGE, mp, mv, nf)
    total = sum(len(c) for c in clouds)
    cap = cap or max(total, 1)
    pts = torch.zeros((cap, nf), dtype=torch.float32, device="cuda")
    if total:
        pts[:total] = torch.from_numpy(np.concatenate(clouds, 0)).cuda()
    off = np.zeros(len(clouds) + 1, np.int32)
    off[1:] = np.cumsum([len(c) for c in clouds])
    buf = ops.VoxelBuffers(cfg, len(clouds), cap, "cuda")
    ops.voxelize(pts, _i32(off), buf)
    nv = _np(buf.num_voxels)
    assert int(nv[-1]) == int(nv[:-1].sum())
    out, base = [], 0
    for f in range(len(clouds)):
        sl = slice(base, base + int(nv[f]))
        out.append(tuple(_np(t[sl]) for t in (buf.voxels, buf.coors, buf.num_points, buf.mean)))
        base += int(nv[f])
    return out


def _check_frames(clouds, got, mp, mv):
    from oracle import cpu as ocpu
    for f, (cloud, (v, c, n, mean)) in enumerate(zip(clouds, got)):
        clean = cloud[~np.isnan(cloud[:, :3]).any(1)]           # NaN points are dropped by the device; the C oracle cannot take them
        ov, oc, on = ocpu.points_to_voxel(clean, fm.VOXEL_SIZE, PC_RANGE, mp, mv)
        assert (c[:, 0] == f).all(), f
        assert np.array_equal(c[:, 1:], oc), f
        assert np.array_equal(n, on), f
        assert np.array_equal(v, ov, equal_nan=True), f
        assert np.array_equal(mean, fm.voxel_mean(ov, on), equal_nan=True), f


@pytest.mark.parametrize("mp,nf", [(1, 3), (5, 4), (7, 5), (5, 3), (7, 4), (1, 4)])
@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_voxelize_cut_payloads_and_mean(mp, nf, delta):
    """max_voxels - 1 / exactly / + 1 distinct cells in every frame (later points of open voxels after the cut), voxels of
    max_points +- 1 and 100 points, an empty frame in the middle, NaN / +-Inf coordinates; both gather kernels"""
    mv = 30
    clouds = [fm.cut_cloud(7 + f + delta, mv, delta, nf=nf, max_points=mp) for f in range(3)]
    clouds[1] = clouds[1][:0]
    clouds.append(fm.clouds_with_edges(4, nf)[0])
    clouds.append(fm.cut_cloud(50 + delta, mv, delta, nf=nf, max_points=mp))
    _check_frames(clouds, _voxelize(clouds, mp, mv, nf), mp, mv)


@pytest.mark.parametrize("cap", fm.WORD_THRESHOLDS)
def test_voxelize_scan_thresholds(cap):
    """point capacities on both sides of the one-CTA / self-prefix / three-launch scan thresholds, with 0, 1, 2047, 2048, 2049 and
    cap points, first points of voxels on the scan-tile boundaries"""
    for count in (0, 1, 2047, 2048, 2049, cap):
        cloud = fm.boundary_cloud(count)
        _check_frames([cloud], _voxelize([cloud], 5, 20000, cap=cap), 5, 20000)


def test_voxelize_300_frames():
    """more frames than one pass of the shared-memory frame-offset loads (256 threads); frames share cells, several are empty"""
    rng = np.random.default_rng(0)
    base = fm.cell_points(fm.random_cells(rng, 20), 0)
    clouds = [base[: (f % 7) * 3] for f in range(300)]
    clouds[150] = fm.cut_cloud(3, 10, 1)
    _check_frames(clouds, _voxelize(clouds, 5, 10), 5, 10)


def test_voxelize_refuses_keys_past_40_bits():
    """batch * cells >= 2^40 would alias the hash keys: refused before any launch, outputs untouched; one frame less is accepted"""
    from sessd_b200 import _lib, ops
    cfg = ops.make_voxel_cfg(fm.VOXEL_SIZE, PC_RANGE, 5, 16)
    cfg.grid[0], cfg.grid[1], cfg.grid[2] = 1 << 14, 1 << 13, 1 << 10            # 2^37 cells
    pts = torch.from_numpy(fm.cell_points(fm.random_cells(np.random.default_rng(0), 8), 0)).cuda()
    for batch, ok in ((8, False), (7, True)):
        off = _i32(np.r_[0, np.full(batch, 8)])                                    # all points in frame 0
        buf = ops.VoxelBuffers(cfg, batch, 8, "cuda")
        buf.num_voxels.fill_(-7)
        buf.coors.fill_(-7)
        torch.cuda.synchronize()
        before = _lib.launch_count()
        if ok:
            ops.voxelize(pts, off, buf)
            assert int(_np(buf.num_voxels)[-1]) == 8
        else:
            with pytest.raises(_lib.SessdError, match="capacity exceeded"):
                ops.voxelize(pts, off, buf)
            assert _lib.launch_count() == before
            assert (_np(buf.num_voxels) == -7).all() and (_np(buf.coors) == -7).all()


# ------------------------------------------------------------------------------------------------------------ rulebooks
def _collision_sites(shape=(5, 40, 48), batch=2, max_rows=500):
    """face sites of every frame plus sites whose hash home slots collide (groups of 3) or sit at cap - 1 (a run that wraps), in
    shuffled row order"""
    cap = fm.hash_capacity(max_rows)
    faces = fm.face_sites(batch, shape, dense=(1,))
    rng = np.random.default_rng(2)
    cand = np.setdiff1d(rng.choice(batch * int(np.prod(shape)), 15000, replace=False), fm.rb_key(faces, shape))
    sel = fm.pick_collisions(cand, cap, groups=30, size=3, wrap=4)
    c = np.concatenate([faces, fm.coors_of(cand[sel], shape)], 0)
    c = c[rng.permutation(len(c))]
    assert len(c) <= max_rows
    return c, shape, batch


def _hash(coors, batch, shape, max_rows, n=None):
    from sessd_b200 import ops
    d = torch.zeros((max_rows, 4), dtype=torch.int32, device="cuda")
    d[:len(coors)] = _i32(coors)
    grid = ops.make_grid(batch, shape)
    n_dev = _n(len(coors) if n is None else n)
    return d, n_dev, grid, ops.hash_build(d, n_dev, max_rows, grid)


def _bitmap_level(d_coors, n_dev, max_rows, grid, index_kind, index, max_out=None):
    """the canonical bitmap-indexed copy of a level: a (1,1,1) s1 strided build (generic kernels) from the given index"""
    from sessd_b200 import ops
    max_out = max_out or max_rows
    bm, scratch = ops.bitmap_alloc(grid, "cuda")
    oc = torch.zeros((max_out, 4), dtype=torch.int32, device="cuda")
    n_out, nbr, status = _n(0), torch.empty((max_out, 1), dtype=torch.int32, device="cuda"), _n(0)
    ops.strided_rulebook(d_coors, n_dev, max_rows, grid, index_kind, index, (1, 1, 1), (1, 1, 1), (0, 0, 0), grid, bm, scratch, oc, n_out,
                         max_out, nbr, status)
    return bm, oc, n_out, nbr, status


def test_hash_table_holds_every_key_in_its_probe_run():
    coors, shape, batch = _collision_sites()
    _d, _nd, _g, table = _hash(coors, batch, shape, 500)
    cap = table.numel()
    keys, vals, home, slots, ok = fm.probe_runs(_np(table), cap)
    want = fm.rb_key(coors, shape)
    assert len(keys) == len(coors) and ok.all()
    assert np.array_equal(want[vals], keys)
    assert (slots != home).sum() >= 30 and (slots < home).any()      # collisions happened, and a run wrapped past cap - 1


@pytest.mark.parametrize("ks", [(3, 3, 3), (1, 1, 1), (3, 1, 1), (1, 3, 3), (5, 5, 5)])
def test_subm_rulebook_hash_and_bitmap_indices(ks):
    from sessd_b200 import ops
    coors, shape, batch = _collision_sites()
    pad = tuple(k // 2 for k in ks)
    max_rows = 500
    d, n_dev, grid, table = _hash(coors, batch, shape, max_rows)
    ref = S.neighbor_table(coors, shape, coors, ks, (1, 1, 1), pad)
    assert np.array_equal(ref, fm.neighbor_table(coors, shape, coors, ks, (1, 1, 1), pad))
    a = ops.subm_rulebook(d, n_dev, max_rows, grid, ks, 0, table)
    b = ops.subm_rulebook(d, n_dev, max_rows, grid, ks, 0, table)
    assert np.array_equal(_np(a)[:len(coors)], ref)
    assert torch.equal(a[:len(coors)], b[:len(coors)])
    # a device count above the capacity is clamped to it
    d2, n2, _g, t2 = _hash(coors, batch, shape, len(coors), n=len(coors) + 1000)
    assert torch.equal(ops.subm_rulebook(d2, n2, len(coors), grid, ks, 0, t2), a[:len(coors)])
    # bitmap index: the canonical copy of the level
    bm, oc, n_out, _nbr, status = _bitmap_level(d, n_dev, max_rows, grid, 0, table)
    canon = coors[np.argsort(fm.rb_key(coors, shape))]
    assert int(_np(n_out)[0]) == len(coors) and int(_np(status)[0]) == 0
    assert np.array_equal(_np(oc)[:len(coors)], canon)
    got = ops.subm_rulebook(oc, n_out, max_rows, grid, ks, 1, bm)
    assert np.array_equal(_np(got)[:len(coors)], S.neighbor_table(canon, shape, canon, ks, (1, 1, 1), pad))


def test_hash_build_refusals():
    from sessd_b200 import _lib, ops
    coors, shape, batch = _collision_sites()
    d, n_dev, grid, table = _hash(coors, batch, shape, 500)
    lib = _lib.lib

    def rc(max_rows, g, cap):
        return lib.sessd_hash_build(ops._p(d), ops._p(n_dev), int(max_rows), g, ops._p(table), int(cap), ops._st())
    assert rc(500, grid, 1536) == -1                                   # not a power of two
    assert rc(500, grid, 512) == -1                                    # < 2 rows
    assert rc(1 << 24, grid, 1 << 25) == -2                            # rows past the 24-bit value field
    assert rc(500, ops.make_grid(1 << 10, (1 << 10, 1 << 10, 1 << 10)), 1024) == -2     # 2^40 cells
    assert rc(500, ops.make_grid(1 << 10, (1 << 10, 1 << 10, (1 << 10) - 1)), 1024) == 0


def _strided(d, n_dev, max_in, in_grid, kind, index, ks, st, pd, out_shape, batch, max_out):
    from sessd_b200 import ops
    og = ops.make_grid(batch, out_shape)
    bm, scratch = ops.bitmap_alloc(og, "cuda")
    oc = torch.zeros((max_out, 4), dtype=torch.int32, device="cuda")
    n_out, status = _n(0), _n(0)
    nbr = torch.empty((max_out, ks[0] * ks[1] * ks[2]), dtype=torch.int32, device="cuda")
    ops.strided_rulebook(d, n_dev, max_in, in_grid, kind, index, ks, st, pd, og, bm, scratch, oc, n_out, max_out, nbr, status)
    return dict(grid=og, bm=bm, coors=oc, n=n_out, nbr=nbr, status=status)


def _check_strided(res, in_coors, in_shape, ks, st, pd, max_out=None):
    ref, oshape = S.strided_out_coors(in_coors, in_shape, ks, st, pd)
    max_out = len(ref) if max_out is None else max_out
    ref = ref[:max_out]
    n = int(_np(res["n"])[0])
    assert n == len(ref)
    assert np.array_equal(_np(res["coors"])[:n], ref)
    assert np.array_equal(_np(res["nbr"])[:n], S.neighbor_table(in_coors, in_shape, ref, ks, st, pd))
    return ref, oshape


STRIDED = [((3, 3, 3), (2, 2, 2), (1, 1, 1)), ((3, 3, 3), (2, 2, 2), (0, 1, 1)), ((3, 1, 1), (2, 1, 1), (0, 0, 0)),
           ((2, 2, 2), (2, 2, 2), (0, 0, 0)), ((3, 3, 3), (1, 2, 2), (1, 1, 1))]


@pytest.mark.parametrize("ks,st,pd", STRIDED)
@pytest.mark.parametrize("kind", [0, 1])
def test_strided_rulebook_faces(ks, st, pd, kind):
    """empty, single-site, face and dense frames, hash- (shuffled rows) or bitmap-indexed input; two builds bitwise equal"""
    coors = fm.face_sites(4, SHAPE, empty=(1,), single=(2,), dense=(3,))
    perm = np.random.default_rng(1).permutation(len(coors))
    max_in = len(coors) + 3
    d, n_dev, grid, table = _hash(coors[perm], 4, SHAPE, max_in)
    if kind == 1:
        index, d, n_dev = _bitmap_level(d, n_dev, max_in, grid, 0, table)[:3]
        src = coors
    else:
        index, src = table, coors[perm]
    oshape = fm.out_shape(SHAPE, ks, st, pd)
    total = len(S.strided_out_coors(src, SHAPE, ks, st, pd)[0])
    r1 = _strided(d, n_dev, max_in, grid, kind, index, ks, st, pd, oshape, 4, total + 10)
    _check_strided(r1, src, SHAPE, ks, st, pd)
    assert int(_np(r1["status"])[0]) == 0
    r2 = _strided(d, n_dev, max_in, grid, kind, index, ks, st, pd, oshape, 4, total + 10)
    for k in ("coors", "nbr"):
        assert torch.equal(r1[k][:total], r2[k][:total]), k
    assert torch.equal(r1["bm"], r2["bm"])
    # zero inputs: zero outputs, no status
    r0 = _strided(d, _n(0), max_in, grid, kind, index, ks, st, pd, oshape, 4, 16)
    assert int(_np(r0["n"])[0]) == 0 and int(_np(r0["status"])[0]) == 0


@pytest.mark.parametrize("words", fm.WORD_THRESHOLDS)
def test_strided_rulebook_scan_thresholds(words):
    """output bitmaps of exactly 16384 / 16385 / 2^21 / 2^21 + 1 words (one-CTA, self-prefix and three-launch scans), sites in the
    first, last and scan-tile-boundary words; then a SubM (1,1,3) lookup through the level's bitmap index"""
    from sessd_b200 import ops
    W = 32 * words
    xs = fm.word_sites(words)
    ic = np.stack([np.zeros_like(xs)] * 3 + [xs], 1).astype(np.int32)
    in_shape = (1, 1, 2 * W - 1)
    d, n_dev, grid, table = _hash(ic, 1, in_shape, len(ic))
    ks, st, pd = (3, 3, 3), (2, 2, 2), (1, 1, 1)
    res = _strided(d, n_dev, len(ic), grid, 0, table, ks, st, pd, (1, 1, W), 1, 4 * len(ic))
    assert lib_words(res["grid"]) == words
    ref, oshape = _check_strided(res, ic, in_shape, ks, st, pd)
    n = len(ref)
    got = ops.subm_rulebook(res["coors"], res["n"], 4 * len(ic), res["grid"], (1, 1, 3), 1, res["bm"])
    assert np.array_equal(_np(got)[:n], S.neighbor_table(ref, oshape, ref, (1, 1, 3), (1, 1, 1), (0, 0, 1)))


def lib_words(grid):
    from sessd_b200 import _lib
    return int(_lib.lib.sessd_bitmap_words(grid))


def test_strided_rulebook_64bit_grid():
    """an output grid of more than 2^32 cells (1 GiB bitmap): the 64-bit enumeration, sites past linear index 2^32"""
    shape = (1, 2, (1 << 30) + 64)
    W = shape[2]
    xs = np.array([0, 31, 32, W - 1, W - 33, (1 << 29) + 5], np.int64)
    c = np.concatenate([np.stack([np.full_like(xs, b), np.zeros_like(xs), np.full_like(xs, y), xs], 1)
                        for b in (0, 1) for y in (0, 1)], 0).astype(np.int32)
    assert fm.rb_key(c, shape).max() >= (1 << 32)
    d, n_dev, grid, table = _hash(c, 2, shape, len(c))
    res = _strided(d, n_dev, len(c), grid, 0, table, (1, 1, 1), (1, 1, 1), (0, 0, 0), shape, 2, len(c))
    assert lib_words(res["grid"]) >= (1 << 27)
    _check_strided(res, c, shape, (1, 1, 1), (1, 1, 1), (0, 0, 0))
    del res
    torch.cuda.empty_cache()


def test_strided_rulebook_refusals():
    from sessd_b200 import _lib, ops
    coors = fm.face_sites(2, SHAPE)
    d, n_dev, grid, table = _hash(coors, 2, SHAPE, len(coors))
    ks, st, pd = (3, 3, 3), (2, 2, 2), (1, 1, 1)
    good = fm.out_shape(SHAPE, ks, st, pd)
    bad_shape = (good[0], good[1], good[2] + 1)
    for batch, shp, what in ((2, bad_shape, "invalid argument"), (3, good, "invalid argument")):
        og = ops.make_grid(batch, shp)
        buf = torch.zeros((64, 4), dtype=torch.int32, device="cuda")
        with pytest.raises(_lib.SessdError, match=what):
            ops.strided_rulebook(d, n_dev, len(coors), grid, 0, table, ks, st, pd, og, buf, buf, buf, _n(0), 16, buf, _n(0))
    big = ops.make_grid(1 << 5, (1, 1 << 6, 1 << 25))                   # exactly 2^31 words
    buf = torch.zeros((64, 4), dtype=torch.int32, device="cuda")
    with pytest.raises(_lib.SessdError, match="capacity exceeded"):
        ops.strided_rulebook(d, n_dev, len(coors), big, 0, table, (1, 1, 1), (1, 1, 1), (0, 0, 0), big, buf, buf, buf, _n(0), 16, buf, _n(0))


# ------------------------------------------------------------------------------------------------------------ overflow
def _frame_coors(cloud):
    from oracle import cpu as ocpu
    from sessd_b200 import synth
    _v, c, _n = ocpu.points_to_voxel(cloud, synth.VOXEL_SIZE, synth.PC_RANGE, 5, 20000)
    return np.concatenate([np.zeros((len(c), 1), np.int32), c], 1).astype(np.int32)


@pytest.mark.parametrize("cut", ["minus1", "half", "none"])
def test_overflowed_level_serves_only_its_kept_sites(cut):
    """level 1 of SpMiddleFHD built with max_out = total - 1 / total / 2 / total: the level holds its first max_out sites in canonical
    order, status is raised, and its SubM rulebook, the next strided rulebook, their tile lists and the dense gather see exactly the kept
    sites -- no rulebook entry reaches past the capacity.  No feature buffer is read."""
    from cases import assert_tile_lists_match
    from sessd_b200 import ops, synth
    c0 = _frame_coors(synth.uniform_cloud(0, 3000))
    shape0 = (41, 1600, 1408)
    ks, st, pd = (3, 3, 3), (2, 2, 2), (1, 1, 1)
    full, shape1 = S.strided_out_coors(c0, shape0, ks, st, pd)
    total = len(full)
    max_out = {"minus1": total - 1, "half": total // 2, "none": total}[cut]
    d, n_dev, grid0, table = _hash(c0, 1, shape0, len(c0))
    L1 = _strided(d, n_dev, len(c0), grid0, 0, table, ks, st, pd, shape1, 1, max_out)
    kept, _ = _check_strided(L1, c0, shape0, ks, st, pd, max_out)
    assert int(_np(L1["status"])[0]) == (1 if max_out < total else 0)
    # SubM rulebook on the level
    sub = ops.subm_rulebook(L1["coors"], L1["n"], max_out, L1["grid"], (3, 3, 3), 1, L1["bm"])
    got = _np(sub)[:max_out]
    assert got.max() < max_out
    assert np.array_equal(got, S.neighbor_table(kept, shape1, kept, (3, 3, 3), (1, 1, 1), (1, 1, 1)))
    tl = ops.rulebook_tile_lists(sub, L1["n"], max_out, ops.alloc_tile_lists(max_out, 27, "cuda"))
    assert_tile_lists_match(_np(tl).view(np.uint32), S.neighbor_table(kept, shape1, kept, (3, 3, 3), (1, 1, 1), (1, 1, 1)), max_out)
    # the next strided rulebook
    shape2 = fm.out_shape(shape1, ks, st, pd)
    cap2 = total * 2
    L2 = _strided(L1["coors"], L1["n"], max_out, L1["grid"], 1, L1["bm"], ks, st, pd, shape2, 1, cap2)
    _check_strided(L2, kept, shape1, ks, st, pd)
    n2 = int(_np(L2["n"])[0])
    assert _np(L2["nbr"])[:n2].max() < max_out
    tl2 = ops.rulebook_tile_lists(L2["nbr"], L2["n"], cap2, ops.alloc_tile_lists(cap2, 27, "cuda"))
    assert_tile_lists_match(_np(tl2).view(np.uint32), S.neighbor_table(kept, shape1, S.strided_out_coors(kept, shape1, ks, st, pd)[0],
                                                                       ks, st, pd), n2)
    # dense gather through the level's index
    C_ = 4
    feat = torch.arange(max_out * C_, dtype=torch.float32, device="cuda").reshape(max_out, C_) + 1
    out = torch.empty((1, shape1[1], shape1[2], C_ * shape1[0]), dtype=torch.float32, device="cuda")
    ops.sparse_to_dense_indexed(feat, L1["bm"], L1["grid"], out)
    ref = np.zeros((1, shape1[1], shape1[2], C_, shape1[0]), np.float32)
    ref[kept[:, 0], kept[:, 2], kept[:, 3], :, kept[:, 1]] = _np(feat)
    assert np.array_equal(_np(out), ref.reshape(out.shape))


def _rulebooks_only(r, coors0, n0):
    """the rulebook builds of SpMiddleRunner.forward, in its order, without any conv"""
    from sessd_b200 import ops
    L0 = r.levels[0]
    cap0 = coors0.shape[0]
    ops.hash_build(coors0, n0, cap0, L0["grid"], L0["index"])
    for p in r.plan:
        lin, lout = r.levels[p["lin"]], r.levels[p["lout"]]
        coors = coors0 if p["lin"] == 0 else lin["coors"]
        n_in, cap_in = (n0, cap0) if p["lin"] == 0 else (lin["n"], lin["cap"])
        if not p["build_rb"]:
            continue
        if p["kind"] == "subm":
            ops.subm_rulebook(coors, n_in, cap_in, lin["grid"], p["ks"], lin["index_kind"], lin["index"], p["nbr"])
        else:
            ops.strided_rulebook(coors, n_in, cap_in, lin["grid"], lin["index_kind"], lin["index"], p["ks"], p["st"], p["pd"], lout["grid"],
                                 lout["index"], lout["scratch"], lout["coors"], lout["n"], lout["cap"], p["nbr"], r.status)


@pytest.mark.parametrize("case", ["uniform20k_level2", "two_frames_level1"])
def test_runner_with_an_overflowed_level(case):
    """SpMiddleRunner with a level capacity below its site count: status raised, counts clamped, every table inside the capacity of
    the level it indexes (checked before any conv runs); per-layer features within 1e-5 of each layer's maximum of the fp64 oracle
    with the same capacities; two runs bitwise equal."""
    from oracle import cpu as ocpu
    from sessd_b200 import synth
    from sessd_b200.runners import SpMiddleRunner
    from sessd_b200 import weights
    if case == "uniform20k_level2":
        clouds = [synth.uniform_cloud(0, 20000)]
        growth = (1.0, 4.0, 4.0, 5.0, 3.0)                 # level 2: 79 992 slots for 103 374 sites
    else:
        clouds = [synth.ring_cloud(3, 6000), synth.uniform_cloud(4, 3000)]
        growth = None
    feats, coors = [], []
    for f, cloud in enumerate(clouds):
        v, c, num = ocpu.points_to_voxel(cloud, synth.VOXEL_SIZE, synth.PC_RANGE, 5, 20000)
        feats.append((v.sum(1) / num[:, None]).astype(np.float32))
        coors.append(np.concatenate([np.full((len(c), 1), f, np.int32), c], 1).astype(np.int32))
    feat, coors = np.concatenate(feats), np.concatenate(coors)
    n = len(coors)
    if growth is None:                                      # level 1 short by 500 sites: frame 1 (last in canonical order) loses them
        total1 = len(S.strided_out_coors(coors, (41, 1600, 1408), (3, 3, 3), (2, 2, 2), (1, 1, 1))[0])
        growth = (1.0, (total1 - 500) / n, 8.0, 8.0, 8.0)
    r = SpMiddleRunner(len(clouds), n, device="cuda", growth=growth)
    layers, _, _ = weights.split_detector_state(weights.random_detector_state(3))
    r.load_weights(layers)
    d_feat, d_coors, n0 = torch.from_numpy(feat).cuda(), _i32(coors), _n(n)
    _rulebooks_only(r, d_coors, n0)
    torch.cuda.synchronize()
    assert int(r.status.item()) == 1
    caps = [lv["cap"] for lv in r.levels]
    counts = [n] + [int(lv["n"].item()) for lv in r.levels[1:]]
    assert all(c <= cap for c, cap in zip(counts[1:], caps[1:]))
    assert any(c == cap for c, cap in zip(counts[1:], caps[1:]))
    if len(clouds) == 2:                                    # the sites dropped from level 1 are all frame 1's
        lv1 = r.levels[1]["coors"][:counts[1]].cpu().numpy()
        full1 = S.strided_out_coors(coors, (41, 1600, 1408), (3, 3, 3), (2, 2, 2), (1, 1, 1))[0]
        assert (lv1[:, 0] == 0).sum() == (full1[:, 0] == 0).sum() and (lv1[:, 0] == 1).sum() < (full1[:, 0] == 1).sum()
    for p in r.plan:
        rows = counts[p["lout"]]
        assert int(p["nbr"][:rows].max()) < counts[p["lin"]], p["rb"]
        assert int(p["nbr"][:rows].min()) >= -1
    params = [dict(weight=l["weight"].numpy(), gamma=l["gamma"].numpy(), beta=l["beta"].numpy(), mean=l["mean"].numpy(),
                   var=l["var"].numpy()) for l in layers]
    trace = []
    ref = S.spmiddle_forward(feat, coors, len(clouds), (1408, 1600, 40), params, np.float64, trace, caps=[None] + caps[1:])
    assert [len(t["coors"]) for t in trace] == [counts[p["lout"]] for p in r.plan]
    d1 = r.forward(d_feat, d_coors, n0).clone()
    torch.cuda.synchronize()
    outs1 = [r.layer_output(li).clone() for li in range(len(r.plan))]
    for li, t in enumerate(trace):
        got = outs1[li][: len(t["coors"])].cpu().numpy().astype(np.float64)
        assert got.shape[0] == counts[r.plan[li]["lout"]]
        scale = np.abs(t["feat"]).max() + 1e-30
        assert np.abs(got - t["feat"]).max() / scale < 1e-5, "layer %d" % li
    got = d1.permute(0, 3, 1, 2).cpu().numpy().astype(np.float64)
    assert np.abs(got - ref).max() / np.abs(ref).max() < 1e-5
    d2 = r.forward(d_feat, d_coors, n0)
    torch.cuda.synchronize()
    assert torch.equal(d1, d2)
    for li, a in enumerate(outs1):
        assert torch.equal(a, r.layer_output(li)), li
