"""CPU checks of tests/frontend_model.py: the crafted inputs reach what they claim (scan thresholds, hash collisions and wraps,
faces, cut counts, batch sizes), the models equal the oracles on every case, and each negative control (a plausible wrong
kernel) changes at least one crafted expectation."""
import numpy as np
import pytest

import frontend_model as fm
from oracle import spconv_ref as S

GENERIC = [((1, 1, 1), (1, 1, 1), (0, 0, 0)), ((3, 1, 1), (1, 1, 1), (1, 0, 0)), ((1, 3, 3), (1, 1, 1), (0, 1, 1)),
           ((5, 5, 5), (1, 1, 1), (2, 2, 2)), ((3, 3, 3), (1, 1, 1), (1, 1, 1))]
STRIDED = [((3, 3, 3), (2, 2, 2), (1, 1, 1)), ((3, 3, 3), (2, 2, 2), (0, 1, 1)), ((3, 1, 1), (2, 1, 1), (0, 0, 0)),
           ((2, 2, 2), (2, 2, 2), (0, 0, 0)), ((3, 3, 3), (1, 2, 2), (1, 1, 1))]
SHAPE = (7, 9, 11)


def _faces():
    return fm.face_sites(4, SHAPE, empty=(1,), single=(2,), dense=(3,))


def _oracle_voxels(cloud, mp, mv):
    from oracle import cpu as ocpu
    cloud = cloud[~np.isnan(cloud[:, :3]).any(1)]            # the C oracle would turn a NaN into an int
    return ocpu.points_to_voxel(cloud, fm.VOXEL_SIZE, fm.RANGE_MIN + (70.4, 40.0, 1.0), mp, mv)


# ------------------------------------------------------------------------------------------------------------ generators
def test_hash_mix_matches_fmix64():
    def fmix(k):
        m = (1 << 64) - 1
        k ^= k >> 33
        k = (k * 0xff51afd7ed558ccd) & m
        k ^= k >> 33
        k = (k * 0xc4ceb9fe1a85ec53) & m
        k ^= k >> 33
        return k & 0xFFFFFFFF
    ks = [0, 1, 2, 12345, (1 << 40) - 1, (1 << 63) + 5]
    assert fm.hash_mix(ks).tolist() == [fmix(k) for k in ks]
    assert [fm.hash_capacity(r) for r in (1, 512, 513, 1000, 4096, 4097)] == [1024, 1024, 2048, 2048, 8192, 16384]


@pytest.mark.parametrize("layout", ["voxel", "rulebook"])
def test_collision_picker_collides_and_wraps(layout):
    rng = np.random.default_rng(1)
    if layout == "voxel":
        cells = fm.random_cells(rng, 100000)
        keys = fm.vox_key(rng.integers(0, 2, len(cells)), cells, fm.GRID)
    else:
        c = fm.coors_of(rng.choice(2 * 5 * 40 * 48, 9000, replace=False), (5, 40, 48))
        keys = fm.rb_key(c, (5, 40, 48))
    cap = 1024
    sel = fm.pick_collisions(keys, cap, groups=24, size=3, wrap=4)
    home = fm.home_slot(keys[sel], cap)
    assert (home[:4] == cap - 1).all()
    assert all(len(set(home[4 + 3 * g: 7 + 3 * g])) == 1 for g in range(24))
    assert len(np.unique(keys[sel])) == len(sel)


def test_face_sites_reach_every_face_edge_and_corner():
    c = _faces()
    d, h, w = SHAPE
    assert set(np.unique(c[:, 0])) == {0, 2, 3}
    assert (c[:, 0] == 2).sum() == 1
    f0 = c[c[:, 0] == 0]
    for z in (0, d - 1):
        for y in (0, h - 1):
            for x in (0, w - 1):
                assert ((f0[:, 1:] == (z, y, x)).all(1)).any()
    for j, s in enumerate(SHAPE):                               # even and odd positions on both sides of every axis
        assert {0, 1, s - 2, s - 1} <= set(f0[:, 1 + j].tolist())
    assert (c[:, 0] == 3).sum() > len(f0)
    assert np.all(np.diff(fm.rb_key(c, SHAPE)) > 0)


@pytest.mark.parametrize("words", fm.WORD_THRESHOLDS)
def test_word_sites_reach_the_scan_thresholds(words):
    W = 32 * words
    assert fm.out_shape((1, 1, 2 * W - 1), (3, 3, 3), (2, 2, 2), (1, 1, 1)) == (1, 1, W)
    xs = fm.word_sites(words)
    ic = np.stack([np.zeros_like(xs), np.zeros_like(xs), np.zeros_like(xs), xs], 1)
    sites, oshape = fm.strided_sites(ic, (1, 1, 2 * W - 1), (3, 3, 3), (2, 2, 2), (1, 1, 1), 1)
    assert oshape == (1, 1, W) and (W + 31) // 32 == words
    ws = set((sites >> 5).tolist())
    assert {0, words - 1} <= ws
    for t in range(1, words // fm.SCAN_TILE + 1):
        assert {t * fm.SCAN_TILE - 1, t * fm.SCAN_TILE} <= ws or t * fm.SCAN_TILE >= words
    assert (xs % 2 == 1).any() and (xs % 2 == 0).any()


@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_cut_clouds_reach_the_cut(delta):
    mv = 40
    cloud = fm.cut_cloud(delta + 5, mv, delta)
    cells, ok = fm.cells_of(cloud, fm.VOXEL_SIZE, fm.RANGE_MIN, fm.GRID)
    assert ok.all() and len(np.unique(fm.vox_key(0, cells, fm.GRID))) == mv + delta
    (v, c, n, _m), = fm.voxelize_batch([cloud], fm.VOXEL_SIZE, fm.RANGE_MIN, fm.GRID, 5, mv)
    assert len(c) == min(mv, mv + delta)
    assert n.max() == 5 and (n == 4).any()
    kept = int(n.sum())
    full = fm.voxelize_batch([cloud], fm.VOXEL_SIZE, fm.RANGE_MIN, fm.GRID, 1000, 10 ** 6)[0][2].sum()
    if delta > 0:
        assert kept < min(full, sum(min(int(x), 5) for x in
                                    np.unique(fm.vox_key(0, cells, fm.GRID), return_counts=True)[1]))
    else:
        assert int(full) == len(cloud)


def test_boundary_cloud_places_first_points_on_tile_edges():
    cloud = fm.boundary_cloud(5000)
    cells, _ = fm.cells_of(cloud, fm.VOXEL_SIZE, fm.RANGE_MIN, fm.GRID)
    key = fm.vox_key(0, cells, fm.GRID)
    first = np.r_[True, key[1:] != key[:-1]]
    assert first[[2047, 2048, 2049]].all() and len(np.unique(key)) == first.sum()


def test_edge_cloud_has_nan_and_inf():
    cloud, nan = fm.clouds_with_edges(3)
    assert nan.sum() == 3 and np.isinf(cloud[:, :3]).sum() == 6
    _cells, ok = fm.cells_of(cloud, fm.VOXEL_SIZE, fm.RANGE_MIN, fm.GRID)
    assert (~ok).sum() == 3 + 6 + 2


# ------------------------------------------------------------------------------------------------------------ models vs oracles
@pytest.mark.parametrize("ks,st,pd", GENERIC)
def test_neighbor_model_matches_oracle(ks, st, pd):
    c = _faces()
    assert np.array_equal(fm.neighbor_table(c, SHAPE, c, ks, st, pd), S.neighbor_table(c, SHAPE, c, ks, st, pd))


@pytest.mark.parametrize("ks,st,pd", STRIDED)
def test_strided_model_matches_oracle(ks, st, pd):
    c = _faces()
    sites, oshape = fm.strided_sites(c, SHAPE, ks, st, pd, 4)
    ref, ref_shape = S.strided_out_coors(c, SHAPE, ks, st, pd)
    assert oshape == ref_shape
    nwords = (4 * int(np.prod(oshape)) + 31) // 32
    for cap in (len(ref), len(ref) - 1, len(ref) // 2, len(ref) + 5):
        rows, n = fm.bitmap_level(sites, nwords, cap)
        oc = fm.level_coors(sites, rows, n, oshape)
        assert np.array_equal(oc, ref[:cap])
        # the level's index answers exactly its kept sites
        nb = fm.level_table(sites, rows, oshape, oc, (3, 3, 3), (1, 1, 1), (1, 1, 1))
        assert np.array_equal(nb, S.neighbor_table(oc, oshape, oc, (3, 3, 3), (1, 1, 1), (1, 1, 1)))
        assert nb.max() < max(cap, 1)
    nb = S.neighbor_table(c, SHAPE, ref, ks, st, pd)
    assert np.array_equal(fm.neighbor_table(c, SHAPE, ref, ks, st, pd), nb)


@pytest.mark.parametrize("mp,nf", [(1, 3), (5, 4), (7, 5), (5, 3), (1, 4)])
@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_voxel_model_matches_oracle(mp, nf, delta):
    mv = 30
    clouds = [fm.cut_cloud(7 + f + delta, mv, delta, nf=nf, max_points=mp) for f in range(3)]
    clouds[1] = clouds[1][:0]                                   # an empty frame in the middle
    edge, _nan = fm.clouds_with_edges(4, nf)
    clouds.append(edge)
    got = fm.voxelize_batch(clouds, fm.VOXEL_SIZE, fm.RANGE_MIN, fm.GRID, mp, mv)
    for cloud, (v, c, n, mean) in zip(clouds, got):
        ov, oc, on = _oracle_voxels(cloud, mp, mv)
        assert np.array_equal(c, oc) and np.array_equal(n, on) and np.array_equal(v, ov, equal_nan=True)


def test_voxel_model_batch_of_300_frames():
    rng = np.random.default_rng(0)
    base = fm.cell_points(fm.random_cells(rng, 20), 0)
    clouds = [base[: (f % 7) * 3] for f in range(300)]          # frames share cells; several are empty
    got = fm.voxelize_batch(clouds, fm.VOXEL_SIZE, fm.RANGE_MIN, fm.GRID, 5, 10)
    for cloud, (v, c, n, _m) in zip(clouds, got):
        ov, oc, on = _oracle_voxels(cloud, 5, 10)
        assert np.array_equal(c, oc) and np.array_equal(n, on) and np.array_equal(v, ov)


# ------------------------------------------------------------------------------------------------------------ negative controls
def _rulebook_expectations(mut):
    c = _faces()
    out = [fm.neighbor_table(c, SHAPE, c, ks, st, pd, mut) for ks, st, pd in GENERIC]
    for ks, st, pd in STRIDED:
        sites, oshape = fm.strided_sites(c, SHAPE, ks, st, pd, 4, mut)
        out.append(sites)
    xs = fm.word_sites(fm.SCAN_SMALL_MAX + 1)
    W = 32 * (fm.SCAN_SMALL_MAX + 1)
    ic = np.stack([np.zeros_like(xs)] * 3 + [xs], 1)
    sites, oshape = fm.strided_sites(ic, (1, 1, 2 * W - 1), (3, 3, 3), (2, 2, 2), (1, 1, 1), 1)
    for cap in (len(sites), len(sites) - 1, len(sites) // 2):
        rows, n = fm.bitmap_level(sites, fm.SCAN_SMALL_MAX + 1, cap, mut)
        oc = fm.level_coors(sites, rows, n, oshape)
        out += [oc, fm.level_table(sites, rows, oshape, oc, (1, 1, 3), (1, 1, 1), (0, 0, 1))]
    return out


def _voxel_expectations(mut):
    a = fm.cut_cloud(11, 30, 1)
    clouds = [a, a[:60]]                                        # the second frame reuses cells of the first
    return [a for fr in fm.voxelize_batch(clouds, fm.VOXEL_SIZE, fm.RANGE_MIN, fm.GRID, 5, 30, mut) for a in fr]


def _differs(a, b):
    return len(a) != len(b) or any(x.shape != y.shape or not np.array_equal(x, y, equal_nan=True) for x, y in zip(a, b))


@pytest.mark.parametrize("mut", ["no_x_bound", "no_yz_bound", "no_parity", "inclusive", "lost_carry", "untruncated"])
def test_rulebook_negative_controls(mut):
    assert _differs(_rulebook_expectations(()), _rulebook_expectations((mut,)))


@pytest.mark.parametrize("mut", ["cut_off_by_one", "keep_last", "no_frame_key"])
def test_voxel_negative_controls(mut):
    assert _differs(_voxel_expectations(()), _voxel_expectations((mut,)))
