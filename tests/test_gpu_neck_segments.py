"""Segment skipping of the SSFA neck + head (csrc/bevskip.cu segment records, the segment path of csrc/bevconv_p2.cuh): the device's
segment records equal the numpy restatement (tests/seg_model.py) on the bench clouds and crafted maps; the neck is bitwise equal to the
dense one from NaN-poisoned buffers; a pixel's value does not depend on the group, slot or CTA that computes it; and a record that
drops or replaces a live segment, leaves a skipped segment unfilled or fills it from the representative of the other v parity is
caught."""
import numpy as np
import pytest
import torch

import seg_model
import skip_model as sm
from test_gpu_neck_skip import PATTERNS, _assert_same, _neck_state, _pattern, _poison

pytestmark = pytest.mark.gpu


def _check_segs(r, occ):
    exp = seg_model.plan(occ)
    for i, name in enumerate(n for n, _, _ in sm.LAUNCHES):
        rec = r.skip.seg_record(i)
        if name in seg_model.TILE_ONLY:
            assert rec is None
            continue
        count, groups, skipped, rep = seg_model.read_seg_record(rec.cpu().numpy())
        e = exp[name]
        assert count == e["count"], name
        assert np.array_equal(groups, e["groups"]), name
        assert np.array_equal(skipped, e["skipped"]), name
        assert rep == e["rep"], name


def _frame(occ, depth=2, seed=13):
    """occ [B, h, w] -> (fp32 NHWC neck input, nonzero exactly on occ; the bitmap index of a level with its sites in slice z = 1; grid)"""
    from sessd_b200 import ops
    batch, h, w = occ.shape
    g = torch.Generator().manual_seed(seed)
    x = torch.zeros((batch, h, w, 128))
    ob, oy, ox = np.nonzero(occ)
    x[ob, oy, ox] = torch.rand((len(ob), 128), generator=g) * 4 + 0.25
    words = -(-batch * depth * h * w // 32)
    bm = np.zeros((words, 2), np.uint32)
    lin = ((ob * depth + 1) * h + oy) * w + ox
    np.bitwise_or.at(bm[:, 0], lin >> 5, (np.uint32(1) << (lin & 31).astype(np.uint32)))
    return x.cuda(), torch.from_numpy(bm.view(np.int32)).cuda(), ops.make_grid(batch, (depth, h, w))


def _runner(batch, hw):
    from oracle import bev_ref
    from sessd_b200.runners import SSFAPlanesRunner
    r = SSFAPlanesRunner(batch, hw, "cuda", skip_constant=True)
    r.load_state(bev_ref.ssfa_random_state(11), bev_ref.head_random_state(12))
    return r


# ----------------------------------------------------------------------------------------------------------- FrameEngine, bench clouds
@pytest.fixture(scope="module")
def engine():
    from sessd_b200.engine import FrameEngine
    from sessd_data import weights
    layers, ssfa, head = weights.bench_detector_state("ring", 0)
    e = FrameEngine(batch=1)
    e.load_weights(layers, ssfa, head, weights.kitti_car_anchors())
    return e


@pytest.mark.parametrize("kind,seed", [("ring", s) for s in range(16)] + [("uniform", s) for s in range(4)])
def test_frame_engine_segment_records(engine, kind, seed):
    from sessd_data import synth
    cloud = synth.ring_cloud(seed, 20000) if kind == "ring" else synth.uniform_cloud(seed, 20000)
    engine.infer([cloud])
    torch.cuda.synchronize()
    last = engine.middle.levels[-1]
    d, h, w = last["grid"].shape[0], last["grid"].shape[1], last["grid"].shape[2]
    occ = sm.occupancy_from_bitmap(last["index"].cpu().numpy(), 1, d, h, w)
    _check_segs(engine.neck, occ)
    if kind == "ring":      # the segments cut more than the tiles on a LiDAR scan's full-resolution layers
        tiles = int(engine.neck.skip.record(0)[0]) * sm.TV
        assert int(engine.neck.skip.seg_record(0)[2]) * seg_model.SLOTS < tiles


# ----------------------------------------------------------------------------------------------------------- crafted maps
@pytest.mark.parametrize("hw", [(200, 176), (48, 64)])
@pytest.mark.parametrize("pattern", PATTERNS)
def test_crafted_maps_segments_bitwise_dense(hw, pattern):
    h, w = hw
    batch = 2 if hw == (48, 64) else 1
    other = {"empty": "centre", "full": "full"}.get(pattern, "empty")
    occ = np.stack([_pattern(pattern, h, w)] + [_pattern(other, h, w)] * (batch - 1))
    r = _runner(batch, hw)
    x, bitmap, grid = _frame(occ)
    r.forward(x)
    dense = _neck_state(r)
    _poison(r, skip_input=False)
    r.forward(x, occupancy=(bitmap, grid))
    torch.cuda.synchronize()
    _assert_same(_neck_state(r), dense)
    _check_segs(r, occ)


# ----------------------------------------------------------------------------------------------------------- records edited on the device
def _blobs(h, w, n, seed):
    rng = np.random.default_rng(seed)
    occ = np.zeros((1, h, w), bool)
    occ[0, rng.integers(0, h, n), rng.integers(0, w, n)] = True
    return occ


def _rerun(r, x):
    """the skipping forward on the records as they are (no new plan), from NaN-poisoned buffers"""
    _poison(r, skip_input=False)
    build = r.skip.build
    r.skip.build = lambda *a: None
    try:
        r.forward(x, occupancy=r._occupancy)
    finally:
        r.skip.build = build
    torch.cuda.synchronize()
    return _neck_state(r)


def _setup(seed):
    occ = _blobs(200, 176, 300, seed)
    r = _runner(1, (200, 176))
    x, bitmap, grid = _frame(occ, seed=seed)
    r._occupancy = (bitmap, grid)
    r.forward(x)
    dense = _neck_state(r)
    _poison(r, skip_input=False)
    r.forward(x, occupancy=r._occupancy)
    torch.cuda.synchronize()
    _assert_same(_neck_state(r), dense)
    return r, x, dense


def _live_slots(r, i):
    """(record, groups view [n, 16] of the device buffer) of segment launch i"""
    rec = r.skip.seg_record(i)
    n = int(rec[2])
    return rec, rec[seg_model.HEADER:seg_model.HEADER + seg_model.SLOTS * n].view(n, seg_model.SLOTS)


def test_segments_permuted_across_groups_and_slots_are_bitwise_equal():
    r, x, dense = _setup(21)
    g = torch.Generator().manual_seed(5)
    for i in range(len(sm.LAUNCHES)):
        if r.skip.seg_record(i) is None:
            continue
        _, groups = _live_slots(r, i)
        flat = groups.reshape(-1)
        cls = torch.where(flat >= 0, flat >> 24, torch.full_like(flat, -1))
        for c in torch.unique(cls[cls >= 0]).tolist():
            pos = torch.nonzero(cls == c).reshape(-1)
            flat[pos] = flat[pos[torch.randperm(len(pos), generator=g).to(pos.device)]]
    _assert_same(_rerun(r, x), dense)


@pytest.mark.parametrize("edit", ["drop", "duplicate"])
def test_segment_record_that_misses_a_live_segment_is_caught(edit):
    r, x, dense = _setup(22)
    _, groups = _live_slots(r, 0)
    assert groups.shape[0] > 1 and int(groups[0, 1]) >= 0
    groups[0, 1] = -1 if edit == "drop" else groups[0, 0]
    with pytest.raises(AssertionError):
        _assert_same(_rerun(r, x), dense)


@pytest.mark.parametrize("edit", ["unfilled", "swapped_parity"])
def test_segment_fill_that_misses_a_segment_or_its_parity_is_caught(edit):
    """conv_0.0 reads the deconvs' period-2 maps: its two v-parity constants differ, so a fill from the wrong parity shows"""
    r, x, dense = _setup(23)
    rec = r.skip.seg_record(r.SKIP_LAUNCHES.index("conv_0.0"))
    rep0, rep1, nskip = int(rec[20]), int(rec[21]), int(rec[1])
    assert rep0 >= 0 and rep1 >= 0 and nskip > 0
    if edit == "unfilled":
        rec[1] = nskip - 1
    else:
        rec[20], rec[21] = rep1, rep0
    with pytest.raises(AssertionError):
        _assert_same(_rerun(r, x), dense)
