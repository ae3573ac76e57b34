"""Constant-region skipping of the SSFA neck + head (csrc/bevskip.cu): bitwise equal to the dense neck, and the device's plan equals the
numpy restatement (tests/skip_model.py).  Inputs: the bench's 16 ring clouds and 4 uniform clouds through FrameEngine, and crafted
occupancy maps (empty, full, single pixels at corners / edges / tile seams, batch 2) through SSFAPlanesRunner with guard bands."""
import numpy as np
import pytest
import torch

import skip_model as sm

pytestmark = pytest.mark.gpu

GUARD = 4096


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.float16 else t.view(torch.int32)


def _neck_state(r):
    s = {"planes:" + k: _bits(v).clone() for k, v in r.planes.items()}
    s.update({"buf:" + k: _bits(v).clone() for k, v in r.buf.items()})
    s["info"] = _bits(r.info).clone()
    return s


def _assert_same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k], b[k]), k


def _poison(r, skip_input=True):
    """overwrite every neck output with NaN so that a tile the skipping run neither computes nor fills cannot pass"""
    for k, v in r.planes.items():
        if not (skip_input and k == "x"):
            v.fill_(float("nan"))
    for v in r.buf.values():
        v.fill_(float("nan"))


def _check_plan(r, occ):
    for i, exp in enumerate(sm.plan(occ)):
        items, skipped, rep = sm.read_record(r.skip.record(i).cpu().numpy())
        assert np.array_equal(items, exp["items"]), exp["name"]
        assert np.array_equal(skipped, exp["skipped"]), exp["name"]
        assert rep[:len(exp["rep"])] == exp["rep"], exp["name"]


# ----------------------------------------------------------------------------------------------------------- FrameEngine, bench clouds
@pytest.fixture(scope="module")
def engines():
    from sessd_b200.engine import FrameEngine
    from sessd_data import weights
    layers, ssfa, head = weights.bench_detector_state("ring", 0)
    anchors = weights.kitti_car_anchors()
    es, ed = FrameEngine(batch=1), FrameEngine(batch=1, skip_constant=False)
    for e in (es, ed):
        e.load_weights(layers, ssfa, head, anchors)
    assert es.neck.skip is not None and ed.neck.skip is None
    return es, ed


@pytest.mark.parametrize("kind,seed", [("ring", s) for s in range(16)] + [("uniform", s) for s in range(4)])
def test_frame_engine_skip_is_bitwise_dense(engines, kind, seed):
    from sessd_data import synth
    es, ed = engines
    cloud = synth.ring_cloud(seed, 20000) if kind == "ring" else synth.uniform_cloud(seed, 20000)
    with torch.cuda.stream(es.stream):
        _poison(es.neck)
    rs, rd = es.infer([cloud])[0], ed.infer([cloud])[0]
    torch.cuda.synchronize()
    _assert_same(_neck_state(es.neck), _neck_state(ed.neck))
    assert torch.equal(_bits(es.d_result), _bits(ed.d_result)) and torch.equal(es.d_meta, ed.d_meta)
    assert np.array_equal(rs["anchor_index"], rd["anchor_index"]) and np.array_equal(rs["box3d_lidar"], rd["box3d_lidar"])
    last = es.middle.levels[-1]
    d, h, w = last["grid"].shape[0], last["grid"].shape[1], last["grid"].shape[2]
    occ = sm.occupancy_from_bitmap(last["index"].cpu().numpy(), 1, d, h, w)
    _check_plan(es.neck, occ)
    if kind == "ring":      # a LiDAR scan leaves empty space: some tiles of the full-resolution layers are skipped
        assert int(es.neck.skip.record(0)[1]) > 0


# ----------------------------------------------------------------------------------------------------------- crafted maps
def _pattern(name, h, w):
    occ = np.zeros((h, w), bool)
    pts = dict(corner_tl=[(0, 0)], corner_tr=[(0, w - 1)], corner_bl=[(h - 1, 0)], corner_br=[(h - 1, w - 1)], edge_top=[(0, w // 2)],
               edge_left=[(h // 2, 0)], edge_bottom=[(h - 1, w // 3)], edge_right=[(h // 3, w - 1)],
               seam_u=[(7, w // 2), (8, w // 2 + 3)], seam_v=[(h // 2, 15), (h // 2 + 5, 16)], seam_uv=[(15, 31), (16, 32)],
               centre=[(h // 2, w // 2)], empty=[])
    if name == "full":
        occ[:] = True
    else:
        for y, x in pts[name]:
            occ[y, x] = True
    return occ


PATTERNS = ["empty", "full", "corner_tl", "corner_tr", "corner_bl", "corner_br", "edge_top", "edge_left", "edge_bottom", "edge_right",
            "seam_u", "seam_v", "seam_uv", "centre"]


def _guarded(t, fill):
    big = torch.full((t.numel() + 2 * GUARD,), fill, dtype=t.dtype, device=t.device)
    return big, big[GUARD:GUARD + t.numel()].view(t.shape)


@pytest.mark.parametrize("hw", [(200, 176), (48, 64)])
@pytest.mark.parametrize("pattern", PATTERNS)
def test_crafted_maps_skip_is_bitwise_dense(hw, pattern):
    from oracle import bev_ref
    from sessd_b200 import ops
    from sessd_b200.runners import SSFAPlanesRunner
    h, w = hw
    batch = 2 if hw == (48, 64) else 1
    other = {"empty": "centre", "full": "full"}.get(pattern, "empty")
    occ = np.stack([_pattern(pattern, h, w)] + [_pattern(other, h, w)] * (batch - 1))
    r = SSFAPlanesRunner(batch, hw, "cuda", skip_constant=True)
    r.load_state(bev_ref.ssfa_random_state(11), bev_ref.head_random_state(12))
    bigs = []
    for dct in (r.planes, r.buf):
        for k in list(dct):
            big, dct[k] = _guarded(dct[k], -1234.0)
            bigs.append(big)
    g = torch.Generator().manual_seed(13)
    x = torch.zeros((batch, h, w, 128))
    ob, oy, ox = np.nonzero(occ)
    x[ob, oy, ox] = torch.rand((len(ob), 128), generator=g) * 4 + 0.25
    x = x.cuda()
    depth = 2
    words = -(-batch * depth * h * w // 32)
    bm = np.zeros((words, 2), np.uint32)
    lin = ((ob * depth + 1) * h + oy) * w + ox                      # sites in slice z = 1
    np.bitwise_or.at(bm[:, 0], lin >> 5, (np.uint32(1) << (lin & 31).astype(np.uint32)))
    bitmap = torch.from_numpy(bm.view(np.int32)).cuda()
    grid = ops.make_grid(batch, (depth, h, w))
    r.forward(x)
    dense = _neck_state(r)
    _poison(r, skip_input=False)
    r.forward(x, occupancy=(bitmap, grid))
    torch.cuda.synchronize()
    _assert_same(_neck_state(r), dense)
    for big in bigs:
        assert bool((big[:GUARD] == -1234.0).all()) and bool((big[-GUARD:] == -1234.0).all())
    _check_plan(r, occ)
    rec0 = r.skip.record(0).cpu().numpy()
    if pattern == "full":
        assert rec0[1] == 0
    else:
        assert rec0[1] > 0
