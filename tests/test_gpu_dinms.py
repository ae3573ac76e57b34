"""DI-NMS on the device (sessd_rotate_weighted_nms, sessd_postprocess with nms_mode 1, FrameEngine) against the reference's outputs
(tests/golden/dinms_cases.npz) and the DI-NMS oracle (oracle/dinms_ref.py through tests/dinms_cases.py)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import dinms_cases as dc

pytestmark = pytest.mark.gpu

# every workspace byte starts as this garbage: a kernel that reads workspace it did not write fails the comparisons (freshly allocated
# device memory is often zero, which would hide such a read)
POISON = 0x5A

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "dinms_cases.npz"))
NAMES = [str(n) for n in GOLD["names"]]


def stored_case(name):
    keys = ("boxes7", "scores", "iou_preds", "labels", "dirs", "anchors", "pre_max")
    c = {k: GOLD["%s__in_%s" % (name, k)] for k in keys}
    c["pre_max"] = int(c["pre_max"])
    return c


def _check_outputs(name, boxes, dirs, labels, scores, selected, keep=None):
    assert np.array_equal(np.asarray(selected, np.int64), GOLD[name + "__selected"]), name
    if keep is not None:
        assert np.array_equal(np.asarray(keep, np.int64), GOLD[name + "__keep"]), name
    assert np.array_equal(np.asarray(labels, np.int64), GOLD[name + "__labels"]), name
    assert np.array_equal(np.asarray(dirs, np.int64), GOLD[name + "__dirs"]), name
    np.testing.assert_allclose(np.asarray(scores, np.float64), GOLD[name + "__scores"], rtol=1e-6, atol=0)
    ref = GOLD[name + "__boxes"]
    got = np.asarray(boxes, np.float64).reshape(-1, 7)
    assert np.array_equal(np.isnan(got), np.isnan(ref)), name
    fin = ~np.isnan(ref)
    np.testing.assert_allclose(got[fin], ref[fin], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("name", NAMES)
def test_box_torch_ops_rotate_weighted_nms_matches_reference(name):
    from det3d.core.bbox import box_torch_ops
    c = stored_case(name)
    t = lambda a, dt=torch.float32: torch.from_numpy(np.ascontiguousarray(a)).to(dt).cuda()
    b7 = t(c["boxes7"]).reshape(-1, 7)
    res = box_torch_ops.rotate_weighted_nms(b7, b7[:, [0, 1, 3, 4, 6]], t(c["dirs"], torch.int64), t(c["labels"], torch.int64),
                                            t(c["scores"]), t(c["iou_preds"]), t(c["anchors"]).reshape(-1, 7), enable_centerness=True,
                                            centerness_pow=2, pre_max_size=c["pre_max"], post_max_size=100, iou_threshold=0.01)
    boxes, dirs, labels, scores, selected = res
    assert boxes.dtype == torch.float64 and scores.dtype == torch.float64
    assert dirs.dtype == labels.dtype == selected.dtype == torch.int64
    _check_outputs(name, boxes.cpu().numpy(), dirs.cpu().numpy(), labels.cpu().numpy(), scores.cpu().numpy(), selected.cpu().numpy())


@pytest.mark.parametrize("name", [n for n in NAMES if n != "empty"])
def test_sessd_rotate_weighted_nms_matches_reference(name):
    from sessd_b200 import ops
    c = stored_case(name)
    n = len(c["scores"])
    t = lambda a, dt=torch.float32: torch.from_numpy(np.ascontiguousarray(a)).to(dt).cuda()
    b7 = t(c["boxes7"]).reshape(-1, 7)
    from sessd_b200._lib import lib
    pre = min(n, c["pre_max"])
    ws = torch.full((lib.sessd_rotate_weighted_nms_workspace_bytes(n, pre),), POISON, dtype=torch.uint8, device="cuda")
    out = ops.rotate_weighted_nms(b7, b7[:, [0, 1, 3, 4, 6]].contiguous(), t(c["scores"]), t(c["iou_preds"]), t(c["labels"], torch.int32),
                                  t(c["dirs"], torch.int32), t(c["anchors"]).reshape(-1, 7), t([n], torch.int32), n, pre,
                                  ops.make_dinms_cfg(), ws=ws)
    k = int(out["count"][0].item())
    g = {key: v[:k].cpu().numpy() for key, v in out.items() if key != "count"}
    _check_outputs(name, g["boxes"], g["dirs"], g["labels"], g["scores"], g["selected"], g["keep"])
    assert int(out["count"][1].item()) >= k


# ------------------------------------------------------------------------------------------------------------------- head path
FRAMES = ("dense_cluster", "recover", "bands", "duplicates", "scene_64", "scene_65")
PLANES = np.array([[1, 0, 0, -45.0], [-1, 0, 0, -1.0], [0, 1, 0, -100.0], [0, -1, 0, -100.0], [0, 0, 1, -50.0], [0, 0, -1, -50.0]],
                  np.float32)


def _model_robust(r):
    if not r["picks"]:
        return True
    cnt = min(abs(c - dc.CNT) for _, c, _, _ in r["picks"])
    a = np.sort(np.asarray(r["adjusted"], np.float64))
    gap = np.min(np.diff(a) / np.maximum(a[1:], 1e-30)) if len(a) > 1 else 1.0
    return cnt > 1e-4 and gap > 1e-6


@pytest.mark.parametrize("use_frustum", [False, True])
def test_postprocess_dinms_matches_model(use_frustum):
    from sessd_b200 import ops
    heads = [dc.crafted_head(dc.cases()[n][0], seed=i) for i, n in enumerate(FRAMES)]
    anchors = heads[0][1]
    h = np.stack([hd for hd, _ in heads])
    B = len(FRAMES)
    cfg = ops.make_post_cfg(batch=B, head_stride=24, nms_pre_max=1000, direction_offset=0.785, use_frustum=use_frustum,
                            nms_type="rotate_weighted_nms")
    buf = ops.PostBuffers(cfg, "cuda")
    assert buf.boxes.shape == (B, 1000, 7)
    buf.ws.fill_(POISON)
    buf.labels.fill_(7)
    planes = torch.from_numpy(np.stack([PLANES] * B)).cuda() if use_frustum else None
    ops.postprocess(torch.from_numpy(h).cuda(), torch.from_numpy(anchors).cuda(), planes, buf)
    torch.cuda.synchronize()
    total = 0
    for b, name in enumerate(FRAMES):
        r = dc.post_frame_dinms(h[b], anchors, dict(nms_pre_max=1000, direction_offset=0.785), PLANES if use_frustum else None)
        assert _model_robust(r), "crafted head %s is not robust" % name
        k = int(buf.count[b].item())
        assert int(buf.aux[b, 0].item()) == r["n"] and int(buf.aux[b, 1].item()) == r["m"]
        assert int(buf.aux[b, 3].item()) == len(r["picks"])
        assert k == r["count"], name
        assert np.array_equal(buf.sel_anchor[b, :int(buf.aux[b, 2].item())].cpu().numpy() >= 0, np.ones(int(buf.aux[b, 2].item()), bool))
        np.testing.assert_allclose(buf.boxes[b, :k].cpu().numpy(), r["boxes"][:k], rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(buf.scores[b, :k].cpu().numpy(), r["scores"][:k], rtol=1e-5, atol=1e-7)
        assert np.all(buf.labels[b, k:].cpu().numpy() == -1)
        total += k
    assert total > 10


def test_engine_graph_dinms_matches_oracle_frame_path():
    """FrameEngine with nms_type rotate_weighted_nms, captured as a graph, on the bench's ring-20k clouds and weights, against the
    oracle frame path (CPU encoder, neck and head, then the DI-NMS model), matched by pick anchor index"""
    from oracle import frame as oframe
    from sessd_b200 import synth, weights
    from sessd_b200.engine import FrameEngine
    anchors = weights.kitti_car_anchors()
    layers, ssfa, head = weights.bench_detector_state("ring", 0)
    lnp = oframe.layers_to_numpy(layers)
    clouds = [synth.ring_cloud(21, 20000), synth.ring_cloud(22, 18000)]
    eng = FrameEngine(batch=2, max_points_per_frame=20000, post_kwargs={"nms_type": "rotate_weighted_nms"})
    eng.load_weights(layers, ssfa, head, anchors)
    eng.post.ws.fill_(POISON)
    eng.capture()
    res = eng.infer(clouds)
    for f, cloud in enumerate(clouds):
        hd = oframe.frame_head(cloud, lnp, ssfa, head)
        h = np.concatenate([hd["box_preds"][0].numpy().reshape(-1, 14), hd["cls_preds"][0].numpy().reshape(-1, 2),
                            hd["dir_cls_preds"][0].numpy().reshape(-1, 4), hd["iou_preds"][0].numpy().reshape(-1, 2),
                            np.zeros((176 * 200, 2), np.float32)], 1)
        r = dc.post_frame_dinms(h, anchors, dict(nms_pre_max=1000))
        assert r["n"] > 100 and r["count"] > 0, "vacuous test: no DI-NMS detections"
        assert _model_robust(r), "tie-degenerate workload: adjusted scores or cnt within tolerance of each other"
        got = res[f]
        assert got["num_candidates"] == r["n"]
        k = r["count"]
        assert np.array_equal(got["anchor_index"], r["anchor"][:k]), "DI-NMS picks differ (matched by anchor index)"
        fin = ~np.isnan(r["boxes"][:k]).any(1)
        np.testing.assert_allclose(got["box3d_lidar"][fin], r["boxes"][:k][fin], rtol=1e-4, atol=1e-4)
        np.testing.assert_allclose(got["scores"], r["scores"][:k], rtol=1e-4, atol=1e-6)


# ------------------------------------------------------------------------------------------------------------------- argument checks
def test_dinms_entries_reject_bad_arguments():
    from sessd_b200 import ops
    from sessd_b200._lib import lib
    cfg = ops.make_dinms_cfg()
    v = C.c_void_p(16)      # never dereferenced: every call below must fail its argument check first
    z = C.c_void_p(0)
    args = [v] * 8
    for i in range(8):
        a = list(args)
        a[i] = z
        if i == 6:          # anchors may be null only without centerness
            continue
        assert lib.sessd_rotate_weighted_nms(*a, 100, 100, C.byref(cfg), v, v, v, v, v, v, v, v, 1 << 30, z) == -1, i
    assert lib.sessd_rotate_weighted_nms(*args[:6], z, args[7], 100, 100, C.byref(cfg), v, v, v, v, v, v, v, v, 1 << 30, z) == -1
    for j in range(8):
        outs = [v] * 8
        outs[j] = z
        if j == 7:          # workspace: null is a workspace error, checked after the arguments
            continue
        assert lib.sessd_rotate_weighted_nms(*args, 100, 100, C.byref(cfg), *outs[:7], v, 1 << 30, z) == -1, j
    assert lib.sessd_rotate_weighted_nms(*args, 5000, 4097, C.byref(cfg), v, v, v, v, v, v, v, v, 1 << 30, z) == -1
    assert lib.sessd_rotate_weighted_nms(*args, 100, 100, None, v, v, v, v, v, v, v, v, 1 << 30, z) == -1
    pc = ops.make_post_cfg(batch=1, nms_pre_max=4097, nms_type="rotate_weighted_nms")
    assert lib.sessd_postprocess(v, v, z, C.byref(pc), v, v, v, v, v, v, v, 1 << 40, z) == -1
    pc = ops.make_post_cfg(batch=1, nms_type="rotate_weighted_nms")
    pc.nms_mode = 2
    assert lib.sessd_postprocess(v, v, z, C.byref(pc), v, v, v, v, v, v, v, 1 << 40, z) == -1
    pc = ops.make_post_cfg(batch=1, nms_type="rotate_weighted_nms")
    assert lib.sessd_postprocess(z, v, z, C.byref(pc), v, v, v, v, v, v, v, 1 << 40, z) == -1
    with pytest.raises(ValueError):
        ops.make_post_cfg(batch=1, nms_type="nms_gpu")
