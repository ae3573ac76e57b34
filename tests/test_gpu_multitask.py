"""Multi-class inference on the device: the head GEMM of three tasks against an fp64 1x1 conv and against one-task runs, the
post-processing of T tasks against T one-task calls (and through them the fp64 oracle of tests/post_model.py), FrameEngine at T = 3
against T = 1, and kitti_test.evaluate with a three-class config."""
import os

import numpy as np
import pytest
import torch

import multitask_cases as mc
import post_model as pm
from test_gpu_postproc_ops import _check, _frame_out, _run

pytestmark = pytest.mark.gpu
PREFIXES = ["tasks.0.", "tasks.1.", "tasks.2."]


def _head_sd(seed, T=3):
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for t in range(T):
        for nm, co in (("conv_box", 14), ("conv_cls", 2), ("conv_dir", 4), ("conv_iou", 2)):
            sd["tasks.%d.%s.weight" % (t, nm)] = torch.randn((co, 128, 1, 1), generator=g) / 11.3
            sd["tasks.%d.%s.bias" % (t, nm)] = 0.1 * torch.randn(co, generator=g)
    return sd


def test_head_three_tasks_one_gemm():
    """T = 3 head output against the fp64 1x1 conv, every task's block against a one-task run with that task's weights (bit for
    bit: the same input planes and per-channel weight splits, and the same K order per output channel), zero padding channels"""
    from sessd_b200.runners import HeadRunner, pack_head
    g = torch.Generator().manual_seed(7)
    x = torch.randn((2, 40, 56, 128), generator=g)
    sd = _head_sd(1)
    r3 = HeadRunner(2, (40, 56), "cuda", num_tasks=3)
    r3.load_state(sd, PREFIXES)
    h3 = r3.forward(x.cuda()).clone().cpu().double()
    assert h3.shape == (2, 40, 56, 72) and r3.HEAD_STRIDE == 72
    w, b = pack_head(sd, PREFIXES, "cpu")
    w2 = w[:, :, 0, 0].double()
    ref = x.double() @ w2.T + b.double()
    tol = 2.0 ** -19 * (x.double().abs() @ w2.abs().T) + 2.0 ** -22 * b.double().abs() + 1e-7
    assert torch.all((h3 - ref).abs() <= tol), float(((h3 - ref).abs() / tol).max())
    for t in range(3):
        r1 = HeadRunner(2, (40, 56), "cuda")
        r1.load_state(sd, PREFIXES[t])
        h1 = r1.forward(x.cuda()).clone().cpu().double()
        blk = h3[..., 24 * t:24 * t + 24]
        assert torch.all(blk[..., 22:] == 0)
        assert torch.equal(blk, h1), (t, float((blk - h1).abs().max()))


def _engine_states():
    from sessd_b200 import weights
    layers, ssfa, head = weights.bench_detector_state("ring", 0)
    head3 = dict(head)
    for t in (1, 2):       # two more tasks from the car head's scale, with their own bias and weights
        for k, v in head.items():
            if k.startswith("tasks.0."):
                nk = k.replace("tasks.0.", "tasks.%d." % t)
                head3[nk] = v * (1.0 - 0.05 * t) if k.endswith("weight") else v + 0.2 * t
    return layers, ssfa, head, head3


def test_engine_three_tasks_car_block_equals_one_task():
    from sessd_b200 import weights
    from sessd_b200.engine import FrameEngine
    from sessd_data import synth
    layers, ssfa, head, head3 = _engine_states()
    anchors = weights.task_anchors(dict(anchor_generators=mc.GENERATORS, tasks=mc.TASKS))
    e1 = FrameEngine(batch=2, max_points_per_frame=20000)
    e1.load_weights(layers, ssfa, head, anchors[0])
    e3 = FrameEngine(batch=2, max_points_per_frame=20000, num_tasks=3)
    e3.load_weights(layers, ssfa, head3, anchors)
    seen = set()
    for seed in (3, 4):
        clouds = [synth.ring_cloud(seed * 10 + f, 20000) for f in range(2)]
        r1, r3 = e1.infer(clouds), e3.infer(clouds)
        for a, b in zip(r1, r3):
            car = b["label_preds"] == 0
            assert np.all(np.diff(b["label_preds"]) >= 0)                   # task order
            assert np.array_equal(a["box3d_lidar"].view(np.uint32), b["box3d_lidar"][car].view(np.uint32))
            assert np.array_equal(a["scores"].view(np.uint32), b["scores"][car].view(np.uint32))
            assert np.array_equal(a["anchor_index"], b["anchor_index"][car]) and np.all(a["label_preds"] == 0)
            assert np.array_equal(b["label_preds"], b["anchor_index"] // 70400)
            seen |= set(b["label_preds"].tolist())
    assert seen == {0, 1, 2}
    # constant-region skipping fills all three blocks: bit-identical to the dense head
    e3d = FrameEngine(batch=2, max_points_per_frame=20000, num_tasks=3, skip_constant=False)
    e3d.load_weights(layers, ssfa, head3, anchors)
    clouds = [synth.ring_cloud(50 + f, 20000) for f in range(2)]
    heads = []
    for e in (e3, e3d):
        e.stage(clouds)
        e.d_points.copy_(e.h_points)
        e.d_off.copy_(e.h_off)
        from sessd_b200 import ops
        ops.voxelize(e.d_points, e.d_off, e.vox)
        heads.append(e.sparse_and_neck().clone())
    torch.cuda.synchronize()
    assert heads[0].shape[-1] == 72 and torch.equal(heads[0], heads[1])


# ------------------------------------------------------------------------------------------------------------ post-processing
def _task_heads():
    """per-task crafted heads (tests/post_model.frame): a task with many candidates, an empty task, a task at exactly nms_post_max
    detections (far-apart boxes), and a copy of the first task (equal scores across tasks)"""
    many, _ = pm.frame(n=300, K=1000, P=20, pattern="chain", seed=1)
    empty, _ = pm.frame(n=0, K=1000, P=20)
    exact, _ = pm.frame(n=20, K=1000, P=20, pattern="far", seed=2)
    return [many, empty, exact, many.copy()]


def _post(heads, anchors, T, nms_type, planes=None, P=20):
    from sessd_b200 import ops
    B = len(heads)
    cfg = ops.make_post_cfg(batch=B, head_stride=24 * T, nms_pre_max=1000, nms_post_max=P, use_frustum=planes is not None,
                            nms_type=nms_type, num_tasks=T)
    Pc = ops.post_capacity(cfg)
    buf = ops.PostBuffers(cfg, "cuda")
    packed = torch.full((B, Pc, 8), float("nan"), device="cuda")
    meta = torch.full((B, 8 + Pc), -7, dtype=torch.int32, device="cuda")
    hd = torch.from_numpy(np.ascontiguousarray(np.stack(heads))).cuda()
    an = torch.from_numpy(np.ascontiguousarray(np.concatenate(anchors))).cuda()
    pl = None if planes is None else torch.from_numpy(np.stack(planes)).cuda()
    ops.postprocess_packed(hd, an, pl, buf, packed, meta, torch.tensor([5, 6][:B], dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    return {k: getattr(buf, k).cpu().numpy() for k in ("boxes", "scores", "labels", "count", "aux", "sel_anchor")} | \
        dict(packed=packed.cpu().numpy(), meta=meta.cpu().numpy())


@pytest.mark.parametrize("nms_type", ["rotate_nms", "rotate_weighted_nms"])
@pytest.mark.parametrize("frustum", [False, True])
def test_tasks_equal_one_task_calls_concatenated(nms_type, frustum):
    tasks = _task_heads()
    T = len(tasks)
    base = pm.kitti_anchors()
    anchors = [base.copy() for _ in range(T)]
    for t in range(T):
        anchors[t][:, 0] += np.float32(0.25 * t)        # every task decodes against its own anchors
    # two frames: the second with the tasks rotated, so a frame's slots do not leak into another's
    frames = [tasks, tasks[1:] + tasks[:1]]
    fr_anchors = anchors
    planes = None
    if frustum:
        pl = np.array([[1, 0, 0, -40], [-1, 0, 0, -100], [0, 1, 0, -100], [0, -1, 0, -100], [0, 0, 1, -100], [0, 0, -1, -100]],
                      np.float32)
        planes = [pl, pl]
    heads = [np.concatenate(f, 1) for f in frames]
    out = _post(heads, fr_anchors, T, nms_type, planes)
    P = out["boxes"].shape[1] // T
    A = base.shape[0]
    for b, f in enumerate(frames):
        singles = [_post([f[t]], [fr_anchors[t]], 1, nms_type, None if planes is None else [planes[b]]) for t in range(T)]
        cnt = [int(s["count"][0]) for s in singles]
        total = sum(cnt)
        assert int(out["count"][b]) == total
        cat = lambda k: np.concatenate([s[k][0][:c] for s, c in zip(singles, cnt)])  # noqa: E731
        assert out["boxes"][b][:total].tobytes() == cat("boxes").tobytes()
        assert out["scores"][b][:total].tobytes() == cat("scores").tobytes()
        assert np.array_equal(out["labels"][b][:total], np.repeat(np.arange(T), cnt))
        assert np.all(out["labels"][b][total:] == -1) and not np.any(out["boxes"][b][total:]) and not np.any(out["scores"][b][total:])
        assert np.array_equal(out["meta"][b][8:8 + total], np.concatenate([s["meta"][0][8:8 + c] + t * A for t, (s, c) in
                                                                            enumerate(zip(singles, cnt))]))
        assert np.all(out["meta"][b][8 + total:] == -1) and not np.any(out["packed"][b][total:])
        assert out["packed"][b][:total, :7].tobytes() == out["boxes"][b][:total].tobytes()
        aux = np.stack([s["aux"][0] for s in singles])
        assert np.array_equal(out["aux"][b * T:(b + 1) * T], aux)
        assert out["meta"][b][:8].tolist() == [total, aux[:, 0].sum(), aux[:, 1].sum(), aux[:, 2].sum(), 5 + b, 0, 0, 0]
        for t, s in enumerate(singles):
            sel = s["sel_anchor"][0]
            assert np.array_equal(out["sel_anchor"][b][t * P:(t + 1) * P], np.where(sel >= 0, sel + t * A, -1))
        if nms_type == "rotate_nms" and b == 0:
            assert cnt[1] == 0 and cnt[0] == cnt[3] > 0 and int(singles[2]["aux"][0][2]) == P     # empty, tie copy, at the cap
            # the one-task calls against the fp64 oracle (tests/post_model.py), hence the T-task call too
            for t, s in enumerate(singles):
                mdl = pm.post_frame(f[t], fr_anchors[t], dict(nms_pre_max=1000, nms_post_max=P),
                                    None if planes is None else planes[b])
                if pm.robust(mdl["ious"], 0.01) and mdl["clear"]:
                    _check(_frame_out(dict(s, sel=s["sel_anchor"]), 0), mdl, 5)


def test_postprocess_rejects_bad_task_layouts():
    import ctypes as C
    from sessd_b200 import ops
    from sessd_b200._lib import lib
    v = C.c_void_p(1)
    for T, stride, hs in ((3, 20, 72), (3, 24, 69), (-1, 24, 24), (65, 24, 24 * 65)):
        c = ops.make_post_cfg(batch=1, head_stride=24)
        c.num_tasks, c.task_stride, c.head_stride = T, stride, hs
        assert lib.sessd_postprocess(v, v, None, C.byref(c), v, v, v, v, v, v, v, 1 << 40, None) == -1, (T, stride, hs)


# ------------------------------------------------------------------------------------------------------------ KITTI evaluation
@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    from sessd_b200.kitti_prep import kitti_data_prep
    from test_gpu_kitti_train import _write_tree
    root = str(tmp_path_factory.mktemp("kitti_multitask"))
    _write_tree(root, n_train=2, n_val=4)
    kitti_data_prep(root)
    return root


def test_kitti_evaluate_three_classes(tree, tmp_path):
    from det3d.datasets import build_dataset
    from sessd_b200 import kitti_test, weights
    cfg = mc.three_class_config(tree)
    cfg.data.samples_per_gpu = 2
    sd = weights.add_task_heads(weights.random_detector_state(0), 3, seed=2)
    ck = str(tmp_path / "three.pth")
    torch.save({"state_dict": sd}, ck)
    results, predictions = kitti_test.evaluate(cfg, ck)
    for key, name in (("results", "official_AP_11"), ("results_2", "official_AP_40")):
        text = results[key][name]
        assert all(n.lower() + " ap" in text.lower() for n in mc.NAMES), text
    assert len(predictions) == 4
    labels = np.concatenate([p["label_preds"].cpu().numpy() for p in predictions.values()])
    assert set(labels.tolist()) == {0, 1, 2}
    ds = build_dataset(cfg.data.val)
    annos = ds.convert_detection_to_kitti_annos(predictions)
    for a in annos:
        tok = str(a["metadata"]["token"]) if "metadata" in a else None
        if tok is None:
            continue
        p = predictions[tok]
        assert set(a["name"].tolist()) <= {mc.NAMES[int(l)] for l in p["label_preds"].cpu().numpy()}
