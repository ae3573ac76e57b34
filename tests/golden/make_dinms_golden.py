"""Generate tests/golden/dinms_cases.npz by running the reference's own DI-NMS Python in place:
box_torch_ops.rotate_weighted_nms (top-k, centerness) and nms_cpu.rotate_weighted_nms_cc (corners, corner_to_standup_nd, numba
iou_jit).  Only the compiled extension det3d.ops.nms.nms (boost::geometry) is stubbed: its IOU_weighted_rotate_non_max_suppression_cpu
is bound to oracle/dinms_ref.dinms_core with the exact fp64 IoUs of tests/dinms_cases.iou_matrix; nms_gpu is stubbed as
make_golden.py does.  The stub checks that the reference's corners are the rectangles the IoUs are taken of.

    python tests/golden/make_dinms_golden.py

Stored per case: the inputs, the reference's adjusted scores (centerness applied, top-k order) and its five outputs.  The margins of
every case (tests/dinms_cases.margins) are asserted here.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "se-ssd_b200"), os.path.join(ROOT, "tests"), HERE]

import make_golden as mg  # noqa: E402
import dinms_cases as dc  # noqa: E402
from oracle import dinms_ref  # noqa: E402

ADJUSTED = {}


def _core(box, corners, standup_iou, thresh, scores, iou_preds, labels, dirs, anchors, cnt_thresh, interval, sigma2, supp, centerness_c):
    assert centerness_c == 0
    b7 = np.asarray(box, np.float32)
    ref = mg._load("bn_check", "det3d/core/bbox/box_np_ops.py").center_to_corner_box2d(b7[:, :2], b7[:, 3:5], b7[:, 6])
    assert np.allclose(ref, corners, atol=1e-5), "rbboxes are not box_preds[:, [0, 1, 3, 4, 6]]"
    ADJUSTED["last"] = np.asarray(scores, np.float32).copy()
    ob, os_, ol, od, keep, _ = dinms_ref.dinms_core(b7, scores, iou_preds, labels, dirs, dc.iou_of_boxes7(b7), cnt_thresh=cnt_thresh,
                                                    dist_edge=tuple(interval), sigma2=tuple(sigma2), suppressed_thresh=supp)
    return [[list(map(float, r)) for r in ob], [float(v) for v in os_], [int(v) for v in ol], [int(v) for v in od], [int(v) for v in keep]]


def main():
    mg.install_det3d_shims()
    sys.modules["det3d.ops.nms"].__path__ = [os.path.join(mg.REF, "det3d/ops/nms")]
    mg._stub("det3d.ops.nms.nms", non_max_suppression_cpu=None, rotate_non_max_suppression_cpu=None,
             IOU_weighted_rotate_non_max_suppression_cpu=_core)
    bn = mg._load("det3d.core.bbox.box_np_ops", "det3d/core/bbox/box_np_ops.py")
    sys.modules["det3d.core.bbox"].box_np_ops = bn
    nc = mg._load("det3d.ops.nms.nms_cpu", "det3d/ops/nms/nms_cpu.py")
    sys.modules["det3d.ops.nms"].nms_cpu = nc
    bt = mg._load("det3d.core.bbox.box_torch_ops", "det3d/core/bbox/box_torch_ops.py")
    torch.Tensor.cuda = lambda self, *a, **k: self          # the wrapper moves its results to the GPU; keep them here
    out = {}
    for name, (c, exempt) in dc.cases().items():
        m_iou, m_cnt, m_dist, m_gap = dc.margins(c, exempt)
        assert m_iou >= 1e-4 and m_cnt >= 1e-4, (name, m_iou, m_cnt)
        if name != "bands":             # bands has its pick exactly at 20.0 m on purpose
            assert m_dist >= 1e-3, (name, m_dist)
        if name not in dc.EQUAL_SCORE_CASES:
            assert m_gap > 1e-5, (name, m_gap)
        n = len(c["scores"])
        t = lambda a, dt=torch.float32: torch.from_numpy(np.ascontiguousarray(a)).to(dt)
        b7 = t(c["boxes7"]).reshape(-1, 7)
        ADJUSTED.pop("last", None)
        res = bt.rotate_weighted_nms(b7, b7[:, [0, 1, 3, 4, 6]], t(c["dirs"], torch.int64), t(c["labels"], torch.int64), t(c["scores"]),
                                     t(c["iou_preds"]), t(c["anchors"]).reshape(-1, 7), enable_centerness=True, centerness_pow=2,
                                     pre_max_size=c["pre_max"], post_max_size=100, iou_threshold=0.01) if n else None
        for k, v in c.items():
            out["%s__in_%s" % (name, k)] = np.asarray(v)
        if res is None:                 # the reference returns None for n == 0 (its caller's unpacking fails there)
            res = (np.zeros((0, 7)), np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0), np.zeros(0, np.int64))
        boxes, dirs, labels, scores, selected = [np.asarray(r) for r in res]
        mine = dc.run_oracle(c)
        assert np.array_equal(selected.astype(np.int64), mine["selected"]), (name, selected, mine["selected"])   # topk ties as the device
        out["%s__adjusted" % name] = ADJUSTED.get("last", np.zeros(0, np.float32))
        out["%s__boxes" % name] = boxes.reshape(-1, 7)
        out["%s__dirs" % name] = dirs.astype(np.int64)
        out["%s__labels" % name] = labels.astype(np.int64)
        out["%s__scores" % name] = scores.astype(np.float64)
        out["%s__selected" % name] = selected.astype(np.int64)
        out["%s__keep" % name] = mine["keep"]
        print("%-18s n=%4d kept=%3d picks=%3d nan=%d margins iou %.1e cnt %.1e dist %.1e gap %.1e" % (
            name, n, len(selected), len(mine["extra"]["picks"]), int(np.isnan(boxes).any(-1).sum()) if len(boxes) else 0,
            m_iou, m_cnt, m_dist, m_gap))
    np.savez_compressed(os.path.join(HERE, "dinms_cases.npz"), names=np.array(list(dc.cases().keys())), **out)


if __name__ == "__main__":
    main()
