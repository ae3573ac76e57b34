"""DI-NMS restated (TEST INFRASTRUCTURE ONLY, never imported by the product): the top-k and centerness of
box_torch_ops.rotate_weighted_nms (det3d/core/bbox/box_torch_ops.py:552-621) and the C core
IOU_weighted_rotate_non_max_suppression_cpu (det3d/ops/nms/nms_cpu.h:173-384), loop for loop, in the core's fp32 arithmetic.

The core receives the IoU of every pair as a dense [k, k] matrix from the caller (the tests build it with the exact fp64 clip of
tests/post_model.py, identical rectangles at exactly 1) and rounds it to fp32, the reference's DType.  The C core's own centerness
(centerness_c == 1) never runs in the reference -- the wrapper passes anchors=None -- and is not restated.
"""
import math

import numpy as np

F32 = np.float32

HEAD_CONSTANTS = dict(cnt_thresh=2.6, dist_edge=(0.0, 20.0, 40.0, 60.0), sigma2=(0.0009, 0.009, 0.1, 1.0), suppressed_thresh=0.3)


def topk_order(scores, pre_max=None):
    """torch.topk order: descending score; equal scores keep the lower index first (the device's key order)"""
    s = np.asarray(scores, np.float64)
    order = np.lexsort((np.arange(s.shape[0]), -s))
    return order if pre_max is None else order[:min(len(order), int(pre_max))]


def centerness(boxes7, anchors, scores, centerness_pow=2):
    """box_torch_ops.py:584-588 in fp32: scores * (1 - softmax(|centre - anchor centre|))^pow over the k boxes"""
    b = np.asarray(boxes7, F32)
    a = np.asarray(anchors, F32)
    dx, dy = np.abs(b[:, 0] - a[:, 0]), np.abs(b[:, 1] - a[:, 1])
    d = np.sqrt(dx * dx + dy * dy).astype(F32)
    e = np.exp((d - d.max()).astype(F32)).astype(F32)
    m = (e / e.sum(dtype=F32)).astype(F32)
    t = (F32(1) - m).astype(F32)
    p = t * t if centerness_pow == 2 else np.power(t, F32(centerness_pow))
    return (np.asarray(scores, F32) * p.astype(F32)).astype(F32)


def dinms_core(boxes7, scores, q, labels, dirs, iou, cnt_thresh=2.6, dist_edge=(0.0, 20.0, 40.0, 60.0), sigma2=(0.0009, 0.009, 0.1, 1.0),
               suppressed_thresh=0.3):
    """nms_cpu.h:173-384 with centerness_c == 0.  boxes7 [k,7], scores [k] (the adjusted scores: they decide the pick order),
    q [k] rectified IoU predictions, labels, dirs [k], iou [k,k] (any float type; rounded to fp32).
    Returns (boxes [K,7] f32, scores [K] f32, labels [K], dirs [K], keep [K] positions, picks) where picks lists, per iteration,
    (idx, cnt, dist, kept)."""
    box = np.asarray(boxes7, F32).reshape(-1, 7)
    s = np.asarray(scores, F32)
    q = np.asarray(q, F32)
    lab = np.asarray(labels)
    n = s.shape[0]
    ov = np.asarray(iou, np.float64).reshape(n, n).astype(F32)
    thr = F32(suppressed_thresh)
    smax = s.max() if n else F32(0)
    with np.errstate(invalid="ignore", divide="ignore"):       # one box: centerness makes its score 0, and 0 / 0 as in the reference
        s_norm = (s / smax).astype(F32)
    supp = np.zeros(n, bool)
    out_b, out_s, out_l, out_d, keep, picks = [], [], [], [], [], []
    while True:
        live = np.nonzero(~supp)[0]
        if live.size == 0:
            break
        idx = int(live[np.argmax(s[live])])                 # strict '>': the first position wins a tie
        dist = F32(math.sqrt(float(box[idx, 0]) ** 2 + float(box[idx, 1]) ** 2))
        supp[idx] = True
        s2 = None
        for k in range(len(dist_edge) - 1):
            if F32(dist_edge[k]) <= dist < F32(dist_edge[k + 1]):
                s2 = F32(sigma2[k])
        avg = np.zeros(7, F32)
        wsum = F32(0)
        score_box = F32(-1)
        cnt = F32(0)
        rec = []
        for j in np.nonzero(ov[idx] > 0)[0]:                 # a pair with IoU <= 0 changes nothing (every test below needs o > 0)
            o = ov[idx, j]
            same = lab[j] == lab[idx]
            if o > 0 and same:
                cnt = F32(cnt + o * q[j])
            if o > thr and same:
                score_box = max(score_box, s_norm[j])
                w = F32(math.exp(-float(F32(1) - o) ** 2 / float(s2))) if s2 is not None else F32(0)
                wq = F32(w * q[j])
                avg = (avg + wq * box[j]).astype(F32)
                wsum = F32(wsum + wq)
            if not supp[j] and o >= thr:                    # IoU >= thr > 0 implies overlapping stand-up boxes
                supp[j] = True
                rec.append(j)
        kept = bool(cnt > F32(cnt_thresh))
        picks.append((idx, float(cnt), float(dist), kept))
        if kept:
            with np.errstate(invalid="ignore", divide="ignore"):
                out_b.append((avg / wsum).astype(F32))
            out_s.append(F32(score_box * smax))
            out_l.append(int(lab[idx]))
            out_d.append(int(np.asarray(dirs)[idx]))
            keep.append(idx)
        else:
            supp[rec] = False
    return (np.array(out_b, F32).reshape(-1, 7), np.array(out_s, F32), np.array(out_l, np.int64), np.array(out_d, np.int64),
            np.array(keep, np.int64), picks)


def rotate_weighted_nms(boxes7, dir_labels, labels, scores, q, anchors, iou_fn, pre_max=None, enable_centerness=True, centerness_pow=2,
                        **constants):
    """the wrapper: top-k, centerness, core.  iou_fn(boxes7 in top-k order) -> [k, k] IoU matrix.  Returns (boxes, dirs, labels,
    scores, selected, extra) with extra = dict(order, adjusted, keep, picks)."""
    c = dict(HEAD_CONSTANTS)
    c.update(constants)
    order = topk_order(scores, pre_max)
    b = np.asarray(boxes7, F32).reshape(-1, 7)[order]
    s = np.asarray(scores, F32)[order]
    if len(order) == 0:
        z = np.zeros(0, np.int64)
        return np.zeros((0, 7), F32), z, z, np.zeros(0, F32), z, dict(order=order, adjusted=s, keep=z, picks=[])
    if enable_centerness:
        s = centerness(b, np.asarray(anchors, F32)[order], s, centerness_pow)
    ob, os_, ol, od, keep, picks = dinms_core(b, s, np.asarray(q, F32)[order], np.asarray(labels)[order], np.asarray(dir_labels)[order],
                                              iou_fn(b), **c)
    return ob, od, ol, os_, order[keep], dict(order=order, adjusted=s, keep=keep, picks=picks)
