"""DI-NMS test inputs and models shared by tests/golden/make_dinms_golden.py, tests/test_dinms_oracle.py and tests/test_gpu_dinms.py.

`iou_matrix` is the exact fp64 BEV IoU of tests/post_model.py over the stand-up-overlapping pairs, with identical rectangles (the
diagonal and duplicate candidates) at exactly 1.  `cases()` builds the crafted stand-alone inputs, each reaching one rule of
nms_cpu.h:173-384; `margins` measures how far a case's decisions lie from their thresholds.  `post_frame_dinms` is one frame of
sessd_postprocess in DI-NMS mode: the post-processing rules of post_model.post_frame around the DI-NMS oracle.
"""
import numpy as np

import post_model as pm
from oracle import dinms_ref

F32 = np.float32
THR, CNT = 0.3, 2.6
EDGES = (0.0, 20.0, 40.0, 60.0)


def iou_matrix(det5):
    """[k, k] fp64 BEV IoU of (x, y, w, l, r) boxes; identical rectangles exactly 1"""
    det5 = np.asarray(det5, F32).reshape(-1, 5)
    k = det5.shape[0]
    m = np.zeros((k, k))
    for (i, j), v in pm.pair_ious(det5).items():
        m[i, j] = m[j, i] = v
    bev = pm.bev_of(det5)
    groups = {}
    for i in range(k):
        groups.setdefault(bev[i].tobytes(), []).append(i)
    for g in groups.values():
        for i in g:
            m[i, g] = 1.0
    return m


def iou_of_boxes7(b7):
    return iou_matrix(np.asarray(b7, F32)[:, [0, 1, 3, 4, 6]])


def margins(case, exempt_pairs=()):
    """(min relative distance of a positive IoU from 0.3, min |cnt - 2.6|, min pick distance from a band edge, min relative gap
    between distinct-by-design adjusted scores), over the case as the oracle runs it"""
    out = run_oracle(case)
    ex = out["extra"]
    b7 = np.asarray(case["boxes7"], F32)[ex["order"]]
    m = iou_of_boxes7(b7) if len(b7) else np.zeros((0, 0))
    order = list(ex["order"])
    exempt = {(order.index(i), order.index(j)) for i, j in exempt_pairs if i in order and j in order}
    exempt |= {(j, i) for i, j in exempt}
    ious = [abs(m[i, j] - THR) / THR for i in range(len(m)) for j in range(len(m)) if i != j and m[i, j] > 0 and (i, j) not in exempt]
    cnts = [abs(c - CNT) for _, c, _, _ in ex["picks"]]
    dists = [min(abs(d - e) for e in EDGES) for _, _, d, _ in ex["picks"]]
    a = np.sort(np.asarray(ex["adjusted"], np.float64))
    gaps = (np.diff(a) / np.maximum(a[1:], 1e-30)) if len(a) > 1 else np.array([1.0])
    return (min(ious, default=1.0), min(cnts, default=1.0), min(dists, default=1.0), float(gaps.min()) if len(gaps) else 1.0)


def run_oracle(case):
    ob, od, ol, os_, sel, extra = dinms_ref.rotate_weighted_nms(case["boxes7"], case["dirs"], case["labels"], case["scores"], case["iou_preds"],
                                                              case["anchors"], iou_of_boxes7, pre_max=case["pre_max"])
    return dict(boxes=ob, dirs=od, labels=ol, scores=os_, selected=sel, keep=extra["keep"], adjusted=extra["adjusted"], extra=extra)


# ------------------------------------------------------------------------------------------------------------------- crafted inputs
def _case(b7, scores, q, labels=None, dirs=None, anchor_off=None, pre_max=1000, seed=0):
    b7 = np.asarray(b7, F32).reshape(-1, 7)
    n = b7.shape[0]
    rng = np.random.default_rng(seed)
    if anchor_off is None:
        anchor_off = rng.uniform(-0.6, 0.6, (n, 2))
    anchors = b7.copy()
    anchors[:, :2] = (b7[:, :2] - np.asarray(anchor_off, np.float64)).astype(F32)
    anchors[:, 3:6] = (1.6, 3.9, 1.56)
    anchors[:, 6] = 0.0
    return dict(boxes7=b7, scores=np.asarray(scores, F32), iou_preds=np.asarray(q, F32),
                labels=np.zeros(n, np.int32) if labels is None else np.asarray(labels, np.int32),
                dirs=rng.integers(0, 2, n).astype(np.int32) if dirs is None else np.asarray(dirs, np.int32),
                anchors=anchors.astype(F32), pre_max=pre_max)


def _box(x, y, w=1.6, l=3.9, r=0.0, z=-1.0, h=1.56):
    return [x, y, z, w, l, h, r]


def _cluster(cx, cy, n, rng, r0=0.0, spread=0.25):
    """n boxes around (cx, cy), the first exactly there; pairwise IoUs well above 0.3"""
    out = [_box(cx, cy, r=r0)]
    for _ in range(n - 1):
        out.append(_box(cx + rng.uniform(-spread, spread), cy + rng.uniform(-spread, spread), r=r0 + rng.uniform(-0.05, 0.05)))
    return out


def _distinct_scores(n, rng, lo=0.35, hi=0.95):
    return np.sort(rng.choice(np.linspace(lo, hi, 20 * n + 1), n, replace=False))[::-1].copy()


def scene(k, seed, pre_max=1000):
    """k boxes in groups of 1-7 on a 5 m grid over the detection range (some groups beyond 60 m), random scores and q"""
    rng = np.random.default_rng(seed)
    b7 = []
    gx, gy = 2.0, -38.0
    while len(b7) < k:
        n = min(int(rng.integers(1, 8)), k - len(b7))
        b7 += _cluster(gx + rng.uniform(-0.5, 0.5), gy + rng.uniform(-0.5, 0.5), n, rng, r0=rng.choice([0.0, 0.3, 1.57]),
                       spread=rng.uniform(0.1, 0.7))
        gx += 5.0
        if gx > 68.0:
            gx, gy = 2.0, gy + 5.0
    b7 = np.asarray(b7)
    perm = rng.permutation(k)
    # score steps of >= 0.3 / k and centre-anchor distances within 2 cm of each other keep the adjusted scores apart by > 1e-5
    sc = rng.choice(np.linspace(0.35, 0.95, 2 * k + 1), k, replace=False)
    ang = rng.uniform(-np.pi, np.pi, k)
    rad = rng.uniform(0.30, 0.32, k)
    off = np.stack([rad * np.cos(ang), rad * np.sin(ang)], 1)
    return _case(b7[perm], sc, rng.uniform(0.55, 1.0, k), anchor_off=off, pre_max=pre_max, seed=seed)


def cases():
    """name -> (case, pairs exempt from the IoU margin)"""
    out = {}
    rng = np.random.default_rng(7)
    # a dense cluster that is kept, two singletons that never are
    b7 = _cluster(15.0, 4.0, 6, rng) + [_box(30.0, -10.0), _box(40.0, 12.0)]
    out["dense_cluster"] = (_case(b7, _distinct_scores(8, rng), rng.uniform(0.8, 0.95, 8), seed=1), ())
    # a pick whose cnt fails (its members are recovered) next to boxes that then form a cluster around its runner-up, which the
    # failed, already suppressed pick joins: it raises the cluster's score_box and enters its average
    b7 = [_box(10.0, -3.0), _box(10.5, -2.97), _box(10.8, -2.99), _box(11.0, -3.03), _box(10.65, -2.95)]
    out["recover"] = (_case(b7, [0.9, 0.8, 0.7, 0.6, 0.5], [0.9, 0.97, 0.97, 0.97, 0.97], seed=2), ())
    # picks in each distance band, one exactly at 20 m ((12, 16)), one beyond 60 m (NaN box)
    b7, sc = [], []
    for i, (x, y) in enumerate(((8.0, 6.0), (12.0, 16.0), (24.5, 18.2), (48.3, 14.1), (63.0, 16.0))):
        b7 += _cluster(x, y, 5, rng, r0=0.2 * i)
        sc += list(np.linspace(0.9 - 0.1 * i, 0.82 - 0.1 * i, 5))
    out["bands"] = (_case(b7, sc, rng.uniform(0.85, 0.98, len(b7)), seed=3), ())
    # axis-aligned dyadic boxes: A meets B at IoU exactly 3/10, whose fp32 value is fl(0.3): B is suppressed but not a member
    A = _box(10.0, 9.0, 4.0, 2.0)
    b7 = [A, _box(10.125, 9.0625, 4.0, 2.0), _box(9.875, 8.9375, 4.0, 2.0), _box(11.5, 9.0, 2.0, 2.5)]
    out["exact_thresh_pair"] = (_case(b7, [0.9, 0.8, 0.7, 0.6], [0.9, 0.9, 0.9, 0.9], seed=4), ((0, 3),))
    # duplicate rectangles inside a kept cluster
    b7 = _cluster(20.0, -8.0, 4, rng)
    b7 = b7 + [list(b7[1]), list(b7[2])]
    out["duplicates"] = (_case(b7, [0.9, 0.85, 0.8, 0.75, 0.7, 0.65], [0.9, 0.8, 0.95, 0.7, 0.85, 0.9], seed=5), ())
    # two labels interleaved in score order over the same objects (suppression ignores labels, clusters do not)
    b7 = _cluster(18.0, 2.0, 8, rng, spread=0.2) + _cluster(26.0, -4.0, 6, rng, spread=0.2)
    out["labels"] = (_case(b7, _distinct_scores(14, rng), rng.uniform(0.9, 1.0, 14), labels=np.arange(14) % 2, seed=6), ())
    # equal input scores and equal centre-anchor distances: equal adjusted scores, the first position wins
    b7 = _cluster(12.0, 5.0, 4, rng) + _cluster(12.0, -15.0, 4, rng)
    sc = [0.8, 0.7, 0.6, 0.5, 0.8, 0.7, 0.6, 0.5]
    off = np.tile([[0.2, 0.1], [0.3, -0.1], [-0.2, 0.25], [0.05, 0.4]], (2, 1))
    out["equal_scores"] = (_case(b7, sc, np.full(8, 0.95), anchor_off=off, seed=7), ())
    # n > pre_max, n = 1, n = 0
    c = scene(50, 11, pre_max=40)
    out["pre_max_cut"] = (c, ())
    out["single"] = (_case([_box(10.0, 0.0)], [0.7], [0.9], seed=8), ())
    out["empty"] = (_case(np.zeros((0, 7)), [], [], seed=9), ())
    # tile and warp edges of the overlap stage and the loop
    for k, seed in ((31, 31), (32, 32), (33, 33), (64, 64), (65, 65), (1000, 1000)):
        out["scene_%d" % k] = (scene(k, seed), ())
    return out


EQUAL_SCORE_CASES = ("equal_scores",)


# ------------------------------------------------------------------------------------------------------------------- head path model
def post_frame_dinms(head, anchors, cfg=None, planes=None):
    """one frame of sessd_postprocess with nms_type rotate_weighted_nms: candidates and top-k as post_model.post_frame, then
    centerness + the DI-NMS loop (oracle) on the decoded boxes, then frustum on the averaged centres, direction flip (averaged yaw,
    the pick's direction label), inclusive range mask, ordered compaction; capacity K = nms_pre_max."""
    c = dict(pm.POST_DEFAULTS)
    c.update(cfg or {})
    K = c["nms_pre_max"]
    h = np.asarray(head, F32)
    A = h.shape[0] * 2
    pix, r = np.arange(A) // 2, np.arange(A) % 2
    logit = h[pix, pm.Head.CLS + r]
    cand = np.nonzero(pm.sigmoid64(logit) >= c["score_thresh"])[0]
    q = (h[pix[cand], pm.Head.IOU + r[cand]] + F32(1)) * F32(0.5)
    q2 = q * q
    score = (pm.sigmoid64(logit[cand]) * (q2 * q2).astype(np.float64)).astype(F32)
    order = pm.score_order(score)[:K]
    sel = cand[order]
    m = len(sel)
    t = h[pix[sel][:, None], 7 * r[sel][:, None] + np.arange(7)[None]]
    box, _ = pm.decode32(t, anchors[sel])
    dirl = (h[pix[sel], pm.Head.DIR + 2 * r[sel] + 1] > h[pix[sel], pm.Head.DIR + 2 * r[sel]]).astype(np.int64)
    out = dict(count=0, n=len(cand), m=m, boxes=np.zeros((K, 7), F32), scores=np.zeros(K, F32), anchor=np.full(K, -1, np.int64), picks=[])
    if m == 0:
        return out
    adj = dinms_ref.centerness(box, anchors[sel], score[order], 2)
    ob, os_, _ol, od, keep, picks = dinms_ref.dinms_core(box, adj, q[order], np.zeros(m, np.int64), dirl, iou_of_boxes7(box),
                                                         **dinms_ref.HEAD_CONSTANTS)
    out.update(picks=picks, adjusted=adj, box=box, nk=len(keep))
    ok = np.ones(len(keep), bool)
    with np.errstate(invalid="ignore"):
        if planes is not None:
            ok &= pm.frustum_ok(ob[:, :3], planes)
        rr = ob[:, 6] - F32(c["direction_offset"])
        opp = (rr > 0) != (od == 1)
        rng = np.asarray(c["post_range"], F32)
        ok &= np.all((ob[:, :3] >= rng[:3]) & (ob[:, :3] <= rng[3:]), 1)
    passed = np.nonzero(ok)[0]
    out["count"] = len(passed)
    for dst, i in enumerate(passed):
        b = ob[i].copy()
        if opp[i]:
            b[6] = b[6] + pm.PI32
        out["boxes"][dst] = b
        out["scores"][dst] = os_[i]
        out["anchor"][dst] = sel[keep[i]]
    return out


def crafted_head(case, seed=0):
    """a head whose candidates decode near the case's boxes (one anchor per box, logits giving the case's score order), with
    iou-head values giving its q; returns (head, anchors)"""
    anchors = pm.kitti_anchors()
    b7 = np.asarray(case["boxes7"], np.float64)
    n = b7.shape[0]
    rng = np.random.default_rng(seed)
    # the anchor whose centre is nearest each box centre, a distinct one per box, rotation 0 (even anchor index)
    used = set()
    idx = []
    for i in range(n):
        col = min(max(int(round(b7[i, 0] / 0.4 - 0.5)), 0), 175)
        row = min(max(int(round((b7[i, 1] + 40.0) / 0.4 - 0.5)), 0), 199)
        a = (row * 176 + col) * 2
        while a in used:
            a = (a + 2) % anchors.shape[0]
        used.add(a)
        idx.append(a)
    idx = np.array(idx)
    enc = pm.encode(b7, anchors[idx])
    s = np.asarray(case["scores"], np.float64)
    logit = np.log(s / (1 - s)).astype(F32) + F32(1.5)
    iou = (2 * np.asarray(case["iou_preds"], np.float64) - 1).astype(F32)
    hd = pm.Head(anchors)
    hd.place(idx, enc, logit, iou, rng.normal(0, 1, (n, 2)).astype(F32))
    return hd.h, anchors
