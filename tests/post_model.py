"""CPU restatement of detection post-processing (csrc/postproc.cu) and exact rotated-box geometry (csrc/rotbox.cuh), with
generators of crafted box sets and head maps.  Used by tests/test_post_model.py (CPU) and tests/test_gpu_postproc_ops.py.

Geometry.  `overlap64` clips the two rotated rectangles exactly in fp64 (Sutherland-Hodgman on the corners the reference's
spin produces, with cos/sin in fp64) and `iou_bev64` / `iou3d64` build the IoUs from it as rotbox.cuh does
(union clamped at 1e-8, the 3-D height overlap clamped at 1e-8 and treated as no overlap there).

NMS.  `greedy` is the suppression rule of nms_cpu.h / box_torch_ops.rotate_nms over a sparse pair list: candidates in score
order (equal scores: lower index first), a kept box suppresses every later box whose IoU with it is >= thr (or > thr), stop
after `cap` kept boxes.  Pairs are only those whose stand-up boxes overlap; the decision uses float32(exact IoU), which is
what the device computes whenever the arithmetic is exact (angle 0, dyadic coordinates) and is otherwise irrelevant because
every crafted pair is robust: its exact IoU is at least MARGIN (relative) away from the threshold, and no corner of an
overlapping pair lies within 1e-3 of the other box's boundary.  `mask_words` /
`scan_words` restate the device's 64-bit suppression words (two 32-bit tile halves per word, the diagonal word's low half
zeroed by the tile below the diagonal, unwritten halves poisoned here) and its block-wise greedy scan; they exist to make
the negative controls of the layout meaningful.

Post-processing.  `post_frame` restates one frame of sessd_postprocess: candidates sigmoid(cls) >= thr, score
sigmoid * q^4 with q = (iou + 1) / 2, top-K, decode, NMS capped at P, frustum (a plane sign >= 0 rejects), direction flip
((r - offset) > 0 differs from dir == 1: add float32(pi)), inclusive range mask, ordered compaction, padding 0 / -1.
x, y, z, r use only IEEE mul/add/sqrt (postproc.cu is compiled with -fmad=false), so they are emulated bit for bit in
numpy float32; w, l, h (expf) and the scores (expf in the sigmoid) are returned in fp64 together with their bounds:

  w = fl(expf(t) * a):          expf is within 2 ulp (CUDA programming guide), i.e. 2^-22 relative, and the product adds
                                one rounding 2^-24:  |w - exp(t) a| <= 5 * 2^-24 * |w|  (first order; we use 5.01 * 2^-24).
  s = fl(fl(1 / fl(1 + expf(-c))) * q4):  expf 2^-22 relative on e, which moves 1 + e by at most 2^-22 relative, plus
                                three roundings (add, IEEE division, product) of 2^-24 each:
                                |s - sigmoid(c) q4| <= 7 * 2^-24 * |s|  (we use 7.01 * 2^-24).  q4 = fl(fl(q q)^2) itself is
                                emulated exactly.
"""
import math

import numpy as np

F32 = np.float32
PI32 = np.float32(np.pi)          # torch.tensor(np.pi).type_as(fp32) == 3.14159265358979323846f
MARGIN = 1e-3                      # relative distance of every crafted pair's IoU from the NMS threshold
U24 = 2.0 ** -24
W_BOUND = 5.01 * U24               # relative bound of decoded w, l, h
S_BOUND = 7.01 * U24               # relative bound of scores


# ------------------------------------------------------------------------------------------------------------ exact geometry
def corners64(b5):
    """[x1, y1, x2, y2, ang] -> the four corners (fp64) of the reference's clockwise spin about the centre, CCW order."""
    x1, y1, x2, y2, a = (float(v) for v in b5[:5])
    cx, cy = (x1 + x2) / 2, (y1 + y2) / 2
    c, s = math.cos(a), math.sin(a)
    return [((px - cx) * c + (py - cy) * s + cx, -(px - cx) * s + (py - cy) * c + cy)
            for px, py in ((x1, y1), (x2, y1), (x2, y2), (x1, y2))]


def _clip(subj, clip):
    out = subj
    n = len(clip)
    for i in range(n):
        if not out:
            break
        ax, ay = clip[i]
        bx, by = clip[(i + 1) % n]
        ex, ey = bx - ax, by - ay
        inp, out = out, []
        k = len(inp)
        for j in range(k):
            px, py = inp[j]
            qx, qy = inp[(j + 1) % k]
            sp = ex * (py - ay) - ey * (px - ax)
            sq = ex * (qy - ay) - ey * (qx - ax)
            if sp >= 0:
                out.append((px, py))
            if (sp >= 0) != (sq >= 0):
                t = sp / (sp - sq)
                out.append((px + t * (qx - px), py + t * (qy - py)))
    return out


def _area(p):
    if len(p) < 3:
        return 0.0
    s = 0.0
    for i in range(len(p)):
        x0, y0 = p[i]
        x1, y1 = p[(i + 1) % len(p)]
        s += x0 * y1 - x1 * y0
    return abs(s) / 2


def overlap64(a5, b5):
    ca, cb = corners64(a5), corners64(b5)
    if _area(ca) == 0.0 or _area(cb) == 0.0:
        return 0.0
    return _area(_clip(ca, cb))


def iou_bev64(a5, b5):
    sa = (float(a5[2]) - float(a5[0])) * (float(a5[3]) - float(a5[1]))
    sb = (float(b5[2]) - float(b5[0])) * (float(b5[3]) - float(b5[1]))
    so = overlap64(a5, b5)
    return so / max(sa + sb - so, 1e-8)


def iou3d64(a7, b7):
    """[x1, y1, z1, x2, y2, z2, ang]"""
    a7 = [float(v) for v in a7]
    b7 = [float(v) for v in b7]
    va = (a7[3] - a7[0]) * (a7[4] - a7[1]) * (a7[5] - a7[2])
    vb = (b7[3] - b7[0]) * (b7[4] - b7[1]) * (b7[5] - b7[2])
    dh = max(min(a7[5], b7[5]) - max(a7[2], b7[2]), 1e-8)
    if dh == 1e-8:
        return 0.0
    vo = overlap64([a7[0], a7[1], a7[3], a7[4], a7[6]], [b7[0], b7[1], b7[3], b7[4], b7[6]]) * dh
    return vo / max(va + vb - vo, 1e-8)


def bev_of(det5):
    """(x, y, w, l, r) float32 -> [x - w/2, y - l/2, x + w/2, y + l/2, r] float32 (iou3d/utils.py, nms_geometry)."""
    d = np.asarray(det5, F32).reshape(-1, 5)
    hw, hl = d[:, 2] / F32(2), d[:, 3] / F32(2)
    return np.stack([d[:, 0] - hw, d[:, 1] - hl, d[:, 0] + hw, d[:, 1] + hl, d[:, 4]], 1).astype(F32)


def standup64(det5):
    """stand-up AABB (fp64) of each rotated (x, y, w, l, r) box"""
    d = np.asarray(det5, np.float64).reshape(-1, 5)
    c, s = np.abs(np.cos(d[:, 4])), np.abs(np.sin(d[:, 4]))
    ex = d[:, 2] / 2 * c + d[:, 3] / 2 * s
    ey = d[:, 2] / 2 * s + d[:, 3] / 2 * c
    return np.stack([d[:, 0] - ex, d[:, 1] - ey, d[:, 0] + ex, d[:, 1] + ey], 1)


def overlapping_pairs(su, pad=1e-4):
    """(i, j), i < j, whose stand-up boxes (padded by `pad`) overlap -- grid hashing, no n^2 work."""
    su = np.asarray(su, np.float64)
    n = su.shape[0]
    if n == 0:
        return []
    cell = max(float(np.max(su[:, 2] - su[:, 0])), float(np.max(su[:, 3] - su[:, 1])), 1e-3) + 2 * pad
    grid = {}
    lo = np.floor((su[:, :2] - pad) / cell).astype(np.int64)
    hi = np.floor((su[:, 2:] + pad) / cell).astype(np.int64)
    for i in range(n):
        for gx in range(lo[i, 0], hi[i, 0] + 1):
            for gy in range(lo[i, 1], hi[i, 1] + 1):
                grid.setdefault((gx, gy), []).append(i)
    pairs = set()
    for members in grid.values():
        for a in range(len(members)):
            i = members[a]
            for b in range(a + 1, len(members)):
                j = members[b]
                if (su[i, 0] - pad < su[j, 2] and su[j, 0] - pad < su[i, 2] and su[i, 1] - pad < su[j, 3] and su[j, 1] - pad < su[i, 3]):
                    pairs.add((min(i, j), max(i, j)))
    return sorted(pairs)


def pair_ious(det5):
    """{(i, j): exact BEV IoU} over the stand-up-overlapping pairs of (x, y, w, l, r) boxes."""
    bev = bev_of(det5)
    return {(i, j): iou_bev64(bev[i], bev[j]) for i, j in overlapping_pairs(standup64(det5))}


def clear_of_boundaries(a5, b5, eps=1e-3):
    """no corner of either [x1, y1, x2, y2, ang] box lies within eps of the other box's boundary.  The reference's
    inside test has a fixed 1e-5 margin, below the fp32 spacing of coordinates beyond 128 m, so near-touching pairs are
    decided by its arithmetic rather than by the geometry."""
    for p, q in ((a5, b5), (b5, a5)):
        cq = corners64(q)
        for vx, vy in corners64(p):
            for i in range(4):
                ax, ay = cq[i]
                ex, ey = cq[(i + 1) % 4][0] - ax, cq[(i + 1) % 4][1] - ay
                L2 = ex * ex + ey * ey
                t = 0.0 if L2 == 0 else min(max(((vx - ax) * ex + (vy - ay) * ey) / L2, 0.0), 1.0)
                if math.hypot(vx - ax - t * ex, vy - ay - t * ey) < eps:
                    return False
    return True


def all_clear(det5, ious):
    """every overlapping pair of the set is clear of the other box's boundary"""
    bev = bev_of(det5)
    return all(clear_of_boundaries(bev[i], bev[j]) for (i, j), v in ious.items() if v > 0)


def robust(ious, thr, margin=MARGIN):
    """every pair decides the same way in exact and in fp32 arithmetic"""
    return all(abs(v - thr) >= margin * thr for v in ious.values())


# ------------------------------------------------------------------------------------------------------------ NMS model
def score_order(scores, ties_high=False):
    """descending score; equal scores (-0 == +0) -> lower index first (or higher, for the negative control)"""
    s = np.asarray(scores, np.float64)
    idx = np.arange(s.shape[0])
    return np.lexsort(((-idx) if ties_high else idx, -s))


def _suppress(v, thr, ge):
    v, thr = F32(v), F32(thr)
    return bool(v >= thr) if ge else bool(v > thr)


def greedy(m, ious, thr, ge=True, cap=None, or_suppressed=False):
    """keep positions (0..m) of the greedy scan over boxes already in score order; ious {(i, j): iou} with i < j."""
    adj = [[] for _ in range(m)]
    for (i, j), v in ious.items():
        if i < m and j < m and _suppress(v, thr, ge):
            adj[i].append(j)
    dead = np.zeros(m, bool)
    keep = []
    cap = m if cap is None else cap
    for i in range(m):
        if len(keep) >= cap:
            break
        if not dead[i]:
            keep.append(i)
        if not dead[i] or or_suppressed:
            for j in adj[i]:
                dead[j] = True
    return keep


def rotate_nms_model(det5, scores, thr, ge=True, pre_max=None, post_max=None, ties_high=False, or_suppressed=False):
    """box_torch_ops.rotate_nms semantics -> kept input indices, best first"""
    n = len(scores)
    order = score_order(scores, ties_high)[: n if pre_max is None else min(n, pre_max)]
    ious = pair_ious(np.asarray(det5, F32)[order])
    keep = greedy(len(order), ious, thr, ge, post_max, or_suppressed)
    return order[keep]


# mask words exactly as post_mask_kernel writes them and greedy_scan reads them
POISON = np.uint64(0xA5A5A5A5A5A5A5A5)


def mask_words(m, K, supp, swap_halves=False):
    """supp: set of (i, j), i < j < m.  Returns [m, ceil(K/64)] uint64 with every unwritten half left poisoned."""
    cbw = (K + 63) // 64
    words = np.full((m, cbw), POISON, np.uint64).view(np.uint32).reshape(m, cbw, 2)
    bits = {}
    for i, j in supp:
        bits[(i, j // 32)] = bits.get((i, j // 32), 0) | (1 << (j % 32))
    nt = (m + 31) // 32
    for rb in range(nt):
        for cb in range(nt):
            if cb < rb:
                if (rb & 1) and cb == rb - 1:
                    for r in range(rb * 32, min(rb * 32 + 32, m)):
                        words[r, cb >> 1, 1 if swap_halves else 0] = 0
                continue
            for r in range(rb * 32, min(rb * 32 + 32, m)):
                words[r, cb >> 1, (cb & 1) ^ int(swap_halves)] = bits.get((r, cb), 0)
    return words.reshape(m, cbw * 2).view(np.uint64)


def scan_words(words, m, cap, drop_last_partial=False, or_suppressed=False):
    """greedy_scan: 64-row blocks, the diagonal word chain resolved serially, kept rows OR-ed into later blocks"""
    nblk = (m // 64) if drop_last_partial else (m + 63) // 64
    remv = [0] * max(words.shape[1], 1)
    keep = []
    for b in range(nblk):
        rows = min(64, m - b * 64)
        cur, kb = remv[b], 0
        for t in range(rows):
            if len(keep) >= cap:
                break
            if not (cur >> t) & 1:
                keep.append(b * 64 + t)
                kb |= 1 << t
                cur |= int(words[b * 64 + t, b])
            elif or_suppressed:
                cur |= int(words[b * 64 + t, b])
                kb |= 1 << t
        if len(keep) >= cap:
            break
        for j in range(b + 1, nblk):
            for t in range(rows):
                if (kb >> t) & 1:
                    remv[j] |= int(words[b * 64 + t, j])
    return keep


def suppress_set(m, ious, thr, ge=True):
    return {(i, j) for (i, j), v in ious.items() if i < m and j < m and _suppress(v, thr, ge)}


# ------------------------------------------------------------------------------------------------------------ box-set generators
CAR_W, CAR_L = F32(1.6), F32(3.9)


def _place_rows(steps, x0=1.0, x1=69.0, y0=-37.0, pitch=6.0):
    """positions along serpentine-free rows: consecutive boxes step by `steps[i]` in x; a row ends at x1"""
    xs, ys = [], []
    x, y = x0, y0
    for i, s in enumerate(steps):
        if i and x + s > x1:
            x, y = x0, y + pitch
        elif i:
            x += s
        xs.append(x)
        ys.append(y)
    return np.array(xs), np.array(ys)


def gen_boxes(pattern, m, seed):
    """(x, y, w, l, r) float32 [m, 5] and a random permutation of score ranks; patterns: chain, cluster, standup, far"""
    rng = np.random.default_rng(seed)
    if pattern == "chain":
        # i overlaps its row neighbours (steps 0.75 or 1.25 m, IoU 0.1 - 0.4) and, when both steps are short, i + 2 (IoU ~0.03)
        xs, ys = _place_rows(rng.choice([0.75, 1.25], m))
        ys = ys + (np.arange(m) % 3) * 0.17                           # no two overlapping boxes share an edge line
        ang = rng.choice([0.0, 0.03, -0.04, np.pi], m)
        w, l = np.full(m, CAR_W), np.full(m, CAR_L)
    elif pattern == "cluster":
        # groups of 2..8 strongly overlapping boxes (IoU > 0.4 inside a group), groups 5 m apart
        sizes = []
        while sum(sizes) < m:
            sizes.append(int(rng.integers(2, 9)))
        sizes[-1] -= sum(sizes) - m
        sizes = [s for s in sizes if s > 0]
        gx, gy = _place_rows(np.full(len(sizes), 5.0))
        ks = [rng.permutation(8)[:s] for s in sizes]                   # distinct offsets inside a group: no shared edge lines
        xs = np.concatenate([np.full(s, x) + k * 0.07 for s, x, k in zip(sizes, gx, ks)])
        ys = np.concatenate([np.full(s, y) + k * 0.05 for s, y, k in zip(sizes, gy, ks)])
        ang = rng.choice([0.0, 0.01, -0.01], m)
        w, l = np.full(m, CAR_W), np.full(m, CAR_L)
    elif pattern == "standup":
        # pairs at 45 degrees, side by side 0.3 m apart: stand-up boxes overlap, rotated boxes do not; every
        # third pair is 0.6 m closer and overlaps
        npair = (m + 1) // 2
        gx, gy = _place_rows(np.full(npair, 6.0))
        d = np.where(np.arange(npair) % 3 == 2, F32(1.3), F32(1.9))
        u = np.array([np.cos(np.pi / 4), -np.sin(np.pi / 4)])       # across the long axis
        v = np.array([u[1], -u[0]]) * 0.2                               # and 0.2 m along it: no shared edge lines
        xs = np.stack([gx, gx + d * u[0] + v[0]], 1).reshape(-1)[:m]
        ys = np.stack([gy, gy + d * u[1] + v[1]], 1).reshape(-1)[:m]
        ang = np.full(m, np.pi / 4)
        w, l = np.full(m, CAR_W), np.full(m, CAR_L)
    elif pattern == "far":
        xs, ys = _place_rows(np.full(m, 5.0))
        ang = rng.uniform(-np.pi, np.pi, m)
        w, l = np.full(m, CAR_W), np.full(m, CAR_L)
    else:
        raise ValueError(pattern)
    det = np.stack([xs, ys, w, l, ang], 1).astype(F32)
    return det, rng.permutation(m)


def exact_threshold_set():
    """axis-aligned boxes with dyadic coordinates: every area and overlap is exact in fp32, so the device's IoU is
    float32(exact).  Box 1 meets box 0 at IoU exactly THR_EXACT; box 2 meets box 1 at a larger IoU."""
    det = np.array([[0, 0, 4, 2, 0], [3, 0, 4, 2, 0], [5.5, 0, 4, 2, 0], [20, 0, 4, 2, 0]], F32)
    return det, F32(2.0 / 14.0)


# ------------------------------------------------------------------------------------------------------------ heads
def kitti_anchors():
    from sessd_data import weights
    return weights.kitti_car_anchors()


def encode(det7, anchors):
    """float32 head values whose decode lands near det7 (x, y, z, w, l, h, r); r exactly when t6 = r - a6 is exact"""
    d = np.asarray(det7, np.float64)
    a = np.asarray(anchors, np.float64)
    diag = np.sqrt(a[:, 4] ** 2 + a[:, 3] ** 2)
    t = np.stack([(d[:, 0] - a[:, 0]) / diag, (d[:, 1] - a[:, 1]) / diag, (d[:, 2] - a[:, 2]) / a[:, 5],
                  np.log(d[:, 3] / a[:, 3]), np.log(d[:, 4] / a[:, 4]), np.log(d[:, 5] / a[:, 5]), d[:, 6] - a[:, 6]], 1)
    return t.astype(F32)


class Head:
    """one frame's head map [A/2, stride] with every anchor a non-candidate until `place` makes it one"""
    CLS, DIR, IOU = 14, 16, 20

    def __init__(self, anchors, stride=24, bg_logit=-8.0):
        self.anchors = anchors
        self.h = np.zeros((anchors.shape[0] // 2, stride), F32)
        self.h[:, self.CLS:self.CLS + 2] = bg_logit

    def place(self, idx, enc, logit, iou, dir_logits=None):
        idx = np.asarray(idx)
        pix, r = idx // 2, idx % 2
        for k in range(7):
            self.h[pix, 7 * r + k] = enc[:, k]
        self.h[pix, self.CLS + r] = logit
        self.h[pix, self.IOU + r] = iou
        if dir_logits is not None:
            self.h[pix, self.DIR + 2 * r] = dir_logits[:, 0]
            self.h[pix, self.DIR + 2 * r + 1] = dir_logits[:, 1]


def iou_for_rank(rank, n):
    """iou-head value whose q = (iou + 1) / 2 falls with the rank: q in (0.5, 1], relative q gaps >= 0.5 / n"""
    q = 1.0 - np.asarray(rank, np.float64) * (0.5 / max(n, 1))
    return (2 * q - 1).astype(F32)


# ------------------------------------------------------------------------------------------------------------ post model
POST_DEFAULTS = dict(score_thresh=0.3, nms_pre_max=1000, nms_post_max=100, nms_iou_thresh=0.01, nms_ge=True,
                     post_range=(0, -40.0, -5.0, 70.4, 40.0, 5.0), direction_offset=0.0)


def sigmoid64(x):
    return 1.0 / (1.0 + np.exp(-np.asarray(x, np.float64)))


def decode32(t, a):
    """x, y, z, r bit-exact (fp32, no FMA); w, l, h as fp64 exp(t) * a and rounded to fp32 for the geometry"""
    t = np.asarray(t, F32)
    a = np.asarray(a, F32)
    diag = np.sqrt(a[:, 4] * a[:, 4] + a[:, 3] * a[:, 3])
    box = np.zeros(t.shape, F32)
    box[:, 0] = t[:, 0] * diag + a[:, 0]
    box[:, 1] = t[:, 1] * diag + a[:, 1]
    box[:, 2] = t[:, 2] * a[:, 5] + a[:, 2]
    whl = np.exp(t[:, 3:6].astype(np.float64)) * a[:, 3:6].astype(np.float64)
    box[:, 3:6] = whl.astype(F32)
    box[:, 6] = t[:, 6] + a[:, 6]
    return box, whl


def frustum_ok(xyz, planes, strict=False):
    """plane sign = ((x a + y b) + z c) + d in fp32 without FMA; sign >= 0 on any plane rejects (> 0 for the control)"""
    xyz = np.asarray(xyz, F32)
    pl = np.asarray(planes, F32).reshape(6, 4)
    ok = np.ones(xyz.shape[0], bool)
    for s in range(6):
        sign = xyz[:, 0] * pl[s, 0] + xyz[:, 1] * pl[s, 1] + xyz[:, 2] * pl[s, 2] + pl[s, 3]
        ok &= ~((sign > 0) if strict else (sign >= 0))
    return ok


def post_frame(head, anchors, cfg=None, planes=None, variant=()):
    """one frame of sessd_postprocess.  variant: negative controls ('gt', 'ties_high', 'or_suppressed', 'cap_after_range',
    'frustum_strict', 'dir_ge').  Returns a dict of the outputs (P-sized, padded) plus fp64 w/l/h and scores."""
    c = dict(POST_DEFAULTS)
    c.update(cfg or {})
    K, P = c["nms_pre_max"], c["nms_post_max"]
    h = np.asarray(head, F32)
    A = h.shape[0] * 2
    pix, r = np.arange(A) // 2, np.arange(A) % 2
    logit = h[pix, Head.CLS + r]
    cand = np.nonzero(sigmoid64(logit) >= c["score_thresh"])[0]
    q = (h[pix[cand], Head.IOU + r[cand]] + F32(1)) * F32(0.5)
    q2 = q * q
    score = sigmoid64(logit[cand]) * (q2 * q2).astype(np.float64)
    n = len(cand)
    order = score_order(score, "ties_high" in variant)[:K]
    sel = cand[order]
    m = len(sel)
    t = h[pix[sel][:, None], 7 * r[sel][:, None] + np.arange(7)[None]]
    box, whl = decode32(t, anchors[sel])
    d0, d1 = h[pix[sel], Head.DIR + 2 * r[sel]], h[pix[sel], Head.DIR + 2 * r[sel] + 1]
    dirl = d1 > d0
    ious = pair_ious(box[:, [0, 1, 3, 4, 6]])
    cap = m if "cap_after_range" in variant else P
    keep = greedy(m, ious, c["nms_iou_thresh"], c["nms_ge"] and "gt" not in variant, cap, "or_suppressed" in variant)
    nk = len(keep)
    kb = box[keep]
    ok = np.ones(nk, bool)
    if planes is not None:
        ok &= frustum_ok(kb[:, :3], planes, "frustum_strict" in variant)
    rr = kb[:, 6] - F32(c["direction_offset"])
    opp = ((rr >= 0) if "dir_ge" in variant else (rr > 0)) != dirl[keep]
    rng = np.asarray(c["post_range"], F32)
    ok &= np.all((kb[:, :3] >= rng[:3]) & (kb[:, :3] <= rng[3:]), 1)
    passed = np.nonzero(ok)[0]
    if "cap_after_range" in variant:
        passed = passed[:P]
        nk = min(nk, P)
    cnt = len(passed)
    out = dict(count=cnt, aux=np.array([n, m, nk, 0], np.int32), sel_anchor=np.full(P, -1, np.int32),
               boxes=np.zeros((P, 7), F32), scores=np.zeros(P, np.float64), labels=np.full(P, -1, np.int32),
               whl=np.zeros((P, 3)), anchor=np.full(P, -1, np.int32), keep=keep, ious=ious, n=n, m=m,
               clear=all_clear(box[:, [0, 1, 3, 4, 6]], ious))
    out["sel_anchor"][:nk] = sel[keep[:nk]]
    for dst, i in enumerate(passed):
        src = keep[i]
        b = box[src].copy()
        if opp[i]:
            b[6] = b[6] + PI32
        out["boxes"][dst] = b
        out["scores"][dst] = score[order[src]]
        out["whl"][dst] = whl[src]
        out["labels"][dst] = 0
        out["anchor"][dst] = sel[src]
    return out


# ------------------------------------------------------------------------------------------------------------ crafted frames
Z0, H0 = F32(-1.0), F32(1.56)


def frame(n, K=1000, P=100, pattern="chain", seed=0, all_anchors=False, tie_levels=None, logit=3.0):
    """A head with n candidates.  Sorted position s < min(n, K) carries box s of the pattern (ranks from its random
    permutation); the other candidates decode to their anchor.  Scores are distinct (relative gaps >= 0.5 / n) unless
    tie_levels quantises them to that many equal values.  Returns (head, cfg)."""
    anchors = kitti_anchors()
    A = anchors.shape[0]
    rng = np.random.default_rng(1000 + seed)
    idx = np.arange(A) if all_anchors else np.sort(rng.choice(A, n, replace=False))
    n = len(idx)
    rank = rng.permutation(n)
    if tie_levels:
        rank = rank * tie_levels // max(n, 1)
    m = min(n, K)
    order = np.lexsort((idx, rank))        # sorted position -> candidate (equal ranks: lower anchor index first)
    hd = Head(anchors)
    enc = np.zeros((n, 7), F32)
    if m:
        det, perm = gen_boxes(pattern, m, seed)
        det = det[np.argsort(perm)]
        d7 = np.stack([det[:, 0], det[:, 1], np.full(m, Z0), det[:, 2], det[:, 3], np.full(m, H0), det[:, 4]], 1)
        enc[order[:m]] = encode(d7, anchors[idx[order[:m]]])
    dirs = rng.normal(0, 1, (n, 2)).astype(F32)
    hd.place(idx, enc, F32(logit), iou_for_rank(rank, n), dirs)
    return hd.h, dict(nms_pre_max=K, nms_post_max=P)


def boundary_frame():
    """range bounds hit exactly, a frustum plane sign of exactly 0, r == direction_offset with equal and unequal dir
    logits, flips either side of a non-zero offset, and P = 10 with the two best boxes out of range and four more boxes behind the cap.
    Returns (head, cfg, planes, {name: sorted position})."""
    anchors = kitti_anchors()
    off = F32(0.785)
    # x, y, z, r, d0, d1 per box, best first; every box is 6 m from the others
    spec = [(-10.0, 0.0, -1.0, 0.2, 0, 1), (-20.0, 0.0, -1.0, 0.2, 0, 1),           # out of range, inside the cap
            (5.0, -30.0, -1.0, off, 0.5, 0.5),                                        # x, y low bounds; r == offset, equal logits
            (12.0, -30.0, -1.0, off, 0.0, 1.0),                                       # r == offset, dir 1 -> flip
            (20.0, -30.0, -1.5, 1.5, 1.0, 0.0), (36.0, -30.0, -0.5, 2.0, 0.0, 1.0),   # z low / high bounds
            (5.0, 30.0, -1.0, -0.3, 0.0, 1.0), (60.0, 0.0, -1.0, 0.0, 0.0, 1.0),      # y / x high bounds
            (50.0, 20.0, -1.0, 0.0, 0.0, 1.0),                                        # frustum sign exactly 0
            (28.0, -30.0, -1.0, -0.3, 0.0, 1.0),
            (44.0, -30.0, -1.0, 0.0, 0, 1), (12.0, 30.0, -1.0, 0.0, 0, 1), (20.0, 30.0, -1.0, 0.0, 0, 1),   # behind the cap
            (30.0, 10.0, -1.0, 0.0, 0, 1)]
    n = len(spec)
    idx = np.array([((int((s[1] + 40) / 0.4) * 176 + int(s[0] / 0.4 if s[0] > 0 else i)) * 2) for i, s in enumerate(spec)])
    an = anchors[idx]
    d7 = np.array([[s[0], s[1], s[2], 1.6, 3.9, 1.56, s[3]] for s in spec], np.float64)
    enc = encode(d7, an)
    enc[:, 6] = (np.array([s[3] for s in spec], F32) - an[:, 6]).astype(F32)     # anchors of rotation 0: r exact
    hd = Head(anchors)
    hd.place(idx, enc, F32(3.0), iou_for_rank(np.arange(n), n), np.array([s[4:6] for s in spec], F32))
    box, _ = decode32(enc, an)
    # range bounds are the decoded centres of boxes 2 (x, y low), 4 (z low), 7 (x high), 6 (y high), 5 (z high): inclusive
    rng_ = (box[2, 0], box[2, 1], box[4, 2], box[7, 0], box[6, 1], box[5, 2])
    # frustum: x + y < x + y of box 8 is inside, so box 8 has sign exactly 0 and is rejected; the other planes are far away
    planes = np.array([[1, 1, 0, -(box[8, 0] + box[8, 1])], [-1, 0, 0, -100], [0, 1, 0, -100], [0, -1, 0, -100], [0, 0, 1, -100],
                       [0, 0, -1, -100]], F32)
    cfg = dict(nms_pre_max=64, nms_post_max=10, post_range=rng_, direction_offset=off)
    return hd.h, cfg, planes, idx
