"""numpy restatement of shape-aware data augmentation (SA-DA, det3d/datasets/utils/sa_da_v2.py: pyramid_augment_v0) for one frame.

  pyramids      get_pyramids: [K, 6, 15] fp32, the box centre then the four corners of one face of center_to_corner_box3d(origin 0.5)
  planes        surface_equ_3d_jitv2 over points_in_pyramids_mask's 5 surfaces, fp32
  in_pyramids   points_in_convex_polygon_3d_jit: inside when every surface sign ((x n0 + y n1) + z n2) + d is < 0, fp32
  fps           the farthest-point contract (start at row 0, fp64 distance sqrt((dx^2 + dy^2) + dz^2) to the nearest pick, ties to the
                lowest row), as the reference's ifp_sample on cKDTree's complete neighbour lists
  sada          the four steps with sessd_b200.sada's draws, returning every stage's rows

The fp32 sin / cos of a box angle are the correctly rounded values; the fixtures use angles where numpy's float32 sin / cos agree.
"""
import numpy as np

from sessd_b200.sada import draw_partners, draw_pick

FACES = np.array([[0, 1, 5, 4], [4, 5, 6, 7], [7, 6, 2, 3], [3, 2, 1, 0], [1, 2, 6, 5], [0, 4, 7, 3]])
SURFACES = [(1, 2, 0), (2, 3, 0), (3, 4, 0), (4, 1, 0), (4, 3, 2)]
NORM = np.array([[0, 0, 0], [0, 0, 1], [0, 1, 1], [0, 1, 0], [1, 0, 0], [1, 0, 1], [1, 1, 1], [1, 1, 0]], np.float32) - np.float32(0.5)


def sincos32(a):
    a = np.asarray(a, np.float32).astype(np.float64)
    return np.sin(a).astype(np.float32), np.cos(a).astype(np.float32)


def pyramids(boxes):
    b = np.asarray(boxes, np.float32).reshape(-1, 7)
    s, c = sincos32(b[:, 6])
    cn = b[:, None, 3:6] * NORM[None]                                         # corners_nd
    x = cn[..., 0] * c[:, None] + cn[..., 1] * s[:, None]                     # einsum with [[c, -s, 0], [s, c, 0], [0, 0, 1]]
    y = cn[..., 0] * -s[:, None] + cn[..., 1] * c[:, None]
    corners = np.stack([x, y, cn[..., 2]], -1) + b[:, None, 0:3]
    out = np.empty((len(b), 6, 15), np.float32)
    for f, order in enumerate(FACES):
        out[:, f] = np.concatenate([b[:, 0:3]] + [corners[:, k] for k in order], 1)
    return out


def planes(pyr):
    P = np.asarray(pyr, np.float32).reshape(-1, 5, 3)
    normals = np.empty((len(P), 5, 3), np.float32)
    d = np.empty((len(P), 5), np.float32)
    for k, (a, b, c) in enumerate(SURFACES):
        u = P[:, a] - P[:, b]
        v = P[:, b] - P[:, c]
        n = np.stack([u[:, 1] * v[:, 2] - u[:, 2] * v[:, 1], u[:, 2] * v[:, 0] - u[:, 0] * v[:, 2], u[:, 0] * v[:, 1] - u[:, 1] * v[:, 0]], 1)
        normals[:, k] = n
        d[:, k] = -P[:, a, 0] * n[:, 0] - P[:, a, 1] * n[:, 1] - P[:, a, 2] * n[:, 2]
    return normals, d


def in_pyramids(points, pyr):
    """[N, P] bool"""
    p = np.asarray(points, np.float32)[:, :3]
    normals, d = planes(pyr)
    inside = np.ones((len(p), len(normals)), bool)
    for k in range(5):
        sign = p[:, None, 0] * normals[None, :, k, 0] + p[:, None, 1] * normals[None, :, k, 1] + p[:, None, 2] * normals[None, :, k, 2]
        sign = sign + d[None, :, k]
        inside &= sign < 0
    return inside


def fps(xyz, k):
    x = np.asarray(xyz, np.float32)[:, :3].astype(np.float64)
    dist = np.full(len(x), np.inf)
    picks, pick = [], 0
    for _ in range(k):
        picks.append(pick)
        dd = x - x[pick]
        dist = np.minimum(dist, np.sqrt((dd[:, 0] * dd[:, 0] + dd[:, 1] * dd[:, 1]) + dd[:, 2] * dd[:, 2]))
        pick = int(np.argmax(dist))
    return np.array(picks, np.int64)


def _ratio(points, q):
    sc = (q[3:6] + q[6:9] + q[9:12] + q[12:]) / np.float32(4.0)
    v0, v1, v2 = q[6:9] - q[3:6], q[12:] - q[3:6], q[0:3] - sc
    a = ((points[:, 0:3] - q[3:6]) * v0).sum(-1) / (v0 * v0).sum()
    b = ((points[:, 0:3] - q[3:6]) * v1).sum(-1) / (v1 * v1).sum()
    g = ((points[:, 0:3] - sc) * v2).sum(-1) / (v2 * v2).sum()
    return a, b, g


def _recover(r, q):
    a, b, g = r
    sc = (q[3:6] + q[6:9] + q[9:12] + q[12:]) / np.float32(4.0)
    v0, v1, v2 = q[6:9] - q[3:6], q[12:] - q[3:6], q[0:3] - sc
    return (a[:, None] * v0 + b[:, None] * v1) + q[3:6] + g[:, None] * v2


def _intensity(w):
    lo, hi = w.min(), w.max()
    return lo, hi, (w - lo) / np.clip(hi - lo, np.float32(1e-6), np.float32(1))


def swap_pair(points, mask_a, mask_b, qa, qb):
    """rows of one pair: the partner's points in pyramid a, then pyramid a's points in the partner"""
    A, B = points[mask_a], points[mask_b]
    lo_a, hi_a, ra = _intensity(A[:, 3])
    lo_b, hi_b, rb = _intensity(B[:, 3])
    new_a = np.concatenate([_recover(_ratio(B, qb), qa), (rb * (hi_a - lo_a) + lo_a)[:, None]], 1)
    new_b = np.concatenate([_recover(_ratio(A, qa), qb), (ra * (hi_b - lo_b) + lo_b)[:, None]], 1)
    return new_a, new_b


def sada(points, boxes, rs, dropout=0.25, sparsity=(0.05, 50), swap=(0.1, 50)):
    """pyramid_augment_v0 on fp32 [N, 4] points and fp32 [K, 7] boxes; returns dict(dropout, sparsify, swap: the rows after each step,
    points: the float32 result)"""
    points = np.asarray(points, np.float32)
    if points.ndim != 2 or points.shape[1] != 4:
        raise ValueError("SA-DA takes [N, 4] points")
    pyr = pyramids(boxes)
    alive = np.arange(len(pyr))
    out = {}
    if dropout is not None and len(pyr) > 0:
        idx, drop = draw_pick(rs, len(pyr), dropout)
        sel = pyr[alive[drop], idx[drop]]
        if len(sel):
            points = points[~in_pyramids(points, sel).any(1)]
        alive = alive[~drop]
    out["dropout"] = points
    if sparsity is not None and len(alive) > 0:
        p, keep = sparsity
        idx, pick = draw_pick(rs, len(alive), p)
        cand = pyr[alive[pick], idx[pick]]
        m = in_pyramids(points, cand)
        valid = m.sum(0) > keep
        if valid.any():
            mv = m[:, valid]
            rest = points[~mv.any(1)]
            sampled = [points[mv[:, i]][fps(points[mv[:, i]], keep)] for i in range(mv.shape[1])]
            points = np.concatenate([rest] + sampled)
        alive = alive[~pick]
    out["sparsify"] = points
    if swap is not None:
        p, thr = swap
        sel = rs.uniform(0, 1, (len(alive),)) <= p
        if sel.any():
            counts = in_pyramids(points, pyr[alive].reshape(-1, 15)).sum(0).reshape(-1, 6)
            pairs = draw_partners(rs, counts, sel, thr)
            if pairs:
                qa = np.stack([pyr[alive[i], j] for i, j, _ in pairs])
                qb = np.stack([pyr[alive[q], j] for _, j, q in pairs])
                m = in_pyramids(points, np.concatenate([qa, qb]))
                res = [points[~m.any(1)]]
                P = len(pairs)
                for t in range(P):
                    res += list(swap_pair(points, m[:, t], m[:, P + t], qa[t], qb[t]))
                points = np.concatenate(res)
    out["swap"] = points
    out["points"] = points.astype(np.float32)
    return out


def preprocess_frame(points, boxes, names, rs, acfg, sa_da, context=-1.0):
    """One labelled frame through Preprocess.__call__ after GT-AUG, with SA-DA between the global scaling and the shuffle (sa_da: a
    sessd_b200.sada.SadaConfig, or None for the chain without it): sessd_b200.augment's host draws, oracle/augment_ref.augment_frame,
    sada, then the shuffle draw sized by the frame after SA-DA.  Returns augment_frame's dict with ``points`` (the student's: SA-DA,
    then shuffled), ``points_sada`` (before the shuffle) and ``draws`` (the frame's FrameDraws)."""
    from oracle import augment_ref
    from sessd_b200 import augment
    points = np.asarray(points, np.float32)
    boxes = np.asarray(boxes, np.float32).reshape(-1, 7)
    valid = np.array([n in acfg.class_names for n in names], bool)
    loc, rot, flip, rotation, scale = augment._labeled_draws(rs, len(boxes), acfg)
    o = augment_ref.augment_frame(points, boxes, valid, dict(loc=loc, rot=rot, flip=flip, rotation=rotation, scale=scale,
                                                              perm=np.arange(len(points))), context)
    s = o["points"]
    if sa_da is not None:
        s = sada(s, o["boxes"], rs, sa_da.dropout, sa_da.sparsity, sa_da.swap)["points"]
    perm = augment._shuffle(rs, len(s), acfg)
    return dict(o, points=s[perm], points_sada=s, draws=augment.FrameDraws(loc, rot, flip, rotation, scale, perm))
