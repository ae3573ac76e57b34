"""numpy restatement of the per-object noise and global augmentation of SE-SSD's training frames, with the reference's rounding.

Stages (det3d/core/sampler/preprocess.py, det3d/datasets/pipelines/preprocess.py:68-175), each a pure function of the frame and the draws:
  noise_per_box        noise_per_box (:579-611) over box_collision_test (:944-1027), in fp64
  point_masks          points_in_convex_polygon_3d_jit over the boxes' surfaces (:634-646), as a box-frame test
  object_transform     points_transform_ / box3d_transform_ (:545-569): the first VALID box holding a point moves it, in fp32
  global_transform     random_flip_v2, global_rotation_v3, global_scaling_v3 (:896-941), in fp32
  augment_frame        the order of Preprocess.__call__ without GT-AUG and SA-DA: noise, valid-box selection, raw twin, global, shuffle

Rounding, traced through the reference:
  * `gt_boxes[:, [0, 1, 3, 4, 6]] + offset` adds a Python list, so numpy promotes the BEV boxes to fp64: corners, draws and the collision
    predicate are fp64.  The 2x2 rotations (`corners @ rot_mat_T`) and the per-point 1x3 @ 3x3 and global N x 3 @ 3x3 rotations are BLAS
    gemm calls; on x86-64 with FMA they evaluate sum_j a_j r_jk as fma(a2, r2k, fma(a1, r1k, a0 r0k)) (checked against the reference by
    tests/golden/make_augment_golden.py).  Those fmas are restated exactly here (fma64 / fma32).
  * points_transform_ works on the fp32 points: `p -= c`, the rotation, `p += c`, then `p += loc` with an fp64 loc (rounded once to
    fp32).  It runs for every point in a valid box even when the box's try is -1 (zero loc, zero angle): (p - c) + c is not always p.
  * The global stages act on fp32 arrays with Python-float draws, which numpy keeps in fp32 (flip: -r + f32(pi); scale: x * f32(s)); the
    rotation matrix is fp32(cos), fp32(sin) of the fp64 angle.
  * Point membership: the reference tests a point against the six face planes of fp64 corners built from fp32 sin / cos of the box angle.
    The same set, for points farther than ~1e-6 from every face, is the box-frame test |R^T (p - c)| < dims / 2 used here (and by the
    kernel).  Points within rounding of a face may fall either way; the fixtures keep every point at least 1e-4 from every face.
"""
from fractions import Fraction

import numpy as np

NUM_TRY = 100


# ---------------------------------------------------------------------------------------------------------------- exact fused multiply-add
def fma64(a, b, c):
    """fp64 fma(a, b, c), correctly rounded (elementwise, through exact rationals)"""
    a, b, c = np.broadcast_arrays(np.asarray(a, np.float64), np.asarray(b, np.float64), np.asarray(c, np.float64))
    out = np.empty(a.shape, np.float64)
    for i in np.ndindex(a.shape):
        out[i] = float(Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i])))
    return out


def fma32(a, b, c):
    """fp32 fma(a, b, c), correctly rounded: a*b is exact in fp64, so the fp64 sum is one rounding away from exact; rounding it again to
    fp32 can only go wrong when that fp64 value is an fp32 midpoint -- those elements are redone through exact rationals"""
    a, b, c = np.broadcast_arrays(np.asarray(a, np.float32), np.asarray(b, np.float32), np.asarray(c, np.float32))
    s = a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)
    out = s.astype(np.float32)
    bits = s.view(np.uint64)
    mid = (bits & np.uint64(0x1FFFFFFF)) == np.uint64(0x10000000)
    for i in zip(*np.nonzero(mid)):
        out[i] = np.float32(float(Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))))
    return out


# ---------------------------------------------------------------------------------------------------------------- collision (fp64)
def bev_boxes(boxes7, context=-1.0):
    """(x, y, w, l, r) in fp64 with w, l enlarged by data_aug_with_context when it is positive (noise_per_object_v4_)"""
    b = np.asarray(boxes7, np.float32)[:, [0, 1, 3, 4, 6]].astype(np.float64)
    if context > 0:
        b[:, 2:4] += np.float64(context)
    return b


def bev_corners(boxes5):
    """box2d_to_corner_jit: [N, 5] fp64 -> [N, 4, 2] fp64, corners (-,-) (-,+) (+,+) (+,-) of (w, l), rotated, plus the centre"""
    boxes5 = np.asarray(boxes5, np.float64)
    nx = np.array([-0.5, -0.5, 0.5, 0.5]); ny = np.array([-0.5, 0.5, 0.5, -0.5])
    cx = boxes5[:, 2:3] * nx; cy = boxes5[:, 3:4] * ny
    s = np.sin(boxes5[:, 4:5]); c = np.cos(boxes5[:, 4:5])
    x = fma64(cy, s, cx * c) + boxes5[:, 0:1]
    y = fma64(cy, c, cx * -s) + boxes5[:, 1:2]
    return np.stack([x, y], axis=-1)


def _contains(a, p):
    for l in range(4):
        for k in range(4):
            k1 = (k + 1) % 4
            vx = -(a[k, 0] - a[k1, 0]); vy = -(a[k, 1] - a[k1, 1])
            cross = vy * (a[k, 0] - p[l, 0])
            cross -= vx * (a[k, 1] - p[l, 1])
            if cross >= 0:
                return False
    return True


def collide(b, q):
    """box_collision_test for one pair of [4, 2] fp64 corner sets (clockwise), operation for operation"""
    b = np.asarray(b, np.float64); q = np.asarray(q, np.float64)
    iw = min(b[:, 0].max(), q[:, 0].max()) - max(b[:, 0].min(), q[:, 0].min())
    if not iw > 0:
        return False
    ih = min(b[:, 1].max(), q[:, 1].max()) - max(b[:, 1].min(), q[:, 1].min())
    if not ih > 0:
        return False
    for k in range(4):
        A, B = b[k], b[(k + 1) % 4]
        for l in range(4):
            C, D = q[l], q[(l + 1) % 4]
            acd = (D[1] - A[1]) * (C[0] - A[0]) > (C[1] - A[1]) * (D[0] - A[0])
            bcd = (D[1] - B[1]) * (C[0] - B[0]) > (C[1] - B[1]) * (D[0] - B[0])
            if acd != bcd:
                abc = (C[1] - A[1]) * (B[0] - A[0]) > (B[1] - A[1]) * (C[0] - A[0])
                abd = (D[1] - A[1]) * (B[0] - A[0]) > (B[1] - A[1]) * (D[0] - A[0])
                if abc != abd:
                    return True
    return _contains(b, q) or _contains(q, b)


def collision_matrix(boxes, qboxes):
    return np.array([[collide(b, q) for q in qboxes] for b in boxes], dtype=bool).reshape(len(boxes), len(qboxes))


def noise_per_box(boxes7, valid, loc_noise, rot_noise, context=-1.0):
    """selected try per box ([M] int32, -1: none / invalid): boxes in index order against the CURRENT corners of every other box"""
    b5 = bev_boxes(boxes7, context)
    m = b5.shape[0]
    sel = -np.ones(m, np.int32)
    if m == 0:
        return sel
    cur = bev_corners(b5)
    for i in range(m):
        if not valid[i]:
            continue
        t = rot_noise.shape[1]
        s = np.sin(rot_noise[i]); c = np.cos(rot_noise[i])
        u = cur[i] - b5[i, :2]                                      # [4, 2]
        x = fma64(u[None, :, 1], s[:, None], u[None, :, 0] * c[:, None])
        y = fma64(u[None, :, 1], c[:, None], u[None, :, 0] * -s[:, None])
        shift = b5[i, :2] + loc_noise[i, :, :2]                     # [T, 2]
        tries = np.stack([x + shift[:, 0:1], y + shift[:, 1:2]], axis=-1)
        for j in range(t):
            if not any(collide(tries[j], cur[k]) for k in range(m) if k != i):
                sel[i] = j
                cur[i] = tries[j]
                break
    return sel


# ---------------------------------------------------------------------------------------------------------------- points / boxes (fp32)
def point_masks(points, boxes7, context=-1.0):
    """[N, M] bool: point n lies inside box m (box-frame test in fp64; see the module docstring)"""
    p = np.asarray(points, np.float32)[:, :3].astype(np.float64)
    b = np.asarray(boxes7, np.float32).astype(np.float64)
    if b.shape[0] == 0 or p.shape[0] == 0:
        return np.zeros((p.shape[0], b.shape[0]), bool)
    dims = b[:, 3:6].copy()
    if context > 0:
        dims[:, 0:2] += np.float64(context)
    c = np.cos(b[:, 6]); s = np.sin(b[:, 6])
    dx = p[:, None, 0] - b[None, :, 0]; dy = p[:, None, 1] - b[None, :, 1]; dz = p[:, None, 2] - b[None, :, 2]
    lx = dx * c - dy * s
    ly = dx * s + dy * c
    return (np.abs(lx) < dims[:, 0] / 2) & (np.abs(ly) < dims[:, 1] / 2) & (np.abs(dz) < dims[:, 2] / 2)


def _rot32(p3, c, s):
    """p3 [N, 3] fp32 @ [[c, -s, 0], [s, c, 0], [0, 0, 1]] (fp32) as the BLAS fma chain"""
    z = np.float32(0); one = np.float32(1)
    x = fma32(p3[:, 2], z, fma32(p3[:, 1], s, p3[:, 0] * c))
    y = fma32(p3[:, 2], z, fma32(p3[:, 1], c, p3[:, 0] * -s))
    zz = fma32(p3[:, 2], one, fma32(p3[:, 1], z, p3[:, 0] * z))
    return np.stack([x, y, zz], axis=1).astype(np.float32)


def select_transform(loc_noise, rot_noise, selected):
    """_select_transform: the selected try's (loc [M, 3], rot [M]) in fp64, zeros for -1"""
    m = len(selected)
    loc = np.zeros((m, 3)); rot = np.zeros(m)
    for i, j in enumerate(selected):
        if j >= 0:
            loc[i] = loc_noise[i, j]; rot[i] = rot_noise[i, j]
    return loc, rot


def object_transform(points, boxes7, valid, masks, loc, rot):
    """points_transform_ + box3d_transform_: returns (points, boxes) fp32 copies"""
    pts = np.array(points, np.float32, copy=True)
    bx = np.array(boxes7, np.float32, copy=True)
    if bx.shape[0] == 0 or pts.shape[0] == 0:
        owner = np.full(pts.shape[0], -1)
    else:
        vm = masks & np.asarray(valid, bool)[None, :]
        owner = np.where(vm.any(1), vm.argmax(1), -1)
    for j in range(bx.shape[0]):
        idx = np.nonzero(owner == j)[0]
        if len(idx) == 0:
            continue
        c32 = np.float32(np.cos(rot[j])); s32 = np.float32(np.sin(rot[j]))
        ctr = bx[j, :3]
        p = pts[idx, :3] - ctr
        p = _rot32(p, c32, s32)
        p = p + ctr
        pts[idx, :3] = (p.astype(np.float64) + loc[j]).astype(np.float32)
    for j in range(bx.shape[0]):
        if valid[j]:
            bx[j, :3] = (bx[j, :3].astype(np.float64) + loc[j]).astype(np.float32)
            bx[j, 6] = np.float32(np.float64(bx[j, 6]) + rot[j])
    return pts, bx


def global_params(flip, rotation, scale):
    """the fp32 constants the global stages use: (cos, sin, scale) as rotation_points_single_angle / global_scaling_v3 round them"""
    return np.float32(np.cos(rotation)), np.float32(np.sin(rotation)), np.float32(scale)


def global_transform(points, boxes7, flip, rotation, scale):
    """random_flip_v2 -> global_rotation_v3 -> global_scaling_v3 on fp32 copies (boxes7 may be None: unlabelled frames)"""
    pts = np.array(points, np.float32, copy=True)
    bx = None if boxes7 is None else np.array(boxes7, np.float32, copy=True)
    c, s, sc = global_params(flip, rotation, scale)
    if flip:
        pts[:, 1] = -pts[:, 1]
        if bx is not None:
            bx[:, 1] = -bx[:, 1]
            bx[:, 6] = -bx[:, 6] + np.float32(np.pi)
    pts[:, :3] = _rot32(pts[:, :3], c, s)
    if bx is not None:
        bx[:, :3] = _rot32(bx[:, :3], c, s)
        bx[:, 6] = bx[:, 6] + np.float32(rotation)
    pts[:, :3] = pts[:, :3] * sc
    if bx is not None:
        bx[:, :6] = bx[:, :6] * sc
    return pts, bx


def augment_frame(points, boxes7, valid, draws, context=-1.0, labeled=True):
    """One frame through Preprocess.__call__'s augmentation without GT-AUG and SA-DA.  draws: dict(loc [M, T, 3], rot [M, T], flip,
    rotation, scale, perm).  Returns dict(selected, masks, points (student, shuffled), points_raw (noised, unshuffled), boxes (valid,
    global), boxes_raw (valid, noised))."""
    points = np.asarray(points, np.float32)
    if not labeled:
        pts = points[draws["perm"]]
        pts, _ = global_transform(pts, None, draws["flip"], draws["rotation"], draws["scale"])
        return dict(points=pts)
    boxes7 = np.asarray(boxes7, np.float32)
    valid = np.asarray(valid, bool)
    sel = noise_per_box(boxes7, valid, draws["loc"], draws["rot"], context)
    masks = point_masks(points, boxes7, context)
    loc, rot = select_transform(draws["loc"], draws["rot"], sel)
    pts, bx = object_transform(points, boxes7, valid, masks, loc, rot)
    bx = bx[valid]
    gp, gb = global_transform(pts, bx, draws["flip"], draws["rotation"], draws["scale"])
    return dict(selected=sel, masks=masks, points=gp[draws["perm"]], points_raw=pts, boxes=gb, boxes_raw=bx)
