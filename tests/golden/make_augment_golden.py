"""Generate tests/golden/augment_cases.npz by running the REFERENCE's own augmentation functions in place on the CPU.

    python tests/golden/make_augment_golden.py

Imports det3d/core/sampler/preprocess.py, det3d/core/bbox/box_np_ops.py and det3d/core/bbox/geometry.py where they lie (numba-compiled,
as in the reference's DataLoader workers) through ``sys.modules`` shims, as make_golden.py does.  Per frame it runs, in the order of
Preprocess.__call__ (det3d/datasets/pipelines/preprocess.py:68-175) without GT-AUG and SA-DA: noise_per_object_v4_ (noise_per_box,
box_collision_test, points_in_convex_polygon_3d_jit, points_transform_, box3d_transform_), the valid-box selection, the raw copy,
random_flip_v2, global_rotation_v3, global_scaling_v3 and the shuffle `np.random.choice(np.arange(n), n, replace=False)`; an unlabelled
frame shuffles first and then flips, rotates and scales its points.  The draws come either from a seeded RandomState through the
reference's own np.random calls (recorded; `seed` >= 0) or are crafted and replayed into those calls (`seed` = -1).

Stored per frame f (prefix "f<f>_"): the inputs (in_points, in_boxes, valid, labeled, context), the draws (loc, rot, flip, rotation, scale, perm,
seed), and the reference's outputs: selected (noise_per_box), masks (points_in_convex_polygon_3d_jit), points_raw / boxes_raw (after the
per-object noise; boxes_raw = the valid boxes), points / boxes (after the global stages; points shuffled).  Collision cases: coll_boxes
[N, 4, 2], coll_qboxes [K, 4, 2] (fp64 corners from box2d_to_corner_jit) and coll_ref (box_collision_test).

Every crafted point is at least MARGIN = 1e-3 (in each box's own frame) from every face plane of every box -- pre-noise boxes, enlarged by
the context where it applies -- so point membership cannot depend on rounding (asserted here; the reference's face-plane test and the
box-frame test of oracle/augment_ref.py agree on every stored point).  The script checks oracle/augment_ref.py against every stored
output before writing.
"""
import contextlib
import importlib.util
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, ROOT)
from oracle import augment_ref  # noqa: E402

MARGIN = 1e-3
CLASS_NAMES = ["Car", "Van"]                 # config class_names with enable_similar_type (pipelines/preprocess.py:56-58)
LOC_STD = [1.0, 1.0, 0.5]
ROT_RANGE = [-0.785, 0.785]
GLOBAL_ROT = [-0.785, 0.785]
GLOBAL_SCALE = [0.95, 1.05]


def _pkg(name):
    m = types.ModuleType(name)
    m.__path__ = [os.path.join(REF, *name.split("."))]
    sys.modules[name] = m
    return m


def _stub(name, **attrs):
    m = types.ModuleType(name)
    for k, v in attrs.items():
        setattr(m, k, v)
    sys.modules[name] = m
    return m


def _load(name, rel):
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
    m = importlib.util.module_from_spec(spec)
    sys.modules[name] = m
    spec.loader.exec_module(m)
    return m


def load_reference():
    for p in ("det3d", "det3d.core", "det3d.core.bbox", "det3d.core.sampler"):
        _pkg(p)
    _stub("spconv")
    _stub("spconv.utils", rbbox_intersection=None, rbbox_iou=None)
    geom = _load("det3d.core.bbox.geometry", "det3d/core/bbox/geometry.py")
    bnp = _load("det3d.core.bbox.box_np_ops", "det3d/core/bbox/box_np_ops.py")
    sys.modules["det3d.core.bbox"].box_np_ops = bnp
    sys.modules["det3d.core.bbox"].geometry = geom
    prep = _load("det3d.core.sampler.preprocess", "det3d/core/sampler/preprocess.py")
    return prep, bnp


@contextlib.contextmanager
def draws_from(source, log):
    """route np.random.normal / uniform / choice to `source` (a RandomState) or, when source is a list, replay its values in order;
    every value handed out is appended to `log`"""
    saved = (np.random.normal, np.random.uniform, np.random.choice)

    def make(name):
        def f(*a, **k):
            v = getattr(source, name)(*a, **k) if isinstance(source, np.random.RandomState) else source.pop(0)
            log.append((name, v))
            return v
        return f
    np.random.normal, np.random.uniform, np.random.choice = make("normal"), make("uniform"), make("choice")
    try:
        yield
    finally:
        np.random.normal, np.random.uniform, np.random.choice = saved


def run_reference(prep, points, boxes, valid, labeled, context, source):
    """one frame through the reference functions; returns (outputs, draws)"""
    log, rec = [], {}
    orig_npb, orig_pic = prep.noise_per_box, prep.points_in_convex_polygon_3d_jit

    def npb(*a):
        rec["selected"] = orig_npb(*a)
        return rec["selected"]

    def pic(*a):
        rec["masks"] = orig_pic(*a)
        return rec["masks"]
    prep.noise_per_box, prep.points_in_convex_polygon_3d_jit = npb, pic
    points = points.copy()
    boxes = boxes.copy()
    out = {}
    try:
        with draws_from(source, log):
            if labeled:
                prep.noise_per_object_v4_(boxes, points, valid, rotation_perturb=ROT_RANGE, center_noise_std=LOC_STD,
                                          global_random_rot_range=[0.0, 0.0], group_ids=None, num_try=100,
                                          data_aug_with_context=context, data_aug_random_drop=-1.0)
                boxes = boxes[valid]
                out["points_raw"], out["boxes_raw"] = points.copy(), boxes.copy()
                boxes, points, _ = prep.random_flip_v2(boxes, points)
                boxes, points, _ = prep.global_rotation_v3(boxes, points, GLOBAL_ROT)
                boxes, points, _ = prep.global_scaling_v3(boxes, points, *GLOBAL_SCALE)
                choice = np.random.choice(np.arange(points.shape[0]), points.shape[0], replace=False)
                points = points[choice]
                out["points"], out["boxes"] = points, boxes
            else:
                choice = np.random.choice(np.arange(points.shape[0]), points.shape[0], replace=False)
                points = points[choice]
                _, points, _ = prep.random_flip_v2(None, points)
                _, points, _ = prep.global_rotation_v3(None, points, GLOBAL_ROT)
                _, points, _ = prep.global_scaling_v3(None, points, *GLOBAL_SCALE)
                out["points"] = points
    finally:
        prep.noise_per_box, prep.points_in_convex_polygon_3d_jit = orig_npb, orig_pic
    if labeled:
        out["selected"] = np.asarray(rec["selected"], np.int32)
        out["masks"] = np.asarray(rec["masks"], bool).reshape(len(points), len(valid))
    vals = [v for _, v in log]
    if labeled:
        d = dict(loc=vals[0], rot=vals[1], flip=bool(vals[2]), rotation=float(vals[3]), scale=float(vals[4]), perm=vals[5])
    else:
        d = dict(loc=np.zeros((0, 100, 3)), rot=np.zeros((0, 100)), perm=vals[0], flip=bool(vals[1]), rotation=float(vals[2]),
                 scale=float(vals[3]))
    return out, d


# ------------------------------------------------------------------------------------------------------------------ crafted frames
def _local(points, boxes, context):
    p = points[:, :3].astype(np.float64)[:, None, :]
    b = boxes.astype(np.float64)
    d = p - b[None, :, :3]
    c, s = np.cos(b[:, 6]), np.sin(b[:, 6])
    lx = d[..., 0] * c - d[..., 1] * s
    ly = d[..., 0] * s + d[..., 1] * c
    dims = b[:, 3:6].copy()
    if context > 0:
        dims[:, :2] += context
    return np.stack([lx, ly, d[..., 2]], -1), dims


def keep_off_faces(points, boxes, context):
    """drop every point within MARGIN of a face plane of any box (in the box's own frame)"""
    if len(boxes) == 0 or len(points) == 0:
        return points
    loc, dims = _local(points, boxes, context)
    gap = np.abs(np.abs(loc) - dims[None] / 2).min(axis=(1, 2))
    return points[gap >= MARGIN]


def inside_points(rs, box, n, context=-1.0):
    """n points inside a box (in its frame, at least 2 * MARGIN from every face)"""
    dims = np.array(box[3:6], np.float64)
    if context > 0:
        dims[:2] += context
    loc = (rs.uniform(-0.5, 0.5, size=(n, 3)) * (dims - 4 * MARGIN))
    c, s = np.cos(box[6]), np.sin(box[6])
    x = loc[:, 0] * c + loc[:, 1] * s + box[0]
    y = -loc[:, 0] * s + loc[:, 1] * c + box[1]
    z = loc[:, 2] + box[2]
    return np.stack([x, y, z, rs.uniform(0, 1, n)], 1).astype(np.float32)


def scene(rs, n_boxes, n_bg, spacing=6.0, jitter=1.0):
    """cars on a jittered grid (no two overlap), background points and points inside every box"""
    cells = [(x, y) for x in np.arange(8.0, 64.0, spacing) for y in np.arange(-32.0, 32.0, spacing)]
    pick = rs.choice(len(cells), n_boxes, replace=False)
    boxes = []
    for k in pick:
        x, y = cells[k]
        boxes.append([x + rs.uniform(-jitter, jitter), y + rs.uniform(-jitter, jitter), -1.0 + rs.uniform(-0.3, 0.3),
                      rs.uniform(1.5, 1.8), rs.uniform(3.5, 4.3), rs.uniform(1.4, 1.7), rs.uniform(-np.pi, np.pi)])
    return np.array(boxes, np.float32).reshape(-1, 7), bg_points(rs, n_bg)


def bg_points(rs, n):
    return np.stack([rs.uniform(0, 70, n), rs.uniform(-40, 40, n), rs.uniform(-3, 1, n), rs.uniform(0, 1, n)], 1).astype(np.float32)


def with_inside(rs, boxes, bg, per_box, context=-1.0):
    pts = [bg] + [inside_points(rs, b, per_box, context) for b in boxes]
    pts = np.concatenate(pts).astype(np.float32)
    pts = pts[rs.permutation(len(pts))]
    return keep_off_faces(pts, boxes, context)


def crafted_frames(rs):
    """(name, points, boxes, names, labeled, context, seed or crafted draws)"""
    frames = []
    # 1. seeded scene: 15 cars, a Van (valid), a Pedestrian and a Cyclist (invalid: block, never move)
    boxes, bg = scene(rs, 19, 2500)
    names = ["Car"] * 15 + ["Van", "Pedestrian", "Cyclist", "Car"]
    frames.append(("scene", with_inside(rs, boxes, bg, 40), boxes, names, True, -1.0, None))
    # 2. crowded: cars 0.35 m apart (most tries collide), a car inside a 30 m Pedestrian box (every try collides: -1), two identical cars
    grid = [[10.0 + 2.0 * i, -6.0 + 4.35 * j, -1.0, 1.6, 4.0, 1.5, 0.0] for i in range(4) for j in range(3)]
    grid += [[40.0, 20.0, -1.0, 30.0, 30.0, 3.0, 0.2], [40.0, 20.0, -1.0, 1.6, 3.9, 1.5, 0.1],
             [20.0, -25.0, -1.0, 1.6, 3.9, 1.5, 0.7], [20.0, -25.0, -1.0, 1.6, 3.9, 1.5, 0.7]]
    boxes = np.array(grid, np.float32)
    names = ["Car"] * 12 + ["Pedestrian", "Car", "Car", "Car"]
    inner = boxes[[i for i in range(len(boxes)) if i != 12]]       # no points inside the 30 m box except around its car
    pts = np.concatenate([bg_points(rs, 1500)] + [inside_points(rs, b, 30) for b in inner]).astype(np.float32)
    frames.append(("crowded", keep_off_faces(pts, boxes, -1.0), boxes, names, True, -1.0, None))
    # 3. crafted draws: a chain (box 1's try 0 hits box 0 only at box 0's new place), overlapping boxes (first valid wins)
    boxes = np.array([[10.0, 0.0, -1.0, 1.6, 4.0, 1.5, 0.0],      # 0: try 0 moves it +5 m in x
                      [20.0, 0.0, -1.0, 1.6, 4.0, 1.5, 0.0],      # 1: try 0 -> (16, 0.3) (hits 0 at 15), try 1 -> x = 23
                      [30.0, 10.0, -1.0, 3.0, 5.0, 2.0, 0.3],     # 2: Pedestrian (invalid) overlapping 3
                      [31.0, 10.5, -1.0, 1.8, 4.2, 1.6, 0.0],     # 3: Car inside 2 -> every try collides with 2 (-1)
                      [40.0, -10.0, -1.0, 2.0, 4.0, 1.6, 0.0],    # 4 / 5: overlapping cars (points in both move with 4)
                      [40.5, -10.0, -1.0, 2.0, 4.0, 1.6, 0.4]], np.float32)
    names = ["Car", "Car", "Pedestrian", "Car", "Car", "Car"]
    m = len(boxes)
    loc = np.zeros((m, 100, 3)); rot = np.zeros((m, 100))
    loc[:, :, 0] = rs.uniform(30, 40, size=(m, 100))              # default tries: far away in x, free -> try 0 unless crafted below
    loc[:, :, 1] = rs.uniform(-0.2, 0.2, size=(m, 100)); loc[:, :, 2] = rs.normal(scale=0.3, size=(m, 100))
    rot[:] = rs.uniform(-0.5, 0.5, size=(m, 100))
    loc[0, 0] = [5.0, 0.0, 0.1]; rot[0, 0] = 0.0
    loc[1, 0] = [-4.0, 0.3, 0.0]; rot[1, 0] = 0.0
    loc[1, 1] = [3.0, 0.5, -0.2]; rot[1, 1] = 0.05
    loc[3] = rs.normal(scale=0.05, size=(100, 3)); rot[3] = rs.uniform(-0.05, 0.05, 100)
    loc[4, :, 0] = loc[4, :, 0] + 40.0                               # 4 moves (far: x + 70 .. 80), 5 then tries x + 30 .. 40
    pts = np.concatenate([bg_points(rs, 800)] + [inside_points(rs, b, 40) for b in boxes]).astype(np.float32)
    pts = keep_off_faces(pts, boxes, -1.0)
    draws = [loc, rot, np.False_, 0.3, 1.02, None]
    frames.append(("chain", pts, boxes, names, True, -1.0, draws))
    # 4. context: boxes enlarged by data_aug_with_context = 1.0 for the collision test and the point membership
    boxes, bg = scene(rs, 10, 1500, spacing=5.0, jitter=0.4)
    frames.append(("context", with_inside(rs, boxes, bg, 30, context=1.0), boxes, ["Car"] * 10, True, 1.0, None))
    # 5. no boxes; 6. empty frame; 7. unlabelled
    frames.append(("no_boxes", bg_points(rs, 700), np.zeros((0, 7), np.float32), [], True, -1.0, None))
    frames.append(("empty", np.zeros((0, 4), np.float32), np.zeros((0, 7), np.float32), [], True, -1.0, None))
    frames.append(("unlabelled", bg_points(rs, 900), np.zeros((0, 7), np.float32), [], False, -1.0, None))
    return frames


def collision_cases(bnp, rs):
    P = np.pi
    pairs = [
        ((0, 0, 2, 4, 0.0), (0, 0, 2, 4, 0.0)),            # identical: no crossing, no strict containment -> no collision
        ((0, 0, 4, 6, 0.3), (0.2, 0.1, 1, 1, 0.5)),        # box contains qbox
        ((0.2, 0.1, 1, 1, 0.5), (0, 0, 4, 6, 0.3)),        # qbox contains box
        ((0, 0, 2, 2, 0.0), (2, 0, 2, 2, 0.0)),            # edge-touching
        ((0, 0, 2, 2, 0.0), (2, 2, 2, 2, 0.0)),            # corner-touching
        ((0, 0, 2, 2, 0.0), (2, 0.5, 2, 1, 0.0)),          # edge-touching, partial edge
        ((0, 0, 1, 6, 0.0), (0, 0, 1, 6, P / 2)),          # crossing (no corner inside the other)
        ((0, 0, 1, 6, P / 4), (2.4, -2.4, 1, 6, P / 4)),   # parallel diagonals: standups overlap, boxes do not
        ((0, 0, 1, 4, P / 4), (2.2, 0, 1, 4, -P / 4)),     # a V: the ends overlap
        ((0, 0, 2, 4, 0.0), (1.5, 0.5, 2, 4, 0.2)),        # partial overlap
        ((0, 0, 2, 4, 0.0), (10, 10, 2, 4, 0.0)),          # far apart
        ((0, 0, 2, 4, 0.0), (1, 0, 2, 4, 0.0)),            # overlap with collinear edges only: the reference finds no collision
    ]
    a = np.array([p[0] for p in pairs], np.float64); b = np.array([p[1] for p in pairs], np.float64)
    ra = np.concatenate([a, np.stack([rs.uniform(0, 12, 40), rs.uniform(0, 12, 40), rs.uniform(1, 3, 40), rs.uniform(2, 5, 40),
                                      rs.uniform(-P, P, 40)], 1)])
    rb = np.concatenate([b, np.stack([rs.uniform(0, 12, 40), rs.uniform(0, 12, 40), rs.uniform(1, 3, 40), rs.uniform(2, 5, 40),
                                      rs.uniform(-P, P, 40)], 1)])
    ca, cb = bnp.box2d_to_corner_jit(ra), bnp.box2d_to_corner_jit(rb)
    return ca, cb


def main():
    prep, bnp = load_reference()
    rs = np.random.RandomState(2024)
    out = {}
    ca, cb = collision_cases(bnp, rs)
    ref = prep.box_collision_test(ca, cb)
    assert np.array_equal(augment_ref.collision_matrix(ca, cb), ref), "oracle collision test differs from the reference"
    assert np.array_equal(augment_ref.bev_corners(np.concatenate([np.zeros((0, 5))])), np.zeros((0, 4, 2)))
    d = np.diag(ref)[:12]
    assert list(d) == [False, True, True, False, False, False, True, False, True, True, False, False], d
    lo = np.maximum(ca[7].min(0), cb[7].min(0)); hi = np.minimum(ca[7].max(0), cb[7].max(0))
    assert (hi > lo).all()                      # case 7: the standup boxes overlap, the boxes do not
    out.update(coll_boxes=ca, coll_qboxes=cb, coll_ref=ref)

    frames = crafted_frames(rs)
    seeds = iter([11, 12, 13, 14, 15, 16, 17])
    flips = []
    for f, (name, pts, boxes, names, labeled, ctx, crafted) in enumerate(frames):
        valid = np.array([n in CLASS_NAMES for n in names], bool)
        if crafted is None:
            seed = next(seeds)
            while True:                         # the first two seeded frames: one unflipped, one flipped
                res, dr = run_reference(prep, pts, boxes, valid, labeled, ctx, np.random.RandomState(seed))
                if f > 1 or dr["flip"] == (f == 1):
                    break
                seed += 100
        else:
            seed = -1
            src = list(crafted)
            src[-1] = np.random.RandomState(99).permutation(len(pts))
            res, dr = run_reference(prep, pts, boxes, valid, labeled, ctx, src)
        flips.append(dr["flip"])
        # the oracle restates every stored output
        orc = augment_ref.augment_frame(pts, boxes, valid, dr, ctx, labeled)
        for k, v in res.items():
            assert np.array_equal(orc[k], v), (name, k, np.abs(orc[k].astype(float) - v.astype(float)).max() if orc[k].shape == v.shape else
                                              (orc[k].shape, v.shape))
        pre = "f%d_" % f
        out.update({pre + "name": name, pre + "in_points": pts, pre + "in_boxes": boxes, pre + "valid": valid, pre + "labeled": labeled,
                    pre + "context": ctx, pre + "seed": seed, pre + "loc": np.asarray(dr["loc"], np.float64),
                    pre + "rot": np.asarray(dr["rot"], np.float64), pre + "flip": dr["flip"], pre + "rotation": dr["rotation"],
                    pre + "scale": dr["scale"], pre + "perm": np.asarray(dr["perm"], np.int64)})
        out.update({pre + k: v for k, v in res.items()})
        sel = res.get("selected", np.zeros(0))
        print("%-10s points %5d boxes %2d  selected %s  flip %d" % (name, len(pts), len(boxes), sel.tolist(), dr["flip"]))
    assert True in flips and False in flips
    out["num_frames"] = len(frames)
    np.savez_compressed(os.path.join(HERE, "augment_cases.npz"), **out)


if __name__ == "__main__":
    main()
