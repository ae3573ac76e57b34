"""Generate tests/golden/sada_cases.npz by running the REFERENCE's own shape-aware augmentation in place on the CPU.

    python tests/golden/make_sada_golden.py

Loads the reference's det3d/datasets/utils/sa_da_v2.py where it lies (with det3d/core/bbox/box_np_ops.py and geometry.py, through the
``sys.modules`` shims of make_augment_golden.py) and installs a stand-in ``ifp`` module: its ``ifp_sample(dists, indices, k)`` is the
farthest-point contract of sessd_b200.sada (start at row 0, the largest distance to the nearest pick, ties to the lowest row), fed by the
real scipy cKDTree's complete neighbour lists.  Each case seeds np.random and runs pyramid_augment_v0 three times: with the dropout
only, with dropout and sparsify, and with all three steps, so the stored rows after each step come from the same draws.

Stored, kept small: each distinct input frame once as a scene (prefix "s<k>_"): points [N, 4] f32, boxes [K, 7] f32, pyramids
[K, 6, 15] (get_pyramids) and mask [N, 6K] (points_in_pyramids_mask of the input points, bit-packed along the rows).  Per case c
(prefix "c<c>_"): name, scene, cfg (dropout, sparsity p, sparsity n, swap p, swap n; NaN = off), seed, the rows after each step as
<step>_keep (the rows of the step before that come first, in order, bit-packed) and <step>_tail (the rows that follow them), and state
(the RandomState's key and position after the full call); ``decode`` rebuilds the rows.  Crafted points lie at least MARGIN (in
box-normalised coordinates) away from every face and every diagonal plane of every pyramid, except in the "diagonal" case, whose points
lie exactly on diagonal planes of an axis-aligned box (every sign there is an exact zero).  Box angles are chosen where numpy's float32
sin / cos equal the correctly rounded values (tests/sada_ref.py).  The script checks tests/sada_ref.py against every stored output
before writing.
"""
import importlib.util
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
ROOT = os.path.dirname(TESTS)
for p in (os.path.join(ROOT, "se-ssd_b200"), TESTS):
    if p not in sys.path:
        sys.path.insert(0, p)
import sada_ref  # noqa: E402

MARGIN = 0.02


def ifp_sample(dists, indices, k):
    n = dists.shape[0]
    d = np.empty((n, n))
    d[np.arange(n)[:, None], indices] = dists
    cur = np.full(n, np.inf)
    picks, pick = [], 0
    for _ in range(k):
        picks.append(pick)
        cur = np.minimum(cur, d[pick])
        pick = int(np.argmax(cur))
    return np.array(picks)


def load_sada():
    spec = importlib.util.spec_from_file_location("make_augment_golden", os.path.join(HERE, "make_augment_golden.py"))
    mag = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mag)
    mag.load_reference()
    sys.modules["ifp"] = types.SimpleNamespace(ifp_sample=ifp_sample)
    for p in ("det3d.datasets", "det3d.datasets.utils"):
        mag._pkg(p)
    return mag._load("det3d.datasets.utils.sa_da_v2", "det3d/datasets/utils/sa_da_v2.py")


def angle(rs, lo=-3.1, hi=3.1):
    """an fp32 angle whose numpy float32 sin / cos are the correctly rounded values"""
    while True:
        a = np.float32(rs.uniform(lo, hi))
        s, c = sada_ref.sincos32(a)
        if np.sin(np.array([a]))[0] == s and np.cos(np.array([a]))[0] == c:
            return a


def box(rs, x, y, z=-1.0, w=1.6, l=3.9, h=1.5, r=None):
    return np.array([x, y, z, w, l, h, angle(rs) if r is None else r], np.float32)


def pyramid_points(rs, b, face, n, intensity=None):
    """n points strictly inside pyramid `face` of box b, MARGIN away from its faces and diagonals (box-normalised coordinates)"""
    out = []
    axis, sign = [(1, -1), (0, 1), (1, 1), (0, -1), (2, 1), (2, -1)][face]
    while len(out) < n:
        q = rs.uniform(-1 + MARGIN, 1 - MARGIN, 3)
        q[axis] = sign * abs(q[axis])
        a = np.abs(q)
        others = [a[i] for i in range(3) if i != axis]
        if a[axis] - max(others) < MARGIN:
            continue
        out.append(q)
    q = np.array(out).reshape(-1, 3) * 0.5 * b[3:6].astype(np.float64)
    c, s = np.cos(np.float64(b[6])), np.sin(np.float64(b[6]))
    x = q[:, 0] * c + q[:, 1] * s + b[0]                        # rotation_3d_in_axis(axis=2): rot_mat_T = [[c, -s], [s, c]]
    y = -q[:, 0] * s + q[:, 1] * c + b[1]
    w = rs.uniform(0, 1, len(q)) if intensity is None else np.full(len(q), intensity)
    return np.stack([x, y, q[:, 2] + b[2], w], 1).astype(np.float32)


def box_points(rs, b, n, intensity=None):
    return np.concatenate([pyramid_points(rs, b, f, k, intensity) for f, k in enumerate(np.broadcast_to(n, 6))])


def scene(rs, n):
    return np.stack([rs.uniform(0, 70, n), rs.uniform(-40, 40, n), rs.uniform(-3, 1, n), rs.uniform(0, 1, n)], 1).astype(np.float32)


def far_from(points, boxes):
    """drop scene points near any box (their pyramid membership is decided by the crafted points alone)"""
    if len(boxes) == 0:
        return points
    d = np.min(np.hypot(points[:, None, 0] - boxes[None, :, 0], points[:, None, 1] - boxes[None, :, 1]), 1)
    return points[d > 4.0]


CAR = (0.25, 0.05, 50, 0.1, 50)


def cases():
    rs = np.random.RandomState(2024)
    out = []
    # no boxes; no points
    out.append(("no_boxes", scene(rs, 300), np.zeros((0, 7), np.float32), CAR, 1))
    b = np.stack([box(rs, 10, 0), box(rs, 20, 5)])
    out.append(("no_points", np.zeros((0, 4), np.float32), b, CAR, 2))
    # dropout: high, and the car values, over a frame of 12 dense boxes
    bs = np.stack([box(rs, 8 + 5 * (i % 6), -12 + 12 * (i // 6)) for i in range(12)])
    pts = np.concatenate([far_from(scene(rs, 2000), bs)] + [box_points(rs, x, 30) for x in bs])
    out.append(("dropout_high", pts, bs, (0.9, None, None, None, None), 3))
    out.append(("car", pts, bs, CAR, 4))
    out.append(("car_b", pts, bs, CAR, 5))
    # the `>` boundary: 50 points in every pyramid of the first box, 51 in the second's
    b2 = np.stack([box(rs, 10, 3), box(rs, 18, -3)])
    pts = np.concatenate([far_from(scene(rs, 500), b2), box_points(rs, b2[0], 50), box_points(rs, b2[1], 51)])
    out.append(("boundary", pts, b2, (None, 1.0, 50, None, None), 6))
    # two overlapping boxes (points in two pyramids), both sparsified
    b3 = np.stack([box(rs, 12, 0, r=np.float32(0.0)), box(rs, 12.4, 0.3, r=angle(rs, 0.2, 0.4))])
    pts = np.concatenate([box_points(rs, b3[0], 80), box_points(rs, b3[1], 80)])
    out.append(("overlap", pts, b3, (None, 1.0, 50, None, None), 7))
    # a self-partner swap: one box
    b4 = box(rs, 15, 2)[None]
    out.append(("self_swap", box_points(rs, b4[0], 60), b4, (None, None, None, 1.0, 50), 8))
    # constant intensity (the clip), two boxes swapping
    b5 = np.stack([box(rs, 10, 4), box(rs, 20, -4)])
    pts = np.concatenate([box_points(rs, b5[0], 60, 0.5), box_points(rs, b5[1], 60, 0.5)])
    out.append(("constant_intensity", pts, b5, (None, None, None, 1.0, 50), 9))
    # two boxes choosing the same partner; sparsify and swap both firing (seeds searched below)
    b6 = np.stack([box(rs, 8 + 6 * i, 0) for i in range(4)])
    pts = np.concatenate([box_points(rs, x, [60, 60, 60, 60, 60, 60]) for x in b6])
    out.append(("same_partner", pts, b6, (None, None, None, 0.6, 50), None))
    out.append(("sparsify_and_swap", pts, b6, (None, 0.5, 50, 0.6, 50), None))
    # points exactly on diagonal planes of an axis-aligned box centred at the origin: every sign is an exact 0 (outside)
    b7 = np.array([[0, 0, 0, 2, 2, 2, 0]], np.float32)
    on = np.array([[0.5, 0.5, 0, 0.3], [-0.5, 0.5, 0.25, 0.6], [0.25, 0, 0.25, 0.9], [0, -0.5, -0.5, 0.1]], np.float32)
    pts = np.concatenate([on, box_points(rs, b7[0], 55)])
    out.append(("diagonal", pts, b7, (None, 1.0, 50, 1.0, 50), 10))
    return out


def kw(cfg):
    d, sp, sn, wp, wn = cfg
    return dict(enable_sa_dropout=d, enable_sa_sparsity=None if sp is None else [sp, sn], enable_sa_swap=None if wp is None else [wp, wn])


def run(sda, points, boxes, cfg, seed):
    k = kw(cfg)
    res = {}
    for name, stage in (("dropout", dict(enable_sa_sparsity=None, enable_sa_swap=None)), ("sparsify", dict(enable_sa_swap=None)),
                        ("swap", {})):
        np.random.seed(seed)
        res[name] = sda.pyramid_augment_v0(boxes, points.copy(), **{**k, **stage})
    res["state"] = np.random.get_state()
    return res


def search(sda, points, boxes, cfg, want):
    for seed in range(100, 2000):
        rs = np.random.RandomState(seed)
        if want(rs, points, boxes, cfg):
            return seed
    raise RuntimeError("no seed found")


def _swap_pairs(rs, points, boxes, cfg):
    """the swap pairs the oracle's draws give (and whether sparsify fired)"""
    d, sp, sn, wp, wn = cfg
    pyr = sada_ref.pyramids(boxes)
    alive = np.arange(len(boxes))
    fired = False
    if sp is not None:
        idx, pick = sada_ref.draw_pick(rs, len(alive), sp)
        m = sada_ref.in_pyramids(points, pyr[alive[pick], idx[pick]])
        fired = bool((m.sum(0) > sn).any())
        if fired:
            mv = m[:, m.sum(0) > sn]
            points = np.concatenate([points[~mv.any(1)]] + [points[mv[:, i]][:sn] for i in range(mv.shape[1])])
        alive = alive[~pick]
    sel = rs.uniform(0, 1, len(alive)) <= wp
    if not sel.any():
        return [], fired
    counts = sada_ref.in_pyramids(points, pyr[alive].reshape(-1, 15)).sum(0).reshape(-1, 6)
    return sada_ref.draw_partners(rs, counts, sel, wn), fired


def encode(prev, out):
    """out as (the rows of prev it starts with, bit-packed; the rows after them): an ordered greedy match, exact by construction"""
    keep = np.zeros(len(prev), bool)
    j = 0
    for i in range(len(prev)):
        if j < len(out) and np.array_equal(prev[i].view(np.uint32), out[j].view(np.uint32)):
            keep[i] = True
            j += 1
    return np.packbits(keep), np.ascontiguousarray(out[j:], np.float32).reshape(-1, 4)


def decode(prev, keep, tail):
    rows = np.unpackbits(keep, count=len(prev)).astype(bool)
    return np.concatenate([np.asarray(prev, np.float32).reshape(-1, 4)[rows], np.asarray(tail, np.float32).reshape(-1, 4)])


def load(path=os.path.join(HERE, "sada_cases.npz")):
    """the stored cases as dicts: name, seed, cfg, points, boxes, pyramids, mask, dropout, sparsify, swap, state_key, state_pos"""
    z = dict(np.load(path))
    out = []
    for c in range(int(z["num_cases"])):
        pre = "c%d_" % c
        sc = "s%d_" % int(z[pre + "scene"])
        case = dict(name=z[pre + "name"], seed=z[pre + "seed"], cfg=z[pre + "cfg"], state_key=z[pre + "state_key"],
                    state_pos=z[pre + "state_pos"], points=z[sc + "points"], boxes=z[sc + "boxes"], pyramids=z[sc + "pyramids"],
                    mask=np.unpackbits(z[sc + "mask"], axis=0, count=int(z[sc + "rows"])).astype(bool))
        prev = case["points"]
        for st in ("dropout", "sparsify", "swap"):
            prev = case[st] = decode(prev, z[pre + st + "_keep"], z[pre + st + "_tail"])
        out.append(case)
    return out


def main():
    sda = load_sada()
    data, scenes = {}, {}
    for c, (name, points, boxes, cfg, seed) in enumerate(cases()):
        if name == "same_partner":
            seed = search(sda, points, boxes, cfg, lambda rs, p, b, f: (lambda pr: len(pr) >= 2 and len({q for _, _, q in pr}) < len(pr))(
                _swap_pairs(rs, p, b, f)[0]))
        elif name == "sparsify_and_swap":
            seed = search(sda, points, boxes, cfg, lambda rs, p, b, f: (lambda r: len(r[0]) > 0 and r[1])(_swap_pairs(rs, p, b, f)))
        res = run(sda, points, boxes, cfg, seed)
        pyr = sda.get_pyramids(boxes)
        mask = sda.points_in_pyramids_mask(points, pyr.reshape(-1, 15)) if len(boxes) else np.zeros((len(points), 0), bool)
        # the oracle reproduces every stored output
        assert np.array_equal(sada_ref.pyramids(boxes), pyr), name
        assert np.array_equal(sada_ref.in_pyramids(points, pyr.reshape(-1, 15)), mask), name
        d, sp, sn, wp, wn = cfg
        rs = np.random.RandomState(seed)
        o = sada_ref.sada(points, boxes, rs, d, None if sp is None else (sp, sn), None if wp is None else (wp, wn))
        for st in ("dropout", "sparsify", "swap"):
            assert o[st].dtype == np.float32 and np.array_equal(o[st], res[st]), (name, st)
        state = rs.get_state()
        assert np.array_equal(state[1], res["state"][1]) and state[2] == res["state"][2], name
        key = points.tobytes() + boxes.tobytes()
        if key not in scenes:
            k = scenes[key] = len(scenes)
            data.update({"s%d_points" % k: points, "s%d_boxes" % k: boxes, "s%d_pyramids" % k: pyr,
                         "s%d_mask" % k: np.packbits(mask, axis=0), "s%d_rows" % k: np.int64(len(points))})
        pre = "c%d_" % c
        data.update({pre + "name": np.array(name), pre + "scene": np.int64(scenes[key]), pre + "seed": np.int64(seed),
                     pre + "cfg": np.array([np.nan if v is None else v for v in cfg], np.float64),
                     pre + "state_key": res["state"][1], pre + "state_pos": np.int64(res["state"][2])})
        prev = points
        for st in ("dropout", "sparsify", "swap"):
            keep, tail = encode(prev, res[st])
            assert np.array_equal(decode(prev, keep, tail), res[st]), (name, st)
            data.update({pre + st + "_keep": keep, pre + st + "_tail": tail})
            prev = res[st]
        print("%-20s N=%5d K=%2d  dropout %5d  sparsify %5d  swap %5d" % (name, len(points), len(boxes), len(res["dropout"]),
                                                                          len(res["sparsify"]), len(res["swap"])))
    data["num_cases"] = np.int64(len(cases()))
    np.savez_compressed(os.path.join(HERE, "sada_cases.npz"), **data)


if __name__ == "__main__":
    main()
