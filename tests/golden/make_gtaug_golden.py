"""Generate tests/golden/gtaug_cases.npz by running the REFERENCE's own GT-database sampling in place on the CPU.

    python tests/golden/make_gtaug_golden.py

Writes a crafted database into a temporary directory -- a dbinfos pickle and one `.bin` per object (fp32 points minus the fp64 box
centre), laid out as det3d/datasets/utils/create_gt_database.py writes them -- and loads the reference's det3d/core/sampler/sample_ops_v2.py,
det3d/core/sampler/preprocess.py and det3d/core/bbox/box_np_ops.py where they lie, through the ``sys.modules`` shims of
make_augment_golden.py.  It builds the reference's DataBaseSamplerV2 with its DataBasePreprocessor (DBFilterByMinNumPoint, then
DBFilterByDifficulty) and, per frame, runs `sample_all` and lines 96-110 of Preprocess.__call__ (remove_points_after_sample through
points_in_rbbox, the concatenations) in place, then the frame's per-object noise, global stages and shuffle through make_augment_golden's
stage runner (Preprocess.__call__ itself is not imported: its module pulls in the dataset, evaluation and SA-DA packages).  Every draw
comes from the global np.random, seeded once, in the reference's order: the samplers' construction shuffles, then per frame GT-AUG's
draws before noise_per_object_v4_'s.  The noise stage gets the pasted boxes as fp32, the dtype the device stages take.

Stored: the database (db_rel_points, db_off, db_count, db_boxes fp64, db_names, db_difficulty, db_num_points_in_gt, db_class = the
pickle's dict order), the config (groups, min points, difficulties, similar type), the seed, per frame f (prefix "f<f>_"): in_points,
in_boxes (fp64), in_names, and the reference's outputs: ids (accepted objects as indices into the stored database, acceptance order),
gt_boxes / gt_names (after GT-AUG), points_pasted, and the later stages' draws and outputs (selected, points, points_raw, boxes,
boxes_raw, loc, rot, flip, rotation, scale, perm).  Every crafted scene point is at least MARGIN = 1e-3 from every face of every box.
The script checks oracle/gt_aug_ref.py against every stored output before writing.
"""
import importlib.util
import os
import pickle
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle import augment_ref, gt_aug_ref  # noqa: E402

MARGIN = 1e-3
SEED = 7
GROUPS = [("Car", 15)]
MIN_POINTS = {"Car": 5}
REMOVED_DIFF = [-1]
SIMILAR = True                                  # Van joins the Car stream: its extra construction shuffle and a zero-point Van
CLASS_NAMES = ["Car", "Van"]


def _augment_golden():
    spec = importlib.util.spec_from_file_location("make_augment_golden", os.path.join(HERE, "make_augment_golden.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def load_sampler_modules():
    mag = _augment_golden()
    prep, bnp = mag.load_reference()
    mag._stub("det3d.utils")
    mag._stub("det3d.utils.check", shape_mergeable=None)
    ops = mag._load("det3d.core.sampler.sample_ops_v2", "det3d/core/sampler/sample_ops_v2.py")
    return prep, bnp, ops


class _Log:
    def info(self, *a):
        pass


def box(x, y, r=0.0, w=1.6, l=3.9, h=1.5, z=-1.0):
    # fp64 values off the fp32 grid, as box_camera_to_lidar leaves them
    return np.array([x + 1e-7 / 3, y - 1e-7 / 7, z + 1e-8, w + 1e-9, l, h, r], np.float64)


def inside(rs, b, n):
    dims = b[3:6] - 4 * MARGIN
    loc = rs.uniform(-0.5, 0.5, size=(n, 3)) * dims
    c, s = np.cos(b[6]), np.sin(b[6])
    x = loc[:, 0] * c + loc[:, 1] * s + b[0]
    y = -loc[:, 0] * s + loc[:, 1] * c + b[1]
    return np.stack([x, y, loc[:, 2] + b[2], rs.uniform(0, 1, n)], 1).astype(np.float32)


def crafted_db(rs):
    cars = [box(10, -10), box(10, 0), box(10, 10), box(20, -10, 0.4), box(20, 0), box(20, 10, -0.3), box(30, -10), box(30, 10),
            box(50, 0.0), box(51.0, 0.5, 0.2),                          # a colliding pair
            box(60.0, -10), box(61.2, -10), box(62.4, -10)]             # a chain: A-B and B-C collide, A-C do not
    infos = {"Car": [], "Pedestrian": [], "Van": [], "Cyclist": []}
    n_pts = [30, 25, 3, 40, 20, 35, 2, 28, 22, 26, 24, 27, 21]          # two under the min-points filter
    diff = [0] * 13
    diff[7] = -1                                                         # one dropped by the difficulty filter
    objs = [("Car", b, n, d) for b, n, d in zip(cars, n_pts, diff)]
    objs += [("Pedestrian", box(40, 5, 0, 0.6, 0.8, 1.7), 10, 0), ("Pedestrian", box(40, -5, 0, 0.6, 0.8, 1.7), 12, 0),
             ("Van", box(30, 0, 0.1, 2.0, 5.0, 2.0), 0, 0), ("Van", box(45, 15, 0.5, 2.0, 5.0, 2.0), 18, 0),
             ("Cyclist", box(40, 15, 0, 0.6, 1.8, 1.7), 8, 0)]
    files = []
    for k, (name, b, n, d) in enumerate(objs):
        pts = inside(rs, b, n) if n else np.zeros((0, 4), np.float32)
        rel = pts.copy()
        rel[:, :3] -= b[:3]                                              # create_gt_database: fp32 points -= fp64 centre
        fn = "gt_database/%06d_%s_%d.bin" % (k, name, k)
        files.append((fn, rel))
        infos[name].append({"name": name, "path": fn, "image_idx": k, "gt_idx": 0, "box3d_lidar": b, "num_points_in_gt": n,
                            "difficulty": d, "group_id": k})
    return infos, files


def off_faces(points, boxes):
    if len(points) == 0 or len(boxes) == 0:
        return points
    p = points[:, :3].astype(np.float64)[:, None, :]
    b = np.asarray(boxes, np.float64)
    d = p - b[None, :, :3]
    c, s = np.cos(b[:, 6]), np.sin(b[:, 6])
    loc = np.stack([d[..., 0] * c - d[..., 1] * s, d[..., 0] * s + d[..., 1] * c, d[..., 2]], -1)
    gap = np.abs(np.abs(loc) - b[None, :, 3:6] / 2).min(axis=(1, 2))
    return points[gap >= MARGIN]


def crafted_frames(rs, db_boxes):
    def scene(n):
        return np.stack([rs.uniform(5, 66, n), rs.uniform(-13, 13, n), rs.uniform(-1.8, -0.2, n), rs.uniform(0, 1, n)], 1).astype(np.float32)
    frames = [("empty", np.zeros((0, 4), np.float32), np.zeros((0, 7)), [])]
    full = [box(2 + 4.5 * (i % 5), -30 - 5 * (i // 5)) for i in range(15)]
    frames.append(("full", scene(300), np.stack(full), ["Car"] * 15))
    peds = [box(x, y, 0, 0.6, 0.8, 1.7) for x, y in ((10, -10), (10, 0), (20, -10), (20, 0), (50, 0), (61.2, -10))]
    frames.append(("ped_block", scene(600), np.stack(peds + [box(20, 10), box(3, 30)]), ["Pedestrian"] * 6 + ["Van", "Car"]))
    for k in range(5):
        m = int(rs.randint(0, 4))
        bx = [box(rs.uniform(0, 60), rs.uniform(25, 35), rs.uniform(-1, 1)) for _ in range(m)]
        frames.append(("scene%d" % k, scene(800), np.stack(bx) if m else np.zeros((0, 7)), ["Car"] * m))
    out = []
    for name, pts, bx, names in frames:
        pts = off_faces(off_faces(pts, bx), db_boxes)
        out.append((name, pts, np.asarray(bx, np.float64).reshape(-1, 7), np.array(names, dtype="<U10")))
    return out


def main():
    prep, bnp, ops = load_sampler_modules()
    mag = _augment_golden()
    rs = np.random.RandomState(2025)
    infos, files = crafted_db(rs)
    all_infos = [i for v in infos.values() for i in v]
    db_boxes = np.stack([i["box3d_lidar"] for i in all_infos])
    frames = crafted_frames(rs, db_boxes)
    with tempfile.TemporaryDirectory() as root:
        os.makedirs(os.path.join(root, "gt_database"))
        for fn, rel in files:
            rel.tofile(os.path.join(root, fn))
        with open(os.path.join(root, "dbinfos_train.pkl"), "wb") as f:
            pickle.dump(infos, f)
        with open(os.path.join(root, "dbinfos_train.pkl"), "rb") as f:
            ref_infos = pickle.load(f)
        gid = {(i["path"]): n for n, i in enumerate(all_infos)}
        log = _Log()
        np.random.seed(SEED)
        prepor = prep.DataBasePreprocessor([prep.DBFilterByMinNumPoint(MIN_POINTS, logger=log),
                                            prep.DBFilterByDifficulty(REMOVED_DIFF, logger=log)])
        sampler = ops.DataBaseSamplerV2(ref_infos, [dict(GROUPS)], prepor, 1.0, [0, 0], logger=log, gt_random_drop=-1.0,
                                        gt_aug_with_context=-1.0, gt_aug_similar_type=SIMILAR)
        streams = {k: s._indices.copy() for k, s in sampler._sampler_dict.items()}
        out = {}
        for f, (name, pts, bx, names) in enumerate(frames):
            sd = sampler.sample_all(root, bx, names, 4, False, gt_group_ids=None, calib=None, targeted_class_names=CLASS_NAMES)
            points, gt_boxes, gt_names = pts.copy(), bx, names
            valid = np.array([n in CLASS_NAMES for n in names], bool)
            ids = np.zeros(0, np.int64)
            if sd is not None:
                gt_names = np.concatenate([gt_names, sd["gt_names"]], axis=0)
                gt_boxes = np.concatenate([gt_boxes, sd["gt_boxes"]])
                valid = np.concatenate([valid, sd["gt_masks"]], axis=0)
                masks = bnp.points_in_rbbox(points, sd["gt_boxes"])
                points = points[np.logical_not(masks.any(-1))]
                points = np.concatenate([sd["points"], points], axis=0)
                # which database objects: match the sampled boxes to the stored ones (every crafted box is distinct)
                ids = np.array([int(np.nonzero((db_boxes == b).all(1))[0][0]) for b in sd["gt_boxes"]], np.int64)
                assert gt_boxes.dtype == np.float64
            res, dr = mag.run_reference(prep, points.astype(np.float32), gt_boxes.astype(np.float32), valid, True, -1.0,
                                        np.random.mtrand._rand)
            pre = "f%d_" % f
            out.update({pre + "name": name, pre + "in_points": pts, pre + "in_boxes": bx, pre + "in_names": names, pre + "ids": ids,
                        pre + "gt_boxes": gt_boxes, pre + "gt_names": gt_names, pre + "points_pasted": points, pre + "valid": valid,
                        pre + "loc": np.asarray(dr["loc"], np.float64), pre + "rot": np.asarray(dr["rot"], np.float64),
                        pre + "flip": dr["flip"], pre + "rotation": dr["rotation"], pre + "scale": dr["scale"],
                        pre + "perm": np.asarray(dr["perm"], np.int64)})
            out.update({pre + k: v for k, v in res.items() if k != "masks"})
            print("%-10s points %4d -> %4d  boxes %2d  accepted %s" % (name, len(pts), len(points), len(bx), ids.tolist()))
    rel = [r for _, r in files]
    cnt = np.array([len(r) for r in rel], np.int64)
    out.update(db_rel_points=np.concatenate(rel), db_count=cnt, db_off=np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.int64),
               db_boxes=db_boxes, db_names=np.array([i["name"] for i in all_infos]), db_difficulty=np.array([i["difficulty"] for i in all_infos]),
               db_num_points_in_gt=np.array([i["num_points_in_gt"] for i in all_infos]), db_class=np.array(list(infos.keys())),
               seed=SEED, num_frames=len(frames), similar=SIMILAR, max_num=GROUPS[0][1], min_points=MIN_POINTS["Car"])
    check_oracle(out)
    np.savez_compressed(os.path.join(HERE, "gtaug_cases.npz"), **out)


def db_infos_from(z):
    """the stored database as a dbinfos dict (dict order of the pickle); 'path' indexes the stored points"""
    infos = {str(c): [] for c in z["db_class"]}
    for k in range(len(z["db_names"])):
        infos[str(z["db_names"][k])].append({"name": str(z["db_names"][k]), "path": "gt_database/%06d_%s_%d.bin" % (k, z["db_names"][k], k),
                                             "image_idx": k, "gt_idx": 0, "box3d_lidar": z["db_boxes"][k],
                                             "num_points_in_gt": int(z["db_num_points_in_gt"][k]), "difficulty": int(z["db_difficulty"][k]),
                                             "group_id": k})
    return infos


def check_oracle(z):
    """oracle/gt_aug_ref.py against every stored output; asserts the crafted cases were reached"""
    infos = db_infos_from(z)
    order = [i["image_idx"] for v in infos.values() for i in v]
    filt = gt_aug_ref.filter_db(infos, {"Car": int(z["min_points"])}, [-1])
    rs = np.random.RandomState(int(z["seed"]))
    g = gt_aug_ref.GtAug(filt, [("Car", int(z["max_num"]))], rs, similar=bool(z["similar"]))
    fid = np.array([i["image_idx"] for i in g.infos])               # oracle global id -> stored database index
    rel = [z["db_rel_points"][o:o + n] for o, n in zip(z["db_off"], z["db_count"])]
    seen = dict(short=False, exact=False, ped=False, pair=False, chain=False, round2=False, removed=False, zero=False, full=False)
    orig_take = gt_aug_ref.Sampler.take

    def take(self, num):
        if self.idx + num > len(self.ind):
            seen["short"] = True
        elif self.idx + num == len(self.ind):
            seen["exact"] = True
        return orig_take(self, num)
    gt_aug_ref.Sampler.take = take
    try:
        for f in range(int(z["num_frames"])):
            pre = "f%d_" % f
            bx, names = z[pre + "in_boxes"], z[pre + "in_names"]
            ids, log = g.sample_frame(bx, names)
            ids = fid[ids]
            assert np.array_equal(ids, z[pre + "ids"]), (f, ids, z[pre + "ids"])
            seen["full"] |= (np.sum(names == "Car") >= 15 and not log)
            seen["round2"] |= len(log) == 2
            for r, (_, cand, acc) in enumerate(log):
                cb = gt_aug_ref.corners(g.boxes[cand], True)
                if r == 1:                              # an object accepted in round 1 blocks a round-2 candidate
                    prev = gt_aug_ref.corners(g.boxes[log[0][1][log[0][2]]], True)
                    seen["chain"] |= any(not acc[a] and any(augment_ref.collide(cb[a], q) for q in prev) for a in range(len(cand)))
                for a in range(len(cand)):
                    for b in range(a + 1, len(cand)):
                        if augment_ref.collide(cb[a], cb[b]):
                            seen["pair"] |= (not acc[a]) and acc[b]
                if "Pedestrian" in list(names):
                    pc = gt_aug_ref.corners(bx[[n == "Pedestrian" for n in names]])
                    seen["ped"] |= any(not acc[a] and any(augment_ref.collide(cb[a], q) for q in pc) for a in range(len(cand)))
            seen["zero"] |= any(z["db_count"][i] == 0 for i in ids)
            pts, boxes, gnames, _ = gt_aug_ref.paste(z[pre + "in_points"], bx, names, ids, rel, z["db_boxes"], z["db_names"])
            assert np.array_equal(pts, z[pre + "points_pasted"]), f
            assert np.array_equal(boxes, z[pre + "gt_boxes"]) and boxes.dtype == z[pre + "gt_boxes"].dtype, f
            assert list(gnames) == list(z[pre + "gt_names"]), f
            seen["removed"] |= len(pts) < len(z[pre + "in_points"]) + sum(z["db_count"][i] for i in ids)
            draws = dict(loc=z[pre + "loc"], rot=z[pre + "rot"], flip=bool(z[pre + "flip"]), rotation=float(z[pre + "rotation"]),
                         scale=float(z[pre + "scale"]), perm=z[pre + "perm"])
            # the rest of the stream: noise_per_object_v4_ then the global stages and the shuffle (sized by the pasted frame)
            assert draws["loc"].shape[0] == len(boxes) and len(draws["perm"]) == len(pts)
            rs_loc = rs.normal(scale=np.array([1.0, 1.0, 0.5], np.float32), size=[len(boxes), 100, 3])
            rs_rot = rs.uniform(-0.785, 0.785, size=[len(boxes), 100])
            assert np.array_equal(rs_loc, draws["loc"]) and np.array_equal(rs_rot, draws["rot"]), f
            assert bool(rs.choice([False, True], replace=False, p=[0.5, 0.5])) == draws["flip"]
            assert float(rs.uniform(-0.785, 0.785)) == draws["rotation"] and float(rs.uniform(0.95, 1.05)) == draws["scale"]
            assert np.array_equal(rs.choice(np.arange(len(pts)), len(pts), replace=False), draws["perm"])
            orc = gt_aug_ref.preprocess_frame(z[pre + "in_points"], bx, names, ids, rel, z["db_boxes"], z["db_names"], CLASS_NAMES, draws)
            for k in ("selected", "points", "points_raw", "boxes", "boxes_raw"):
                assert np.array_equal(orc[k], z[pre + k]), (f, k)
    finally:
        gt_aug_ref.Sampler.take = orig_take
    del order
    missing = [k for k, v in seen.items() if not v]
    assert not missing, "crafted cases not reached: %s" % missing


if __name__ == "__main__":
    main()
