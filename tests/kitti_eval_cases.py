"""Seeded synthetic KITTI sets for the evaluation tests: infos (calibration, image size, ground-truth annotations) and lidar-frame
detections.  Every overlap a case produces (2D, BEV, 3D, and detection-over-DontCare) is kept at least MARGIN away from every
min overlap the evaluation uses, so fp32 rounding differences between implementations cannot flip a match."""
import numpy as np

from oracle import kitti_eval_ref as ref

MARGIN = 1e-4
CLASSES = ["Car", "Pedestrian", "Cyclist"]
THRESHOLDS = sorted({0.25, 0.5, 0.7} | set(np.linspace(0.5, 0.95, 10).tolist()) | set(np.linspace(0.25, 0.7, 10).tolist()))
_SIZES = {"Car": (1.6, 3.9, 1.56), "Van": (1.9, 5.0, 2.1), "Pedestrian": (0.6, 0.8, 1.73), "Person_sitting": (0.6, 0.8, 1.2),
          "Cyclist": (0.6, 1.76, 1.73)}


def calib(rng):
    a = rng.uniform(-0.01, 0.01, 3)
    r0 = np.eye(4)
    r0[:3, :3] = np.array([[1, -a[2], a[1]], [a[2], 1, -a[0]], [-a[1], a[0], 1]])
    tr = np.eye(4)
    tr[:3, :3] = np.array([[0, -1, 0], [0, 0, -1], [1, 0, 0]], dtype=np.float64)
    tr[:3, 3] = [rng.uniform(-0.01, 0.01), rng.uniform(-0.08, -0.06), rng.uniform(-0.3, -0.25)]
    p2 = np.eye(4)
    p2[:3, :] = [[721.5377, 0, 609.5593, 44.85728], [0, 721.5377, 172.854, 0.2163791], [0, 0, 1, 0.002745884]]
    return {"R0_rect": r0, "Tr_velo_to_cam": tr, "P2": p2}


def exact_calib():
    """R0_rect = I and a Tr_velo_to_cam that only permutes axes: camera (x, y, z) = lidar (-y, -z, x) with no rounding, so boxes
    placed edge to edge in lidar stay edge to edge in camera coordinates."""
    tr = np.eye(4)
    tr[:3, :3] = np.array([[0, -1, 0], [0, 0, -1], [1, 0, 0]], dtype=np.float64)
    c = calib(np.random.default_rng(0))
    return {"R0_rect": np.eye(4), "Tr_velo_to_cam": tr, "P2": c["P2"]}


# frame kind 4: a car and a detection that shares its camera-BEV edge x = -0.5 (extent along camera x is l = 4, along z is w = 1.75;
# every value is exact in fp32)
EDGE_GT = np.array([20.0, 2.5, -1.0, 1.75, 4.0, 1.5, 0.0], np.float32)
EDGE_DT = np.array([20.0, -1.5, -1.0, 1.75, 4.0, 1.5, 0.0], np.float32)


def _lidar_box(rng, name, x=None, y=None):
    w, l, h = _SIZES[name]
    s = rng.uniform(0.9, 1.1, 3)
    x = rng.uniform(5, 45) if x is None else x
    y = rng.uniform(-0.45, 0.45) * x if y is None else y
    return np.array([x, y, -1.0, w * s[0], l * s[1], h * s[2], rng.uniform(-np.pi, np.pi)], np.float32)


def _gt_annos(info, lidar, names, rng):
    a = ref.convert_frame(lidar, np.ones(len(lidar), np.float32), np.arange(len(lidar)), info, list(names))
    keep = len(a["name"])
    assert keep == len(lidar), "ground truth must project into the image"
    a = {k: v for k, v in a.items() if k != "score"}
    # alpha as the reference's conversion forms it: numpy's fp32 atan2 of fp32 scalars
    a["alpha"] = np.array([np.float64(-np.arctan2(-b[1], b[0])) + r for b, r in zip(lidar, a["rotation_y"])])
    a["name"] = np.array(list(names))
    a["occluded"] = rng.integers(0, 3, len(lidar)).astype(np.int64)
    a["truncated"] = rng.choice([0.0, 0.1, 0.2, 0.4, 0.6], len(lidar)).astype(np.float64)
    return a


def _add_dontcare(a, boxes):
    n = len(boxes)
    a = dict(a)
    a["name"] = np.concatenate([a["name"], ["DontCare"] * n])
    a["bbox"] = np.concatenate([a["bbox"].reshape(-1, 4), np.asarray(boxes, np.float64).reshape(-1, 4)])
    for k, v in (("alpha", -10.0), ("rotation_y", -10.0), ("truncated", -1.0)):
        a[k] = np.concatenate([a[k], np.full(n, v)])
    a["occluded"] = np.concatenate([a["occluded"], np.full(n, -1, np.int64)])
    a["location"] = np.concatenate([a["location"].reshape(-1, 3), np.full((n, 3), -1000.0)])
    a["dimensions"] = np.concatenate([a["dimensions"].reshape(-1, 3), np.full((n, 3), -1.0)])
    return a


def _near_threshold(ov):
    ov = np.asarray(ov).ravel()
    return np.array([np.min(np.abs(v - np.array(THRESHOLDS))) < MARGIN for v in ov], bool)


def _bad_dets(info, det, gt):
    """Indices of the frame's detections (after conversion) with an overlap near a min overlap; and the converted annotation."""
    a = ref.convert_frame(det["box3d_lidar"], det["scores"], det["label_preds"], info, CLASSES)
    d, g = ref.records(a, "score"), ref.records(gt, "truncated")
    bad = np.zeros(len(d), bool)
    for m in range(3):
        ov = ref.overlaps_frame(m, d, g)
        if ov.size:
            bad |= _near_threshold(ov).reshape(ov.shape).any(1)
    dc = ref.dontcare_boxes(gt)
    if len(dc) and len(d):
        bad |= _near_threshold(ref.box2d_overlap(d[:, :4], dc, 0)).reshape(len(d), len(dc)).any(1)
    return a, bad


def _clean(info, det, gt):
    """Drop detections whose overlaps sit near a threshold (maps converted indices back to the input boxes)."""
    for _ in range(10):
        a, bad = _bad_dets(info, det, gt)
        if not bad.any():
            return det
        # converted annotations keep input order among kept boxes: find the input indices of the kept ones
        b = det["box3d_lidar"]
        kept = [j for j in range(len(b)) if len(ref.convert_frame(b[j:j + 1], det["scores"][j:j + 1], det["label_preds"][j:j + 1],
                                                                  info, CLASSES)["name"])]
        drop = {kept[i] for i in np.nonzero(bad)[0]}
        keep = np.array([j for j in range(len(b)) if j not in drop], np.int64)
        det = {k: (v[keep] if isinstance(v, np.ndarray) else v) for k, v in det.items()}
    raise AssertionError("could not keep overlaps off the thresholds")


def make_set(seed, num_frames, max_dets=30, special=True):
    """(infos, detections) with detections {image_idx str: {box3d_lidar [n,7] f32, scores [n] f32, label_preds [n] i64,
    metadata}} as numpy arrays.  `special` adds the crafted frames (empty, DontCare only, neighbours, identical and edge-touching
    boxes, detections outside the image, tied scores)."""
    rng = np.random.default_rng(seed)
    infos, dets = [], {}
    gt_names = ["Car", "Car", "Car", "Van", "Pedestrian", "Person_sitting", "Car"] + ([] if special else ["Cyclist"])
    for f in range(num_frames):
        info = {"image": {"image_idx": 1000 + f, "image_shape": np.array([375, 1242], np.int32)}, "calib": calib(rng)}
        kind = f % 8 if special else 7
        ng = 0 if kind in (0, 1) else int(rng.integers(1, 9))
        names = [gt_names[i] for i in rng.integers(0, len(gt_names), ng)]
        if kind == 4:
            info["calib"] = exact_calib()
            names[0] = "Car"
        lidar = np.stack([_lidar_box(rng, n) for n in names]) if ng else np.zeros((0, 7), np.float32)
        if kind == 4:
            lidar[0] = EDGE_GT
        gt = _gt_annos(info, lidar, names, rng) if ng else {k: v for k, v in ref.convert_frame(lidar, [], [], info, CLASSES).items()
                                                            if k != "score"}
        if not ng:
            gt["occluded"], gt["truncated"] = np.zeros(0, np.int64), np.zeros(0)
        if kind in (1, 2):
            gt = _add_dontcare(gt, [[100.0 + 50 * kind, 150.0, 180.0 + 50 * kind, 230.0]])
        info["annos"] = gt
        boxes, labels = [], []
        for j, n in enumerate(names):
            if rng.uniform() < 0.2 and not (kind in (3, 4) and j == 0):
                continue
            b = lidar[j].copy()
            if kind == 3 and j == 0:
                pass                                                        # identical to the ground truth
            elif kind == 4 and j == 0:
                b = EDGE_DT.copy()                                          # shares an edge with the ground truth
            else:
                b[:2] += rng.normal(0, 0.25, 2)
                b[3:6] *= rng.uniform(0.9, 1.1, 3)
                b[6] += rng.normal(0, 0.1)
            boxes.append(b)
            labels.append({"Car": 0, "Van": 0, "Pedestrian": 1, "Person_sitting": 1}.get(n, 2))
        if kind != 0:
            for _ in range(int(rng.integers(0, max_dets - len(boxes) + 1))):
                boxes.append(_lidar_box(rng, CLASSES[int(rng.integers(0, 3))]))
                labels.append(int(rng.integers(0, 3)))
        if kind == 5:                                                       # outside the image: behind the camera, far to the side
            boxes += [np.array([-10, 0, -1, 1.6, 3.9, 1.5, 0.3], np.float32), np.array([4, 30, -1, 1.6, 3.9, 1.5, 0.0], np.float32)]
            labels += [0, 0]
        n = len(boxes)
        scores = rng.uniform(0.05, 1.0, n).astype(np.float32)
        if kind == 6 and n > 2:
            scores[: n // 2] = np.float32(0.5)                              # tied scores
        det = {"box3d_lidar": np.stack(boxes).astype(np.float32) if n else np.zeros((0, 7), np.float32), "scores": scores,
               "label_preds": np.asarray(labels, np.int64), "metadata": {"image_idx": 1000 + f}}
        infos.append(info)
        dets[str(1000 + f)] = _clean(info, det, gt)
    return infos, dets


def dt_annos_of(infos, dets):
    out = []
    for info in infos:
        d = dets[str(info["image"]["image_idx"])]
        a = ref.convert_frame(d["box3d_lidar"], d["scores"], d["label_preds"], info, CLASSES)
        a["metadata"] = d["metadata"]
        out.append(a)
    return out


GT_KEYS = ("name", "truncated", "occluded", "alpha", "bbox", "dimensions", "location", "rotation_y")
CALIB_KEYS = ("R0_rect", "Tr_velo_to_cam", "P2")
DET_KEYS = ("box3d_lidar", "scores", "label_preds")


def golden_inputs(infos, dets):
    """npz entries holding a set's inputs: per frame the image index and shape, calibration, ground truth and lidar detections."""
    out = {}
    for f, info in enumerate(infos):
        out["image%d_idx" % f] = np.int64(info["image"]["image_idx"])
        out["image%d_shape" % f] = np.asarray(info["image"]["image_shape"])
        for k in CALIB_KEYS:
            out["calib%d_%s" % (f, k)] = np.asarray(info["calib"][k])
        for k in GT_KEYS:
            v = info["annos"][k]
            out["gt%d_%s" % (f, k)] = np.asarray(v).astype(str) if k == "name" else np.asarray(v)
        d = dets[str(info["image"]["image_idx"])]
        for k in DET_KEYS:
            out["det%d_%s" % (f, k)] = np.asarray(d[k])
    return out


def load_golden(path):
    """(npz, infos, detections, dt_annos) of the golden fixture, every input and output as stored."""
    g = np.load(path)
    infos, dets, dt_annos = [], {}, []
    for f in range(int(g["frames"])):
        idx = int(g["image%d_idx" % f])
        gt = {k: g["gt%d_%s" % (f, k)] for k in GT_KEYS}
        gt["bbox"], gt["location"], gt["dimensions"] = gt["bbox"].reshape(-1, 4), gt["location"].reshape(-1, 3), gt["dimensions"].reshape(-1, 3)
        infos.append({"image": {"image_idx": idx, "image_shape": g["image%d_shape" % f]},
                      "calib": {k: g["calib%d_%s" % (f, k)] for k in CALIB_KEYS}, "annos": gt})
        dets[str(idx)] = dict({k: g["det%d_%s" % (f, k)] for k in DET_KEYS}, metadata={"image_idx": idx})
        a = {k: g["dt%d_%s" % (f, k)] for k in ("bbox", "alpha", "location", "dimensions", "rotation_y", "score", "name")}
        a["bbox"], a["location"], a["dimensions"] = a["bbox"].reshape(-1, 4), a["location"].reshape(-1, 3), a["dimensions"].reshape(-1, 3)
        dt_annos.append(a)
    return g, infos, dets, dt_annos
