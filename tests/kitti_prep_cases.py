"""A seeded, crafted KITTI tree for the data-preparation tests: ImageSets, training/ and testing/ with calib, label_2, velodyne and
minimal valid image_2 PNGs.  `write_tree(root)` writes it and returns the split ids.

The cases: the four KITTI image sizes with distinct calibrations (non-zero P2 translation, non-identity R0_rect); points behind the
sensor, beyond the far clip and past each image edge; DontCare lines between objects; a label file with scores and an empty one;
difficulty boundaries (bbox height exactly 40 and 25, each occlusion and truncation threshold); overlapping boxes that share points; a box
that straddles the frustum and one wholly behind the sensor (0 points); test frames without labels; several classes.  Every point is at
least MARGIN from every frustum and box plane (both the label boxes and the h/2-lower boxes _calculate_num_points_in_gt counts in).
"""
import os
import struct
import zlib

import numpy as np

from oracle import kitti_prep_ref as ref

MARGIN = 1e-4
SIZES = [(375, 1242), (370, 1224), (374, 1238), (376, 1241)]
SPLITS = {"train": [0, 1, 2, 4, 6], "val": [3, 5], "test": [0, 1]}
USED_CLASSES = ["Car", "Pedestrian", "Cyclist"]


def png(h, w):
    """a minimal valid 1x1-pixel-row-per-line grayscale PNG of the given size"""
    def chunk(t, d):
        return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d) & 0xFFFFFFFF)
    raw = b"".join(b"\x00" + b"\x00" * w for _ in range(h))
    return (b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 0, 0, 0, 0)) + chunk(b"IDAT", zlib.compress(raw))
            + chunk(b"IEND", b""))


def calib(rs, k):
    f = 721.5377 + 3.1 * k
    p2 = np.array([[f, 0, 609.5593 + k, 44.85728 + k], [0, f, 172.854 - k, 0.2163791], [0, 0, 1, 0.002745884]])
    a = 0.01 * (k + 1)
    r0 = np.array([[np.cos(a), -np.sin(a), 0.0], [np.sin(a), np.cos(a), 0.0], [0.0, 0.0, 1.0]]) @ \
        np.array([[1.0, 0.0, 0.0], [0.0, np.cos(a / 2), -np.sin(a / 2)], [0.0, np.sin(a / 2), np.cos(a / 2)]])
    tr = np.array([[7.533745e-03, -9.999714e-01, -6.166020e-04, -4.069766e-03], [1.480249e-02, 7.280733e-04, -9.998902e-01, -7.631618e-02],
                   [9.998621e-01, 7.523790e-03, 1.480755e-02, -2.717806e-01]])
    tr[:, 3] += rs.uniform(-0.05, 0.05, 3)
    p0 = p2.copy(); p0[:, 3] = 0
    p1 = p2.copy(); p1[0, 3] = -387.5744
    p3 = p2.copy(); p3[0, 3] = -337.2877
    imu = np.array([[9.999976e-01, 7.553071e-04, -2.035826e-03, -8.086759e-01], [-7.854027e-04, 9.998898e-01, -1.482298e-02, 3.195559e-01],
                    [2.024406e-03, 1.482454e-02, 9.998881e-01, -7.997231e-01]])

    def line(n, m):
        return n + ": " + " ".join("%.12e" % v for v in np.ravel(m))
    text = "\n".join([line("P0", p0), line("P1", p1), line("P2", p2), line("P3", p3), line("R0_rect", r0), line("Tr_velo_to_cam", tr),
                      line("Tr_imu_to_velo", imu)]) + "\n"
    return text, {"P2": np.vstack([p2, [0, 0, 0, 1]]), "R0_rect": np.pad(r0, ((0, 1), (0, 1))) + np.diag([0, 0, 0, 1.0]),
                  "Tr_velo_to_cam": np.vstack([tr, [0, 0, 0, 1]])}


# (name, truncated, occluded, alpha, bbox, h w l, x y z (camera), ry): the crafted label lines per training frame
def objects(k):
    car = lambda x, z, ry=0.3, top=150.0, h=40.0, o=0, t=0.0, name="Car": (name, t, o, -1.2, (500.0, top, 600.0, top + h),
                                                                            (1.52, 1.63, 3.9), (x, 1.7, z), ry)
    dc = ("DontCare", -1, -1, -10, (700.0, 160.0, 720.0, 180.0), (-1, -1, -1), (-1000, -1000, -1000), -10)
    if k == 0:   # difficulty boundaries, DontCare between objects, overlapping boxes
        return [car(-2.0, 12.0, h=40.0), dc, car(-1.0, 13.0, ry=0.9, h=40.01), car(3.0, 20.0, h=25.0, o=1, t=0.3), dc,
                car(5.0, 30.0, h=25.01, o=2, t=0.5), car(-6.0, 18.0, o=3, t=0.15), car(1.0, 40.0, t=0.16, name="Van"),
                ("Pedestrian", 0.0, 0, 0.1, (300.0, 140.0, 330.0, 220.0), (1.75, 0.6, 0.8), (-4.0, 1.6, 9.0), 1.1)]
    if k == 1:   # straddles the frustum's right edge; wholly behind the sensor
        return [car(9.0, 10.0, ry=-0.4), car(0.0, -10.0), ("Cyclist", 0.2, 1, 0.3, (800.0, 150.0, 850.0, 210.0), (1.7, 0.6, 1.8),
                                                           (2.5, 1.6, 14.0), -1.3)]
    if k == 2:   # empty label file
        return []
    return [car(-3.0 + k, 15.0 + k, ry=0.2 * k), dc, car(2.0, 25.0 + k, ry=-0.5, name="Pedestrian" if k % 2 else "Car")]


def label_text(objs, scores=False):
    lines = []
    for i, (n, t, o, al, bb, hwl, xyz, ry) in enumerate(objs):
        v = [n, "%.2f" % t, "%d" % o, "%.2f" % al] + ["%.2f" % x for x in bb] + ["%.2f" % x for x in hwl] + ["%.2f" % x for x in xyz] + \
            ["%.2f" % ry]
        if scores:
            v.append("%.4f" % (0.5 + 0.01 * i))
        lines.append(" ".join(v))
    return "".join(l + "\n" for l in lines)


def _anno(text, keep_dontcare=True):
    """the geometry of a label text as the parser reads it"""
    rows = [l.split(" ") for l in text.splitlines() if keep_dontcare or not l.startswith("DontCare")]
    f = lambda a, b: np.array([[float(v) for v in r[a:b]] for r in rows], np.float64).reshape(len(rows), b - a)
    return {"name": np.array([r[0] for r in rows]), "location": f(11, 14), "dimensions": f(8, 11)[:, [2, 0, 1]],
            "rotation_y": f(14, 15).reshape(-1), "difficulty": np.zeros(len(rows), np.int32)}


def _clear(points, pl):
    """points at least MARGIN from every plane of pl [K, 6, 4]"""
    if len(pl) == 0 or len(points) == 0:
        return points
    p = points[:, :3].astype(np.float64)
    s = np.einsum("nc,kfc->nkf", p, pl[..., :3]) + pl[None, :, :, 3]
    d = np.abs(s) / np.linalg.norm(pl[..., :3], axis=-1)[None]
    return points[(d >= MARGIN).all(axis=(1, 2))]


def cloud(rs, n, boxes):
    az = rs.uniform(-np.pi, np.pi, n)
    r = rs.uniform(2.0, 110.0, n)                                   # past the 100 m far clip too
    pts = np.stack([r * np.cos(az), r * np.sin(az), rs.uniform(-2.5, 1.5, n), rs.uniform(0, 1, n)], 1)
    extra = [pts]
    for b in boxes:                                                  # dense points inside every box
        m = 60
        loc = rs.uniform(-0.5, 0.5, (m, 3)) * b[3:6]
        c, s = np.cos(b[6]), np.sin(b[6])
        extra.append(np.stack([loc[:, 0] * c - loc[:, 1] * s + b[0], loc[:, 0] * s + loc[:, 1] * c + b[1], loc[:, 2] + b[2],
                               rs.uniform(0, 1, m)], 1))
    return np.concatenate(extra).astype(np.float32)


def write_tree(root, seed=2026, points=3000):
    rs = np.random.RandomState(seed)
    os.makedirs(os.path.join(root, "ImageSets"), exist_ok=True)
    for s, ids in SPLITS.items():
        with open(os.path.join(root, "ImageSets", s + ".txt"), "w") as f:
            f.write("".join("%06d\n" % i for i in ids))
    n_train = max(SPLITS["train"] + SPLITS["val"]) + 1
    for part, count in (("training", n_train), ("testing", max(SPLITS["test"]) + 1)):
        for d in ("calib", "label_2", "velodyne", "image_2"):
            os.makedirs(os.path.join(root, part, d), exist_ok=True)
        for k in range(count):
            h, w = SIZES[(k + (part == "testing")) % 4]
            with open(os.path.join(root, part, "image_2", "%06d.png" % k), "wb") as f:
                f.write(png(h, w))
            text, cal = calib(rs, k + 10 * (part == "testing"))
            with open(os.path.join(root, part, "calib", "%06d.txt" % k), "w") as f:
                f.write(text)
            objs = objects(k) if part == "training" else []
            text = label_text(objs, scores=(k == 4))
            if part == "training":
                with open(os.path.join(root, part, "label_2", "%06d.txt" % k), "w") as f:
                    f.write(text)
            info = {"annos": _anno(text), "calib": cal}
            boxes = ref.db_boxes(info)[0] if objs else np.zeros((0, 7))
            pts = cloud(rs, points, boxes)
            pl = [ref.frustum_planes(cal["R0_rect"], cal["Tr_velo_to_cam"], cal["P2"], (h, w))[None], ref.box_planes(boxes)]
            if objs:
                pl.append(ref.box_planes(ref.count_boxes(info)))
            for q in pl:
                pts = _clear(pts, q)
            pts.tofile(os.path.join(root, part, "velodyne", "%06d.bin" % k))
    return SPLITS
