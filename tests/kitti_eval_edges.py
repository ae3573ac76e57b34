"""Crafted KITTI evaluation frames that sit on the evaluation's decision edges, built directly as annotation dicts.

Each frame holds one decision and is named after it: an overlap exactly at a min overlap, a difficulty cut-off, a matching
precedence rule, a DontCare rule, a threshold rule or an AOS delta.  Every bbox, location, dimension, alpha and score is an exact
value chosen here.  Boxes that take part in a BEV / 3D decision have ry = 0 and dyadic sizes, so every fp32 corner, clip vertex
and triangle area is exact and the only rounding left is the reference's own: the fp64 quotient stored as fp32.
tests/golden/make_kitti_eval_golden.py asserts each crafted condition on the reference's own intermediate values, and that the
simulated BEV / 3D overlaps equal the oracle's bit for bit.

`CHECKS[name]` lists the decision of a frame: (metric, class code, difficulty, min overlap, [(tp, fp) per threshold]) as the
frame gives it when it is evaluated alone.  Competing detections carry different alphas, so the AOS shows which one matched.
Objects that take no part in a BEV / 3D decision get 1 m cubes of their own, far apart, so they overlap nothing there.
"""
import numpy as np

from oracle import kitti_eval_ref as ref

CLASSES = ["Car", "Pedestrian", "Cyclist"]
CODES = [0, 1, 10]
CAR, PED, CYC = 0, 1, 10
COCO_CAR = np.linspace(0.5, 0.95, 10)
COCO_PED = np.linspace(0.25, 0.7, 10)
NEXT = np.nextafter
F32_ABOVE_HALF = float(np.nextafter(np.float32(0.5), np.float32(1)))
# first fp32 above 0.5 as a stored BEV / 3D overlap: the GT 0.5 x 5 and the detection 0.5 x 4 shifted along x by X_SHIFT overlap
# in 0.375000030 x 4 = 1.500000119 of a union 3.0 (a small search over dyadic sizes; the clip's crossings at x = 0.25 are exact)
X_SHIFT = 4194303 / 33554432


class _Frame:
    def __init__(self):
        self.gt, self.dt, self.k = [], [], 0

    def _far(self):
        self.k += 1
        return (0.0, 1.0, 100.0 + 8.0 * self.k), (1.0, 1.0, 1.0)

    def g(self, name, bbox, loc=None, dims=None, alpha=0.0, trunc=0.0, occ=0):
        if loc is None:
            loc, dims = self._far()
        if name == "DontCare":
            loc, dims, alpha, trunc, occ = (-1000.0, -1000.0, -1000.0), (-1.0, -1.0, -1.0), -10.0, -1.0, -1
        self.gt.append(dict(name=name, bbox=bbox, location=loc, dimensions=dims, rotation_y=-10.0 if name == "DontCare" else 0.0,
                            alpha=alpha, truncated=trunc, occluded=occ))
        return self

    def d(self, name, bbox, score, loc=None, dims=None, alpha=0.0):
        if loc is None:
            loc, dims = self._far()
        self.dt.append(dict(name=name, bbox=bbox, location=loc, dimensions=dims, rotation_y=0.0, alpha=alpha, score=score))
        return self

    def clear(self, name="Car", score=0.3, x=1000.0):
        """A GT and an identical detection that match in 2D only: it gives the frame a threshold below the decision's score."""
        return self.g(name, [x, 0.0, x + 100.0, 100.0]).d(name, [x, 0.0, x + 100.0, 100.0], score)

    def annos(self):
        gt = {"name": np.array([o["name"] for o in self.gt]),
              "truncated": np.array([o["truncated"] for o in self.gt], np.float64),
              "occluded": np.array([o["occluded"] for o in self.gt], np.int64)}
        dt = {"name": np.array([o["name"] for o in self.dt]), "score": np.array([o["score"] for o in self.dt], np.float32)}
        for a, objs in ((gt, self.gt), (dt, self.dt)):
            a["alpha"] = np.array([o["alpha"] for o in objs], np.float64)
            a["bbox"] = np.array([o["bbox"] for o in objs], np.float64).reshape(-1, 4)
            a["dimensions"] = np.array([o["dimensions"] for o in objs], np.float64).reshape(-1, 3)
            a["location"] = np.array([o["location"] for o in objs], np.float64).reshape(-1, 3)
            a["rotation_y"] = np.array([o["rotation_y"] for o in objs], np.float64)
        return gt, dt


def _bev_pair(f, gt_ld, dt_ld, score, name="Car", dt_x=0.0, dt_y=1.0, h=2.0, gt_bbox=(0.0, 0.0, 100.0, 100.0)):
    """A GT (l, w) and a detection (l, w) centred at camera (0, 20) / (dt_x, 20); their 2D boxes do not overlap."""
    f.g(name, list(gt_bbox), (0.0, 1.0, 20.0), (gt_ld[0], h, gt_ld[1]))
    return f.d(name, [500.0, 0.0, 600.0, 100.0], score, (dt_x, dt_y, 20.0), (dt_ld[0], h, dt_ld[1]))


def _bev_clear(f, score=0.3, name="Car"):
    """A GT and an identical detection that match in BEV / 3D only (4 x 2 x 2 at camera z = 40)."""
    f.g(name, [2000.0, 0.0, 2100.0, 100.0], (0.0, 1.0, 40.0), (4.0, 2.0, 2.0))
    return f.d(name, [2500.0, 0.0, 2600.0, 100.0], score, (0.0, 1.0, 40.0), (4.0, 2.0, 2.0))


def _2d_iou(name, y1):
    """GT [100, 0, 200, 100] and a detection [100, 0, 200, y1] at score 0.9 (2D IoU y1 / 100), plus a clear pair at 0.3."""
    return _Frame().g(name, [100.0, 0.0, 200.0, 100.0]).d(name, [100.0, 0.0, 200.0, y1], 0.9, alpha=0.5).clear(name)


def build():
    """(names, gt_annos, dt_annos, checks, conditions).  conditions[name]: the crafted values the generator asserts on the
    reference's intermediates: ("ov", metric, dt, gt, value) an overlap, ("ov_lt", metric, dt, gt, value) an overlap below a value
    (fp32 storage), ("dc", dt, dc, value) a detection-over-DontCare overlap, ("h_gt", gt, value) / ("h_dt", dt, value) a box
    height, ("n_thr", value) the number of thresholds of the frame's check."""
    frames, checks, cond = {}, {}, {}

    def add(name, f, chk, c=()):
        frames[name], checks[name], cond[name] = f, chk, list(c)

    # ---- 2D overlap exactly at the min overlap (fp64), and just above it
    above = 70.0 + 2.0 ** -7
    add("2d_iou_eq_0.7_car_no_match", _2d_iou("Car", 70.0), [(0, CAR, 0, 0.7, [(1, 1)])], [("ov", 0, 0, 0, 0.7)])
    add("2d_iou_above_0.7_car_match", _2d_iou("Car", above), [(0, CAR, 0, 0.7, [(1, 0), (2, 0)])])
    add("2d_iou_eq_0.5_ped_no_match", _2d_iou("Pedestrian", 50.0), [(0, PED, 0, 0.5, [(1, 1)])], [("ov", 0, 0, 0, 0.5)])
    add("2d_iou_above_0.5_ped_match", _2d_iou("Pedestrian", 50.0 + 2.0 ** -7), [(0, PED, 0, 0.5, [(1, 0), (2, 0)])])
    # ---- COCO grid: np.linspace puts 0.9, 0.45 and 0.65 one ulp below their decimals, so these exact IoUs match
    add("2d_iou_0.9_car_coco_match", _2d_iou("Car", 90.0), [(0, CAR, 0, COCO_CAR[8], [(1, 0), (2, 0)])], [("ov", 0, 0, 0, 0.9)])
    add("2d_iou_0.65_ped_coco_match", _2d_iou("Pedestrian", 65.0), [(0, PED, 0, COCO_PED[8], [(1, 0), (2, 0)])],
        [("ov", 0, 0, 0, 0.65)])
    # the car grid holds 0.65 itself: a tie there, not a match
    add("2d_iou_eq_0.65_car_coco_no_match", _2d_iou("Car", 65.0), [(0, CAR, 0, COCO_CAR[3], [(1, 1)])], [("ov", 0, 0, 0, 0.65)])
    add("2d_iou_0.45_ped_coco_match", _2d_iou("Pedestrian", 45.0), [(0, PED, 0, COCO_PED[4], [(1, 0), (2, 0)])],
        [("ov", 0, 0, 0, 0.45)])
    # ---- BEV / 3D overlaps exactly at the min overlap, stored as fp32
    f = _bev_clear(_bev_pair(_Frame(), (3.0, 6.0), (2.25, 4.0), 0.9))
    add("bev_3d_eq_0.5_no_match", f, [(1, CAR, 0, 0.5, [(1, 1)]), (2, CAR, 0, 0.5, [(1, 1)])],
        [("ov", 1, 0, 0, 0.5), ("ov", 2, 0, 0, 0.5)])
    f = _bev_clear(_bev_pair(_Frame(), (2.0, 5.0), (1.75, 4.0), 0.9))
    add("bev_3d_fp32_0.7_no_match", f, [(1, CAR, 1, 0.7, [(1, 1)]), (2, CAR, 1, 0.7, [(1, 1)])],
        [("ov", 1, 0, 0, float(np.float32(0.7))), ("ov_lt", 1, 0, 0, 0.7), ("ov", 2, 0, 0, float(np.float32(0.7)))])
    f = _bev_clear(_bev_pair(_Frame(), (0.5, 5.0), (0.5, 4.0), 0.9, dt_x=X_SHIFT))
    add("bev_3d_first_fp32_above_0.5_match", f, [(1, CAR, 0, 0.5, [(1, 0), (2, 0)]), (2, CAR, 0, 0.5, [(1, 0), (2, 0)])],
        [("ov", 1, 0, 0, F32_ABOVE_HALF), ("ov", 2, 0, 0, F32_ABOVE_HALF)])
    # 13 / 20 = 0.65 stored as fp32 0.6499999762 misses the pedestrian COCO 0.6499999999999999 that the fp64 value would pass
    f = _bev_clear(_bev_pair(_Frame(), (4.0, 5.0), (3.25, 4.0), 0.9, name="Pedestrian"), name="Pedestrian")
    add("bev_fp32_0.65_ped_coco_no_match", f, [(1, PED, 0, COCO_PED[8], [(1, 1)]), (2, PED, 0, COCO_PED[8], [(1, 1)])],
        [("ov", 1, 0, 0, float(np.float32(0.65))), ("ov_lt", 1, 0, 0, COCO_PED[8])])
    # identical BEV boxes that touch in height: BEV IoU 1, 3D overlap 0 (iw == 0)
    f = _bev_clear(_bev_pair(_Frame(), (2.0, 4.0), (2.0, 4.0), 0.9, dt_y=-1.0))
    add("3d_touching_in_height", f, [(1, CAR, 0, 0.7, [(1, 0), (2, 0)]), (2, CAR, 0, 0.7, [(1, 1)])],
        [("ov", 1, 0, 0, 1.0), ("ov", 2, 0, 0, 0.0)])

    # ---- difficulty cut-offs: a Car GT and an identical detection (TP when the GT is valid, absorbed when it is ignored)
    def cut(name, bbox, check, c, **kw):
        f = _Frame().g("Car", bbox, **kw).d("Car", list(bbox), 0.9, alpha=0.5).clear()
        add(name, f, check, c)

    cut("gt_h_eq_40_ignored_easy", [0.0, 0.0, 100.0, 40.0], [(0, CAR, 0, 0.7, [(1, 0)]), (0, CAR, 1, 0.7, [(1, 0), (2, 0)])],
        [("h_gt", 0, 40.0)])
    cut("gt_h_above_40_valid_easy", [0.0, 0.0, 100.0, NEXT(40.0, 41.0)], [(0, CAR, 0, 0.7, [(1, 0), (2, 0)])],
        [("h_gt", 0, NEXT(40.0, 41.0))])
    cut("gt_h_eq_25_ignored_moderate", [0.0, 0.0, 100.0, 25.0], [(0, CAR, 1, 0.7, [(1, 0)]), (0, CAR, 2, 0.7, [(1, 0)])],
        [("h_gt", 0, 25.0)])
    cut("gt_h_above_25_valid_moderate", [0.0, 0.0, 100.0, NEXT(25.0, 26.0)], [(0, CAR, 1, 0.7, [(1, 0), (2, 0)])],
        [("h_gt", 0, NEXT(25.0, 26.0))])
    for t, diff in ((0.15, 0), (0.3, 1), (0.5, 2)):
        cut("trunc_eq_%g_valid_diff%d" % (t, diff), [0.0, 0.0, 100.0, 100.0], [(0, CAR, diff, 0.7, [(1, 0), (2, 0)])], (),
            trunc=t)
        cut("trunc_above_%g_ignored_diff%d" % (t, diff), [0.0, 0.0, 100.0, 100.0], [(0, CAR, diff, 0.7, [(1, 0)])], (),
            trunc=NEXT(t, 1.0))
    for occ in range(4):
        cut("occluded_%d" % occ, [0.0, 0.0, 100.0, 100.0],
            [(0, CAR, d, 0.7, [(1, 0), (2, 0)] if occ <= d else [(1, 0)]) for d in range(3)], (), occ=occ)

    # detection height: the pair matches in BEV (identical 3D boxes); its 2D box height decides whether it is short
    def det_h(name, h, short_diffs, c):
        f = _Frame()
        f.g("Car", [0.0, 0.0, 100.0, 100.0], (0.0, 1.0, 20.0), (4.0, 2.0, 2.0))
        f.d("Car", [500.0, 0.0, 600.0, h], 0.9, (0.0, 1.0, 20.0), (4.0, 2.0, 2.0))
        _bev_clear(f)
        add(name, f, [(1, CAR, d, 0.7, [(1, 0)] if d in short_diffs else [(1, 0), (2, 0)]) for d in range(3)], c)

    det_h("dt_h_eq_40_not_short", 40.0, (), [("h_dt", 0, 40.0)])
    det_h("dt_h_below_40_short_easy", NEXT(40.0, 0.0), (0,), [("h_dt", 0, NEXT(40.0, 0.0))])
    det_h("dt_h_eq_25_not_short", 25.0, (0,), [("h_dt", 0, 25.0)])
    det_h("dt_h_below_25_short", NEXT(25.0, 0.0), (0, 1, 2), [("h_dt", 0, NEXT(25.0, 0.0))])

    # ---- match precedence
    # in BEV / 3D: a short detection (2D height 20) with the higher overlap (1.0, score 0.9), then a normal one above the min
    # overlap (7 / 8, score 0.5).  Pass 1 takes the higher score, the short one, so this GT gives no threshold; pass 2 at the clear
    # pair's 0.3 lets the normal one displace it.
    f = _Frame().g("Car", [0.0, 0.0, 100.0, 100.0], (0.0, 1.0, 20.0), (4.0, 2.0, 2.0))
    f.d("Car", [500.0, 0.0, 600.0, 20.0], 0.9, (0.0, 1.0, 20.0), (4.0, 2.0, 2.0), alpha=1.0)
    f.d("Car", [700.0, 0.0, 800.0, 100.0], 0.5, (0.0, 1.0, 20.0), (4.0, 2.0, 1.75))
    _bev_clear(f)
    add("short_then_normal_normal_wins_pass2", f, [(1, CAR, 0, 0.7, [(2, 0)]), (2, CAR, 2, 0.7, [(2, 0)])],
        [("ov", 1, 0, 0, 1.0), ("ov", 1, 1, 0, 0.875), ("h_dt", 0, 20.0)])

    # bit-identical overlaps: detections j = 5 and 37 (one lane, two mask words) and j = 5 and 6 (two lanes), equal scores
    for name, pair in (("tie_same_lane_j5_j37", (5, 37)), ("tie_two_lanes_j5_j6", (5, 6))):
        f = _Frame().g("Car", [0.0, 0.0, 100.0, 100.0], alpha=0.0)
        for j in range(max(pair) + 2):
            if j in pair:
                f.d("Car", [0.0, 0.0, 100.0, 90.0], 0.6, alpha=0.0 if j == pair[0] else 1.5)
            else:
                f.d("Cyclist", [200.0 + 110 * j, 0.0, 300.0 + 110 * j, 100.0], 0.5)
        f.clear(score=0.3, x=6000.0)
        add(name, f, [(0, CAR, 0, 0.7, [(1, 1), (2, 1)])])
    # equal scores in pass 1: GT 1 overlaps detections a and b equally; GT 2 overlaps only b.  The first (a) must go to GT 1.
    f = _Frame().g("Pedestrian", [0.0, 0.0, 100.0, 100.0]).g("Pedestrian", [0.0, 40.0, 100.0, 140.0])
    f.d("Pedestrian", [0.0, 0.0, 100.0, 60.0], 0.6, alpha=0.0).d("Pedestrian", [0.0, 40.0, 100.0, 100.0], 0.6, alpha=1.0)
    add("tie_equal_scores_pass1_first_wins", f, [(0, PED, 0, 0.5, [(2, 0), (2, 0)])], [("ov", 0, 0, 0, 0.6), ("ov", 0, 1, 0, 0.6)])
    # neighbour classes: a Van GT under Car and a Person_sitting GT under Pedestrian absorb their detection; a Van detection
    # under Car is neither TP nor FP
    f = _Frame().g("Van", [0.0, 0.0, 100.0, 100.0]).d("Car", [0.0, 0.0, 100.0, 100.0], 0.9).clear()
    add("van_gt_absorbs_car", f, [(0, CAR, 0, 0.7, [(1, 0)])])
    f = _Frame().g("Person_sitting", [0.0, 0.0, 100.0, 100.0]).d("Pedestrian", [0.0, 0.0, 100.0, 100.0], 0.9).clear("Pedestrian")
    add("person_sitting_gt_absorbs_ped", f, [(0, PED, 0, 0.5, [(1, 0)])])
    f = _Frame().g("Car", [0.0, 0.0, 100.0, 100.0]).d("Van", [0.0, 0.0, 100.0, 100.0], 0.9).clear()
    add("van_det_under_car_neither", f, [(0, CAR, 0, 0.7, [(1, 0)])])

    # ---- DontCare (2D only): criterion-0 overlap of the detection over the region
    def dc(name, regions, check, c=(), extra=None):
        f = _Frame().clear().d("Car", [600.0, 0.0, 700.0, 100.0], 0.9)
        for r in regions:
            f.g("DontCare", r)
        if extra:
            extra(f)
        add(name, f, check, c)

    # with a pair that matches in BEV / 3D only: there the detection over DontCare stays an FP, since DontCare is a 2D rule
    dc("dontcare_eq_0.7_not_absorbed", [[600.0, 0.0, 700.0, 70.0]],
       [(0, CAR, 0, 0.7, [(1, 2)]), (1, CAR, 0, 0.7, [(1, 2)]), (2, CAR, 0, 0.7, [(1, 2)])], [("dc", 1, 0, 0.7)], _bev_clear)
    dc("dontcare_above_0.7_absorbed", [[600.0, 0.0, 700.0, above]],
       [(0, CAR, 0, 0.7, [(1, 1)]), (1, CAR, 0, 0.7, [(1, 2)]), (2, CAR, 0, 0.7, [(1, 2)])], [], _bev_clear)
    dc("dontcare_two_regions_absorb_once", [[600.0, 0.0, 700.0, 100.0], [590.0, 0.0, 710.0, 100.0]],
       [(0, CAR, 0, 0.7, [(1, 0)])])
    # the TP (score 0.8) and a detection below the threshold (0.2) both lie in a DontCare region: neither is absorbed
    f = _Frame().g("Car", [0.0, 0.0, 100.0, 100.0]).d("Car", [0.0, 0.0, 100.0, 100.0], 0.8)
    f.d("Car", [300.0, 0.0, 400.0, 100.0], 0.2).g("DontCare", [0.0, 0.0, 400.0, 100.0])
    add("dontcare_skips_assigned_and_below_threshold", f, [(0, CAR, 0, 0.7, [(1, 0)])])

    # ---- NaN precision: GTs Van then Car; A (0.9) overlaps only the Van and lies over DontCare; X (0.5) overlaps both and the
    # Van more than A.  Pass 1: Van takes A, Car takes X (threshold 0.5).  Pass 2 at 0.5: Van takes X, Car is missed, DontCare
    # absorbs A: tp + fp == 0.
    f = _Frame().g("Van", [0.0, 100.0, 100.0, 200.0], alpha=0.0).g("Car", [0.0, 110.0, 100.0, 210.0], alpha=0.0)
    f.d("Car", [0.0, 90.0, 100.0, 190.0], 0.9, alpha=1.0).d("Car", [0.0, 105.0, 100.0, 205.0], 0.5, alpha=2.0)
    f.g("DontCare", [0.0, 90.0, 100.0, 190.0])
    add("nan_precision_tp_fp_zero", f, [(0, CAR, 0, 0.7, [(0, 0)])], [("ov", 0, 1, 0, 19 / 21), ("ov", 0, 0, 0, 9 / 11)])

    # ---- thresholds
    # tied scores exactly at the threshold: three TPs and an FP at 0.5 are all kept (the test is `<`)
    f = _Frame()
    for i in range(3):
        f.g("Car", [120.0 * i, 0.0, 120.0 * i + 100, 100.0]).d("Car", [120.0 * i, 0.0, 120.0 * i + 100, 100.0], 0.5)
    f.d("Car", [600.0, 0.0, 700.0, 100.0], 0.5).clear(score=0.25)
    add("tied_scores_at_threshold", f, [(0, CAR, 0, 0.7, [(3, 1), (3, 1), (3, 1), (4, 1)])])
    # more than 41 TPs: 50 pairs with distinct scores, so get_thresholds skips and caps at 41
    f = _Frame()
    scores = [(100 - i) / 128.0 for i in range(50)]
    for i in range(50):
        x = 110.0 * i
        f.g("Car", [x, 0.0, x + 100, 100.0]).d("Car", [x, 0.0, x + 100, 100.0], scores[i], alpha=0.25 * (i % 7))
    thr = ref.thresholds(scores, 50)
    add("fifty_tps", f, [(0, CAR, 0, 0.7, [(sum(s >= t for s in scores), 0) for t in thr])], [("n_thr", 41)])
    # a class with detections and no valid GT (Cyclist): no thresholds
    f = _Frame().d("Cyclist", [0.0, 0.0, 100.0, 100.0], 0.7).g("Car", [0.0, 0.0, 100.0, 100.0])
    add("no_valid_gt_with_detections", f, [(0, CYC, 0, 0.5, [])])

    # ---- AOS deltas 0, pi, -pi, 2 pi
    f = _Frame()
    for i, da in enumerate((0.0, np.pi, -np.pi, 2 * np.pi)):
        x = 110.0 * i
        f.g("Car", [x, 0.0, x + 100, 100.0], alpha=0.0).d("Car", [x, 0.0, x + 100, 100.0], 0.9 - 0.1 * i, alpha=-da)
    add("aos_deltas", f, [(0, CAR, 0, 0.7, [(1, 0), (2, 0), (3, 0), (4, 0)])])

    names = list(frames)
    gts, dts = zip(*(frames[n].annos() for n in names))
    return names, list(gts), list(dts), checks, cond


def min_overlaps_ref():
    """[12, 3, 3] min overlaps as the reference forms them for CLASSES: the official moderate and easy sets, then the COCO grid."""
    mod = np.array([[0.7, 0.5, 0.5, 0.7, 0.7, 0.7, 0.7, 0.5, 0.5, 0.5, 0.5]] * 3)
    easy = np.array([[0.7, 0.5, 0.5, 0.7, 0.7, 0.7, 0.7, 0.5, 0.25, 0.25, 0.5],
                     [0.5, 0.25, 0.25, 0.5, 0.5, 0.5, 0.5, 0.25, 0.25, 0.25, 0.25],
                     [0.5, 0.25, 0.25, 0.5, 0.5, 0.5, 0.5, 0.25, 0.25, 0.25, 0.25]])
    off = np.stack([mod, easy], 0)[:, :, CODES]
    rng = {0: [0.5, 0.95, 10], 1: [0.25, 0.7, 10], 10: [0.25, 0.7, 10]}
    coco = np.zeros([10, 3, len(CODES)])
    for j, c in enumerate(CODES):
        for i in range(3):
            start, stop, num = rng[c]
            coco[:, i, j] = np.linspace(start, stop, int(num))
    return np.concatenate([off, coco], 0)


GT_KEYS = ("name", "truncated", "occluded", "alpha", "bbox", "dimensions", "location", "rotation_y")
DT_KEYS = ("name", "score", "alpha", "bbox", "dimensions", "location", "rotation_y")


def load_edges(path):
    """(npz, frame names, gt_annos, dt_annos) of kitti_eval_edges.npz."""
    g = np.load(path)
    names = [str(n) for n in g["names"]]
    gts = [{k: g["gt%d_%s" % (f, k)] for k in GT_KEYS} for f in range(len(names))]
    dts = [{k: g["dt%d_%s" % (f, k)] for k in DT_KEYS} for f in range(len(names))]
    return g, names, gts, dts


def golden_checks(g, names):
    """[(frame index, frame name, key prefix)] of the per-frame checks stored in the golden."""
    out = []
    for f, name in enumerate(names):
        q = 0
        while "c%d_%d_config" % (f, q) in g:
            out.append((f, name, "c%d_%d" % (f, q)))
            q += 1
    return out


def aos_bound(n_tp):
    """Largest difference between two AOS curve points computed with different fp64 cos implementations.

    Each similarity term is (1 + cos(delta)) / 2 with cos within 2 ulp of the exact value on the device (CUDA's fp64 cos) and
    within 1 ulp in numpy: the cos values differ by at most 3 ulp <= 3 * 2^-52, the term by at most 2^-50 after `1 +` and the
    halving round.  Both sides add the terms in the same order (ground truth within a frame, then frames), so over n TPs the
    sum differs by at most n * 2^-50 from the terms plus n * 2^-52 per partial-sum rounding, n^2 * 2^-52 in all.  A curve point
    divides the sum by tp + fp >= n and rounds once more, and the suffix max keeps the bound:
    |d aos| <= 2^-50 + n * 2^-52 + 2^-53 <= (4 + n) * 2^-52."""
    return (4 + n_tp) * 2.0 ** -52


def map_aos_bound(n_tp):
    """The R11 / R40 AOS average: at most 40 points of aos_bound each, 40 additions in [0, 40] (2^-47 each), then / 40 * 100."""
    return 100 * (aos_bound(n_tp) + 40 * 2.0 ** -47)


# ------------------------------------------------------------------------------------------------ capacity frames
CAPACITY_COUNTS = (0, 1, 31, 32, 33, 127, 128, 129, 255, 256, 991, 992, 993, 1023, 1024)
GT_BOX = np.array([20.0, 0.0, -1.0, 1.6, 3.9, 1.5, 0.0], np.float32)


def capacity_set(seed=3):
    """(infos, dets, kind): one frame per CAPACITY_COUNTS entry, a frame with 1024 detections and no ground truth, one with 300
    ground-truth boxes (Car, Pedestrian, Van) and 4 DontCare regions, and two frames whose conversion drops detections.

    kind[f] is "count" for the counted frames: every detection lies in front of the camera and inside the image, so the frame
    keeps exactly its capacity, and the evaluation sees each listed count.  Each holds one valid Car GT (GT_BOX, not occluded or
    truncated) and the GT box itself as its last detection, at j = n - 1 (mask word 31, lane 31 at 1024), with the frame's
    unique highest score.  The fillers lie left of the GT in the image and overlap it by less than 0.1; their rotations include fp32 pi,
    -pi, 3 pi and -3 pi, the limit_period boundary.  kind "drop": 40 and 1024 input detections of which one in 8 lies outside
    the image and is dropped (the kept count is below the capacity) and one in 8 lies behind the camera, where it still
    projects into the image and is kept; the matching detection is again last."""
    from kitti_eval_cases import _add_dontcare, _gt_annos, exact_calib
    rng = np.random.default_rng(seed)
    infos, dets, kind = [], {}, []
    edge_ry = np.array([np.pi, -np.pi, 3 * np.pi, -3 * np.pi], np.float32)

    def frame(idx, gt_lidar, gt_names, n_det, what, dontcare=(), drop=False):
        info = {"image": {"image_idx": idx, "image_shape": np.array([375, 1242], np.int32)}, "calib": exact_calib()}
        if len(gt_lidar):
            gt = _gt_annos(info, np.asarray(gt_lidar, np.float32), gt_names, rng)
            if len(gt_lidar) == 1:
                gt["occluded"], gt["truncated"] = np.zeros(1, np.int64), np.zeros(1)
        else:
            gt = {k: np.zeros((0, 4) if k == "bbox" else (0, 3) if k in ("location", "dimensions") else 0)
                  for k in GT_KEYS}
            gt["name"] = np.array([], dtype="<U8")
            gt["occluded"] = np.zeros(0, np.int64)
        if len(dontcare):
            gt = _add_dontcare(gt, dontcare)
        info["annos"] = gt
        boxes = np.zeros((n_det, 7), np.float32)
        k = np.arange(n_det)
        boxes[:, 0] = 12.0 + (k % 37)
        boxes[:, 1] = 3.0 + 0.1 * boxes[:, 0] * ((k // 37) % 3) / 3.0
        boxes[:, 2] = -1.0
        boxes[:, 3:6] = (0.6, 0.8, 1.7)
        boxes[:, 6] = edge_ry[k % 4]
        if drop:
            boxes[k % 8 == 7, :2] = (4.0, 30.0)                              # far to the side, outside the image: dropped
            boxes[k % 8 == 5, 0] = -12.0                 # behind the camera: it still projects into the image, and is kept
        labels = (k % 3 == 0).astype(np.int64)                               # Car and Pedestrian fillers
        scores = rng.permutation(np.linspace(0.05, 0.95, max(n_det, 1)))[:n_det].astype(np.float32)
        if n_det and len(gt_lidar) == 1:
            boxes[-1], labels[-1], scores[-1] = GT_BOX, 0, np.float32(0.99)
        infos.append(info)
        kind.append(what)
        dets[str(idx)] = {"box3d_lidar": boxes, "scores": scores, "label_preds": labels, "metadata": {"image_idx": idx}}

    for i, n in enumerate(CAPACITY_COUNTS):
        frame(3000 + i, [GT_BOX], ["Car"], n, "count")
    frame(3100, [], [], 1024, "count")
    many = np.zeros((300, 7), np.float32)
    j = np.arange(300)
    many[:, 0] = 15.0 + 0.2 * j
    many[:, 1] = -0.2 * many[:, 0] * ((j % 5) - 2) / 2.0
    many[:, 2] = -1.0
    many[:, 3:6] = (1.6, 3.9, 1.5)
    many[:, 6] = 0.01 * j
    frame(3101, many, ["Car", "Pedestrian", "Van"] * 100, 64, "count",
          dontcare=[[0.0, 150.0, 200.0, 250.0], [300.0, 150.0, 400.0, 250.0], [600.0, 160.0, 640.0, 200.0], [0.0, 0.0, 50.0, 50.0]])
    frame(3200, [GT_BOX], ["Car"], 40, "drop", drop=True)
    frame(3201, [GT_BOX], ["Car"], 1024, "drop", drop=True)
    return infos, dets, kind


# ------------------------------------------------------------------------------------------------ conversion edges
CONV_IMAGE = (375, 1000)


def conversion_set():
    """(infos, dets, expected): one frame of lidar detections on the conversion's edges, with an exact calibration: R0_rect = I,
    Tr_velo_to_cam permutes the axes (camera = lidar (-y, -z, x)) and P2 = [[500, 0, 600, 0], [0, 500, 200, 0], [0, 0, 1, 0]].
    Every box has w = l = 2 and h = 1.5 at lidar z = -1 (camera bottom y = 1.75), so with ry = 0 its camera corners are exact
    and u = 500 X / Z + 600 is exact where it is finite.

    0  u0 == W: corners X in {8, 10}, Z in {8, 10}; the smallest u is 10000 / 10 = 1000, the image width, and the box is kept
    1  u1 == 0: X in {-14, -12}, Z in {8, 10}; the largest u is 0, and the box is kept
    2  a corner on the camera plane with U = 0: X in {-2, 0}, Z in {0, 2}; u = 0 / 0 is NaN, so the min and max are NaN (the
       npmin rule) and the NaN comparisons keep the box
    3  corners on the camera plane with U > 0: u = +inf there, clipped to the image width; the box is kept
    4  behind the camera, projecting into the image: kept
    5  behind the camera, projecting left of the image: dropped
    6-9  ry = fp32 pi, -pi, 3 pi, -3 pi at 20 m, the limit_period boundary

    expected: the kept inputs and the crafted bbox values the generator asserts on the reference's conversion."""
    from kitti_eval_cases import exact_calib
    c = exact_calib()
    p2 = np.eye(4)
    p2[:3, :] = [[500.0, 0, 600, 0], [0, 500.0, 200, 0], [0, 0, 1.0, 0]]
    info = {"image": {"image_idx": 4000, "image_shape": np.array(CONV_IMAGE, np.int32)},
            "calib": {"R0_rect": c["R0_rect"], "Tr_velo_to_cam": c["Tr_velo_to_cam"], "P2": p2},
            "annos": {k: (np.zeros((0, 4)) if k == "bbox" else np.zeros((0, 3)) if k in ("location", "dimensions")
                          else np.zeros(0, np.int64) if k == "occluded" else np.zeros(0)) for k in GT_KEYS}}
    info["annos"]["name"] = np.array([], dtype="<U8")
    xy = [(9, -9), (9, 13), (1, 1), (1, -1.5), (-5, 0), (-5, -20), (20, -2), (20, 0), (20, 2), (20, 4)]
    ry = [0, 0, 0, 0, 0, 0, np.pi, -np.pi, 3 * np.pi, -3 * np.pi]
    boxes = np.array([[x, y, -1.0, 2.0, 2.0, 1.5, r] for (x, y), r in zip(xy, ry)], np.float32)
    det = {"box3d_lidar": boxes, "scores": np.linspace(0.9, 0.45, len(boxes)).astype(np.float32),
           "label_preds": np.arange(len(boxes)) % 2, "metadata": {"image_idx": 4000}}
    W = float(CONV_IMAGE[1])
    expected = {"kept": [0, 1, 2, 3, 4, 6, 7, 8, 9], "bbox": {0: (0, W), 1: (2, 0.0), 2: (0, np.nan), 3: (2, W)}}
    return [info], {"4000": det}, expected


def conversion_golden(g):
    """(info, det, dt_anno): the conversion-edge frame's inputs and the reference's conversion, as kitti_eval_edges.npz stores them."""
    info = {"image": {"image_idx": 4000, "image_shape": g["cvin_image_shape"]},
            "calib": {k: g["cvin_" + k] for k in ("R0_rect", "Tr_velo_to_cam", "P2")}}
    det = {k: g["cvin_" + k] for k in ("box3d_lidar", "scores", "label_preds")}
    anno = {k: g["cv_" + k] for k in ("bbox", "alpha", "location", "dimensions", "rotation_y", "score", "name")}
    return info, det, anno
