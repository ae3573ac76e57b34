"""numpy restatement of the KITTI object evaluation (official R11 / R40, COCO-style AP, AOS) and of the detection -> camera
annotation conversion, written from their definitions; the device version is csrc/kitti_eval.cu.

Rounding follows the reference's types step by step (listed at the top of csrc/kitti_eval.cu): fp64 for 2D overlaps, matching and
thresholds; the rotated-box clip in fp32 with its triangle areas summed in fp64 and every BEV / 3D overlap rounded to fp32.
The rotated-box clip is vectorised over all box pairs; everything else is plain loops, so this is meant for test-sized sets.
"""
import numpy as np

CLASS_NAMES = ("car", "pedestrian", "bicycle", "truck", "bus", "trailer", "construction_vehicle", "motorcycle", "barrier",
               "traffic_cone", "cyclist")
MIN_HEIGHT = (40, 25, 25)
MAX_OCCLUSION = (0, 1, 2)
MAX_TRUNCATION = (0.15, 0.3, 0.5)
N_PTS = 41
f4, f8 = np.float32, np.float64


# ------------------------------------------------------------------------------------------------ overlaps
def box2d_overlap(b, q, criterion=-1):
    """[N, K] fp64 overlap of boxes b [N, 4] against q [K, 4]; criterion -1 IoU, 0 over b's area."""
    b = np.asarray(b, f8).reshape(-1, 4)
    q = np.asarray(q, f8).reshape(-1, 4)
    out = np.zeros((len(b), len(q)))
    for k in range(len(q)):
        qa = (q[k, 2] - q[k, 0]) * (q[k, 3] - q[k, 1])
        for n in range(len(b)):
            iw = min(b[n, 2], q[k, 2]) - max(b[n, 0], q[k, 0])
            if iw > 0:
                ih = min(b[n, 3], q[k, 3]) - max(b[n, 1], q[k, 1])
                if ih > 0:
                    ba = (b[n, 2] - b[n, 0]) * (b[n, 3] - b[n, 1])
                    ua = ba + qa - iw * ih if criterion == -1 else ba
                    out[n, k] = iw * ih / ua
    return out


def _corners(r):
    """r [P, 5] fp32 -> x [P, 4], y [P, 4] fp32, corner order (-,-) (-,+) (+,+) (+,-) rotated clockwise for positive angles."""
    ca, sa = np.cos(r[:, 4].astype(f8)).astype(f4), np.sin(r[:, 4].astype(f8)).astype(f4)     # correctly rounded fp32
    hx, hy = r[:, 2] / f4(2), r[:, 3] / f4(2)
    cx = np.stack([-hx, -hx, hx, hx], 1)
    cy = np.stack([-hy, hy, hy, -hy], 1)
    x = ca[:, None] * cx + sa[:, None] * cy + r[:, 0:1]
    y = -sa[:, None] * cx + ca[:, None] * cy + r[:, 1:2]
    return x, y


def _inside(px, py, qx, qy):
    ab0, ab1 = qx[:, 1] - qx[:, 0], qy[:, 1] - qy[:, 0]
    ad0, ad1 = qx[:, 3] - qx[:, 0], qy[:, 3] - qy[:, 0]
    ap0, ap1 = px - qx[:, 0], py - qy[:, 0]
    abab, abap = ab0 * ab0 + ab1 * ab1, ab0 * ap0 + ab1 * ap1
    adad, adap = ad0 * ad0 + ad1 * ad1, ad0 * ap0 + ad1 * ap1
    return (abab >= abap) & (abap >= 0) & (adad >= adap) & (adap >= 0)


def _crossing(x1, y1, x2, y2, i, j):
    A0, A1, B0, B1 = x1[:, i], y1[:, i], x1[:, (i + 1) % 4], y1[:, (i + 1) % 4]
    C0, C1, D0, D1 = x2[:, j], y2[:, j], x2[:, (j + 1) % 4], y2[:, (j + 1) % 4]
    BA0, BA1, DA0, CA0, DA1, CA1 = B0 - A0, B1 - A1, D0 - A0, C0 - A0, D1 - A1, C1 - A1
    acd = DA1 * CA0 > CA1 * DA0
    bcd = (D1 - B1) * (C0 - B0) > (C1 - B1) * (D0 - B0)
    abc = CA1 * BA0 > BA1 * CA0
    abd = DA1 * BA0 > BA1 * DA0
    ok = (acd != bcd) & (abc != abd)
    DC0, DC1 = D0 - C0, D1 - C1
    ABBA, CDDC = A0 * B1 - B0 * A1, C0 * D1 - D0 * C1
    DH = BA1 * DC0 - BA0 * DC1
    with np.errstate(divide="ignore", invalid="ignore"):
        return ok, (ABBA * DC0 - BA0 * CDDC) / DH, (ABBA * DC1 - BA1 * CDDC) / DH


def rbox_inter(r1, r2, with_count=False):
    """Intersection areas (fp64) of rotated boxes r1 [P, 5] and r2 [P, 5] (x, y, dx, dy, angle; rounded to fp32); with_count also
    returns the number of clip vertices of each pair."""
    r1, r2 = np.asarray(r1, f4).reshape(-1, 5), np.asarray(r2, f4).reshape(-1, 5)
    P = len(r1)
    x1, y1 = _corners(r1)
    x2, y2 = _corners(r2)
    cand_x, cand_y, cand_ok = [], [], []
    for i in range(4):
        cand_x += [x1[:, i], x2[:, i]]
        cand_y += [y1[:, i], y2[:, i]]
        cand_ok += [_inside(x1[:, i], y1[:, i], x2, y2), _inside(x2[:, i], y2[:, i], x1, y1)]
    for i in range(4):
        for j in range(4):
            ok, cx, cy = _crossing(x1, y1, x2, y2, i, j)
            cand_x.append(cx)
            cand_y.append(cy)
            cand_ok.append(ok)
    ok = np.stack(cand_ok, 1)
    order = np.argsort(~ok, axis=1, kind="stable")                      # kept candidates first, in candidate order
    px = np.take_along_axis(np.stack(cand_x, 1), order, 1).astype(f4)
    py = np.take_along_axis(np.stack(cand_y, 1), order, 1).astype(f4)
    n = ok.sum(1)
    valid = np.arange(24)[None, :] < n[:, None]
    sx, sy = np.zeros(P, f4), np.zeros(P, f4)
    for k in range(24):
        sx = np.where(valid[:, k], sx + px[:, k], sx)
        sy = np.where(valid[:, k], sy + py[:, k], sy)
    with np.errstate(divide="ignore", invalid="ignore"):
        sx = (sx.astype(f8) / np.maximum(n, 1)).astype(f4)
        sy = (sy.astype(f8) / np.maximum(n, 1)).astype(f4)
        v0, v1 = px - sx[:, None], py - sy[:, None]
        d = np.sqrt(v0 * v0 + v1 * v1)
        v0, v1 = v0 / d, v1 / d
    vs = np.where(v1 < 0, f4(-2) - v0, v0)
    vs = np.where(valid, vs, np.inf).astype(f4)
    srt = np.argsort(vs, axis=1, kind="stable")                         # the insertion sort is stable
    px, py = np.take_along_axis(px, srt, 1), np.take_along_axis(py, srt, 1)
    area = np.zeros(P, f8)
    for k in range(22):
        with np.errstate(invalid="ignore"):                              # slots past the polygon hold NaN / inf
            t = (px[:, 0] - px[:, k + 2]) * (py[:, k + 1] - py[:, k + 2]) - (py[:, 0] - py[:, k + 2]) * (px[:, k + 1] - px[:, k + 2])
        area = np.where(k < n - 2, area + np.abs(t.astype(f8) / 2.0), area)
    return (area, n) if with_count else area


def _bev(rec, z_axis):
    a, b = [i for i in range(3) if i != z_axis]
    return np.stack([rec[:, 5 + a], rec[:, 5 + b], rec[:, 8 + a], rec[:, 8 + b], rec[:, 11]], 1)


def overlaps_frame(metric, dt, gt, z_axis=1, z_center=1.0):
    """[n_dt, n_gt] fp64 overlaps of one frame.  dt / gt: records [n, 13] (bbox 4, alpha, location 3, dimensions 3, ry, score or
    truncation)."""
    nd, ng = len(dt), len(gt)
    if metric == 0:
        return box2d_overlap(dt[:, :4], gt[:, :4])
    if nd == 0 or ng == 0:
        return np.zeros((nd, ng))
    jj, ii = np.meshgrid(np.arange(nd), np.arange(ng), indexing="ij")
    bg, bd = _bev(gt, z_axis).astype(f4)[ii.ravel()], _bev(dt, z_axis).astype(f4)[jj.ravel()]
    inter = rbox_inter(bg, bd)                                           # GT first, as the reference's swapped operands put it
    if metric == 1:
        a12 = (bg[:, 2] * bg[:, 3] + bd[:, 2] * bd[:, 3]).astype(f8)
        with np.errstate(divide="ignore", invalid="ignore"):
            return (inter / (a12 - inter)).astype(f4).astype(f8).reshape(nd, ng)
    rinc = inter.astype(f4).reshape(nd, ng)
    out = rinc.copy()
    up = 1 - z_center
    for j in range(nd):
        for i in range(ng):
            if rinc[j, i] > 0:
                lj, dj, li, di = dt[j, 5:8], dt[j, 8:11], gt[i, 5:8], gt[i, 8:11]
                min_z = min(lj[z_axis] + dj[z_axis] * up, li[z_axis] + di[z_axis] * up)
                max_z = max(lj[z_axis] - dj[z_axis] * z_center, li[z_axis] - di[z_axis] * z_center)
                iw = min_z - max_z
                if iw > 0:
                    inc = iw * f8(rinc[j, i])
                    out[j, i] = inc / (dj[0] * dj[1] * dj[2] + di[0] * di[1] * di[2] - inc)
                else:
                    out[j, i] = 0.0
    return out.astype(f8)


# ------------------------------------------------------------------------------------------------ annotations -> flags
def name_code(name):
    n = str(name).lower()
    if n in CLASS_NAMES:
        return CLASS_NAMES.index(n)
    return {"person_sitting": 11, "van": 12}.get(n, -1)


def records(anno, last):
    n = len(anno["name"])
    r = np.zeros((n, 13))
    if n:
        r[:, 0:4], r[:, 4], r[:, 5:8] = anno["bbox"], anno["alpha"], anno["location"]
        r[:, 8:11], r[:, 11], r[:, 12] = anno["dimensions"], anno["rotation_y"], anno[last]
    return r


def gt_flags(anno, cls, diff):
    out = []
    for i, name in enumerate(anno["name"]):
        code = name_code(name)
        valid = 1 if code == cls else (0 if (cls == 1 and code == 11) or (cls == 0 and code == 12) else -1)
        h = anno["bbox"][i][3] - anno["bbox"][i][1]
        ign = anno["occluded"][i] > MAX_OCCLUSION[diff] or anno["truncated"][i] > MAX_TRUNCATION[diff] or h <= MIN_HEIGHT[diff]
        out.append(0 if valid == 1 and not ign else (1 if valid == 0 or (ign and valid == 1) else -1))
    return np.array(out, dtype=np.int64)


def dt_flags(anno, cls, diff):
    out = []
    for i, name in enumerate(anno["name"]):
        if abs(anno["bbox"][i][3] - anno["bbox"][i][1]) < MIN_HEIGHT[diff]:
            out.append(1)
        else:
            out.append(0 if name_code(name) == cls else -1)
    return np.array(out, dtype=np.int64)


def dontcare_boxes(anno):
    return np.array([b for n, b in zip(anno["name"], anno["bbox"]) if n == "DontCare" or n == "ignore"], f8).reshape(-1, 4)


# ------------------------------------------------------------------------------------------------ matching
def match(ov, gt, dt, ig, idt, dc, metric, min_ov, thresh=0.0, compute_fp=False, aos=False):
    """One frame: (tp, fp, similarity or -1, TP scores in GT order).  ov [n_dt, n_gt]."""
    nd = len(dt)
    assigned = np.zeros(nd, bool)
    below = (dt[:, 12] < thresh) if compute_fp else np.zeros(nd, bool)
    tp = fp = 0
    sim = 0.0
    scores = []
    for i in range(len(gt)):
        if ig[i] == -1:
            continue
        best, best_key, taken_ignored = -1, None, False
        for j in np.nonzero((idt != -1) & ~assigned & ~below & (ov[:, i] > min_ov))[0] if nd else ():
            if not compute_fp:
                if dt[j, 12] > -10000000 and (best < 0 or dt[j, 12] > best_key):
                    best, best_key = j, dt[j, 12]
            elif idt[j] == 0 and (best < 0 or taken_ignored or ov[j, i] > best_key):
                best, best_key, taken_ignored = j, ov[j, i], False
            elif idt[j] == 1 and best < 0:
                best, best_key, taken_ignored = j, 0.0, True
        if best < 0:
            continue
        if ig[i] == 1 or idt[best] == 1:
            assigned[best] = True
            continue
        tp += 1
        scores.append(dt[best, 12])
        if aos:
            sim += (1.0 + np.cos(gt[i, 4] - dt[best, 4])) / 2.0
        assigned[best] = True
    if not compute_fp:
        return tp, 0, -1, scores
    free = ~(assigned | (idt == -1) | (idt == 1) | below)
    fp = int(free.sum())
    if metric == 0 and len(dc):
        odc = box2d_overlap(dt[:, :4], dc, 0)
        for c in range(len(dc)):
            for j in range(nd):
                if free[j] and not assigned[j] and odc[j, c] > min_ov:
                    assigned[j] = True
                    fp -= 1
    return tp, fp, (sim if (tp > 0 or fp > 0) else -1), scores


def thresholds(scores, num_gt):
    s = np.sort(np.asarray(scores, f8))[::-1]
    cur, out = 0.0, []
    for i in range(len(s)):
        lr = (i + 1) / num_gt
        rr = (i + 2) / num_gt if i < len(s) - 1 else lr
        if (rr - cur) < (cur - lr) and i < len(s) - 1:
            continue
        out.append(s[i])
        cur += 1 / (N_PTS - 1.0)
    return out


def eval_config(ovs, gts, dts, gt_annos, dt_annos, dcs, metric, cls, diff, min_ov, aos):
    """(thresholds, precision [41], aos [41]) of one (metric, class, difficulty, min overlap)."""
    igs = [gt_flags(a, cls, diff) for a in gt_annos]
    ids = [dt_flags(a, cls, diff) for a in dt_annos]
    num_valid = sum(int((g == 0).sum()) for g in igs)
    tp_scores = []
    for f in range(len(gts)):
        tp_scores += match(ovs[f], gts[f], dts[f], igs[f], ids[f], dcs[f], metric, min_ov)[3]
    thr = thresholds(tp_scores, num_valid)
    pr = np.zeros((len(thr), 3))
    for f in range(len(gts)):
        for t, th in enumerate(thr):
            tp, fp, sim, _ = match(ovs[f], gts[f], dts[f], igs[f], ids[f], dcs[f], metric, min_ov, th, True, aos)
            pr[t, 0] += tp
            pr[t, 1] += fp
            if sim != -1:
                pr[t, 2] += sim
    prec, orient, th = np.zeros(N_PTS), np.zeros(N_PTS), np.zeros(N_PTS)
    th[:len(thr)] = thr
    with np.errstate(divide="ignore", invalid="ignore"):
        for t in range(len(thr)):
            prec[t] = pr[t, 0] / (pr[t, 0] + pr[t, 1])
            if aos:
                orient[t] = pr[t, 2] / (pr[t, 0] + pr[t, 1])
    for t in range(len(thr)):
        prec[t] = np.max(prec[t:])
        if aos:
            orient[t] = np.max(orient[t:])
    return th, prec, orient


def map_r11(p):
    s = 0
    for i in range(0, p.shape[-1], 4):
        s = s + p[..., i]
    return s / 11 * 100


def map_r40(p):
    s = 0
    for i in range(1, p.shape[-1]):
        s = s + p[..., i]
    return s / 40 * 100


def evaluate(gt_annos, dt_annos, classes, difficultys, min_overlaps, aos_metrics=(0,), z_axis=1, z_center=1.0):
    """Same layout as sessd_b200.kitti_eval.evaluate: {metric: {"precision", "orientation", "thresholds" [C, D, K, 41],
    "map" [C, D, K, 4]}}."""
    gts = [records(a, "truncated") for a in gt_annos]
    dts = [records(a, "score") for a in dt_annos]
    dcs = [dontcare_boxes(a) for a in gt_annos]
    K, C, D = min_overlaps.shape[0], len(classes), len(difficultys)
    res = {}
    for metric in range(3):
        ovs = [overlaps_frame(metric, d, g, z_axis, z_center) for d, g in zip(dts, gts)]
        out = {k: np.zeros((C, D, K, N_PTS)) for k in ("precision", "orientation", "thresholds")}
        for m, cls in enumerate(classes):
            for l, diff in enumerate(difficultys):
                for k in range(K):
                    th, p, o = eval_config(ovs, gts, dts, gt_annos, dt_annos, dcs, metric, cls, diff, min_overlaps[k, metric, m],
                                           metric in aos_metrics)
                    out["thresholds"][m, l, k], out["precision"][m, l, k], out["orientation"][m, l, k] = th, p, o
        out["map"] = np.stack([map_r11(out["precision"]), map_r40(out["precision"]), map_r11(out["orientation"]),
                               map_r40(out["orientation"])], -1)
        out["overlaps"] = ovs
        res[metric] = out
    return res


# ------------------------------------------------------------------------------------------------ lidar detections -> annotations
def convert_frame(boxes, scores, labels, info, class_names):
    """One frame of KittiDataset.convert_detection_to_kitti_annos: lidar boxes [n, 7] fp32 -> annotation dict (no metadata)."""
    b = np.array(boxes, dtype=f4).reshape(-1, 7)
    keys = ("name", "truncated", "occluded", "alpha", "bbox", "dimensions", "location", "rotation_y", "score")
    out = {k: [] for k in keys}
    if len(b):
        period = f4(2 * np.pi)
        b[:, 6] = b[:, 6] - np.floor(b[:, 6] / period + f4(0.5)) * period
        b[:, 2] = b[:, 2] - b[:, 5] / f4(2)
        c = info["calib"]
        m = np.asarray(c["R0_rect"]) @ np.asarray(c["Tr_velo_to_cam"])
        xyz = np.concatenate([b[:, :3].astype(f8), np.ones((len(b), 1))], 1) @ m.T
        cam = np.concatenate([xyz[:, :3], b[:, 4:5], b[:, 5:6], b[:, 3:4], b[:, 6:7]], 1).astype(f8)
        bits = np.array([[(o >> 2) & 1, (o >> 1) & 1, o & 1] for o in (0, 1, 3, 2, 4, 5, 7, 6)], f8) - np.array([0.5, 1.0, 0.5])
        corners = cam[:, None, 3:6] * bits[None]
        rc, rs = np.cos(cam[:, 6])[:, None], np.sin(cam[:, 6])[:, None]
        X = corners[..., 0] * rc + corners[..., 2] * rs + cam[:, 0:1]
        Y = corners[..., 1] + cam[:, 1:2]
        Z = -corners[..., 0] * rs + corners[..., 2] * rc + cam[:, 2:3]
        P = np.asarray(c["P2"])
        U = X * P[0, 0] + Y * P[0, 1] + Z * P[0, 2]
        V = X * P[1, 0] + Y * P[1, 1] + Z * P[1, 2]
        W = X * P[2, 0] + Y * P[2, 1] + Z * P[2, 2]
        u, v = U / W, V / W
        bbox = np.stack([u.min(1), v.min(1), u.max(1), v.max(1)], 1)
        H, Wd = info["image"]["image_shape"][:2]
        for j in range(len(b)):
            if bbox[j, 0] > Wd or bbox[j, 1] > H or bbox[j, 2] < 0 or bbox[j, 3] < 0:
                continue
            bb = np.array([max(bbox[j, 0], 0), max(bbox[j, 1], 0), min(bbox[j, 2], Wd), min(bbox[j, 3], H)], f8)
            out["bbox"].append(bb)
            out["alpha"].append(f8(-f4(np.arctan2(-f8(b[j, 1]), f8(b[j, 0])))) + cam[j, 6])   # fp32 atan2, correctly rounded
            out["dimensions"].append(cam[j, 3:6])
            out["location"].append(cam[j, :3])
            out["rotation_y"].append(cam[j, 6])
            out["name"].append(class_names[int(labels[j])])
            out["truncated"].append(0.0)
            out["occluded"].append(0)
            out["score"].append(f4(scores[j]))
    if not out["name"]:
        return {"name": np.array([]), "truncated": np.array([]), "occluded": np.array([]), "alpha": np.array([]),
                "bbox": np.zeros([0, 4]), "dimensions": np.zeros([0, 3]), "location": np.zeros([0, 3]), "rotation_y": np.array([]),
                "score": np.array([])}
    return {k: np.stack(v) for k, v in out.items()}
