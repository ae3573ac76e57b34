"""KITTI official (R11, R40) and COCO-style AP with AOS, computed on the device (sessd_b200.kitti_eval, csrc/kitti_eval.cu).

Same signatures, keys and text as det3d/datasets/kitti/eval.py of the reference: every function returns
{"result": str, "detail": dict}.  `gt_annos` / `dt_annos` are lists of per-frame annotation dicts (bbox, alpha, location,
dimensions, rotation_y, name, plus truncated / occluded for ground truth and score for detections).
"""
import numpy as np

from sessd_b200.kitti_eval import CLASS_NAMES, DeviceDT, DeviceGT, Frames, evaluate

_MOD = [0.7, 0.5, 0.5, 0.7, 0.7, 0.7, 0.7, 0.5, 0.5, 0.5, 0.5]
_EASY = ([0.7, 0.5, 0.5, 0.7, 0.7, 0.7, 0.7, 0.5, 0.25, 0.25, 0.5],
         [0.5, 0.25, 0.25, 0.5, 0.5, 0.5, 0.5, 0.25, 0.25, 0.25, 0.25])
# [overlap set, metric, class]: the moderate set for all metrics, then the easy set (its own 2D row)
OFFICIAL_OVERLAPS = np.stack([np.array([_MOD] * 3), np.array([_EASY[0], _EASY[1], _EASY[1]])], axis=0)
# class -> (first, last, count) of the COCO-style min-overlap grid
COCO_RANGES = {c: ((0.5, 0.95, 10) if CLASS_NAMES[c] in ("car", "truck", "bus", "trailer", "construction_vehicle") else (0.25, 0.7, 10))
               for c in range(len(CLASS_NAMES))}
_METRICS = ("bbox", "bev", "3d")


def _class_ints(current_classes):
    if not isinstance(current_classes, (list, tuple)):
        current_classes = [current_classes]
    return [CLASS_NAMES.index(c.lower()) if isinstance(c, str) else int(c) for c in current_classes]


def _has_alpha(dt_annos):
    """AOS is reported when the first frame with detections carries a real alpha (the label files' -10 means none)."""
    for a in dt_annos:
        if len(a["alpha"]):
            return bool(a["alpha"][0] != -10)
    return False


def _coco_overlaps(classes):
    mo = np.zeros([10, 3, len(classes)])
    for j, c in enumerate(classes):
        first, last, num = COCO_RANGES[c]
        mo[:, :, j] = np.linspace(first, last, int(num))[:, None]
    return mo


def _frames(gt_annos, dt_annos):
    return Frames(DeviceGT(gt_annos), DeviceDT.from_annos(dt_annos))


def _line(text):
    return text + "\n"


def _fmt(values):
    return ", ".join("%.2f" % v for v in values)


def format_official(ret, classes, min_overlaps, compute_aos, col, k0=0):
    """Result text and detail of the official AP (col 0: R11, col 1: R40) from `evaluate` output; sets k0, k0 + 1, ..."""
    result, detail = "", {}
    for j, cls in enumerate(classes):
        name = CLASS_NAMES[cls]
        detail[name] = {}
        for i in range(min_overlaps.shape[0]):
            ov = min_overlaps[i, :, j]
            aps = [ret[m]["map"][j, :, k0 + i, col] for m in range(3)]
            for m in range(3):
                detail[name]["%s@%.2f" % (_METRICS[m], ov[m])] = aps[m].tolist()
            result += _line("%s AP(Average Precision)@%.2f, %.2f, %.2f:" % (name, ov[0], ov[1], ov[2]))
            result += _line("bbox AP:" + _fmt(aps[0])) + _line("bev  AP:" + _fmt(aps[1])) + _line("3d   AP:" + _fmt(aps[2]))
            if compute_aos:
                aos = ret[0]["map"][j, :, k0 + i, col + 2]
                detail[name]["aos"] = aos.tolist()
                result += _line("aos  AP:" + _fmt(aos))
    return {"result": result, "detail": detail}


def format_coco(ret, classes, compute_aos, k0=0):
    """COCO-style text and detail: the R11 AP averaged over the 10 min-overlap sets k0 ... k0 + 9."""
    means = [ret[m]["map"][:, :, k0:k0 + 10, 0].mean(-1) for m in range(3)]
    aos = ret[0]["map"][:, :, k0:k0 + 10, 2].mean(-1)
    result, detail = "", {}
    for j, cls in enumerate(classes):
        name = CLASS_NAMES[cls]
        first, last, num = COCO_RANGES[cls]
        step = (last - first) / (num - 1)
        result += _line("%s coco AP@%.2f:%.2f:%.2f:" % (name, first, step, last))
        for m, label in enumerate(("bbox AP:", "bev  AP:", "3d   AP:")):
            result += _line(label + _fmt(means[m][j, :3]))
        detail[name] = {_METRICS[m]: means[m][j].tolist() for m in range(3)}
        if compute_aos:
            detail[name]["aos"] = aos[j].tolist()
            result += _line("aos  AP:" + _fmt(aos[j, :3]))
    return {"result": result, "detail": detail}


def _official(gt_annos, dt_annos, current_classes, difficultys, z_axis, z_center, col):
    classes = _class_ints(current_classes)
    mo = OFFICIAL_OVERLAPS[:, :, classes]
    aos = _has_alpha(dt_annos)
    ret = evaluate(_frames(gt_annos, dt_annos), classes, list(difficultys), mo, (0,) if aos else (), z_axis, z_center)
    return format_official(ret, classes, mo, aos, col)


def get_official_eval_result(gt_annos, dt_annos, current_classes, difficultys=(0, 1, 2), z_axis=1, z_center=1.0):
    """Official KITTI AP at 11 recall points (R11) for 2D, BEV, 3D and AOS."""
    return _official(gt_annos, dt_annos, current_classes, difficultys, z_axis, z_center, 0)


def get_official_eval_result_v2(gt_annos, dt_annos, current_classes, difficultys=(0, 1, 2), z_axis=1, z_center=1.0):
    """Official KITTI AP at 40 recall points (R40)."""
    return _official(gt_annos, dt_annos, current_classes, difficultys, z_axis, z_center, 1)


def get_coco_eval_result(gt_annos, dt_annos, current_classes, z_axis=1, z_center=1.0):
    """COCO-style AP: R11 AP averaged over 10 min overlaps per class (0.5:0.05:0.95 for cars, 0.25:0.05:0.7 otherwise)."""
    classes = _class_ints(current_classes)
    aos = _has_alpha(dt_annos)
    ret = evaluate(_frames(gt_annos, dt_annos), classes, [0, 1, 2], _coco_overlaps(classes), (0,) if aos else (), z_axis, z_center)
    return format_coco(ret, classes, aos)


def evaluate_all(frames, current_classes, compute_aos, z_axis=1, z_center=1.0):
    """R11, R40 and COCO results of one device run over the 2 official and the 10 COCO min-overlap sets."""
    classes = _class_ints(current_classes)
    mo = np.concatenate([OFFICIAL_OVERLAPS[:, :, classes], _coco_overlaps(classes)], axis=0)
    ret = evaluate(frames, classes, [0, 1, 2], mo, (0,), z_axis, z_center)
    off = OFFICIAL_OVERLAPS[:, :, classes]
    return (format_official(ret, classes, off, compute_aos, 0), format_official(ret, classes, off, compute_aos, 1),
            format_coco(ret, classes, compute_aos, k0=2))
