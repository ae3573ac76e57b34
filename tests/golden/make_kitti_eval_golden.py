"""Generate tests/golden/kitti_eval_cases.npz by running the REFERENCE's own KITTI evaluation in place.

    NUMBA_ENABLE_CUDASIM=1 python tests/golden/make_kitti_eval_golden.py          # kitti_eval_cases.npz
    NUMBA_ENABLE_CUDASIM=1 python tests/golden/make_kitti_eval_golden.py edges    # kitti_eval_edges.npz

Imports det3d/datasets/kitti/{eval,kitti,kitti_common}.py, det3d/datasets/utils/eval.py, det3d/ops/nms/nms_gpu.py and
det3d/core/bbox/box_np_ops.py where they lie, through ``sys.modules`` shims for the compiled / optional modules they import
(det3d.utils.buildtools.pybind11_build, det3d.ops.nms.nms, spconv.utils, skimage, tqdm, the dataset base class).  The numba CUDA
simulator runs ``rotate_iou_gpu_eval`` without a GPU; it evaluates scalar expressions in Python floats, so the cases keep every
overlap at least kitti_eval_cases.MARGIN away from every min overlap (asserted here on the reference's own overlaps).

Stored: the inputs (per frame the calibration, image size, ground truth and lidar detections), the converted dt_annos, the
per-frame overlap matrices of each metric, and the result strings and detail values of get_official_eval_result, get_official_eval_result_v2, get_coco_eval_result and
KittiDataset.evaluation.

`edges` runs the reference on the crafted decision frames of tests/kitti_eval_edges.py instead.  These frames sit exactly on the
evaluation's edges, so it asserts each crafted condition on the reference's own values, and it asserts that the simulated BEV /
3D overlaps equal the fp32 oracle's bit for bit: the simulator computes in Python floats, so this equality shows that every
intermediate of these frames is exact.  Stored: the inputs, the per-frame overlaps, the min overlaps, eval_class_v3's thresholds /
precision / orientation over the whole set, the three result functions' output, and for each frame's checks, run on that frame
alone, compute_statistics_jit's (tp, fp, similarity) at every threshold and eval_class_v3's curves.  It also stores the
reference's conversion of the conversion-edge frame (kitti_eval_edges.conversion_set), with its inputs.
"""
import importlib.util
import json
import os
import pickle
import sys
import tempfile
import types

os.environ.setdefault("NUMBA_ENABLE_CUDASIM", "1")
import numpy as np  # noqa: E402
import torch  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from kitti_eval_cases import CLASSES, THRESHOLDS, MARGIN, golden_inputs, make_set  # noqa: E402

SEED, FRAMES = 7, 48


def _pkg(name):
    m = types.ModuleType(name)
    m.__path__ = [os.path.join(REF, *name.split("."))]
    sys.modules[name] = m
    return m


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


def _load(name, rel):
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
    m = importlib.util.module_from_spec(spec)
    sys.modules[name] = m
    spec.loader.exec_module(m)
    return m


class _Reg:
    def register_module(self, cls):
        return cls


class _PointCloudDataset:
    def __init__(self, root_path, info_path, pipeline=None, test_mode=False, **kwargs):
        self._root_path, self._info_path, self.pipeline, self.test_mode = root_path, info_path, pipeline, test_mode


def _memo(fn):
    """The reference's rotate_iou_gpu_eval, run once per distinct input: every result function recomputes the same overlaps, and the
    simulator takes minutes per call.  Returns a copy, since box3d_overlap writes into the array it gets."""
    cache = {}

    def wrapped(boxes, query_boxes, criterion=-1, device_id=0):
        key = (boxes.dtype.str, boxes.shape, boxes.tobytes(), query_boxes.dtype.str, query_boxes.shape, query_boxes.tobytes(), criterion)
        if key not in cache:
            cache[key] = fn(boxes, query_boxes, criterion, device_id)
        return cache[key].copy()

    return wrapped


def install_shims():
    for p in ("det3d", "det3d.core", "det3d.core.bbox", "det3d.ops", "det3d.ops.nms", "det3d.utils", "det3d.utils.buildtools",
              "det3d.datasets", "det3d.datasets.kitti", "det3d.datasets.utils"):
        _pkg(p)
    _stub("det3d.utils.buildtools.pybind11_build", load_pb11=None)
    _stub("det3d.ops.nms.nms", non_max_suppression=None)
    _stub("spconv")
    _stub("spconv.utils", rbbox_iou=None, rbbox_intersection=None)
    _stub("skimage", io=None)
    _stub("tqdm", tqdm=lambda x, *a, **k: x)
    _stub("det3d.datasets.registry", DATASETS=_Reg())
    _stub("det3d.datasets.custom", PointCloudDataset=_PointCloudDataset)
    _load("det3d.core.bbox.geometry", "det3d/core/bbox/geometry.py")
    sys.modules["det3d.core.bbox"].box_np_ops = _load("det3d.core.bbox.box_np_ops", "det3d/core/bbox/box_np_ops.py")
    nms_gpu = _load("det3d.ops.nms.nms_gpu", "det3d/ops/nms/nms_gpu.py")
    nms_gpu.rotate_iou_gpu_eval = _memo(nms_gpu.rotate_iou_gpu_eval)
    _load("det3d.datasets.utils.eval", "det3d/datasets/utils/eval.py")
    ev = _load("det3d.datasets.kitti.eval", "det3d/datasets/kitti/eval.py")
    _load("det3d.datasets.kitti.kitti_common", "det3d/datasets/kitti/kitti_common.py")
    kitti = _load("det3d.datasets.kitti.kitti", "det3d/datasets/kitti/kitti.py")
    return ev, kitti, sys.modules["det3d.datasets.utils.eval"]


def _torch_dets(dets):
    return {k: {"box3d_lidar": torch.from_numpy(v["box3d_lidar"].copy()), "scores": torch.from_numpy(v["scores"].copy()),
                "label_preds": torch.from_numpy(v["label_preds"].copy()), "metadata": v["metadata"]} for k, v in dets.items()}


def main():
    ev, kitti, ueval = install_shims()
    infos, dets = make_set(SEED, FRAMES)
    with tempfile.TemporaryDirectory() as tmp:
        info_path = os.path.join(tmp, "infos.pkl")
        with open(info_path, "wb") as f:
            pickle.dump(infos, f)
        ds = kitti.KittiDataset(tmp, info_path, class_names=CLASSES)
        results, dt_annos = ds.evaluation(_torch_dets(dets))
    gt_annos = ds.ground_truth_annotations
    out = {"seed": SEED, "frames": FRAMES, "dataset_results": json.dumps(results)}
    overlaps = {}
    for metric in range(3):
        ovs = ueval.calculate_iou_partly(dt_annos, gt_annos, metric, 50, z_axis=1, z_center=1.0)[0]
        for f, o in enumerate(ovs):
            v = np.asarray(o, np.float64)
            near = np.array([np.min(np.abs(x - np.array(THRESHOLDS))) for x in v.ravel()]) if v.size else np.zeros(0)
            assert (near >= MARGIN).all(), ("overlap near a min overlap", metric, f)
            overlaps["ov%d_%d" % (metric, f)] = v
    for name, fn in (("official", ev.get_official_eval_result), ("official_v2", ev.get_official_eval_result_v2),
                     ("coco", ev.get_coco_eval_result)):
        r = fn(gt_annos, dt_annos, CLASSES, z_axis=1, z_center=1.0)
        out[name + "_result"] = r["result"]
        out[name + "_detail"] = json.dumps(r["detail"])
        print(r["result"])
    for f, a in enumerate(dt_annos):
        for k in ("bbox", "alpha", "location", "dimensions", "rotation_y", "score"):
            out["dt%d_%s" % (f, k)] = np.asarray(a[k])
        out["dt%d_name" % f] = np.asarray(a["name"]).astype(str)
    out.update(golden_inputs(infos, dets))
    out.update(overlaps)
    np.savez_compressed(os.path.join(HERE, "kitti_eval_cases.npz"), **out)
    print("kitti_eval_cases.npz:", FRAMES, "frames,", sum(len(a["name"]) for a in dt_annos), "detections")


def _frame_stats(ev, ueval, gt, dt, metric, cls, diff, min_ov):
    """The reference's eval_class_v3 steps on one frame for one config: (thresholds, [(tp, fp, similarity)] per threshold)."""
    ov = ueval.calculate_iou_partly([dt], [gt], metric, 50, z_axis=1, z_center=1.0)[0][0]
    gd, dd, igs, ids, dcs, _, nv = ueval.prepare_data([gt], [dt], cls, difficulty=diff, clean_data=ev.clean_data)
    tps = ueval.compute_statistics_jit(ov, gd[0], dd[0], igs[0], ids[0], dcs[0], metric, min_overlap=min_ov, thresh=0.0,
                                       compute_fp=False)[4]
    thr = np.array(ev.get_thresholds(np.array(tps.tolist()), nv))
    stats = [ueval.compute_statistics_jit(ov, gd[0], dd[0], igs[0], ids[0], dcs[0], metric, min_overlap=min_ov, thresh=t,
                                          compute_fp=True, compute_aos=True) for t in thr]
    return thr, np.array([(s[0], s[1], s[3]) for s in stats], np.float64).reshape(-1, 3)


def main_edges():
    """tests/golden/kitti_eval_edges.npz from the crafted decision frames of tests/kitti_eval_edges.py."""
    from kitti_eval_edges import CLASSES as E_CLASSES, CODES, build, min_overlaps_ref
    from oracle import kitti_eval_ref as ref
    ev, kitti, ueval = install_shims()
    names, gts, dts, checks, cond = build()
    mo = min_overlaps_ref()
    out = {"names": np.array(names), "min_overlaps": mo}
    for f, (g, d) in enumerate(zip(gts, dts)):
        for k, v in g.items():
            out["gt%d_%s" % (f, k)] = v
        for k, v in d.items():
            out["dt%d_%s" % (f, k)] = v
    # per-frame overlaps of the whole set; the simulator evaluates in Python floats, so equality with the fp32 oracle proves every
    # intermediate of these frames exact
    ovs = {}
    for metric in range(3):
        for f, o in enumerate(ueval.calculate_iou_partly(dts, gts, metric, 50, z_axis=1, z_center=1.0)[0]):
            v = np.asarray(o, np.float64)
            orc = ref.overlaps_frame(metric, ref.records(dts[f], "score"), ref.records(gts[f], "truncated"))
            assert np.array_equal(v, orc), ("simulator and oracle overlaps differ", names[f], metric)
            ovs[(metric, f)] = out["ov%d_%d" % (metric, f)] = v
    # every crafted condition, on the reference's own values
    for f, name in enumerate(names):
        for c in cond[name]:
            if c[0] == "ov":
                assert ovs[(c[1], f)][c[2], c[3]] == c[4], (name, c, ovs[(c[1], f)][c[2], c[3]])
            elif c[0] == "ov_lt":
                assert ovs[(c[1], f)][c[2], c[3]] < c[4], (name, c)
            elif c[0] == "dc":
                dc = np.stack([b for n, b in zip(gts[f]["name"], gts[f]["bbox"]) if n == "DontCare"]).astype(np.float64)
                assert ueval.image_box_overlap(dts[f]["bbox"], dc, 0)[c[1], c[2]] == c[3], (name, c)
            elif c[0] == "h_gt":
                assert gts[f]["bbox"][c[1], 3] - gts[f]["bbox"][c[1], 1] == c[2], (name, c)
            elif c[0] == "h_dt":
                assert abs(dts[f]["bbox"][c[1], 3] - dts[f]["bbox"][c[1], 1]) == c[2], (name, c)
    for t in (0.15, 0.3, 0.5):
        assert np.nextafter(t, 1.0) > t
    # each decision frame alone, one config per check: compute_statistics_jit at every threshold and eval_class_v3's curves
    for f, name in enumerate(names):
        for q, (metric, cls, diff, min_ov, want) in enumerate(checks[name]):
            thr, st = _frame_stats(ev, ueval, gts[f], dts[f], metric, cls, diff, min_ov)
            assert [(int(a), int(b)) for a, b, _ in st] == want, (name, metric, cls, diff, st, want)
            for c in cond[name]:
                if c[0] == "n_thr":
                    assert len(thr) == c[1], (name, len(thr))
            m1 = np.zeros([1, 3, 1])
            m1[0, metric, 0] = min_ov
            r = ev.eval_class_v3([gts[f]], [dts[f]], [cls], [diff], metric, m1, compute_aos=metric == 0, z_axis=1, z_center=1.0)
            if want and all(a + b == 0 for a, b in want[:1]):
                assert np.isnan(r["precision"][0, 0, 0, 0]), name
            key = "c%d_%d" % (f, q)
            out[key + "_config"] = np.array([metric, cls, diff], np.int64)
            out[key + "_min_overlap"] = np.float64(min_ov)
            out[key + "_stats"] = st
            for k in ("thresholds", "precision", "orientation"):
                out[key + "_" + k] = r[k][0, 0, 0]
    # the whole set: eval_class_v3 per metric over the official and COCO min overlaps, and the three result functions
    for metric in range(3):
        r = ev.eval_class_v3(gts, dts, CODES, [0, 1, 2], metric, mo, compute_aos=metric == 0, z_axis=1, z_center=1.0)
        for k in ("thresholds", "precision", "orientation"):
            out["set%d_%s" % (metric, k)] = r[k]
    for name, fn in (("official", ev.get_official_eval_result), ("official_v2", ev.get_official_eval_result_v2),
                     ("coco", ev.get_coco_eval_result)):
        r = fn(gts, dts, E_CLASSES, z_axis=1, z_center=1.0)
        out[name + "_result"] = r["result"]
        out[name + "_detail"] = json.dumps(r["detail"])
        print(r["result"])
    # the conversion edges: KittiDataset.convert_detection_to_kitti_annos on one frame, each crafted bbox value asserted
    from kitti_eval_edges import conversion_set
    cinfos, cdets, expect = conversion_set()
    with tempfile.TemporaryDirectory() as tmp:
        info_path = os.path.join(tmp, "infos.pkl")
        with open(info_path, "wb") as fh:
            pickle.dump(cinfos, fh)
        conv = kitti.KittiDataset(tmp, info_path, class_names=E_CLASSES).convert_detection_to_kitti_annos(_torch_dets(cdets))[0]
    d = cdets["4000"]
    assert len(conv["name"]) == len(expect["kept"]), conv["name"]
    for i, (col, v) in expect["bbox"].items():
        got = conv["bbox"][expect["kept"].index(i), col]
        assert (np.isnan(got) if np.isnan(v) else got == v), (i, col, got)
    for k in ("box3d_lidar", "scores", "label_preds"):
        out["cvin_" + k] = d[k]
    for k in ("R0_rect", "Tr_velo_to_cam", "P2"):
        out["cvin_" + k] = cinfos[0]["calib"][k]
    out["cvin_image_shape"] = cinfos[0]["image"]["image_shape"]
    for k in ("bbox", "alpha", "location", "dimensions", "rotation_y", "score"):
        out["cv_" + k] = np.asarray(conv[k])
    out["cv_name"] = np.asarray(conv["name"]).astype(str)
    np.savez_compressed(os.path.join(HERE, "kitti_eval_edges.npz"), **out)
    print("kitti_eval_edges.npz:", len(names), "frames,", sum(len(c) for c in checks.values()), "checks")


if __name__ == "__main__":
    if sys.argv[1:] == ["edges"]:
        main_edges()
    else:
        main()
