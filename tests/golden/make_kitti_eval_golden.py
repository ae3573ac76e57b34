"""Generate tests/golden/kitti_eval_cases.npz by running the REFERENCE's own KITTI evaluation in place.

    NUMBA_ENABLE_CUDASIM=1 python tests/golden/make_kitti_eval_golden.py

Imports det3d/datasets/kitti/{eval,kitti,kitti_common}.py, det3d/datasets/utils/eval.py, det3d/ops/nms/nms_gpu.py and
det3d/core/bbox/box_np_ops.py where they lie, through ``sys.modules`` shims for the compiled / optional modules they import
(det3d.utils.buildtools.pybind11_build, det3d.ops.nms.nms, spconv.utils, skimage, tqdm, the dataset base class).  The numba CUDA
simulator runs ``rotate_iou_gpu_eval`` without a GPU; it evaluates scalar expressions in Python floats, so the cases keep every
overlap at least kitti_eval_cases.MARGIN away from every min overlap (asserted here on the reference's own overlaps).

Stored: the inputs (per frame the calibration, image size, ground truth and lidar detections), the converted dt_annos, the
per-frame overlap matrices of each metric, and the result strings and detail values of get_official_eval_result, get_official_eval_result_v2, get_coco_eval_result and
KittiDataset.evaluation.
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


if __name__ == "__main__":
    main()
