"""KittiDataset mirror (det3d/datasets/kitti/kitti.py): frame loading and evaluation.

``__getitem__`` / ``get_sensor_data`` build the reference's ``res`` dict and run the config pipeline's host stages, the two loaders of
pipelines/loading.py (one ``np.fromfile``, the camera -> lidar boxes, the calibration frustum).  The pipeline's device stages
(``Preprocess``, ``Voxelization``, ``AssignTarget``, ``Reformat``) are run per batch by ``det3d.datasets.loader.build_dataloader``
(sessd_b200.kitti_loader), which reads their configs from ``device_stages``.  Evaluation (ground truth, detection -> KITTI camera
annotations, ``evaluation``) runs on the device (sessd_b200.kitti_eval)."""
import pickle

import numpy as np

from det3d.utils import build_from_cfg
from sessd_b200 import kitti_eval as ke

from ..registry import DATASETS, PIPELINES
from .eval import _has_alpha, evaluate_all

HOST_STAGES = ("LoadPointCloudFromFile", "LoadPointCloudAnnotations")
DEVICE_STAGES = ("Preprocess", "Voxelization", "AssignTarget", "Reformat")


@DATASETS.register_module
class KittiDataset:
    NumPointFeatures = 4

    def __init__(self, root_path, info_path, cfg=None, pipeline=None, class_names=None, test_mode=False, **kwargs):
        assert info_path is not None
        self._root_path = root_path
        self._info_path = info_path
        self.pipeline = pipeline
        self.test_mode = test_mode
        self._host_stages, self.device_stages = _split_pipeline(pipeline or [])
        # the frames' mode: the pipeline's Preprocess sets it (the reference's val split is built without test_mode)
        pre = self.device_stages.get("Preprocess")
        self.mode = pre["cfg"]["mode"] if pre is not None else ("val" if test_mode else "train")
        with open(info_path, "rb") as f:
            self._kitti_infos = pickle.load(f)
        self._num_point_features = KittiDataset.NumPointFeatures
        self._class_names = class_names
        self.CLASSES = class_names
        self.labeled = kwargs.get("labeled", True)
        self.plane_dir = root_path + "/training/planes"
        self._device_gt = None       # packed ground truth; it does not change between epochs
        self._device_calib = None

    def __len__(self):
        return len(self._kitti_infos)

    @property
    def num_point_features(self):
        return self._num_point_features

    @property
    def ground_truth_annotations(self):
        if "annos" not in self._kitti_infos[0]:
            return None
        return [info["annos"] for info in self._kitti_infos]

    def _gt(self):
        if self._device_gt is None:
            self._device_gt = ke.DeviceGT(self.ground_truth_annotations)
        return self._device_gt

    def _frames_of(self, detection, partial):
        gt_idx = [str(info["image"]["image_idx"]) for info in self._kitti_infos]
        keys = list(detection.keys()) if partial else gt_idx
        if partial:
            calib = ke.DeviceCalib([self._kitti_infos[gt_idx.index(k)] for k in keys])
        else:
            if self._device_calib is None:
                self._device_calib = ke.DeviceCalib(self._kitti_infos)
            calib = self._device_calib
        dets = [(detection[k]["box3d_lidar"], detection[k]["scores"], detection[k]["label_preds"]) for k in keys]
        dt, labels = ke.convert_detections(dets, calib, self._class_names)
        return keys, dt, labels

    def _annos(self, detection, keys, dt, labels):
        annos = ke.dt_annos_from_device(dt, labels, self._class_names)
        for a, k in zip(annos, keys):
            a["metadata"] = detection[k]["metadata"]
        return annos

    def convert_detection_to_kitti_annos(self, detection, partial=False):
        """detection: {image_idx string: {"box3d_lidar", "scores", "label_preds", "metadata"}}, tensors on any device.  Boxes whose
        image box lies outside the image are dropped, the rest clipped to it."""
        keys, dt, labels = self._frames_of(detection, partial)
        return self._annos(detection, keys, dt, labels)

    def evaluation(self, detections, output_dir=None, get_results=True):
        """KITTI camera boxes: z_axis 1, z_center 1.0.  Returns (results, dt_annos); nothing is copied to the host before the
        kernels have run, then one copy brings the curves back and one builds dt_annos."""
        keys, dt, labels = self._frames_of(detections, False)
        results = None
        if get_results:
            frames = ke.Frames(self._gt(), dt)
            official, official_2, coco = evaluate_all(frames, self._class_names, True, z_axis=1, z_center=1.0)
        dt_annos = self._annos(detections, keys, dt, labels)
        if get_results:
            if not _has_alpha(dt_annos):
                official, official_2, coco = (_drop_aos(r) for r in (official, official_2, coco))
            results = {"results": {"official_AP_11": official["result"]},
                       "results_2": {"official_AP_40": official_2["result"]},
                       "detail": {"eval.kitti": {"official": official["detail"], "coco": coco["detail"]}}}
        return results, dt_annos

    def __getitem__(self, idx):
        return self.get_sensor_data(idx)

    def get_sensor_data(self, idx, with_image=False, with_gp=False, by_index=False):
        """The reference's ``res`` dict of frame ``idx`` (by_index: ``idx`` is an image index) after the host stages: points, calib with
        the image frustum, the lidar / camera annotations, and ``mode`` as the pipeline's Preprocess sets it.  A labelled train-mode frame also carries ``gt_boxes`` / ``gt_names`` with
        DontCare / ignore dropped, the first step of the reference's Preprocess, which the device batch builder takes."""
        if self.pipeline is None:
            raise NotImplementedError("KittiDataset: built without a pipeline, so nothing loads its frames (pass the config's "
                                      "pipeline list)")
        if with_gp or with_image:
            raise NotImplementedError("road planes and camera images are not loaded (the SE-SSD car config uses neither)")
        if by_index:
            idx = [int(info["image"]["image_idx"]) for info in self._kitti_infos].index(idx)
        info = self._kitti_infos[idx]
        res = {
            "type": "KittiDataset",
            "lidar": {"type": "lidar", "points": None, "ground_plane": None, "annotations": None, "names": None, "targets": None},
            "metadata": {"image_prefix": self._root_path, "num_point_features": KittiDataset.NumPointFeatures,
                         "image_idx": info["image"]["image_idx"], "image_shape": info["image"]["image_shape"],
                         "token": str(info["image"]["image_idx"])},
            "calib": None,
            "cam": {"annotations": None},
            "mode": "val" if self.test_mode else "train",
        }
        res.update({"labeled": self.labeled})
        for stage in self._host_stages:
            res, info = stage(res, info)
        res["mode"] = self.mode
        anno = res["lidar"]["annotations"]
        if res["mode"] == "train" and res["labeled"] and anno is not None:
            names = np.array(anno["names"]).reshape(-1)
            keep = np.array([i for i, n in enumerate(names) if n not in ("DontCare", "ignore")], dtype=np.int64)
            res["lidar"]["gt_boxes"], res["lidar"]["gt_names"] = anno["boxes"][keep], names[keep]
        return res


def _split_pipeline(pipeline):
    """the config pipeline -> (host stage objects, {device stage type: its config dict}); any other stage type is a ValueError"""
    host, device = [], {}
    for stage in pipeline:
        kind = stage["type"]
        if kind in HOST_STAGES:
            host.append(build_from_cfg(stage, PIPELINES))
        elif kind in DEVICE_STAGES:
            device[kind] = stage
        else:
            raise ValueError("KittiDataset: pipeline stage %r is neither a host loader %s nor a device stage %s"
                             % (kind, HOST_STAGES, DEVICE_STAGES))
    return host, device


def _drop_aos(r):
    lines = [ln for ln in r["result"].split("\n") if not ln.startswith("aos  AP:")]
    detail = {c: {k: v for k, v in d.items() if k != "aos"} for c, d in r["detail"].items()}
    return {"result": "\n".join(lines), "detail": detail}
