"""The two pipeline transforms that sit on the per-frame hot path (reference: det3d/datasets/pipelines/preprocess.py:178-232 and
:235-358).  Transforms are ``(res, info) -> (res, info)``.  Dataset I/O and the reference's ``Preprocess`` are not registered here: the
per-object noise, global flip / rotation / scaling, shuffle and teacher twin run on the device through ``sessd_b200.augment`` (its own entry
point), GT-database sampling (GT-AUG) runs there too when ``build_train_batch`` is given a ``db_sampler`` (det3d.core.sampler), and
shape-aware augmentation (SA-DA) when it is given ``sa_da`` (sessd_b200.sada).  No ``Preprocess`` is registered: frame loading is not
mirrored, and a DataLoader worker cannot hold the CUDA context those stages need."""
import numpy as np

from det3d.builder import build_anchor_generator, build_box_coder, build_similarity_metric
from det3d.core.anchor.target_assigner import TargetAssigner
from det3d.core.bbox import box_np_ops
from det3d.core.input.voxel_generator import VoxelGenerator

from ..registry import PIPELINES


def _dict_select(dict_, inds):
    """reference preprocess.py:22-27"""
    for k, v in dict_.items():
        if isinstance(v, dict):
            _dict_select(v, inds)
        else:
            dict_[k] = v[inds]


def filter_gt_box_outside_range(gt_boxes, limit_range):
    """Mask of the GT boxes that have at least one BEV corner STRICTLY inside the rectangle limit_range = [x0, y0, x1, y1]
    (reference det3d/core/sampler/preprocess.py:138-148: center_to_corner_box2d + points_in_convex_polygon_jit, whose test
    `cross >= 0 -> outside` makes points on the boundary count as outside)."""
    gt_boxes = np.asarray(gt_boxes)
    if gt_boxes.shape[0] == 0:
        return np.zeros((0,), dtype=np.bool_)
    corners = box_np_ops.center_to_corner_box2d(gt_boxes[:, [0, 1]], gt_boxes[:, [3, 4]], gt_boxes[:, -1])      # [N, 4, 2]
    x0, y0, x1, y1 = [float(v) for v in limit_range]
    inside = (corners[..., 0] > x0) & (corners[..., 0] < x1) & (corners[..., 1] > y0) & (corners[..., 1] < y1)
    return inside.any(axis=1)


@PIPELINES.register_module
class Voxelization(object):
    def __init__(self, **kwargs):
        cfg = kwargs.get("cfg", None)
        self.range, self.voxel_size = cfg.range, cfg.voxel_size
        self.max_points_in_voxel, self.max_voxel_num = cfg.max_points_in_voxel, cfg.max_voxel_num
        self.far_points_first = cfg.get("far_points_first", False)
        self.voxel_generator = VoxelGenerator(point_cloud_range=self.range, voxel_size=self.voxel_size,
                                              max_num_points=self.max_points_in_voxel, max_voxels=self.max_voxel_num)

    def _pack(self, points):
        voxels, coordinates, num_points = self.voxel_generator.generate(points)
        return dict(voxels=voxels, coordinates=coordinates, num_points=num_points,
                    num_voxels=np.array([voxels.shape[0]], dtype=np.int64), shape=self.voxel_generator.grid_size)

    def __call__(self, res, info):
        if res.get("mode") == "train" and res.get("labeled", False):
            # reference :199-205: drop the GT boxes with no BEV corner inside the point-cloud range BEFORE target assignment
            gt = res["lidar"]["annotations"]
            pc_range = np.asarray(self.voxel_generator.point_cloud_range)
            _dict_select(gt, filter_gt_box_outside_range(gt["gt_boxes"], pc_range[[0, 1, 3, 4]]))
            res["lidar"]["annotations"] = gt
        res["lidar"]["voxels"] = self._pack(res["lidar"]["points"])
        if "points_raw" in res["lidar"]:                      # SE-SSD teacher branch: un-augmented copy (:218-230)
            res["lidar"]["voxels_raw"] = self._pack(res["lidar"]["points_raw"])
        return res, info


@PIPELINES.register_module
class AssignTarget(object):
    def __init__(self, **kwargs):
        cfg = kwargs["cfg"]
        ta_cfg = cfg.target_assigner
        self.tasks = ta_cfg.tasks
        generators = [build_anchor_generator(a) for a in ta_cfg.anchor_generators]
        self.target_class_names = [g.class_name for g in generators]
        self.enable_similar_type = cfg.get("enable_similar_type", False)
        self.target_class_ids = [1, 2] if self.enable_similar_type else [1]
        similarity = build_similarity_metric(ta_cfg.region_similarity_calculator)
        fraction = ta_cfg.sample_positive_fraction
        fraction = None if fraction < 0 else fraction
        self.target_assigners, start = [], 0
        for task in self.tasks:
            self.target_assigners.append(TargetAssigner(box_coder=build_box_coder(cfg.box_coder),
                                                        anchor_generators=generators[start:start + task.num_class],
                                                        region_similarity_calculator=similarity, positive_fraction=fraction,
                                                        sample_size=ta_cfg.sample_size))
            start += task.num_class
        self.out_size_factor = cfg.out_size_factor
        feature_map_size = [1, 200, 176]                          # hard-coded in the reference as well (:283)
        self.anchor_dicts_by_task = [a.generate_anchors_dict(feature_map_size) for a in self.target_assigners]

    def _assign(self, gt_dict):
        mask = np.zeros(gt_dict["gt_classes"].shape, dtype=np.bool_)
        for cid in self.target_class_ids:
            mask |= gt_dict["gt_classes"] == cid
        boxes = gt_dict["gt_boxes"][mask]
        boxes[:, -1] = box_np_ops.limit_period(boxes[:, -1], offset=0.5, period=np.pi * 2)
        gt_dict["gt_boxes"], gt_dict["gt_classes"], gt_dict["gt_names"] = [boxes], [gt_dict["gt_classes"][mask]], [gt_dict["gt_names"][mask]]
        out = {}
        for i, assigner in enumerate(self.target_assigners):
            out = assigner.assign_v2(self.anchor_dicts_by_task[i], gt_dict["gt_boxes"][i], anchors_mask=None,
                                     gt_classes=gt_dict["gt_classes"][i], gt_names=gt_dict["gt_names"][i],
                                     enable_similar_type=self.enable_similar_type)
        return {"labels": [out["labels"]], "reg_targets": [out["bbox_targets"]], "reg_weights": [out["bbox_outside_weights"]],
                "positive_gt_id": [out["positive_gt_id"]]}

    def __call__(self, res, info):
        anchors = [d[self.target_class_names[i]]["anchors"].reshape([-1, 7]) for i, d in enumerate(self.anchor_dicts_by_task)]
        targets, targets_raw = {"anchors": anchors}, {"anchors": list(anchors)}
        if res["mode"] == "train" and res.get("labeled", True):
            targets.update(self._assign(res["lidar"]["annotations"]))
            if "annotations_raw" in res["lidar"]:
                targets_raw.update(self._assign(res["lidar"]["annotations_raw"]))
        res["lidar"]["targets"], res["lidar"]["targets_raw"] = targets, targets_raw
        return res, info
