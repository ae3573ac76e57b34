"""GT-database sampling (GT-AUG), under the reference's names (det3d/core/sampler/sample_ops_v2.py): ``DataBaseSamplerV2``.

Selection -- which database objects a frame takes -- runs on the host, draw for draw as the reference: one ``BatchSampler`` per class in
the infos' dict order (each shuffles at construction), ``sample_all``'s count ``round(rate * (max_num - #gt named exactly like the
group))``, at most two rounds, and ``sample_class_v2``'s acceptance over the BEV corners of ``center_to_corner_box2d`` with the collision
predicate of the device kernels (``sessd_gtaug_select_host``).  ``select`` returns the accepted database ids; ``sample_all`` returns the
reference's dict.  The database is owned by the sampler: ``load_database`` reads every filtered object's file once into one host array
(and, on demand, one device buffer with a single host-to-device copy); later frames read no files.

Dtypes, as the reference has them: box3d_lidar rows are float64 (box_camera_to_lidar of the fp32 labels through fp64 matrices,
create_gt_database.py:60-110), so the sampled boxes, the offset-added dims (a Python list: numpy promotes to float64) and every corner are
float64; a frame's own boxes keep the dtype they come in (their corners are computed in it and promoted when concatenated).  Object points
are fp32; ``s_points[:, :3] += box3d_lidar[:3]`` rounds fp32(double(rel) + centre).
"""
import os

import numpy as np

from . import preprocess as prep


def _corners_2d(centers, dims, angles):
    """center_to_corner_box2d (box_np_ops.py:512-532) with its own operations: corners_nd(origin 0.5) in dims' dtype, rotation_2d's
    einsum, then the centres added in place"""
    norm = np.stack(np.unravel_index(np.arange(4), [2, 2]), axis=1).astype(dims.dtype)[[0, 1, 3, 2]]
    norm = norm - np.array(0.5, dtype=dims.dtype)
    corners = dims.reshape([-1, 1, 2]) * norm.reshape([1, 4, 2])
    s, c = np.sin(angles), np.cos(angles)
    corners = np.einsum("aij,jka->aik", corners, np.stack([[c, -s], [s, c]]))
    corners += centers.reshape([-1, 1, 2])
    return corners


class DataBaseSamplerV2:
    def __init__(self, db_infos, groups, db_prepor=None, rate=1.0, global_rot_range=None, logger=None, gt_random_drop=-1.0,
                 gt_aug_with_context=-1.0, gt_aug_similar_type=False, random_state=np.random):
        if gt_random_drop > 0:
            raise NotImplementedError("gt_random_drop > 0 is not supported (the SE-SSD car config does not use it)")
        if gt_aug_with_context > 0:
            raise NotImplementedError("gt_aug_with_context > 0 is not supported (the SE-SSD car config does not use it)")
        if db_prepor is not None:
            db_infos = db_prepor(db_infos)
        self.db_infos = db_infos
        self._rate = rate
        self._groups = groups
        self._rs = random_state
        self.gt_point_random_drop = gt_random_drop
        self.gt_aug_with_context = gt_aug_with_context
        self._sample_classes, self._sample_max_nums = [], []
        for group_info in groups:
            self._sample_classes += list(group_info.keys())
            self._sample_max_nums += list(group_info.values())
        # global object ids: the filtered infos of every class, in dict order
        self._infos = [info for v in db_infos.values() for info in v]
        gid = {id(info): i for i, info in enumerate(self._infos)}
        self._sampler_dict, self._sampler_ids = {}, {}
        for k, v in db_infos.items():
            self._sampler_dict[k] = prep.BatchSampler(v, k, random_state=random_state)
        if gt_aug_similar_type:
            self._sampler_dict["Car"] = prep.BatchSampler(db_infos["Car"] + db_infos["Van"], "Car", random_state=random_state)
        for k, s in self._sampler_dict.items():
            self._sampler_ids[k] = np.array([gid[id(info)] for info in s._sampled_list], np.int64)
        self.boxes = (np.stack([np.asarray(i["box3d_lidar"]) for i in self._infos]) if self._infos else np.zeros((0, 7)))
        self.names = np.array([i["name"] for i in self._infos])
        self.root_path = None
        self._points = None
        self._device = {}

    def _set_random_state(self, rs):
        """the RandomState every class stream draws from"""
        self._rs = rs
        for s in self._sampler_dict.values():
            s._rs = rs

    # ------------------------------------------------------------------------------------------------ the resident database
    def load_database(self, root_path=None, num_point_features=4):
        """read every object's file once: points [P_db, F] f32 relative to the centre, offset / count per object"""
        if self._points is not None:
            return
        root = root_path if root_path is not None else self.root_path
        if root is None:
            raise ValueError("DataBaseSamplerV2: no root path for the database files")
        parts = [np.fromfile(os.path.join(str(root), i["path"]), dtype=np.float32).reshape(-1, num_point_features) for i in self._infos]
        self.counts = np.array([len(p) for p in parts], np.int64)
        self.offsets = np.concatenate([[0], np.cumsum(self.counts)[:-1]]).astype(np.int64) if parts else np.zeros(0, np.int64)
        self._points = np.concatenate(parts + [np.zeros((0, num_point_features), np.float32)])

    def device_database(self, device="cuda"):
        """the database on the device (one host-to-device copy): dict(points [P_db, 4] f32, off / count [N] i32, boxes [N, 7] f64)"""
        import torch
        key = str(device)
        if key not in self._device:
            self.load_database()
            if self._points.shape[1] != 4:
                raise ValueError("the device database holds 4-feature points")
            if len(self._points) >= 2 ** 31:
                raise ValueError("the database has too many points for int32 offsets")
            from sessd_b200.augment import _pack, _unpack
            buf, layout = _pack([self._points, self.offsets.astype(np.int32), self.counts.astype(np.int32),
                                 self.boxes.astype(np.float64)])
            dev = torch.from_numpy(buf).to(device)
            pts, off, cnt, bx = _unpack(dev, layout)
            self._device[key] = dict(points=pts, off=off, count=cnt, boxes=bx)
        return self._device[key]

    # ------------------------------------------------------------------------------------------------ selection
    def sample_class_v2(self, name, num, gt_boxes):
        """reference :238-276, returning the accepted global ids in sampler order"""
        from sessd_b200 import ops
        ids = self._sampler_ids[name][self._sampler_dict[name]._sample(num)]
        sp_boxes = self.boxes[ids]
        num_gt = gt_boxes.shape[0]
        boxes = np.concatenate([gt_boxes, sp_boxes], axis=0).copy()
        sp_new = boxes[num_gt:]
        gt_bv = _corners_2d(gt_boxes[:, 0:2], gt_boxes[:, 3:5], gt_boxes[:, -1])
        sp_bv = _corners_2d(sp_new[:, 0:2], sp_new[:, 3:5] + [0.0, 0.0], sp_new[:, -1])
        total = np.concatenate([gt_bv, sp_bv], axis=0)
        return ids[ops.gtaug_select_host(total, num_gt)]

    def select(self, gt_boxes, gt_names):
        """sample_all's selection (reference :67-108): the accepted global ids of one frame, in acceptance order"""
        gt_boxes = np.asarray(gt_boxes)
        nums = []
        for class_name, max_num in zip(self._sample_classes, self._sample_max_nums):
            n = int(max_num - np.sum([n == class_name for n in gt_names]))
            nums.append(np.round(self._rate * n).astype(np.int64))
        out, all_gt = [], gt_boxes
        for class_name, sampled_num in zip(self._sample_classes, nums):
            times = 0
            while sampled_num > 0 and times < 2:
                acc = self.sample_class_v2(class_name, sampled_num, all_gt)
                out.append(acc)
                if len(acc) > 0:
                    all_gt = np.concatenate([all_gt, self.boxes[acc]], axis=0)
                sampled_num -= len(acc)
                times += 1
        return np.concatenate(out + [np.zeros(0, np.int64)]).astype(np.int64)

    def sample_all(self, root_path, gt_boxes, gt_names, num_point_features, random_crop=False, gt_group_ids=None, calib=None,
                   targeted_class_names=None, with_road_plane_cam=None):
        """reference :67-192: dict(gt_names, difficulty, gt_boxes, points, gt_masks, group_ids) in numpy, or None when nothing is
        accepted"""
        if random_crop:
            raise NotImplementedError("random_crop is not supported (the SE-SSD car config does not use it)")
        if with_road_plane_cam is not None:
            raise NotImplementedError("with_road_plane_cam is not supported (the SE-SSD car config does not use it)")
        self.load_database(root_path, num_point_features)
        ids = self.select(gt_boxes, gt_names)
        if len(ids) == 0:
            return None
        pts = []
        for i in ids:
            s = self._points[self.offsets[i]:self.offsets[i] + self.counts[i]].copy()
            s[:, :3] += self.boxes[i][:3]
            pts.append(s)
        n_gt = np.asarray(gt_boxes).shape[0]
        return {"gt_names": self.names[ids], "difficulty": np.array([self._infos[i]["difficulty"] for i in ids]),
                "gt_boxes": self.boxes[ids], "points": np.concatenate(pts, axis=0), "gt_masks": np.ones((len(ids),), dtype=np.bool_),
                "group_ids": np.arange(n_gt, n_gt + len(ids))}
