"""Generate tests/golden/kitti_prep_cases.npz by running the REFERENCE's own KITTI data preparation in place on the CPU.

    python tests/golden/make_kitti_prep_golden.py

Writes the crafted tree of tests/kitti_prep_cases.py into a temporary directory and runs, where they lie, the reference's
det3d/datasets/kitti/kitti_common.py (get_kitti_image_info, _calculate_num_points_in_gt, _create_reduced_point_cloud) and
det3d/datasets/utils/create_gt_database.py (create_groundtruth_database, driven by the reference's LoadPointCloudFromFile and
LoadPointCloudAnnotations of det3d/datasets/pipelines/loading.py), with numba and the ``sys.modules`` shims of make_augment_golden.py, a
`skimage.io` stub that returns the PNG's shape and a minimal stand-in for KittiDataset that builds the reference's `res` dict and runs the
two pipeline stages.  The info pickles are written as create_kitti_info_file writes them (its split files are read from the tree).

Stored: every file the reference wrote (key "file:<relative path>" -> its bytes as uint8), the reference's frustum and box planes
(surface_equ_3d_jitv2) per training / testing frame ("planes_frustum:<part>/<idx>", "planes_count:<idx>", "planes_db:<idx>"), and
the reference's points_in_rbbox masks of the database boxes ("mask_db:<idx>").  The angles of the crafted boxes are checked to have
np.sin / np.cos equal to math.sin / math.cos on this host.
"""
import importlib.util
import math
import os
import pickle
import sys
import tempfile
import types
from pathlib import Path

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
import kitti_prep_cases as cases  # noqa: E402


def _augment_golden():
    spec = importlib.util.spec_from_file_location("make_augment_golden", os.path.join(HERE, "make_augment_golden.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def load_reference():
    mag = _augment_golden()
    _, bnp = mag.load_reference()
    geom = sys.modules["det3d.core.bbox.geometry"]
    for p in ("det3d.datasets", "det3d.datasets.kitti", "det3d.datasets.utils", "det3d.datasets.pipelines"):
        mag._pkg(p)
    sys.modules["det3d.core"].box_np_ops = bnp

    def imread(path):
        with open(path, "rb") as f:
            head = f.read(24)
        assert head[:8] == b"\x89PNG\r\n\x1a\n" and head[12:16] == b"IHDR"
        return np.zeros((int.from_bytes(head[20:24], "big"), int.from_bytes(head[16:20], "big")), np.uint8)
    mag._stub("skimage", io=mag._stub("skimage.io", imread=imread))
    kc = mag._load("det3d.datasets.kitti.kitti_common", "det3d/datasets/kitti/kitti_common.py")
    sys.modules["det3d.datasets.kitti"].kitti_common = kc
    mag._stub("pycocotools", mask=mag._stub("pycocotools.mask"))
    mag._stub("det3d.torchie", Config=None)
    reg = types.SimpleNamespace(register_module=lambda c: c)
    mag._stub("det3d.datasets.registry", PIPELINES=reg)
    loading = mag._load("det3d.datasets.pipelines.loading", "det3d/datasets/pipelines/loading.py")

    class KittiStandIn:
        """the parts of the reference's KittiDataset create_groundtruth_database uses: len() and get_sensor_data -> the pipeline"""

        def __init__(self, info_path, root_path, test_mode, pipeline):
            with open(info_path, "rb") as f:
                self.infos = pickle.load(f)
            self.root = root_path
            self.stages = [loading.LoadPointCloudFromFile(**{k: v for k, v in pipeline[0].items() if k != "type"}),
                           loading.LoadPointCloudAnnotations(**{k: v for k, v in pipeline[1].items() if k != "type"})]

        def __len__(self):
            return len(self.infos)

        def get_sensor_data(self, idx):
            info = self.infos[idx]
            res = {"type": "KittiDataset", "lidar": {"type": "lidar", "points": None, "annotations": None},
                   "metadata": {"image_prefix": self.root, "num_point_features": 4, "image_idx": info["image"]["image_idx"],
                                "image_shape": info["image"]["image_shape"], "token": str(info["image"]["image_idx"])},
                   "calib": None, "cam": {"annotations": None}, "mode": "val"}
            for s in self.stages:
                res, info = s(res, info)
            return res
    mag._stub("det3d.datasets.dataset_factory", get_dataset=lambda name: KittiStandIn)
    cgd = mag._load("det3d.datasets.utils.create_gt_database", "det3d/datasets/utils/create_gt_database.py")
    return kc, cgd, bnp, geom


def main():
    kc, cgd, bnp, geom = load_reference()
    out = {}
    with tempfile.TemporaryDirectory() as root:
        splits = cases.write_tree(root)
        tr = kc.get_kitti_image_info(root, True, True, True, True, splits["train"], relative_path=True)
        kc._calculate_num_points_in_gt(root, tr, True)
        va = kc.get_kitti_image_info(root, True, True, True, True, splits["val"], relative_path=True)
        kc._calculate_num_points_in_gt(root, va, True)
        te = kc.get_kitti_image_info(root, False, False, True, True, splits["test"], relative_path=True)
        for name, obj in (("kitti_infos_train.pkl", tr), ("kitti_infos_val.pkl", va), ("kitti_infos_trainval.pkl", tr + va),
                          ("kitti_infos_test.pkl", te)):
            with open(os.path.join(root, name), "wb") as f:
                pickle.dump(obj, f)
        for part in ("training", "testing"):
            os.makedirs(os.path.join(root, part, "velodyne_reduced"))
        for name in ("train", "val", "test"):
            kc._create_reduced_point_cloud(root, os.path.join(root, "kitti_infos_%s.pkl" % name))
        cgd.create_groundtruth_database("KITTI", root, Path(root) / "kitti_infos_train.pkl", used_classes=cases.USED_CLASSES)
        for info in tr + va + te:
            part = "training" if "annos" in info else "testing"
            idx = info["image"]["image_idx"]
            cal = info["calib"]
            fr = bnp.get_valid_frustum(cal["R0_rect"], cal["Tr_velo_to_cam"], cal["P2"], info["image"]["image_shape"])
            n, d = geom.surface_equ_3d_jitv2(fr[:, :, :3, :])
            out["planes_frustum:%s/%d" % (part, idx)] = np.concatenate([n, d[..., None]], -1)[0]
            if part == "training":
                a = info["annos"]
                num = len([x for x in a["name"] if x != "DontCare"])
                cam = np.concatenate([a["location"][:num], a["dimensions"][:num], a["rotation_y"][:num, None]], axis=1)
                cb = bnp.box_camera_to_lidar(cam, cal["R0_rect"], cal["Tr_velo_to_cam"])
                out["planes_count:%d" % idx] = _ref_planes(bnp, geom, cb)
                r = cb[:, 6]
                assert (np.array_equal(np.sin(r), [math.sin(v) for v in r]) and np.array_equal(np.cos(r), [math.cos(v) for v in r])), \
                    "numpy's vector sin / cos differ from the correctly rounded values: pick other fixture angles"
        for info in tr:
            idx = info["image"]["image_idx"]
            a, cal = kc.remove_dontcare(info["annos"]), info["calib"]
            b = np.concatenate([a["location"], a["dimensions"], a["rotation_y"][:, None]], axis=1).astype(np.float32)
            b = bnp.box_camera_to_lidar(b, cal["R0_rect"], cal["Tr_velo_to_cam"])
            bnp.change_box3d_center_(b, [0.5, 0.5, 0], [0.5, 0.5, 0.5])
            out["planes_db:%d" % idx] = _ref_planes(bnp, geom, b)
            red = np.fromfile(os.path.join(root, "training", "velodyne_reduced", "%06d.bin" % idx), np.float32).reshape(-1, 4)
            out["mask_db:%d" % idx] = bnp.points_in_rbbox(red, b) if len(b) else np.zeros((len(red), 0), bool)
        for dp, _, files in os.walk(root):
            for fn in files:
                full = os.path.join(dp, fn)
                rel = os.path.relpath(full, root)
                if rel.split(os.sep)[0] in ("ImageSets",) or os.sep + "image_2" in full or os.sep + "velodyne" + os.sep in full:
                    continue
                if os.sep + "calib" + os.sep in full or os.sep + "label_2" + os.sep in full:
                    continue
                with open(full, "rb") as f:
                    out["file:" + rel.replace(os.sep, "/")] = np.frombuffer(f.read(), np.uint8)
    print("\n".join("%-50s %d" % (k, v.size) for k, v in sorted(out.items()) if k.startswith("file:")))
    np.savez_compressed(os.path.join(HERE, "kitti_prep_cases.npz"), **out)


def _ref_planes(bnp, geom, boxes):
    if len(boxes) == 0:
        return np.zeros((0, 6, 4))
    c = bnp.center_to_corner_box3d(boxes[:, :3], boxes[:, 3:6], boxes[:, -1], origin=(0.5, 0.5, 0.5), axis=2)
    n, d = geom.surface_equ_3d_jitv2(bnp.corner_to_surfaces_3d(c)[:, :, :3, :])
    return np.concatenate([n, d[..., None]], -1)


if __name__ == "__main__":
    main()
