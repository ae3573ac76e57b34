"""KITTI data preparation on the CPU: the host parsing and planes of sessd_b200.kitti_prep and the numpy oracle against the reference's
outputs on the crafted tree (tests/golden/kitti_prep_cases.npz, from tests/golden/make_kitti_prep_golden.py)."""
import io
import os
import pickle

import numpy as np
import pytest

import kitti_prep_cases as cases
from oracle import kitti_prep_ref as ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kitti_prep_cases.npz")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = tmp_path_factory.mktemp("kitti")
    cases.write_tree(str(root))
    return root


def _pkl(g, name):
    return pickle.load(io.BytesIO(g["file:" + name].tobytes()))


def assert_same(a, b, path="info"):
    """equal keys (in order), types, dtypes and values"""
    assert type(a) is type(b), (path, type(a), type(b))
    if isinstance(a, dict):
        assert list(a.keys()) == list(b.keys()), path
        for k in a:
            assert_same(a[k], b[k], "%s.%s" % (path, k))
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            assert_same(x, y, "%s[%d]" % (path, i))
    elif isinstance(a, np.ndarray):
        assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b), path
    else:
        assert a == b, path
        if isinstance(a, np.generic):
            assert a.dtype == b.dtype, path


def test_label_calib_png_and_difficulty_parsing(golden, tree):
    from sessd_b200 import kitti_prep
    for split, training in (("train", True), ("val", True), ("test", False)):
        want = _pkl(golden, "kitti_infos_%s.pkl" % split)
        for w in want:
            got = kitti_prep.image_info(str(tree), w["image"]["image_idx"], training, training, True, True)
            if training:
                got["annos"]["num_points_in_gt"] = w["annos"]["num_points_in_gt"]
            assert_same(got, w)
    with pytest.raises(ValueError):
        kitti_prep.png_shape(str(tree / "training" / "calib" / "000000.txt"))
    with pytest.raises(FileNotFoundError, match="train.txt"):
        kitti_prep.imageset_ids(str(tree / "nowhere"), "train")


def test_difficulty_boundaries_reached(golden):
    d = _pkl(golden, "kitti_infos_train.pkl")[0]["annos"]["difficulty"]
    assert set(d.tolist()) >= {0, 1, 2, -1}


def test_host_planes_equal_the_reference(golden):
    from sessd_b200 import kitti_prep
    for split in ("train", "val", "test"):
        for info in _pkl(golden, "kitti_infos_%s.pkl" % split):
            part = "training" if "annos" in info else "testing"
            idx = info["image"]["image_idx"]
            c = info["calib"]
            fr = kitti_prep.frustum_planes(c["R0_rect"], c["Tr_velo_to_cam"], c["P2"], info["image"]["image_shape"])
            assert np.array_equal(fr, golden["planes_frustum:%s/%d" % (part, idx)])
            if part == "training":
                assert np.array_equal(kitti_prep.box_planes(kitti_prep.info_boxes(info)), golden["planes_count:%d" % idx])
                if split == "train":
                    assert np.array_equal(kitti_prep.box_planes(kitti_prep.db_boxes(info)[0]), golden["planes_db:%d" % idx])


def test_oracle_reproduces_every_output(golden, tree):
    db = _pkl(golden, "dbinfos_train.pkl")
    seen = {"zero": False, "shared": False}
    for split in ("train", "val", "test"):
        for info in _pkl(golden, "kitti_infos_%s.pkl" % split):
            part = "training" if "annos" in info else "testing"
            idx = info["image"]["image_idx"]
            raw = np.fromfile(str(tree / info["point_cloud"]["velodyne_path"]), np.float32).reshape(-1, 4)
            c = info["calib"]
            red = ref.reduce_frame(raw, c["R0_rect"], c["Tr_velo_to_cam"], c["P2"], info["image"]["image_shape"])
            assert red.tobytes() == golden["file:%s/velodyne_reduced/%06d.bin" % (part, idx)].tobytes()
            assert np.array_equal(ref.frustum_planes(c["R0_rect"], c["Tr_velo_to_cam"], c["P2"], info["image"]["image_shape"]),
                                  golden["planes_frustum:%s/%d" % (part, idx)])
            if part == "testing":
                continue
            assert_same(ref.num_points_in_gt(red, info), info["annos"]["num_points_in_gt"])
            if split != "train":
                continue
            boxes = ref.db_boxes(info)[0]
            assert np.array_equal(ref.inside(red, ref.box_planes(boxes)), golden["mask_db:%d" % idx])
            m = golden["mask_db:%d" % idx]
            seen["shared"] |= bool((m.sum(1) > 1).any())
            for i, (name, rows, n, box, diff) in enumerate(ref.db_objects(red, info)):
                key = "file:gt_database/%d_%s_%d.bin" % (idx, name, i)
                assert rows.tobytes() == golden[key].tobytes(), key
                seen["zero"] |= n == 0
                if name in cases.USED_CLASSES:
                    e = [x for x in db[name] if x["image_idx"] == idx and x["gt_idx"] == i][0]
                    assert e["num_points_in_gt"] == n and np.array_equal(e["box3d_lidar"], box) and e["difficulty"] == diff
    assert all(seen.values()), seen
