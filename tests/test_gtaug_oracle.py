"""CPU: GT-database sampling.  The numpy restatement (oracle/gt_aug_ref.py) and the det3d.core.sampler mirror against the reference's own
DataBaseSamplerV2 run on a crafted database (tests/golden/gtaug_cases.npz, made by tests/golden/make_gtaug_golden.py), and
build_dbsampler on the unchanged reference config."""
import copy
import importlib.util
import os
import pickle

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "gtaug_cases.npz")


def load():
    return dict(np.load(GOLDEN))


def _golden():
    """tests/golden/make_gtaug_golden.py as a module (its oracle check and the database layout)"""
    spec = importlib.util.spec_from_file_location("make_gtaug_golden", os.path.join(ROOT, "tests", "golden", "make_gtaug_golden.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def db_infos_from(z):
    return _golden().db_infos_from(z)


def check_oracle(z):
    return _golden().check_oracle(z)


def write_database(z, root):
    """the stored database laid out as create_gt_database writes it: dbinfos pickle + one .bin per object"""
    infos = db_infos_from(z)
    os.makedirs(os.path.join(root, "gt_database"), exist_ok=True)
    for v in infos.values():
        for i in v:
            k = i["image_idx"]
            z["db_rel_points"][z["db_off"][k]:z["db_off"][k] + z["db_count"][k]].tofile(os.path.join(root, i["path"]))
    path = os.path.join(root, "dbinfos_train.pkl")
    with open(path, "wb") as f:
        pickle.dump(infos, f)
    return path, infos


def rest_of_frame(rs, z, pre):
    """the frame's draws after GT-AUG (noise, global, shuffle), so the next frame's reshuffles see the reference's stream"""
    m, n = len(z[pre + "gt_boxes"]), len(z[pre + "points_pasted"])
    rs.normal(scale=np.array([1.0, 1.0, 0.5], np.float32), size=[m, 100, 3]); rs.uniform(-0.785, 0.785, size=[m, 100])
    rs.choice([False, True], replace=False, p=[0.5, 0.5]); rs.uniform(-0.785, 0.785); rs.uniform(0.95, 1.05)
    rs.choice(np.arange(n), n, replace=False)


def mirror_sampler(z, infos, rs):
    from det3d.core.sampler import DataBasePreprocessor, DataBaseSamplerV2, DBFilterByDifficulty, DBFilterByMinNumPoint
    prepor = DataBasePreprocessor([DBFilterByMinNumPoint({"Car": int(z["min_points"])}), DBFilterByDifficulty([-1])])
    return DataBaseSamplerV2(copy.deepcopy(infos), [dict(Car=int(z["max_num"]))], prepor, 1.0, [0, 0],
                             gt_aug_similar_type=bool(z["similar"]), random_state=rs)


def test_oracle_reproduces_the_reference_fixture():
    check_oracle(load())                          # every stored stage, bit for bit, and every crafted case reached


def test_mirror_sampler_indices_and_sample_all_match_the_reference(tmp_path):
    z = load()
    _, infos = write_database(z, str(tmp_path))
    rs = np.random.RandomState(int(z["seed"]))
    s = mirror_sampler(z, infos, rs)
    for f in range(int(z["num_frames"])):
        pre = "f%d_" % f
        bx, names = z[pre + "in_boxes"], list(z[pre + "in_names"])
        ret = s.sample_all(str(tmp_path), bx, names, 4)
        rest_of_frame(rs, z, pre)
        ids = z[pre + "ids"]
        if len(ids) == 0:
            assert ret is None
            continue
        n = sum(int(z["db_count"][i]) for i in ids)
        assert np.array_equal(ret["gt_boxes"], z[pre + "gt_boxes"][len(bx):]) and ret["gt_boxes"].dtype == np.float64
        assert list(ret["gt_names"]) == list(z[pre + "gt_names"][len(bx):])
        assert np.array_equal(ret["points"], z[pre + "points_pasted"][:n])
        assert ret["gt_masks"].all() and list(ret["group_ids"]) == list(range(len(bx), len(bx) + len(ids)))


def test_mirror_select_returns_the_reference_ids_with_resets():
    z = load()
    s = mirror_sampler(z, db_infos_from(z), np.random.RandomState(int(z["seed"])))
    fid = np.array([i["image_idx"] for i in s._infos])
    rs = s._rs
    for f in range(int(z["num_frames"])):
        pre = "f%d_" % f
        assert np.array_equal(fid[s.select(z[pre + "in_boxes"], list(z[pre + "in_names"]))], z[pre + "ids"]), f
        rest_of_frame(rs, z, pre)


def test_host_draws_follow_the_reference_stream():
    """the builder's host order -- per frame, the sampler's draws, then draw_augmentation sized by the pasted frame -- against the draws
    the reference made on the same seed (the pasted sizes taken from the fixture)"""
    z = load()
    from sessd_b200.augment import AugmentConfig, draw_augmentation
    rs = np.random.RandomState(int(z["seed"]))
    s = mirror_sampler(z, db_infos_from(z), rs)
    cfg = AugmentConfig()
    for f in range(int(z["num_frames"])):
        pre = "f%d_" % f
        s.select(z[pre + "in_boxes"], list(z[pre + "in_names"]))
        d = draw_augmentation(rs, [(len(z[pre + "points_pasted"]), len(z[pre + "gt_boxes"]), True)], cfg).frames[0]
        assert np.array_equal(d.loc, z[pre + "loc"]) and np.array_equal(d.rot, z[pre + "rot"])
        assert (d.flip, d.rotation, d.scale) == (bool(z[pre + "flip"]), float(z[pre + "rotation"]), float(z[pre + "scale"]))
        assert np.array_equal(d.perm, z[pre + "perm"])


def test_build_dbsampler_reads_the_reference_config(tmp_path):
    from test_augment_oracle import reference_config
    from det3d.builder import build_dbsampler
    z = load()
    path, _ = write_database(z, str(tmp_path))
    cfg = reference_config().db_sampler
    cfg.db_info_path = path
    s = build_dbsampler(cfg, random_state=np.random.RandomState(0))
    assert s._sample_classes == ["Car"] and s._sample_max_nums == [15] and s._rate == 1.0
    kept = [i for i in s.db_infos["Car"]]
    assert all(i["num_points_in_gt"] >= 5 and i["difficulty"] != -1 for i in kept)
    assert len(kept) == int(((z["db_names"] == "Car") & (z["db_num_points_in_gt"] >= 5) & (z["db_difficulty"] != -1)).sum())
    assert set(s._sampler_dict) == {"Car", "Pedestrian", "Van", "Cyclist"}       # no similar type in the car config
    s.load_database()                                                              # the files beside the pickle
    assert s._points.shape == (int(z["db_count"][[i["image_idx"] for i in s._infos]].sum()), 4)


@pytest.mark.parametrize("key", ["gt_random_drop", "gt_aug_with_context"])
def test_unused_options_raise(key):
    from det3d.core.sampler import DataBaseSamplerV2
    with pytest.raises(NotImplementedError):
        DataBaseSamplerV2({"Car": []}, [dict(Car=15)], **{key: 0.5})


def test_sample_all_rejects_unsupported_arguments():
    from det3d.core.sampler import DataBaseSamplerV2
    s = DataBaseSamplerV2({"Car": []}, [dict(Car=15)], random_state=np.random.RandomState(0))
    with pytest.raises(NotImplementedError):
        s.sample_all("/", np.zeros((0, 7)), [], 4, random_crop=True)
    with pytest.raises(NotImplementedError):
        s.sample_all("/", np.zeros((0, 7)), [], 4, with_road_plane_cam=(0, 1, 0, 1))
