"""CPU: the numpy restatement of the training augmentation (oracle/augment_ref.py) against the reference's own functions
(tests/golden/augment_cases.npz, made by tests/golden/make_augment_golden.py), and the host draws of sessd_b200.augment against the draws
the reference functions make on the same seed."""
import json
import os

import numpy as np
import pytest

from oracle import augment_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "augment_cases.npz")


def load_frames():
    z = np.load(GOLDEN)
    frames = []
    for f in range(int(z["num_frames"])):
        pre = "f%d_" % f
        d = {k[len(pre):]: z[k] for k in z.files if k.startswith(pre)}
        d["draws"] = dict(loc=d["loc"], rot=d["rot"], flip=bool(d["flip"]), rotation=float(d["rotation"]), scale=float(d["scale"]),
                          perm=d["perm"])
        frames.append(d)
    return z, frames


def reference_config():
    """the upstream config's values (tests/golden/reference_config.json); its two constructed objects (the neck's logger, the head's box
    coder) are not data and are taken from the repo's config, as test_compat does"""
    from det3d.torchie import Config
    d = json.load(open(os.path.join(ROOT, "tests", "golden", "reference_config.json")))
    ours = Config.fromfile(os.path.join(ROOT, "examples", "second", "configs", "config.py"))
    d["model"]["neck"]["logger"] = ours.model.neck.logger
    d["model"]["bbox_head"]["box_coder"] = ours.model.bbox_head.box_coder
    return Config(d)


def test_collision_matrix_matches_reference():
    z, _ = load_frames()
    got = augment_ref.collision_matrix(z["coll_boxes"], z["coll_qboxes"])
    assert np.array_equal(got, z["coll_ref"])
    # the crafted pairs on the diagonal: identical boxes and overlaps with only collinear edges do not collide in the reference
    assert list(np.diag(z["coll_ref"])[:12]) == [False, True, True, False, False, False, True, False, True, True, False, False]


@pytest.mark.parametrize("frame", range(7))
def test_frame_stages_match_reference(frame):
    _, frames = load_frames()
    d = frames[frame]
    got = augment_ref.augment_frame(d["in_points"], d["in_boxes"], d["valid"], d["draws"], float(d["context"]), bool(d["labeled"]))
    keys = ["points"] + (["selected", "masks", "points_raw", "boxes_raw", "boxes"] if d["labeled"] else [])
    for k in keys:
        assert got[k].dtype == d[k].dtype and np.array_equal(got[k], d[k]), (str(d["name"]), k)


def test_crafted_frames_reach_the_cases_they_are_for():
    _, frames = load_frames()
    by = {str(d["name"]): d for d in frames}
    sel = by["chain"]["selected"]
    assert list(sel) == [0, 1, -1, -1, 0, 0]        # box 1 skips the try that only box 0's NEW place blocks; 2 invalid; 3 always collides
    assert (by["crowded"]["selected"] == -1).sum() >= 3
    masks, valid = by["chain"]["masks"], by["chain"]["valid"]
    assert (masks[:, 4] & masks[:, 5]).any() and (masks[:, 2] & masks[:, 3]).any() and not valid[2]
    assert {bool(d["flip"]) for d in frames if d["labeled"] and len(d["in_points"])} == {False, True}
    assert not by["unlabelled"]["labeled"] and len(by["empty"]["in_points"]) == 0 and len(by["no_boxes"]["in_boxes"]) == 0


def test_config_drives_the_augmentation():
    from sessd_b200.augment import AugmentConfig
    cfg = reference_config()
    a = AugmentConfig.from_config(cfg)
    assert a.class_names == ("Car", "Van") and list(cfg.train_preprocessor.class_names) == ["Car"]      # the config's list is not mutated
    assert a.gt_loc_noise == (1.0, 1.0, 0.5) and a.gt_rot_noise == (-0.785, 0.785) and a.global_rot_noise == (-0.785, 0.785)
    assert a.global_scale_noise == (0.95, 1.05) and a.data_aug_with_context == -1.0 and a.shuffle_points
    assert a.target_class_ids == (1, 2) and a.range_bev == (0.0, -40.0, 70.4, 40.0)


def test_draws_follow_the_reference_call_order():
    """draw_augmentation on RandomState(seed) hands out, value for value, what the reference's np.random calls drew on that seed"""
    from sessd_b200.augment import AugmentConfig, draw_augmentation
    a = AugmentConfig.from_config(reference_config())
    _, frames = load_frames()
    seeded = [d for d in frames if int(d["seed"]) >= 0]
    assert len(seeded) >= 5 and any(not d["labeled"] for d in seeded)
    for d in seeded:
        got = draw_augmentation(np.random.RandomState(int(d["seed"])), [(len(d["in_points"]), len(d["in_boxes"]), bool(d["labeled"]))], a)
        g = got.frames[0]
        if d["labeled"]:
            assert np.array_equal(g.loc, d["loc"]) and np.array_equal(g.rot, d["rot"])
        assert g.flip == bool(d["flip"]) and g.rotation == float(d["rotation"]) and g.scale == float(d["scale"])
        assert np.array_equal(g.perm, d["perm"])
        assert got.transformation() == [dict(flipped=g.flip, noise_rotation=g.rotation, noise_scale=g.scale)]


def test_exact_fma_helpers():
    rs = np.random.RandomState(0)
    a, b, c = (rs.randn(2000) * 3).astype(np.float32), rs.randn(2000).astype(np.float32), rs.randn(2000).astype(np.float32)
    from fractions import Fraction
    want = np.array([np.float32(float(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(w)))) for x, y, w in zip(a, b, c)])
    assert np.array_equal(augment_ref.fma32(a, b, c), want)
    a64, b64, c64 = rs.randn(50), rs.randn(50), rs.randn(50)
    assert np.array_equal(augment_ref.fma64(a64, b64, c64),
                          [float(Fraction(x) * Fraction(y) + Fraction(w)) for x, y, w in zip(a64, b64, c64)])
