"""CPU: shape-aware augmentation (SA-DA).  The numpy restatement (tests/sada_ref.py) and the host draws of sessd_b200.sada against the
reference's own pyramid_augment_v0 run on crafted frames (tests/golden/sada_cases.npz, made by tests/golden/make_sada_golden.py)."""
import importlib.util
import os

import numpy as np
import pytest

import sada_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "sada_cases.npz")


def load():
    """tests/golden/make_sada_golden.py's ``load``: the stored cases, decoded"""
    spec = importlib.util.spec_from_file_location("make_sada_golden", os.path.join(ROOT, "tests", "golden", "make_sada_golden.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m.load(GOLDEN)


def stage_cfg(cfg):
    d, sp, sn, wp, wn = [None if np.isnan(v) else float(v) for v in cfg]
    return d, None if sp is None else (sp, int(sn)), None if wp is None else (wp, int(wn))


CASES = load()


@pytest.mark.parametrize("case", CASES, ids=[str(c["name"]) for c in CASES])
def test_pyramids_and_membership(case):
    pyr = sada_ref.pyramids(case["boxes"])
    assert np.array_equal(pyr, case["pyramids"])
    assert np.array_equal(sada_ref.in_pyramids(case["points"], pyr.reshape(-1, 15)), case["mask"])


@pytest.mark.parametrize("case", CASES, ids=[str(c["name"]) for c in CASES])
def test_stages_and_random_state(case):
    rs = np.random.RandomState(int(case["seed"]))
    out = sada_ref.sada(case["points"], case["boxes"], rs, *stage_cfg(case["cfg"]))
    for st in ("dropout", "sparsify", "swap"):
        assert out[st].dtype == np.float32
        assert np.array_equal(out[st], case[st]), st
    _, key, pos = rs.get_state()[:3]
    assert np.array_equal(key, case["state_key"]) and pos == int(case["state_pos"])


def test_cases_cover_the_crafted_conditions():
    by = {str(c["name"]): c for c in CASES}
    assert len(by["no_points"]["swap"]) == 0 and len(by["no_boxes"]["boxes"]) == 0
    b = by["boundary"]["mask"].sum(0).reshape(-1, 6)
    assert (b[0] == 50).all() and (b[1] == 51).all() and len(by["boundary"]["sparsify"]) == len(by["boundary"]["points"]) - 1
    assert (by["overlap"]["mask"].sum(1) > 1).any()
    assert len(by["self_swap"]["swap"]) > len(by["self_swap"]["points"])          # the self partner duplicates points
    assert len(np.unique(by["constant_intensity"]["points"][:, 3])) == 1
    s = by["sparsify_and_swap"]
    assert len(s["sparsify"]) != len(s["dropout"]) and not np.array_equal(s["swap"], s["sparsify"])


def test_fps_contract_ties_go_to_the_lowest_row():
    x = np.array([[0, 0, 0], [1, 0, 0], [-1, 0, 0], [1, 0, 0], [0, 2, 0]], np.float32)
    assert sada_ref.fps(x, 4).tolist() == [0, 4, 1, 2]


def test_rejects_other_widths():
    with pytest.raises(ValueError):
        sada_ref.sada(np.zeros((3, 5), np.float32), np.zeros((0, 7), np.float32), np.random.RandomState(0))


def test_chain_without_sada_is_the_existing_preprocess_frame():
    """the chained oracle with sa_da off draws and computes what draw_augmentation + augment_ref.augment_frame do"""
    from oracle import augment_ref
    from sessd_b200 import augment
    from test_augment_oracle import reference_config
    acfg = augment.AugmentConfig.from_config(reference_config())
    rs = np.random.RandomState(4)
    pts = np.concatenate([rs.uniform([0, -40, -3, 0], [70, 40, 1, 1], (3000, 4))]).astype(np.float32)
    boxes = np.stack([[10 + 8 * i, -5 + 3 * i, -1, 1.6, 3.9, 1.5, 0.3 * i] for i in range(5)]).astype(np.float32)
    names = np.array(["Car", "Van", "Car", "Pedestrian", "Car"])
    rs1, rs2 = np.random.RandomState(8), np.random.RandomState(8)
    chained = [sada_ref.preprocess_frame(pts, boxes, names, rs1, acfg, None) for _ in range(2)]
    draws = augment.draw_augmentation(rs2, [(len(pts), len(boxes), True)] * 2, acfg)
    for c, f in zip(chained, draws.frames):
        o = augment_ref.augment_frame(pts, boxes, np.array([n in acfg.class_names for n in names]),
                                      dict(loc=f.loc, rot=f.rot, flip=f.flip, rotation=f.rotation, scale=f.scale, perm=f.perm))
        assert np.array_equal(c["points"], o["points"]) and np.array_equal(c["points_raw"], o["points_raw"])
        assert np.array_equal(c["boxes"], o["boxes"]) and np.array_equal(c["draws"].perm, f.perm)
    assert np.array_equal(rs1.get_state()[1], rs2.get_state()[1]) and rs1.get_state()[2] == rs2.get_state()[2]
