"""DI-NMS oracle (oracle/dinms_ref.py) against the reference's own rotate_weighted_nms, run in place by
tests/golden/make_dinms_golden.py on the crafted cases of tests/dinms_cases.py."""
import os

import numpy as np
import pytest

import dinms_cases as dc
import post_model as pm

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "dinms_cases.npz"))
NAMES = [str(n) for n in GOLD["names"]]


def stored_case(name):
    keys = ("boxes7", "scores", "iou_preds", "labels", "dirs", "anchors", "pre_max")
    c = {k: GOLD["%s__in_%s" % (name, k)] for k in keys}
    c["pre_max"] = int(c["pre_max"])
    return c


def test_fixture_covers_the_crafted_cases():
    assert NAMES == list(dc.cases().keys())
    for name in NAMES:
        c, _ = dc.cases()[name]
        s = stored_case(name)
        for k in ("boxes7", "scores", "iou_preds", "labels", "dirs", "anchors"):
            assert np.array_equal(np.asarray(c[k]), s[k]), (name, k)


@pytest.mark.parametrize("name", NAMES)
def test_oracle_reproduces_reference(name):
    c = stored_case(name)
    got = dc.run_oracle(c)
    sel = GOLD[name + "__selected"]
    assert np.array_equal(got["selected"], sel)
    assert np.array_equal(got["keep"], GOLD[name + "__keep"])
    assert np.array_equal(got["labels"], GOLD[name + "__labels"])
    assert np.array_equal(got["dirs"], GOLD[name + "__dirs"])
    assert np.array_equal(got["scores"].astype(np.float64), GOLD[name + "__scores"])
    np.testing.assert_array_equal(got["boxes"].astype(np.float64), GOLD[name + "__boxes"])     # NaN where the reference has NaN
    adj = GOLD[name + "__adjusted"]
    if len(c["scores"]):
        np.testing.assert_allclose(got["adjusted"], adj, rtol=1e-6, atol=0)


def test_cases_reach_their_rules():
    by = {n: dc.run_oracle(stored_case(n)) for n in NAMES}
    picks = {n: by[n]["extra"]["picks"] for n in NAMES}
    assert [k for _, _, _, k in picks["recover"]] == [False, True]                 # recovered, then a cluster of its own
    assert picks["recover"][1][0] != 0 and by["recover"]["scores"][0] == by["recover"]["adjusted"].max()   # score_box from the failed pick
    assert [round(d, 6) for _, _, d, _ in picks["bands"]][1] == 20.0
    nan = np.isnan(by["bands"]["boxes"]).any(1)
    assert nan.tolist() == [False, False, False, False, True]                       # the pick at 65 m
    assert len(picks["exact_thresh_pair"]) == 1 and len(by["exact_thresh_pair"]["keep"]) == 1
    assert len(by["single"]["keep"]) == 0 and len(by["empty"]["keep"]) == 0
    assert len(set(by["labels"]["labels"].tolist())) >= 1 and len(picks["labels"]) > 2
    a = by["equal_scores"]["adjusted"]
    assert a[0] == a[1]                                                             # the two picks tie; the first position wins
    assert by["equal_scores"]["keep"].tolist()[:2] == [0, 1]
    assert len(stored_case("pre_max_cut")["scores"]) > stored_case("pre_max_cut")["pre_max"]


def test_exact_threshold_pair_is_fl_point3():
    c = stored_case("exact_thresh_pair")
    m = dc.iou_of_boxes7(c["boxes7"])
    assert np.float32(m[0, 3]) == np.float32(0.3)
    # a member would move the average: B's box (x 11.5) is not in it
    box = dc.run_oracle(c)["boxes"][0]
    assert abs(box[0] - 10.0) < 1e-3


@pytest.mark.parametrize("name", [n for n in NAMES if n.startswith("scene") or n in ("dense_cluster", "bands", "labels")])
def test_oracle_ious_match_the_reference_clip(name):
    """the fp64 IoUs against the reference's iou3d CPU twin (oracle.cpu.boxes_iou_bev, fp32) on the pairs away from touching"""
    from oracle import cpu as ocpu
    b7 = stored_case(name)["boxes7"]
    det5 = b7[:, [0, 1, 3, 4, 6]]
    bev = pm.bev_of(det5)
    ours = dc.iou_matrix(det5)
    ref = ocpu.boxes_iou_bev(bev, bev)
    ious = pm.pair_ious(det5)
    checked = 0
    for (i, j), v in ious.items():
        if v > 0 and pm.clear_of_boundaries(bev[i], bev[j]):
            assert abs(ref[i, j] - ours[i, j]) <= 1e-5 * max(ours[i, j], 1e-3) + 1e-6, (i, j, ref[i, j], ours[i, j])
            checked += 1
    assert checked > 0
