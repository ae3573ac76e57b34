"""CPU checks of tests/post_model.py: the model equals the oracle on every crafted case (so the margins hold), the crafted
cases reach the shapes the device code is structured around, and each negative control (a plausible wrong kernel) changes
at least one crafted result."""
import numpy as np
import pytest
import torch

import post_model as pm

M_SWEEP = [1, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128, 129, 1000]
THRS = [0.01, 0.1, 0.3]


def _box_cases():
    for m in M_SWEEP:
        for pat in ("chain", "cluster"):
            yield pat, m, m
    for pat in ("standup", "far"):
        yield pat, 200, 7


def _oracle_keep(det, scores, thr, ge=True):
    from oracle import cpu as ocpu
    order = pm.score_order(scores)
    dets = np.concatenate([det[order], np.asarray(scores, np.float32)[order, None]], 1)
    return order[ocpu.rotate_nms_cc(dets, thr, ge=ge)]


@pytest.mark.parametrize("pat,m,seed", list(_box_cases()))
def test_nms_model_matches_oracle_and_margins_hold(pat, m, seed):
    det, perm = pm.gen_boxes(pat, m, seed)
    scores = ((m - perm) / m).astype(np.float32)
    ious = pm.pair_ious(det)
    assert pm.all_clear(det, ious)
    for thr in THRS:
        assert pm.robust(ious, thr), (pat, m, thr)
        assert np.array_equal(pm.rotate_nms_model(det, scores, thr), _oracle_keep(det, scores, thr))


def test_exact_threshold_set_is_exact():
    from oracle import cpu as ocpu
    det, thr = pm.exact_threshold_set()
    bev = pm.bev_of(det)
    assert np.float32(pm.iou_bev64(bev[0], bev[1])) == thr
    assert ocpu.boxes_iou_bev(bev[:2], bev[:2])[0, 1] == thr       # fp32 arithmetic lands on the same value
    scores = np.array([0.9, 0.8, 0.7, 0.6], np.float32)
    for ge in (True, False):
        assert np.array_equal(pm.rotate_nms_model(det, scores, thr, ge), _oracle_keep(det, scores, thr, ge))
    assert pm.rotate_nms_model(det, scores, thr, True).tolist() == [0, 2, 3]
    assert pm.rotate_nms_model(det, scores, thr, False).tolist() == [0, 1, 3]


def _sorted_suppressions(pat, m, seed, thr=0.01):
    det, perm = pm.gen_boxes(pat, m, seed)
    order = np.argsort(perm)
    ious = pm.pair_ious(det[order])
    return pm.suppress_set(m, ious, thr), ious


def test_crafted_sets_reach_every_mask_position():
    """suppression pairs in both word halves, across 64-row blocks, and at tile rows / columns 0, 31, 32, 63"""
    rows, cols, halves, cross, diag_blk = set(), set(), set(), 0, 0
    for pat, m, seed in _box_cases():
        supp, _ = _sorted_suppressions(pat, m, seed)
        for i, j in supp:
            rows.add(i % 64)
            cols.add(j % 64)
            halves.add((j % 64) // 32)
            cross += (i // 64) != (j // 64)
            diag_blk += (i // 64) == (j // 64) and (i % 64) < 32 <= (j % 64)
    assert {0, 31, 32, 63} <= rows and {0, 31, 32, 63} <= cols
    assert halves == {0, 1} and cross > 100 and diag_blk > 10


@pytest.mark.parametrize("pat,m,seed", [c for c in _box_cases() if c[1] <= 129 or c[0] == "chain"])
def test_mask_word_layout_restatement(pat, m, seed):
    """the restated words (unwritten halves poisoned) scanned block-wise give the plain greedy result: the scan never reads
    a half no tile wrote"""
    supp, ious = _sorted_suppressions(pat, m, seed)
    K = max(m, 1000)
    for cap in (m, max(1, m // 3)):
        assert pm.scan_words(pm.mask_words(m, K, supp), m, cap) == pm.greedy(m, ious, 0.01, True, cap)


# ------------------------------------------------------------------------------------------------------------ frames
FRAME_SWEEP = [dict(n=n, K=1000, P=100) for n in (999, 1000, 1001, 1023, 1024, 1025, 2049)] + \
              [dict(n=m, K=1000, P=100, pattern=("chain", "cluster")[i % 2]) for i, m in enumerate(M_SWEEP[:-1])] + \
              [dict(n=50, K=1, P=1), dict(n=100, K=33, P=100, pattern="cluster"), dict(n=1500, K=1000, P=100, tie_levels=1),
               dict(n=600, K=500, P=100, tie_levels=40, pattern="cluster"),
               dict(n=99, K=1000, P=100, pattern="far"), dict(n=100, K=1000, P=100, pattern="far"),
               dict(n=101, K=1000, P=100, pattern="far"), dict(n=2, K=1000, P=1, pattern="far"),
               dict(n=70400, K=16384, P=4096, all_anchors=True)]


def _predict(h, cfg):
    from oracle import bev_ref
    an = pm.kitti_anchors()
    t = torch.from_numpy(h)
    c = dict(pm.POST_DEFAULTS)
    c.update(cfg)
    return bev_ref.predict_frame(t[:, 0:14].reshape(-1, 7), t[:, 14:16].reshape(-1), t[:, 16:20].reshape(-1, 2), t[:, 20:22].reshape(-1),
                                 torch.from_numpy(an), nms_pre=c["nms_pre_max"], nms_post=c["nms_post_max"], nms_thr=c["nms_iou_thresh"],
                                 post_range=c["post_range"], direction_offset=float(c["direction_offset"]), return_aux=True)


@pytest.mark.parametrize("kw", FRAME_SWEEP, ids=lambda kw: "-".join("%s%s" % (k, v) for k, v in kw.items()))
def test_post_model_matches_predict_frame(kw):
    h, cfg = pm.frame(**kw)
    o = pm.post_frame(h, pm.kitti_anchors(), cfg)
    assert pm.robust(o["ious"], 0.01) and o["clear"]
    boxes, scores, _l, aux = _predict(h, cfg)
    assert o["n"] == aux["n_candidates"] == kw["n"]
    nk = o["aux"][2]
    assert np.array_equal(o["sel_anchor"][:nk], aux["nms_selected_anchor"].numpy())
    assert np.array_equal(o["anchor"][:o["count"]], aux["final_anchor"].numpy())
    np.testing.assert_array_equal(o["boxes"][:o["count"], [0, 1, 2, 6]], boxes.numpy()[:, [0, 1, 2, 6]])
    np.testing.assert_allclose(o["scores"][:o["count"]], scores.numpy(), rtol=2e-7)


def test_frame_sweep_reaches_its_shapes():
    an = pm.kitti_anchors()
    ms, nks = set(), []
    for kw in FRAME_SWEEP:
        h, cfg = pm.frame(**kw)
        o = pm.post_frame(h, an, cfg)
        ms.add(o["m"])
        nks.append((o["aux"][2], kw["P"], len(pm.greedy(o["m"], o["ious"], 0.01))))
    assert set(M_SWEEP) <= ms | {1000}
    # uncapped keep counts P - 1, P and P + 1 (P = 100), and P + 1 at P = 1
    unc = {(u - P) for _nk, P, u in nks}
    assert {-1, 0, 1} <= unc


def test_boundary_frame_hits_every_boundary():
    an = pm.kitti_anchors()
    h, cfg, planes, idx = pm.boundary_frame()
    o = pm.post_frame(h, an, cfg, planes)
    assert o["aux"][2] == cfg["nms_post_max"] and o["n"] > cfg["nms_post_max"]
    kept = set(o["anchor"][:o["count"]].tolist())
    assert {idx[2], idx[4], idx[5], idx[6], idx[7]} <= kept               # on the inclusive range bounds
    assert idx[8] not in kept and idx[8] in o["sel_anchor"]                # frustum sign 0 rejects
    b = o["boxes"][:o["count"]]
    assert b[0, 6] == np.float32(cfg["direction_offset"])                  # r == offset, equal logits: label 0, no flip
    assert b[1, 6] == np.float32(cfg["direction_offset"]) + pm.PI32        # r == offset, dir 1: flip


# ------------------------------------------------------------------------------------------------------------ negative controls
def _differs(a, b):
    return any(not np.array_equal(np.asarray(a[k]), np.asarray(b[k])) for k in ("count", "aux", "sel_anchor", "boxes", "anchor"))


def test_negative_controls_nms():
    changed = dict(or_suppressed=False, swap=False, drop_last=False, gt=False, ties_high=False)
    for pat, m, seed in _box_cases():
        supp, ious = _sorted_suppressions(pat, m, seed)
        good = pm.greedy(m, ious, 0.01)
        changed["or_suppressed"] |= pm.greedy(m, ious, 0.01, or_suppressed=True) != good
        if m <= 1000:
            K = max(m, 1000)
            changed["swap"] |= pm.scan_words(pm.mask_words(m, K, supp, swap_halves=True), m, m) != good
            changed["drop_last"] |= pm.scan_words(pm.mask_words(m, K, supp), m, m, drop_last_partial=True) != good
    det, thr = pm.exact_threshold_set()
    sc = np.array([0.9, 0.8, 0.7, 0.6], np.float32)
    changed["gt"] = pm.rotate_nms_model(det, sc, thr, True).tolist() != pm.rotate_nms_model(det, sc, thr, False).tolist()
    h, cfg = pm.frame(n=1500, K=1000, P=100, tie_levels=1)
    an = pm.kitti_anchors()
    changed["ties_high"] = _differs(pm.post_frame(h, an, cfg), pm.post_frame(h, an, cfg, variant=("ties_high",)))
    assert all(changed.values()), changed


@pytest.mark.parametrize("variant", ["cap_after_range", "frustum_strict", "dir_ge", "or_suppressed"])
def test_negative_controls_post(variant):
    an = pm.kitti_anchors()
    h, cfg, planes, _idx = pm.boundary_frame()
    frames = [(h, cfg, planes)] + [pm.frame(**kw) + (None,) for kw in FRAME_SWEEP]
    assert any(_differs(pm.post_frame(h_, an, c_, p_), pm.post_frame(h_, an, c_, p_, variant=(variant,))) for h_, c_, p_ in frames)
