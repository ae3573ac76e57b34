"""CPU checks of tests/train_ops_model.py before any GPU time is spent: the fp32 emulations of the training-signal kernels pass every
bound on every crafted case, and each planted mistake (MUTANTS) fails at least one case -- the bounds are neither too loose nor too
tight."""
import numpy as np
import pytest

import train_ops_model as tm


@pytest.fixture(scope="module")
def head_cases():
    cases = []
    for name, head, anc, labels, targets, cfg in tm.head_cases():
        rl, rg = tm.head_loss_ref(head, anc, labels, targets, cfg)
        lb, gb = tm.head_loss_bounds(head, anc, labels, targets, cfg)
        cases.append((name, head, anc, labels, targets, cfg, rl, rg, lb, gb))
    return cases


def test_head_loss_emulation_within_bounds(head_cases):
    worst = [0.0, 0.0]
    for name, head, anc, labels, targets, cfg, rl, rg, lb, gb in head_cases:
        losses, grad = tm.head_loss_emul(head, anc, labels, targets, cfg)
        rv, rgr = tm.head_loss_violations(losses, grad, rl, rg, lb, gb)
        assert rv <= 1.0 and rgr <= 1.0, (name, rv, rgr)
        worst = [max(worst[0], rv), max(worst[1], rgr)]
        assert np.array_equal(losses[:, 6], (labels > 0).sum(1)) and np.array_equal(losses[:, 7], (labels == 0).sum(1))
    print("head loss emulation: worst error / bound, losses %.3g, gradient %.3g" % tuple(worst))


@pytest.mark.parametrize("mutant", tm.MUTANTS)
def test_head_loss_mutant_fails_a_bound(head_cases, mutant):
    failed = []
    for name, head, anc, labels, targets, cfg, rl, rg, lb, gb in head_cases:
        losses, grad = tm.head_loss_emul(head, anc, labels, targets, cfg, mutant=mutant)
        rv, rgr = tm.head_loss_violations(losses, grad, rl, rg, lb, gb)
        if rv > 1.0 or rgr > 1.0:
            failed.append(name)
    assert failed, mutant


def test_head_cases_reach_their_edges(head_cases):
    """the crafted values are really in the cases: every logit on every label, knee residuals, yaw + pi, direction boundary"""
    seen = set()
    for name, head, anc, labels, targets, cfg, *_ in head_cases:
        x = head[..., 14:16].reshape(labels.shape)
        for v in tm.LOGITS:
            for lab in (-1, 0, 1):
                if ((x == v) & (labels == lab)).any():
                    seen.add((float(v), lab))
        rot = targets[..., 6] + anc[None, :, 6]
        if ((rot == np.float32(cfg.dir_offset)) & (labels > 0)).any():
            seen.add(("dir_boundary", cfg.dir_offset))
        box = head[..., :14].reshape(labels.shape + (7,))
        if ((box[..., :6] == tm.KNEE) & (targets[..., :6] == 0) & (labels[..., None] > 0)).any():
            seen.add("knee")
    assert {(float(v), lab) for v in tm.LOGITS for lab in (-1, 0, 1)} <= seen
    assert {("dir_boundary", 0.0), ("dir_boundary", 0.78), "knee"} <= seen


# ------------------------------------------------------------------------------------------------ ODIoU fp64 restatement
def test_odiou_restatement_matches_reference_golden_and_host_twin(golden_dir):
    """odiou_ref (fp64, autograd) vs the reference's odiou_3D values (golden: the reference's fp32 numpy loops, 2e-4 as
    tests/test_odiou.py) and vs the kernel's host twin within odiou_bounds: value on every pair, all 7 gradient components where the
    minimising hull edge is unique.  The exactly identical pair (50) is excluded from the golden comparison: the reference's polygon
    routine returns IoU 1/3 there (tests/test_odiou.py)."""
    import os
    from cases import odiou_pairs
    from sessd_b200 import ops
    g, q = odiou_pairs()
    v, gr, uniq = tm.odiou_ref(g, q)
    ref = np.load(os.path.join(golden_dir, "odiou_case.npz"))
    keep = np.arange(len(g)) != 50
    np.testing.assert_allclose(v[keep], ref["odiou"][keep], atol=2e-4, rtol=0)
    assert abs(v[50]) < 1e-12
    hv, hg = ops.odiou_pairs_host(g, q)
    vb, gb = tm.odiou_bounds(g, q, gr)
    rv = np.abs(hv - v) / vb
    rg = (np.abs(hg - gr) / gb[:, None])[uniq]
    assert rv.max() <= 1.0 and rg.max() <= 1.0, (rv.max(), rg.max())
    assert uniq[:48].sum() >= 30                                  # most generic pairs are compared on the gradient
    print("odiou host twin vs fp64: worst error / bound, value %.3g, gradient %.3g" % (rv.max(), rg.max()))


# ------------------------------------------------------------------------------------------------ IoU-prediction loss
@pytest.fixture(scope="module")
def iou_pred_cases():
    cases = []
    for name, head, anc, labels, targets, sigma, w_iou in tm.iou_pred_cases():
        rs, rg, info = tm.iou_pred_ref(head, anc, labels, targets, sigma, w_iou)
        sb, gb = tm.iou_pred_bounds(info)
        cases.append((name, head, anc, labels, targets, sigma, w_iou, rs, rg, sb, gb))
    return cases


def test_iou_pred_twin_within_bounds(iou_pred_cases):
    """the fp32 twin (the C oracle's decode and overlap, the kernel's operation order) within iou_pred_bounds of the fp64 reference, and its
    per-frame sums equal oracle.loss_ref.iou_pred_loss (the reference's arithmetic) within the same bound"""
    import torch
    from oracle import loss_ref
    worst = [0.0, 0.0]
    for name, head, anc, labels, targets, sigma, w_iou, rs, rg, sb, gb in iou_pred_cases:
        sums, grad = tm.iou_pred_emul(head, anc, labels, targets, sigma, w_iou)
        rv, rgr = tm.iou_pred_violations(sums, grad, rs, rg, sb, gb)
        assert rv <= 1.0 and rgr <= 1.0, (name, rv, rgr)
        worst = [max(worst[0], rv), max(worst[1], rgr)]
        h = torch.from_numpy(head)
        box, _, _ = loss_ref.split_head(h)
        o = loss_ref.iou_pred_loss(h[..., 20:22].reshape(labels.shape), box, torch.from_numpy(anc), torch.from_numpy(labels).long(),
                                   torch.from_numpy(targets), sigma=sigma).numpy()
        assert (np.abs(o - rs) <= sb).all(), (name, o, rs, sb)
    print("iou prediction twin: worst error / bound, sums %.3g, gradient %.3g" % tuple(worst))


@pytest.mark.parametrize("mutant", tm.IP_MUTANTS)
def test_iou_pred_mutant_fails_a_bound(iou_pred_cases, mutant):
    failed = []
    for name, head, anc, labels, targets, sigma, w_iou, rs, rg, sb, gb in iou_pred_cases:
        sums, grad = tm.iou_pred_emul(head, anc, labels, targets, sigma, w_iou, mutant=mutant)
        rv, rgr = tm.iou_pred_violations(sums, grad, rs, rg, sb, gb)
        if rv > 1.0 or rgr > 1.0:
            failed.append(name)
    assert failed, mutant


def test_iou_pred_npos_clamp_is_unobservable(iou_pred_cases):
    """only positives read 1 / num_pos, so a frame without positives never uses the clamp max(num_pos, 1): dropping it changes nothing
    here (the head loss's negatives do read it, and its mutant is caught there)"""
    for name, head, anc, labels, targets, sigma, w_iou, *_ in iou_pred_cases:
        a = tm.iou_pred_emul(head, anc, labels, targets, sigma, w_iou)
        b = tm.iou_pred_emul(head, anc, labels, targets, sigma, w_iou, mutant="no_npos_clamp")
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), name


def test_iou_pred_cases_reach_their_edges(iou_pred_cases):
    """positives at anchor 0, A - 1 and past the grid-stride wrap, an empty frame, batch 5, strides 22 / 24 / 32, sigma 3 / 1, w_iou 1 /
    0.5, A = 37 890 and 70 400; every crafted pair; iou head values at the knee, one ulp either side and d = 0 on exact -1 targets; the
    exact-(-1) pairs really are -1 in fp64; the -104 encoding underflows to a zero-size box"""
    seen = set()
    for name, head, anc, labels, targets, sigma, w_iou, rs, rg, *_ in iou_pred_cases:
        B, A = labels.shape
        pos = labels > 0
        seen |= {("A", A), ("stride", head.shape[2]), ("sigma", sigma), ("w_iou", w_iou), ("B", B)}
        if (pos.sum(1) == 0).any():
            seen.add("empty")
        if pos[:, 0].any() and pos[:, A - 1].any() and pos[:, tm.IP_CTA_SPAN:].any():
            seen.add(("wrap", A))
        _, _, info = tm.iou_pred_ref(head, anc, labels, targets, sigma, w_iou)
        t = 2 * info["iou"] - 1
        k = np.float32(1) / np.float32(sigma * sigma)
        hv = head[info["b"], info["a"] // 2, 20 + info["r"]]
        on = t == -1.0
        for v, tag in ((np.float32(-1), "d0"), (np.float32(-1) + k, "knee+"), (np.float32(-1) - k, "knee-")):
            if (on & (hv == v)).any():
                seen.add((tag, sigma))
            if (on & (hv == np.nextafter(v, np.float32(2)))).any() and (on & (hv == np.nextafter(v, np.float32(-2)))).any():
                seen.add((tag + "ulp", sigma))
        q = info["q"]
        e3 = head[info["b"], info["a"] // 2, 7 * info["r"] + 3]
        if (e3 == -104).any() and np.exp(np.float32(-104)) == 0:                     # the fp32 decode's width is exactly 0
            seen.add("zero_size")
        if (np.abs(q[:, :2]).max(1) > 39).any() and (q[:, 0] > 69).any():
            seen.add("far")
    want = {("A", 37890), ("A", 70400), ("stride", 22), ("stride", 24), ("stride", 32), ("sigma", 3.0), ("sigma", 1.0), ("w_iou", 1.0),
            ("w_iou", 0.5), ("B", 5), "empty", ("wrap", 37890), ("wrap", 70400), "zero_size", "far"}
    want |= {(tag, s) for s in (3.0, 1.0) for tag in ("d0", "knee+", "knee-", "knee+ulp", "knee-ulp")}
    assert want <= seen, want - seen
    names = [n for n, _, _ in tm.iou_pred_pairs()]
    assert {"identical", "yaw_plus_pi", "yaw_plus_half_pi_wl_swapped", "disjoint_bev", "no_height_overlap", "touching_faces", "contained",
            "corner_on_edge", "pedestrian", "enc_dims_plus5", "enc_dims_minus5", "enc_dims_minus104"} <= set(names)
