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
