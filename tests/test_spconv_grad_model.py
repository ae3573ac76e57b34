"""CPU checks of the weight-gradient model and bounds (tests/spconv_grad_model.py) and of the fp64 train-mode restatement."""
import numpy as np
import pytest
import torch

from oracle.spconv_grad_ref import conv_backward_from_nbr
from spconv_grad_model import WgradCase, ratio, torch_conv, wgrad_chunks
from test_gpu_spconv_ops import crafted_nbr


def test_item_decomposition_matches_the_library():
    from sessd_b200 import ops
    for max_out in (1, 127, 128, 129, 20000, 70000, 600000):
        for kvol in (1, 3, 27):
            chunks, tpi = wgrad_chunks(max_out, kvol)
            assert ops.wgrad_items(max_out, kvol) == kvol * chunks
            assert (chunks - 1) * tpi < -(-max_out // 128) <= chunks * tpi


def _case(cin, cout, seed, n_out=3000, kvol=27):
    rng = np.random.default_rng(seed)
    nbr = crafted_nbr("full", n_out, kvol, 1500, seed)
    nbr[rng.random(nbr.shape) < 0.4] = -1           # ~ 77 pairs per tile and offset: rounds of 64 + 13 (stale slots reachable)
    x = rng.standard_normal((1500, cin)).astype(np.float32)
    g = rng.standard_normal((n_out, cout)).astype(np.float32)
    return WgradCase(nbr, n_out, n_out, x, g)


@pytest.mark.parametrize("cin,cout", [(32, 32), (64, 64)])
def test_wgrad_bounds_hold_for_exact_emulation_and_catch_wrong_kernels(cin, cout):
    """positive control: the exact emulation is within the fp64 bound; negative controls: each wrong kernel exceeds the emulation bound
    and the fp64 bound (ratio > 1).  The smallest ratios are printed."""
    c = _case(cin, cout, cin + cout)
    truth, emul = c.truth(), c.emul()
    assert ratio(emul, truth, c.tol_fp64()) <= 1.0
    assert ratio(truth.astype(np.float32), truth, c.tol_rows()) <= 1.0
    wrong = {"dropped pair": c.wrong_dropped_pair(), "swapped offsets": c.wrong_swapped_offsets(), "no cross products": c.wrong_no_cross(),
             "missed clear": c.wrong_stale_slots(), "partial twice": c.wrong_reduce("twice"), "partial lost": c.wrong_reduce("lost")}
    for name, w in wrong.items():
        re, rf = ratio(w, emul, c.tol_emul()), ratio(w, truth, c.tol_fp64())
        print("%-18s emul %.3g  fp64 %.3g" % (name, re, rf))
        assert re > 1.0 and rf > 1.0, name


def test_rows_bound_catches_a_dropped_pair():
    c = _case(16, 16, 3)
    truth = c.truth()
    x, g = c.x.astype(np.float64), c.g.astype(np.float64)
    items = dict(c.items)
    key = max(items, key=lambda kc: len(items[kc][0]))
    pairs, s = items[key]
    items[key] = (pairs[1:], s)
    wrong = c.per_offset(lambda i, o: x[i].T @ g[o], items)
    assert ratio(wrong, truth, c.tol_rows()) > 1.0


def test_train_restatement_conv_gradients_equal_the_pinned_oracle():
    """torch autograd through torch_conv (the restatement's conv) == conv_backward_from_nbr (pinned to dense autograd)"""
    rng = np.random.default_rng(0)
    for n_out, n_in, kvol in ((300, 200, 27), (50, 400, 3)):
        # every (input row, offset) feeds at most one output row, as in a real rulebook (transpose_nbr)
        nbr = np.stack([rng.permutation(n_in)[:n_out] if n_out <= n_in else np.r_[rng.permutation(n_in), np.full(n_out - n_in, -1)]
                        for _ in range(kvol)], 1)
        nbr[rng.random(nbr.shape) < 0.5] = -1
        x = torch.from_numpy(rng.standard_normal((n_in, 8))).requires_grad_(True)
        w = torch.from_numpy(rng.standard_normal((kvol, 8, 16))).requires_grad_(True)
        g = rng.standard_normal((n_out, 16))
        torch_conv(x, nbr, w).backward(torch.from_numpy(g))
        gx, gw = conv_backward_from_nbr(x.detach().numpy(), nbr, w.detach().numpy(), g)
        np.testing.assert_allclose(x.grad.numpy(), gx, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(w.grad.numpy(), gw, rtol=1e-12, atol=1e-12)
