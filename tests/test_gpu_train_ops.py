"""The training-signal kernels one operator at a time against fp64 references on crafted inputs (bounds and their derivation:
tests/train_ops_model.py).

* sessd_head_loss: every crafted head case of train_ops_model.head_cases() -- logits up to +-100 on every label, smooth-L1 knee
  residuals, yaw + pi, direction targets on the boundary, empty / ignored / ragged frames over a batch of 5, A from 2 to 70 400, head
  strides 22 / 24 / 32, non-default loss parameters.  Values and every gradient entry within the derived bound; the gradient buffer is
  poisoned with NaN first, so every channel must be written (iou and padding: exactly 0); the values-only call gives bit-identical
  losses; two runs are bitwise equal; the counts are exact.
* sessd_axpby / sessd_grad_sqnorm / sessd_adamw_clip_ema_step on plain tensors of sizes that reach the float4 tails and the
  single-chunk norm, against fp64 or the same fp32 expression evaluated by torch.  The C entry points are called on buffers 4-8
  elements longer than n (n = 0 included: a valid pointer, nothing to do), so writes past n would show.
* sessd_iou_pred_loss: every crafted case of train_ops_model.iou_pred_cases() against the fp64 aligned 3-D IoU reference and the fp32
  twin, on a NaN-filled gradient; an odd anchor count is refused before any launch.
* sessd_odiou_loss: where the positives sit (anchor 0, A - 1, past the grid-stride wrap), an empty frame, a clamped prediction and
  accumulation into a pre-filled gradient, against the host twin of odiou.cuh."""
import numpy as np
import pytest
import torch

import train_ops_model as tm

pytestmark = pytest.mark.gpu


def _d(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _head_loss_poisoned(head, anc, labels, targets, cfg, with_grad=True, w_iou=None):
    """sessd_head_loss (then sessd_iou_pred_loss when w_iou is given) into NaN-filled outputs"""
    from sessd_b200 import _lib, ops
    B, A = labels.shape
    h, a, lab, tg = _d(head), _d(anc), _d(labels), _d(targets)
    losses = torch.full((B, 8), float("nan"), device="cuda")
    grad = torch.full_like(h, float("nan")) if with_grad else None
    ws = torch.empty((_lib.lib.sessd_head_loss_workspace_bytes(B),), dtype=torch.uint8, device="cuda")
    c = cfg
    _lib.check(_lib.lib.sessd_head_loss(ops._p(h), ops._p(a), ops._p(lab), ops._p(tg), B, A, 2, head.shape[2], float(c.alpha), float(c.sigma),
                                        float(c.dir_offset), float(c.pos_cls_weight), float(c.neg_cls_weight), float(c.w_cls),
                                        float(c.w_loc), float(c.w_dir), ops._p(losses), ops._p(grad), ops._p(ws), ws.numel(), ops._st()),
               "sessd_head_loss")
    if w_iou is not None:
        ws2 = torch.empty((_lib.lib.sessd_iou_pred_loss_workspace_bytes(B),), dtype=torch.uint8, device="cuda")
        _lib.check(_lib.lib.sessd_iou_pred_loss(ops._p(h), ops._p(a), ops._p(lab), ops._p(tg), B, A, 2, head.shape[2], float(c.sigma),
                                                float(w_iou), ops._p(losses), ops._p(grad), ops._p(ws2), ws2.numel(), ops._st()),
                   "sessd_iou_pred_loss")
    torch.cuda.synchronize()
    return losses.cpu().numpy(), (grad.cpu().numpy() if with_grad else None)


def test_head_loss_crafted_cases_within_fp64_bounds():
    worst = [0.0, 0.0]
    for name, head, anc, labels, targets, cfg in tm.head_cases():
        rl, rg = tm.head_loss_ref(head, anc, labels, targets, cfg)
        lb, gb = tm.head_loss_bounds(head, anc, labels, targets, cfg)
        losses, grad = _head_loss_poisoned(head, anc, labels, targets, cfg)
        assert np.isfinite(grad).all(), name                                 # every channel written
        assert not grad[..., 20:].any(), name                                # iou head and padding: exact zeros
        rv, rgr = tm.head_loss_violations(losses, grad, rl, rg, lb, gb)
        assert rv <= 1.0 and rgr <= 1.0, (name, rv, rgr)
        worst = [max(worst[0], rv), max(worst[1], rgr)]
        assert np.array_equal(losses[:, 6], (labels > 0).sum(1).astype(np.float32)), name
        assert np.array_equal(losses[:, 7], (labels == 0).sum(1).astype(np.float32)), name
        values_only, _ = _head_loss_poisoned(head, anc, labels, targets, cfg, with_grad=False)
        assert np.array_equal(values_only[:, [0, 1, 2, 3, 4, 6, 7]], losses[:, [0, 1, 2, 3, 4, 6, 7]]), name
        again, grad2 = _head_loss_poisoned(head, anc, labels, targets, cfg)
        assert np.array_equal(again[:, [0, 1, 2, 3, 4, 6, 7]], losses[:, [0, 1, 2, 3, 4, 6, 7]]) and np.array_equal(grad2, grad), name
    print("head loss: worst error / bound, losses %.3g, gradient %.3g" % tuple(worst))


# ------------------------------------------------------------------------------------------------ IoU-prediction loss
def test_iou_pred_crafted_cases_within_fp64_bounds():
    """sessd_iou_pred_loss behind sessd_head_loss on every case of train_ops_model.iou_pred_cases() (degenerate pairs, knee residuals,
    positives at anchor 0, A - 1 and past the grid-stride wrap, an empty frame, a ragged batch of 5, strides 22 / 24 / 32, sigma 3 / 1,
    w_iou 1 / 0.5), into a NaN-filled gradient: the iou channels of the positives within iou_pred_bounds of the fp64 reference and within
    twice that of the fp32 twin, those of every other anchor exactly 0; every other gradient channel and every other loss column
    bit-identical to the run without the IoU term; losses[:, 5] within the sum bound; two runs bitwise equal."""
    worst = [0.0, 0.0, 0.0]
    keep = [0, 1, 2, 3, 4, 6, 7]
    for name, head, anc, labels, targets, sigma, w_iou in tm.iou_pred_cases():
        cfg = tm.HeadCfg(sigma=sigma)
        rs, rg, info = tm.iou_pred_ref(head, anc, labels, targets, sigma, w_iou)
        sb, gb = tm.iou_pred_bounds(info)
        es, eg = tm.iou_pred_emul(head, anc, labels, targets, sigma, w_iou)
        base, gbase = _head_loss_poisoned(head, anc, labels, targets, cfg)
        losses, grad = _head_loss_poisoned(head, anc, labels, targets, cfg, w_iou=w_iou)
        assert np.isfinite(grad).all() and np.isfinite(losses).all(), name
        pos = labels > 0
        assert not grad[..., 20:22].reshape(labels.shape)[~pos].any(), name
        other = np.ones(head.shape[2], bool)
        other[20:22] = False
        assert np.array_equal(grad[..., other], gbase[..., other]), name
        assert np.array_equal(losses[:, keep], base[:, keep]), name
        assert (losses[~pos.any(1), 5] == 0).all(), name
        g_iou = np.zeros_like(grad)
        sel = (info["b"], info["a"] // 2, 20 + info["r"])
        g_iou[sel] = grad[sel]
        rv, rgr = tm.iou_pred_violations(losses[:, 5], g_iou, rs, rg, sb, gb)
        assert rv <= 1.0 and rgr <= 1.0, (name, rv, rgr)
        ts, tg_ = tm.iou_pred_violations(losses[:, 5], g_iou, es.astype(np.float64), eg.astype(np.float64), sb, gb, scale=2.0)
        assert ts <= 1.0 and tg_ <= 1.0, (name, ts, tg_)
        worst = [max(worst[0], rv), max(worst[1], rgr), max(worst[2], ts, tg_)]
        again, grad2 = _head_loss_poisoned(head, anc, labels, targets, cfg, w_iou=w_iou)
        assert np.array_equal(again, losses) and np.array_equal(grad2, grad), name
    print("iou prediction device: worst error / bound, sums %.3g, gradient vs fp64 %.3g, vs twin (2x bound) %.3g" % tuple(worst))


def test_iou_pred_refuses_odd_anchor_count():
    """num_anchors not a multiple of anchors_per_loc: SESSD_EINVAL before any launch (the outputs keep their fill)"""
    from sessd_b200 import _lib, ops
    B, A, S = 2, 7, 24
    h = torch.zeros((B, A // 2 + 1, S), device="cuda")
    a = torch.zeros((A + 1, 7), device="cuda")
    lab = torch.ones((B, A + 1), dtype=torch.int32, device="cuda")
    tg = torch.zeros((B, A + 1, 7), device="cuda")
    losses = torch.full((B, 8), 7.0, device="cuda")
    grad = torch.full_like(h, 7.0)
    ws = torch.empty((_lib.lib.sessd_iou_pred_loss_workspace_bytes(B),), dtype=torch.uint8, device="cuda")
    rc = _lib.lib.sessd_iou_pred_loss(ops._p(h), ops._p(a), ops._p(lab), ops._p(tg), B, A, 2, S, 3.0, 1.0, ops._p(losses), ops._p(grad),
                                      ops._p(ws), ws.numel(), ops._st())
    torch.cuda.synchronize()
    assert rc == -1                                                              # SESSD_EINVAL
    assert bool((losses == 7.0).all()) and bool((grad == 7.0).all())
    rc = _lib.lib.sessd_iou_pred_loss(ops._p(h), ops._p(a), ops._p(lab), ops._p(tg), B, A + 1, 2, S, 3.0, 1.0, ops._p(losses), ops._p(grad),
                                      ops._p(ws), ws.numel(), ops._st())
    torch.cuda.synchronize()
    assert rc == 0


# ------------------------------------------------------------------------------------------------ optimiser kernels
SIZES = (0, 1, 3, 5, 16383, 16384, 16385, 5 * 16384 + 3)


def _spread(n, seed):
    """fp32 values with magnitudes spread over 2^-40 .. 2^40 and random signs"""
    rng = np.random.default_rng(seed)
    e = rng.uniform(-40, 40, n)
    return (np.exp2(e) * rng.choice([-1.0, 1.0], n)).astype(np.float32)


@pytest.mark.parametrize("n", SIZES)
def test_axpby_tails(n):
    from sessd_b200 import _lib
    from sessd_b200.train import _p, _st
    rng = np.random.default_rng(n)
    y0 = rng.standard_normal(n + 8).astype(np.float32)
    x0 = rng.standard_normal(n + 8).astype(np.float32)
    a, b = np.float32(0.999), np.float32(1.0 - 0.999)
    for with_x in (True, False):
        y, x = _d(y0), _d(x0)
        _lib.check(_lib.lib.sessd_axpby(_p(y), _p(x) if with_x else _p(None), float(a), float(b), n, _st(y)), "sessd_axpby")
        got = y.cpu().numpy()
        yd, xd = y0[:n].astype(np.float64), (x0[:n].astype(np.float64) if with_x else np.zeros(n))
        # fmaf(a, y, b * x): one rounding of b x, one of the fma
        ref = a.astype(np.float64) * yd + b.astype(np.float64) * xd
        bound = 2 * tm.U * (np.abs(a * yd) + 2 * np.abs(b * xd))
        assert (np.abs(got[:n] - ref) <= bound).all(), (n, with_x)
        assert np.array_equal(got[n:], y0[n:]), (n, with_x)                   # nothing past n is touched


def _norm(buf, n, max_norm=35.0):
    """sessd_grad_sqnorm over the first n elements of buf -> device tensor [total_norm, clip_coef]"""
    from sessd_b200 import _lib
    from sessd_b200.train import _p, _st
    ws = torch.zeros(_lib.lib.sessd_grad_sqnorm_workspace_bytes(n), dtype=torch.uint8, device="cuda")
    out = torch.empty(2, dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib.sessd_grad_sqnorm(_p(buf), n, float(max_norm), _p(out), _p(ws), _st(buf)), "sessd_grad_sqnorm")
    return out


@pytest.mark.parametrize("n", SIZES)
def test_grad_norm_spread_values(n):
    x = _spread(n, 100 + n)
    buf = torch.full((n + 4,), 1e30, dtype=torch.float32, device="cuda")       # past n: would dominate the norm if read
    buf[:n] = _d(x)
    out1 = _norm(buf, n).cpu().numpy()
    out2 = _norm(buf, n).cpu().numpy()
    assert np.array_equal(out1, out2)
    ref = np.sqrt(np.sum(x.astype(np.float64) ** 2))
    ulp = np.spacing(np.float32(ref)) if ref > 0 else 0.0
    assert abs(float(out1[0]) - ref) <= ulp, (n, out1[0], ref)
    t = torch.tensor(float(out1[0]), dtype=torch.float32)
    coef = torch.clamp((t + 1e-6).reciprocal() * 35.0, max=1.0)                 # clip_grad_norm_'s arithmetic on the fp32 norm
    assert float(out1[1]) == float(coef), (n, out1[1], float(coef))


@pytest.mark.parametrize("bad", ("inf", "nan"))
def test_grad_norm_non_finite(bad):
    from sessd_b200.train import grad_norm
    x = _spread(16385, 7)
    x[1234] = np.float32(bad)
    out = grad_norm(_d(x), 35.0).cpu().numpy()
    g = torch.from_numpy(x.copy()).requires_grad_(False)
    holder = torch.nn.Parameter(torch.zeros_like(g))
    holder.grad = g
    total = torch.nn.utils.clip_grad_norm_([holder], 35.0)
    coef = torch.clamp((total + 1e-6).reciprocal() * 35.0, max=1.0)
    np.testing.assert_equal(out[0], np.float32(total))
    np.testing.assert_equal(out[1], np.float32(coef))


@pytest.mark.parametrize("n", SIZES)
def test_adamw_clip_ema_tails(n):
    """one clipped AdamW + EMA step: every element against the kernel's fp32 expression evaluated in fp64 from the same fp32 inputs"""
    from sessd_b200 import _lib
    from sessd_b200.train import _p, _st
    rng = np.random.default_rng(1000 + n)
    p0, g0 = rng.standard_normal(n + 4).astype(np.float32), (rng.standard_normal(n + 4) * 30).astype(np.float32)
    m0, v0 = (rng.standard_normal(n + 4) * 0.1).astype(np.float32), (rng.random(n + 4) * 0.01).astype(np.float32)
    e0 = rng.standard_normal(n + 4).astype(np.float32)
    p, g, m, v, e = (_d(a) for a in (p0, g0, m0, v0, e0))
    norm = _norm(g, n)
    lr, b1, b2, eps, wd, step, alpha = 3e-3, 0.9, 0.99, 1e-8, 0.01, 3, 0.75
    _lib.check(_lib.lib.sessd_adamw_clip_ema_step(_p(p), _p(g), _p(m), _p(v), n, lr, b1, b2, eps, wd, step, _p(norm[1:]), _p(e), alpha,
                                                  _st(p)), "sessd_adamw_clip_ema_step")
    got = [a.cpu().numpy() for a in (p, g, m, v, e)]
    for a, a0 in zip(got, (p0, g0, m0, v0, e0)):
        assert np.array_equal(a[n:], a0[n:])                                 # nothing past n is touched
    coef = float(norm[1].cpu()) if n else 1.0
    f = np.float64
    lr, b1, b2, eps, wd = (float(np.float32(c)) for c in (lr, b1, b2, eps, wd))      # the kernel's fp32 constants
    gi = g0[:n].astype(f) * coef
    mi = m0[:n] + (1 - b1) * (gi - m0[:n])
    vi = b2 * v0[:n].astype(f) + (1 - b2) * gi * gi
    bc1, bc2s = 1 - b1 ** step, np.sqrt(1 - b2 ** step)
    pi = p0[:n] * (1 - lr * wd) - lr / bc1 * (mi / (np.sqrt(vi) / bc2s + eps))
    ei = alpha * e0[:n] + (1 - alpha) * pi
    # per element a chain of <= 8 roundings of terms no larger than the listed magnitudes (the constants are rounded to fp32 once)
    u8 = 8 * tm.U
    np.testing.assert_array_less(np.abs(got[1][:n] - gi), u8 * np.abs(gi) + 1e-30)
    np.testing.assert_array_less(np.abs(got[2][:n] - mi), u8 * (np.abs(m0[:n]) + np.abs(gi)) + 1e-30)
    np.testing.assert_array_less(np.abs(got[3][:n] - vi), u8 * (np.abs(vi)) + 1e-30)
    denom = np.sqrt(vi) / bc2s + eps
    # the step inherits mi's absolute error (a cancellation of m and g), so it is counted on |m| + |g|
    step_mag = lr / bc1 * (np.abs(mi) + np.abs(m0[:n]) + np.abs(gi)) / denom
    np.testing.assert_array_less(np.abs(got[0][:n] - pi), u8 * (np.abs(p0[:n]) + 4 * step_mag) + 1e-30)
    np.testing.assert_array_less(np.abs(got[4][:n] - ei), u8 * (np.abs(e0[:n]) + np.abs(p0[:n]) + 4 * step_mag) + 1e-30)


# ------------------------------------------------------------------------------------------------ ODIoU on the device
def test_odiou_device_vs_fp64_and_host_twin():
    """sessd_odiou_loss on every pair of cases.odiou_pairs (generic, disjoint, contained, identical, perpendicular, no height overlap,
    far-rotated) placed into a head: near the origin (small R / S: tight bounds), at anchor 0, at A - 1 and past the grid-stride wrap
    (132 CTAs x 128 threads); a frame without positives; a prediction decoding beyond +-200 m; a pre-filled gradient.  Against the fp64
    restatement (train_ops_model.odiou_ref, decode and Jacobian in fp64, 1 / num_pos, w / batch) within odiou_bounds, and against the
    host twin of odiou.cuh on the same decoded boxes within twice that (both are within the bound of fp64).  Pairs whose minimising hull
    edge is not unique within rounding are compared on the value only.  The kernel must ADD to the box channels of the positives and
    leave everything else, the empty frame included, untouched; the clamped component's gradient is exactly 0."""
    from cases import odiou_pairs
    from sessd_b200 import ops
    A, B, S, w_od = 70400, 3, 24, 2.0
    anc = tm._anchors(A)
    g_boxes, q_boxes = odiou_pairs()
    near = [((iy * 176) + ix) * 2 + r for iy in (99, 100) for ix in range(0, 14) for r in (0, 1)]
    pos = [0, A - 1, 132 * 128, 132 * 128 + 1, 2 * 132 * 128 + 7] + near
    npair = len(pos)
    labels = np.zeros((B, A), np.int32)
    targets = np.zeros((B, A, 7), np.float32)
    rng = np.random.default_rng(3)
    head = (rng.standard_normal((B, A // 2, S)) * 0.3).astype(np.float32)
    for b in (0, 2):
        sel = (np.arange(npair) + 11 * b) % len(g_boxes)                       # every pair, the degenerate ones included
        for i, a in enumerate(pos):
            labels[b, a] = 1
            c = g_boxes[sel[i], :2].round()
            ga, qa = g_boxes[sel[i]].copy(), q_boxes[sel[i]].copy()
            ga[:2] = anc[a, :2] + (ga[:2] - c)                                  # near the anchor, as the assigner's positives are
            qa[:2] = anc[a, :2] + (qa[:2] - c)
            diag = np.sqrt(anc[a, 4] ** 2 + anc[a, 3] ** 2)
            enc = lambda x: np.float32([(x[0] - anc[a, 0]) / diag, (x[1] - anc[a, 1]) / diag, (x[2] - anc[a, 2]) / anc[a, 5],   # noqa: E731
                                        np.log(x[3] / anc[a, 3]), np.log(x[4] / anc[a, 4]), np.log(x[5] / anc[a, 5]), x[6] - anc[a, 6]])
            targets[b, a] = enc(ga)
            head[b, a // 2, 7 * (a % 2):7 * (a % 2) + 7] = enc(qa)
    clamped = pos[2]
    head[0, clamped // 2, 7 * (clamped % 2)] = np.float32(60.0)                   # x decodes to ~ 60 * 4.2 m > 200 m
    losses, grad0 = ops.head_loss(_d(head), _d(anc), _d(labels), _d(targets), w_loc=0.0)
    prefill = torch.from_numpy(rng.standard_normal(head.shape).astype(np.float32)).cuda()
    grad = grad0 + prefill
    base = grad.clone()
    sums = ops.odiou_loss(_d(head), _d(anc), _d(labels), _d(targets), losses, grad, w_odiou=w_od)
    torch.cuda.synchronize()
    delta = (grad - base).cpu().numpy()
    base = base.cpu().numpy()
    assert not delta[..., 14:].any()                                              # only the box channels change
    assert not delta[1].any() and float(sums[1]) == 0.0                             # the frame without positives
    p = np.array(pos)
    an = anc[p].astype(np.float64)
    diag = np.sqrt(an[:, 4] ** 2 + an[:, 3] ** 2)
    worst = [0.0, 0.0, 0.0]
    for b in (0, 2):
        enc = np.stack([head[b, a // 2, 7 * (a % 2):7 * (a % 2) + 7] for a in p]).astype(np.float64)
        tg = targets[b, p].astype(np.float64)
        dec = lambda e: np.stack([e[:, 0] * diag + an[:, 0], e[:, 1] * diag + an[:, 1], e[:, 2] * an[:, 5] + an[:, 2],   # noqa: E731
                                  np.exp(e[:, 3]) * an[:, 3], np.exp(e[:, 4]) * an[:, 4], np.exp(e[:, 5]) * an[:, 5], e[:, 6] + an[:, 6]], 1)
        qb, gb = dec(enc), dec(tg)
        v, gq, uniq = tm.odiou_ref(gb, qb)
        vb, gbnd = tm.odiou_bounds(gb, qb, gq)
        jac = np.stack([diag, diag, an[:, 5], qb[:, 3], qb[:, 4], qb[:, 5], np.ones(npair)], 1)
        scale = w_od / B / npair
        # per-frame sum: the values' bounds + the fixed-order reduction of terms <= |v| / npair
        # (<= 5 grid-stride steps, 5 shuffle levels, 4 warps, 132 block partials)
        err = abs(float(sums[b]) - v.sum() / npair)
        bound = vb.sum() / npair + 146 * tm.U * np.abs(v).sum() / npair
        assert err <= bound, (b, err, bound)
        worst[0] = max(worst[0], err / bound)
        got = np.stack([delta[b, a // 2, 7 * (a % 2):7 * (a % 2) + 7] for a in p]).astype(np.float64)
        pre = np.stack([base[b, a // 2, 7 * (a % 2):7 * (a % 2) + 7] for a in p]).astype(np.float64)
        # the kernel's own product chain (4 roundings), the Jacobian's (expf 4u + product) and the pre-fill's add-then-subtract
        slack = 8 * tm.U * np.abs(gq * jac * scale) + 4 * tm.U * (np.abs(pre) + np.abs(got))
        gbound = (gbnd[:, None] * np.abs(jac) * scale + slack)[uniq]
        r = (np.abs(got - gq * jac * scale)[uniq] / gbound).max()
        assert r <= 1.0, (b, r)
        worst[1] = max(worst[1], r)
        hv, hg = ops.odiou_pairs_host(gb.astype(np.float32), qb.astype(np.float32))
        r = (np.abs(got - hg * jac * scale)[uniq] / (2 * gbound)).max()
        assert r <= 1.0, (b, r)
        worst[2] = max(worst[2], r)
        others = np.ones(A // 2, bool)
        others[p // 2] = False
        assert not delta[b, others].any()
    c0 = 7 * (clamped % 2)
    assert delta[0, clamped // 2, c0] == 0.0                                      # clamped x: exactly zero gradient
    assert np.abs(delta[0, clamped // 2, c0 + 1:c0 + 7]).max() > 0               # the other components still learn
    print("odiou device: worst error / bound, sums %.3g, gradient vs fp64 %.3g, vs host twin %.3g" % tuple(worst))
