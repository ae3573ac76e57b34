"""fp64 references, fp32 numpy emulations and error bounds of the SE-SSD supervised head loss (csrc/headloss.cu), the IoU-prediction
loss (csrc/iou3d.cu) and the ODIoU loss (csrc/odiou.cuh, odiou.cu); shared by tests/test_train_ops_model.py (CPU) and tests/test_gpu_train_ops.py.

Notation: u = 2^-24 (fp32 unit roundoff); an fp32 operation rounds its exact result r to r (1 + e), |e| <= u; one ulp of r is at most
2u |r|.  expf / logf / log1pf / sinf / cosf of CUDA (and numpy's float32 versions in the emulations) are within 2 ulp = 4u relative.
Every bound below is first order in u with the second-order terms either written out (where an operand can be as small as u) or
absorbed by rounding the constants up.

Supervised head loss (sessd_head_loss), per anchor, against fp64 autograd through oracle/loss_ref on the same fp32 inputs
-----------------------------------------------------------------------------------------------------------------------------
focal term, x = logit, t in {0, 1}, p = 1 / (1 + exp(-x)), pt = t p + (1 - t)(1 - p), om = 1 - pt, ce = max(x, 0) - x t + log1p(exp(-|x|)):
  * p: expf (4u), the add (u), the division (u): |dp| <= 6u p.  (1 - p) is then an ABSOLUTE error of 6u p + u: on a confident anchor
    it is a cancellation, and the reference (fp32 torch) has it too.  om = 1 - pt takes one or two such subtractions:
        E_om = 8u   (absolute).                                    [t = 1: 6u p + u;  t = 0: 6u p + u + u, rounded up]
    At x = -8 on a negative anchor om = p = 3.4e-4, so the focal weight om^2 carries ~4e-4 relative error: a relative bar would
    fail there for a reason that is not a bug.
  * ce: max(x, 0) - x t is exact in the kernel (t is exactly 0 or 1) but is counted as an absolute error u |x| (the cancellation of
    two operands of size |x|); log1p(exp(-|x|)) = L takes expf's 4u through log1p (d log1p(y) = dy / (1 + y) <= L dy / y), log1pf's
    4u and the add:    E_ce = u |x| + 10u L + 2u ce.
  * value om^2 aw ce w (aw = alpha or 1 - alpha: 2u, including the fp32 rounding of alpha; w = class weight / num_pos: 2u):
        |d cls| <= w aw [(2 om E_om + E_om^2) ce + om^2 E_ce] + 10u |cls|.
  * gradient g = w aw (T2 - s T1), s = 2t - 1, T1 = 2 om q ce, q = p (1 - p), T2 = om^2 (p - t): (1 - p) and (p - t) are absolute
    errors again, E_q = 7u p + 7u q, E_pt = 7u:
        dT1 <= 2 [E_om q ce + om E_q ce + om q E_ce + E_om E_q ce] + 6u |T1|
        dT2 <= (2 om E_om + E_om^2) |p - t| + (om + E_om)^2 E_pt + 4u |T2|
        |d g| <= w aw (dT1 + dT2) + 10u w aw (|T1| + |T2|), then x w_cls / batch: + 2u |g|.
  * at x == 0 exactly the autograd of clamp + abs returns the subgradient 1 - t instead of the derivative p - t = 0.5 - t of this
    smooth function; the fp64 reference is therefore taken at x = 1e-300 there (the same value to 1e-300, differentiable).
box term (positives only, rw = 1 / num_pos, knee k = 1 / sigma^2, fp32(k) in the kernel, k in the fp64 reference):
  * x..h: d = b - t is one rounding, E_d = u |d|; the gradient f'(d) = sigma^2 d or sign(d) is continuous at the knee, so a residual
    within E_d (or within |fp32(k) - k| <= u k) of the knee changes it by <= sigma^2 (E_d + u k):
        |d g_j| <= rw (sigma^2 (E_d + u k)) w_loc / batch + 4u |g_j|
  * yaw: d = sin a cos b - cos a sin b (4 transcendental 4u, two products, the subtraction -- or one fma):
        E_d = 12u (|sa cb| + |ca sb|) + u |d|,  chain = cos a cos b + sin a sin b,  E_c = 12u (|ca cb| + |sa sb|) + u
        |d g_6| <= rw (sigma^2 (E_d + u k) |chain| + min(sigma^2 |d|, 1) E_c + sigma^2 E_d E_c) w_loc / batch + 4u |g_6|
    value per component: rw (min(sigma^2 |d|, 1) E_d + sigma^2 E_d^2) + 4u |loc_j|.
direction term (2-way softmax CE, target from the fp32 sum rot_gt = t_6 + a_6 compared with fp32(dir_offset), as the reference's
fp32 tensors do; the fp64 reference takes the same fp32 target): l_min - m rounds (u |l0 - l1|), expf 4u, the sum, logf 4u, m + log
and lse - l_t (cancellation of operands of size |m|):
        value:    E = rw (2u (|l0| + |l1|) + 12u + 2u ce_dir)
        gradient: |d g_i| <= rw ((14u + 2u |l0 - l1|) s_i + 4u [i = target]) w_dir / batch + 4u |g_i|
per-frame sums: each partial sum the kernel forms is a sum of a subset of the terms through at most D additions: <= 4 grid-stride
steps per thread at A <= 74 * 256 * 4, + 7 box components, 5 shuffle levels, 8 warps, 74 block partials => D = 98 and
        |d S| <= sum_a E_a + D u sum_a |term_a|.
The iou and padding channels of the gradient are written as exact zeros; counts are exact.

IoU-prediction loss (sessd_iou_pred_loss, iou_pred_loss_kernel in csrc/iou3d.cu), per positive, against iou_pred_ref
---------------------------------------------------------------------------------------------------------------------
iou_pred_ref decodes the prediction and the target in fp64 (second_box_decode), builds the BEV rectangles [x -+ w/2, y -+ l/2] rotated
clockwise by r as rb_spin does (not the ODIoU corner convention), takes their exact convex intersection (_od_inter_area), the height
overlap about the z centres and the union clamped at 1e-7, then smooth-L1 of the iou head value h against the constant 2 IoU - 1 with
weight rw = 1 / max(num_pos, 1); the gradient into channel 20 + r is scaled by w_iou / B.  With R = the largest |x|, |y| of the two
centres and the anchor's plus half the larger BEV diagonal:
  * decode: diag = sqrtf(l^2 + w^2) (2 products, the add, sqrtf: 3u), x = e diag + x_a: 4u |e diag| + u |x| <= 9u R; w = expf(e) w_a:
    5u relative; r = e + r_a: u |r|.
  * corners: x -+ w/2, the recomputed centre, p - c, cosf / sinf (2 ulp each, argument error u |r|), two products, the sum and + c: the
    absolute error of every corner coordinate is a cancellation between centres up to ~70 m and offsets of 0.25-2 m, counted on R:
        E_p = u R (24 + |r_q| + |r_g|).
  * area: the intersection of two convex polygons whose edges each move by <= E_p changes by <= E_p per unit length of its boundary, and
    that boundary is no longer than the smaller perimeter P_min; a crossing of two nearly parallel edges is ill-conditioned along the
    edges (~ 1 / sin of the angle) but moves inside the thin wedge between them, so it stays within the same band.  rb_inside admits a
    corner up to m = 1e-5 outside the other rectangle (its margin), which adds at most m x P_min -- counted only where some corner lies
    within m + 2 E_p of the other rectangle's boundary.  The shoelace fan sums <= 24 cross products of differences <= D (the smaller
    BEV diagonal): 72u D^2.
        E_A = (2 E_p + [near] m) P_min + 72u D^2.
  * height: z -+ h/2 per box (decode of z and h, the half, the add): E_zb = u (2 |z| + |z_a| + 3h); E_ih = 2 max(E_zb) + u ih.
  * ov3 = ov ih: E_ov3 = E_A ih + ov E_ih + E_A E_ih + u ov ih; volumes (three 5u dimensions, two products): 17u v; the union's two adds:
    E_Un = 19u (v_q + v_g) + E_ov3; the quotient: E_I = (E_ov3 + IoU E_Un) / (Un - E_Un) + u IoU; the target 2 IoU - 1: E_t = 2 E_I + u.
  * smooth-L1 of d = h - t: E_d = E_t + u |d|.  The gradient sigma^2 d or sign(d) is continuous at the knee k = 1 / sigma^2 (fp32(k) in
    the kernel: + u k) but its sign flips at d = 0, so the bar is absolute:
        |d g| <= rw (w_iou / B) sigma^2 (E_d + u k) + 4u |g|,     value: rw (min(sigma^2 |d|, 1) E_d + sigma^2 E_d^2 + u k) + 4u |f|.
  * per-frame sums: <= ceil(A / 18 944) grid-stride steps per thread (74 CTAs x 256), 5 shuffle levels, 8 warps, 74 block partials:
        |d S| <= sum E_f + (ceil(A / 18 944) + 87) u sum |f|.
A disjoint pair or a pair without height overlap has IoU exactly 0 in both fp32 and fp64 (target exactly -1); an encoded dimension of
-104 underflows expf to a zero-size box (target -1 up to the shoelace term).  The fp32 twin iou_pred_emul (the C oracle's decode and
overlap) passes these bounds; IP_MUTANTS are the planted mistakes each of which fails at least one crafted case.

ODIoU: odiou_ref (fp64 restatement of odiou.cuh) and odiou_bounds, derived in its docstring.  The optimiser kernels' references and
bounds sit beside their tests (tests/test_gpu_train_ops.py).
"""
import numpy as np
import torch

from oracle import loss_ref

U = 2.0 ** -24
D_SUM = 98


class HeadCfg:
    def __init__(self, alpha=0.25, sigma=3.0, dir_offset=0.0, pos_cls_weight=1.0, neg_cls_weight=1.0, w_cls=1.0, w_loc=2.0, w_dir=0.2):
        self.alpha, self.sigma, self.dir_offset = alpha, sigma, dir_offset
        self.pos_cls_weight, self.neg_cls_weight = pos_cls_weight, neg_cls_weight
        self.w_cls, self.w_loc, self.w_dir = w_cls, w_loc, w_dir


def _split(head):
    B, P, S = head.shape
    return head[..., :14].reshape(B, 2 * P, 7), head[..., 14:16].reshape(B, 2 * P), head[..., 16:20].reshape(B, 2 * P, 2)


def dir_target(anchors, targets, dir_offset):
    """direction class of every anchor as the reference's fp32 tensors compute it: (fp32(t_6 + a_6) - fp32(offset)) > 0"""
    rot = targets[..., 6].astype(np.float32) + anchors[None, :, 6].astype(np.float32)
    return (rot - np.float32(dir_offset)) > np.float32(0)


# ------------------------------------------------------------------------------------------------ fp64 reference
def head_loss_ref(head, anchors, labels, targets, cfg):
    """fp64 autograd through oracle/loss_ref.  Returns (losses [B, 5] = cls, loc, dir, cls_pos, cls_neg, grad [B, P, S]) as float64 numpy:
    grad is d/d head of (w_cls cls + w_loc loc + w_dir dir) summed over frames / batch."""
    B = head.shape[0]
    h0 = torch.from_numpy(head.astype(np.float64))
    x0 = h0[..., 14:16]
    h0[..., 14:16] = torch.where(x0 == 0, torch.full_like(x0, 1e-300), x0)          # see the module docstring (x == 0)
    h = h0.requires_grad_(True)
    box, cls, dr = loss_ref.split_head(h)
    lab = torch.from_numpy(labels.astype(np.int64))
    tg = torch.from_numpy(targets.astype(np.float64))
    cls_w, reg_w, cared = loss_ref.loss_weights(lab, cfg.pos_cls_weight, cfg.neg_cls_weight, torch.float64)
    t = (lab * cared.type_as(lab)).double()
    c = loss_ref.sigmoid_focal(cls, t, cls_w, cfg.alpha)
    loc = loss_ref.smooth_l1_sin(box, tg, reg_w, cfg.sigma)
    tgt = torch.from_numpy(dir_target(anchors, targets, cfg.dir_offset).astype(np.int64))
    dce = torch.nn.functional.cross_entropy(dr.reshape(-1, 2), tgt.reshape(-1), reduction="none").view(reg_w.shape) * reg_w
    total = (cfg.w_cls * c.sum() + cfg.w_loc * loc.sum() + cfg.w_dir * dce.sum()) / B
    total.backward()
    pos, neg = (lab > 0).double(), (lab == 0).double()
    L = torch.stack([c.sum(1), loc.sum((1, 2)), dce.sum(1), (c * pos).sum(1), (c * neg).sum(1)], 1)
    return L.detach().numpy(), h.grad.numpy().copy()


# ------------------------------------------------------------------------------------------------ bounds
def head_loss_bounds(head, anchors, labels, targets, cfg):
    """(loss bound [B, 5], gradient bound [B, P, S]) of the module docstring, evaluated on fp64 values of the inputs."""
    B, P, S = head.shape
    A = 2 * P
    u = U
    box, x, dr = (a.astype(np.float64) for a in _split(head))
    tg = targets.astype(np.float64)
    pos, neg = labels > 0, labels == 0
    npos = np.maximum(pos.sum(1), 1).astype(np.float64)[:, None]
    t = pos.astype(np.float64)
    w = np.where(pos, cfg.pos_cls_weight, np.where(neg, cfg.neg_cls_weight, 0.0)) / npos
    aw = np.where(pos, cfg.alpha, 1.0 - cfg.alpha)
    with np.errstate(over="ignore"):
        p = 1.0 / (1.0 + np.exp(-x))
        q = 1.0 / (1.0 + np.exp(x))
    om = np.where(pos, q, p)                                          # 1 - pt, evaluated without cancellation
    L = np.log1p(np.exp(-np.abs(x)))
    ce = np.maximum(x, 0) - x * t + L
    E_om = 8 * u
    E_ce = u * np.abs(x) + 10 * u * L + 2 * u * ce
    cls = om * om * aw * ce * w
    cls_err = w * aw * ((2 * om * E_om + E_om ** 2) * ce + om * om * E_ce) + 10 * u * np.abs(cls)
    pq = p * q
    E_q = 7 * u * p + 7 * u * pq
    T1 = 2 * om * pq * ce
    T2 = om * om * (p - t)
    dT1 = 2 * (E_om * pq * ce + om * E_q * ce + om * pq * E_ce + E_om * E_q * ce) + 6 * u * np.abs(T1)
    dT2 = (2 * om * E_om + E_om ** 2) * np.abs(p - t) + (om + E_om) ** 2 * 7 * u + 4 * u * np.abs(T2)
    g_cls = w * aw * (T2 - (2 * t - 1) * T1)
    gb_cls = (w * aw * (dT1 + dT2) + 10 * u * w * aw * (np.abs(T1) + np.abs(T2))) * cfg.w_cls / B + 2 * u * np.abs(g_cls) * cfg.w_cls / B

    rw = pos / npos
    s2, k = cfg.sigma ** 2, 1.0 / cfg.sigma ** 2
    d = box[..., :6] - tg[..., :6]
    Ed = u * np.abs(d)
    fp = np.where(np.abs(d) <= k, s2 * d, np.sign(d))
    loc_terms = np.where(np.abs(d) <= k, 0.5 * s2 * d * d, np.abs(d) - 0.5 * k) * rw[..., None]
    loc_err = rw[..., None] * (np.minimum(s2 * np.abs(d), 1) * Ed + s2 * Ed ** 2) + 4 * u * np.abs(loc_terms)
    gb_box = np.zeros((B, A, 7))
    gb_box[..., :6] = rw[..., None] * s2 * (Ed + u * k) * cfg.w_loc / B + 4 * u * np.abs(fp * rw[..., None]) * cfg.w_loc / B
    sa, ca, sb, cb = np.sin(box[..., 6]), np.cos(box[..., 6]), np.sin(tg[..., 6]), np.cos(tg[..., 6])
    d6 = sa * cb - ca * sb
    chain = ca * cb + sa * sb
    Ed6 = 12 * u * (np.abs(sa * cb) + np.abs(ca * sb)) + u * np.abs(d6)
    Ec = 12 * u * (np.abs(ca * cb) + np.abs(sa * sb)) + u
    fp6 = np.where(np.abs(d6) <= k, s2 * d6, np.sign(d6))
    g6 = fp6 * chain * rw
    gb_box[..., 6] = rw * (s2 * (Ed6 + u * k) * np.abs(chain) + np.minimum(s2 * np.abs(d6), 1) * Ec + s2 * Ed6 * Ec) * cfg.w_loc / B \
        + 4 * u * np.abs(g6) * cfg.w_loc / B
    t6 = np.where(np.abs(d6) <= k, 0.5 * s2 * d6 * d6, np.abs(d6) - 0.5 * k) * rw
    loc_err6 = rw * (np.minimum(s2 * np.abs(d6), 1) * Ed6 + s2 * Ed6 ** 2) + 4 * u * np.abs(t6)

    tgt = dir_target(anchors, targets, cfg.dir_offset)
    l0, l1 = dr[..., 0], dr[..., 1]
    m = np.maximum(l0, l1)
    lse = m + np.log(np.exp(l0 - m) + np.exp(l1 - m))
    ce_dir = lse - np.where(tgt, l1, l0)
    dir_err = rw * (2 * u * (np.abs(l0) + np.abs(l1)) + 12 * u + 2 * u * ce_dir)
    sm = np.stack([np.exp(l0 - lse), np.exp(l1 - lse)], -1)
    onehot = np.stack([~tgt, tgt], -1).astype(np.float64)
    g_dir = (sm - onehot) * rw[..., None]
    gb_dir = rw[..., None] * ((14 * u + 2 * u * np.abs(l0 - l1))[..., None] * sm + 4 * u * onehot) * cfg.w_dir / B \
        + 4 * u * np.abs(g_dir) * cfg.w_dir / B

    gb = np.zeros((B, P, S))
    gb[..., :14] = gb_box.reshape(B, P, 14)
    gb[..., 14:16] = gb_cls.reshape(B, P, 2)
    gb[..., 16:20] = gb_dir.reshape(B, P, 4)
    dir_terms = ce_dir * rw
    mags = [np.abs(cls), np.abs(loc_terms).sum(-1) + np.abs(t6), np.abs(dir_terms)]
    errs = [cls_err, loc_err.sum(-1) + loc_err6, dir_err]
    lb = np.zeros((B, 5))
    for j in range(3):
        lb[:, j] = errs[j].sum(1) + D_SUM * u * mags[j].sum(1)
    for j, sel in ((3, pos), (4, neg)):
        lb[:, j] = (errs[0] * sel).sum(1) + D_SUM * u * (mags[0] * sel).sum(1)
    return lb, gb


# ------------------------------------------------------------------------------------------------ fp32 emulation of headloss_kernel
MUTANTS = ("dir_ge", "no_batch_div", "no_npos_clamp", "wrong_slot", "wrong_frame")


def head_loss_emul(head, anchors, labels, targets, cfg, mutant=None):
    """numpy fp32, the kernel's operation order (per-frame sums by np.sum in fp32: within the D_SUM model).  `mutant` plants one of
    MUTANTS.  Returns (losses [B, 8] float32, grad [B, P, S] float32)."""
    f = np.float32
    B, P, S = head.shape
    A = 2 * P
    box, x, dr = _split(head)
    if mutant == "wrong_slot":                                        # reads the logit of the other anchor of the pixel
        x = x.reshape(B, P, 2)[..., ::-1].reshape(B, A)
    pos, neg = labels > 0, labels == 0
    cnt = pos.sum(1).astype(f)
    pos_norm = cnt if mutant == "no_npos_clamp" else np.maximum(cnt, f(1))
    inv_b = f(1) if mutant == "no_batch_div" else f(1) / f(B)
    pn = pos_norm[:, None]
    t = pos.astype(f)
    one = f(1)
    with np.errstate(over="ignore", divide="ignore", invalid="ignore"):
        w = np.where(pos, f(cfg.pos_cls_weight), np.where(neg, f(cfg.neg_cls_weight), f(0))).astype(f) / pn
        p = one / (one + np.exp(-x))
        ce = np.maximum(x, f(0)) - x * t + np.log1p(np.exp(-np.abs(x)))
        pt = t * p + (one - t) * (one - p)
        om = one - pt
        al = f(cfg.alpha)
        aw = t * al + (one - t) * (one - al)
        cls = om * om * aw * ce * w
        g_cls = w * aw * (f(-2) * om * (f(2) * t - one) * p * (one - p) * ce + om * om * (p - t))
        rw = np.where(pos, one / pn, f(0)).astype(f)
        sig = f(cfg.sigma)
        inv_s2 = one / (sig * sig)
        d = np.empty_like(box)
        chain = np.ones_like(box)
        d[..., :6] = box[..., :6] - targets[..., :6]
        sa, ca, sb, cb = np.sin(box[..., 6]), np.cos(box[..., 6]), np.sin(targets[..., 6]), np.cos(targets[..., 6])
        d[..., 6] = sa * cb - ca * sb
        chain[..., 6] = ca * cb + sa * sb
        ad = np.abs(d)
        small = ad <= inv_s2
        sd = ad * sig
        loc = np.where(small, f(0.5) * sd * sd, ad - f(0.5) * inv_s2) * rw[..., None]
        g_box = np.where(small, sig * sig * d, np.sign(d).astype(f)) * chain * rw[..., None]
        rot = targets[..., 6] + anchors[None, :, 6]
        cls_t = (rot - f(cfg.dir_offset)) >= f(0) if mutant == "dir_ge" else (rot - f(cfg.dir_offset)) > f(0)
        l0, l1 = dr[..., 0], dr[..., 1]
        m = np.maximum(l0, l1)
        e0, e1 = np.exp(l0 - m), np.exp(l1 - m)
        lse = m + np.log(e0 + e1)
        dce = (lse - np.where(cls_t, l1, l0)) * rw
        g_dir = np.stack([(e0 / (e0 + e1) - np.where(cls_t, f(0), one)) * rw, (e1 / (e0 + e1) - np.where(cls_t, one, f(0))) * rw], -1)
    g_box = np.where(pos[..., None], g_box, f(0))
    g_dir = np.where(pos[..., None], g_dir, f(0))
    loc = np.where(pos[..., None], loc, f(0))
    dce = np.where(pos, dce, f(0))
    grad = np.zeros((B, P, S), f)
    grad[..., :14] = (g_box * f(cfg.w_loc) * inv_b).reshape(B, P, 14)
    grad[..., 14:16] = (g_cls * f(cfg.w_cls) * inv_b).reshape(B, P, 2)
    grad[..., 16:20] = (g_dir * f(cfg.w_dir) * inv_b).reshape(B, P, 4)
    losses = np.zeros((B, 8), f)
    losses[:, 0] = cls.sum(1, dtype=f)
    losses[:, 1] = loc.sum((1, 2), dtype=f)
    losses[:, 2] = dce.sum(1, dtype=f)
    losses[:, 3] = np.where(pos, cls, f(0)).sum(1, dtype=f)
    losses[:, 4] = np.where(neg, cls, f(0)).sum(1, dtype=f)
    losses[:, 6] = cnt
    losses[:, 7] = neg.sum(1)
    if mutant == "wrong_frame":
        losses[:, :6] = np.roll(losses[:, :6], 1, 0)
    return losses, grad


def head_loss_violations(losses, grad, ref_losses, ref_grad, lb, gb):
    """(worst ratio |got - ref| / bound over losses, over the gradient); non-finite results count as infinite"""
    def ratio(got, ref, bound):
        got = got.astype(np.float64)
        err = np.abs(got - ref)
        r = np.where(err == 0, 0.0, err / np.maximum(bound, 1e-300))
        r[~np.isfinite(got)] = np.inf
        return float(r.max()) if r.size else 0.0
    return ratio(losses[:, :5], ref_losses, lb), ratio(grad, ref_grad, gb)


# ------------------------------------------------------------------------------------------------ crafted cases
LOGITS = np.float32([0, 1e-3, -1e-3, 8, -8, 20, -20, 88, -88, 100, -100])
KNEE = np.float32(1.0 / 9.0)


def _anchors(A):
    from oracle import anchors as oa
    anc = oa.create_anchors_3d_range().reshape(-1, 7)
    return np.ascontiguousarray(anc[:A])


def make_head_case(B, A, stride, seed, cfg, frames=None):
    """head [B, A/2, stride], anchors [A, 7], labels [B, A], targets [B, A, 7] with the crafted values of the module's test plan.
    frames: per frame one of "mixed" (default), "no_pos", "ignored", or an int number of positives (ragged counts)."""
    rng = np.random.default_rng(seed)
    P = A // 2
    anc = _anchors(A)
    head = (rng.standard_normal((B, P, stride)) * 0.5).astype(np.float32)
    labels = np.zeros((B, A), np.int32)
    targets = (rng.standard_normal((B, A, 7)) * 0.4).astype(np.float32)
    frames = frames or ["mixed"] * B
    for b, kind in enumerate(frames):
        if kind == "no_pos":
            labels[b] = np.where(rng.random(A) < 0.1, -1, 0)
        elif kind == "ignored":
            labels[b] = -1
        elif isinstance(kind, int):
            labels[b] = np.where(rng.random(A) < 0.1, -1, 0)
            labels[b, rng.choice(A, min(kind, A), replace=False)] = 1
        else:
            labels[b] = rng.choice([-1, 0, 1], A, p=[0.1, 0.7, 0.2])
    box, x, dr = (a.copy() for a in _split(head))
    # logits: every crafted value on every label, cycling through the anchors
    idx = np.arange(A)
    x[:] = np.where(idx % 3 == 0, LOGITS[idx // 3 % len(LOGITS)], x)
    knees = np.float32([0, KNEE, -KNEE, np.nextafter(KNEE, np.float32(1)), np.nextafter(KNEE, np.float32(0)),
                        -np.nextafter(KNEE, np.float32(1)), -np.nextafter(KNEE, np.float32(0))])
    off32 = np.float32(cfg.dir_offset)
    for b in range(B):
        pa = np.nonzero(labels[b] > 0)[0]
        for n, a in enumerate(pa):
            kind = n % 5
            if kind == 0:                                             # box residuals at / next to the smooth-L1 knee, and 0
                targets[b, a, :6] = 0
                box[b, a, :6] = knees[(n // 5 + np.arange(6)) % len(knees)]
            elif kind == 1:                                           # predicted yaw = target yaw + pi
                box[b, a, 6] = targets[b, a, 6] + np.float32(np.pi)
            elif kind == 2:                                           # direction target exactly on the boundary, or 1 ulp off it
                want = [off32, np.nextafter(off32, np.float32(1)), np.nextafter(off32, np.float32(-1))][n // 5 % 3]
                targets[b, a, 6] = want - anc[a, 6]                   # exact on the yaw-0 anchors, within an ulp on the others
            elif kind == 3:                                           # prediction == target: d = 0 (yaw: sin/cos product cancellation)
                box[b, a] = targets[b, a]
    out = head.copy()
    out[..., :14] = box.reshape(B, P, 14)
    out[..., 14:16] = x.reshape(B, P, 2)
    out[..., 16:20] = dr.reshape(B, P, 4)
    return out, anc, labels, targets


def head_cases():
    """(name, head, anchors, labels, targets, cfg) of the crafted head-loss cases"""
    out = []
    d = HeadCfg()
    nd = HeadCfg(alpha=0.3, pos_cls_weight=1.7, neg_cls_weight=0.6, w_cls=1.3, w_loc=0.7, w_dir=0.45)
    out.append(("a2_s24",) + make_head_case(2, 2, 24, 1, d, ["mixed", "ignored"]) + (d,))
    out.append(("a258_s22",) + make_head_case(3, 258, 22, 2, nd) + (nd,))
    out.append(("a258_s32_off0",) + make_head_case(2, 258, 32, 3, d) + (d,))
    off = HeadCfg(dir_offset=0.78)
    out.append(("a258_s24_off078",) + make_head_case(2, 258, 24, 4, off) + (off,))
    out.append(("a37890_s24_ragged5",) + make_head_case(5, 74 * 256 * 2 + 2, 24, 5, nd, [0, 3, "no_pos", 700, "ignored"]) + (nd,))
    out.append(("a70400_s32",) + make_head_case(2, 70400, 32, 6, off, ["mixed", 1]) + (off,))
    return out


# ------------------------------------------------------------------------------------------------ ODIoU: fp64 restatement of odiou.cuh
ODIOU_HALF_PI = 3.1415926 / 2.0                                   # the reference's literal (odious.py:597-648)


def _od_corners(x, y, w, l, r):
    cs, sn = torch.cos(r), torch.sin(r)
    dxcos, dxsin, dycos, dysin = w * cs * 0.5, w * sn * 0.5, l * cs * 0.5, l * sn * 0.5
    return [(-dxcos - dysin + x, dxsin - dycos + y), (-dxcos + dysin + x, dxsin + dycos + y),
            (dxcos + dysin + x, -dxsin + dycos + y), (dxcos - dysin + x, -dxsin - dycos + y)]


def _od_inter_area(clip, subj, zero):
    """Sutherland-Hodgman clip of subj against the clockwise rectangle clip, shoelace area (torch or numpy scalars)"""
    a = list(subj)
    for e in range(4):
        if not a:
            break
        p0, p1 = clip[e], clip[(e + 1) % 4]
        ex, ey = p1[0] - p0[0], p1[1] - p0[1]
        b = []
        for i in range(len(a)):
            s, t = a[i], a[(i + 1) % len(a)]
            cs = ex * (s[1] - p0[1]) - ey * (s[0] - p0[0])
            ct = ex * (t[1] - p0[1]) - ey * (t[0] - p0[0])
            ins, int_ = cs.item() <= 0.0, ct.item() <= 0.0
            if ins:
                b.append(s)
            if ins != int_:
                k = cs / (cs - ct)
                b.append((s[0] + k * (t[0] - s[0]), s[1] + k * (t[1] - s[1])))
        a = b
    if len(a) < 3:
        return zero
    s2 = zero
    for i in range(len(a)):
        p, q = a[i], a[(i + 1) % len(a)]
        s2 = s2 + (p[0] * q[1] - q[0] * p[1])
    return abs(s2) * 0.5


def _od_mbr_diag(pts, zero):
    """diagonal of the minimum-area rectangle aligned with a convex-hull edge of the 8 points (monotone chain on the values)"""
    v = [(p[0].item(), p[1].item()) for p in pts]
    idx = sorted(range(8), key=lambda i: v[i])

    def cross(o, a, b):
        return (v[a][0] - v[o][0]) * (v[b][1] - v[o][1]) - (v[a][1] - v[o][1]) * (v[b][0] - v[o][0])
    hull = []
    for i in idx:
        while len(hull) >= 2 and cross(hull[-2], hull[-1], i) <= 0:
            hull.pop()
        hull.append(i)
    lower = len(hull) + 1
    for i in reversed(idx[:-1]):
        while len(hull) >= lower and cross(hull[-2], hull[-1], i) <= 0:
            hull.pop()
        hull.append(i)
    hull.pop()
    h = len(hull)
    best, best_area, areas = zero, np.inf, []
    if h < 2:
        return best, areas
    for e in range(h):
        p, q = pts[hull[e]], pts[hull[(e + 1) % h]]
        ang = torch.abs(torch.fmod(torch.atan2(q[1] - p[1], q[0] - p[0]), ODIOU_HALF_PI))
        r00, r01, r10 = torch.cos(ang), torch.cos(ang - ODIOU_HALF_PI), torch.cos(ang + ODIOU_HALF_PI)
        rx = [r00 * pts[k][0] + r01 * pts[k][1] for k in hull]
        ry = [r10 * pts[k][0] + r00 * pts[k][1] for k in hull]
        mnx = mxx = rx[0]
        mny = mxy = ry[0]
        for k in range(1, h):
            mnx = rx[k] if float(rx[k]) < float(mnx) else mnx
            mxx = rx[k] if float(rx[k]) > float(mxx) else mxx
            mny = ry[k] if float(ry[k]) < float(mny) else mny
            mxy = ry[k] if float(ry[k]) > float(mxy) else mxy
        dx, dy = mxx - mnx, mxy - mny
        area = float(dx) * float(dy)
        areas.append(area)
        if area < best_area:
            best_area, best = area, torch.sqrt(dx * dx + dy * dy)
    return best, areas


def odiou_ref(gboxes, qboxes):
    """fp64 restatement of odiou_pair (odiou.cuh) with autograd: (value [n], d value / d q [n, 7], unique [n] bool).  unique is False
    where a second hull edge's bounding rectangle is within 1e-4 relative of the minimum: the minimiser is then not unique within
    rounding and an fp32 evaluation may take the other edge (same value, different gradient)."""
    n = len(gboxes)
    val, grad, uniq = np.zeros(n), np.zeros((n, 7)), np.ones(n, bool)
    for i in range(n):
        gi = np.asarray(gboxes[i], np.float64)
        q = torch.tensor(np.asarray(qboxes[i], np.float64), requires_grad=True)
        if not ((gi[3:6] > 0).all() and bool((q[3:6] > 0).all())):
            continue
        g = [torch.tensor(float(np.clip(c, -200.0, 200.0)), dtype=torch.float64) for c in gi]
        qc = torch.clamp(q, -200.0, 200.0)
        qq = [qc[j] for j in range(7)]
        zero = qc.sum() * 0.0
        angle = 1.25 * (1.0 - torch.abs(torch.cos(qq[6] - g[6])))
        cg = _od_corners(g[0], g[1], g[3], g[4], g[6])
        cq = _od_corners(qq[0], qq[1], qq[3], qq[4], qq[6])
        inter = _od_inter_area(cg, cq, zero)
        center2 = (g[0] - qq[0]) ** 2 + (g[1] - qq[1]) ** 2 + (g[2] - qq[2]) ** 2
        diag, areas = _od_mbr_diag(cg + cq, zero)
        top = qq[2] + 0.5 * qq[5] if float(qq[2] + 0.5 * qq[5]) < float(g[2] + 0.5 * g[5]) else g[2] + 0.5 * g[5]
        bot = qq[2] - 0.5 * qq[5] if float(qq[2] - 0.5 * qq[5]) > float(g[2] - 0.5 * g[5]) else g[2] - 0.5 * g[5]
        ih = top - bot
        if float(ih) < 0:
            ih = zero
        diag3 = diag * diag + ih * ih + 1e-7
        inc = ih * inter
        iou = inc / (g[3] * g[4] * g[5] + qq[3] * qq[4] * qq[5] - inc)
        od = 1.0 - iou + center2 / diag3 + angle
        od.backward()
        val[i], grad[i] = float(od), q.grad.numpy()
        a = np.sort(np.asarray(areas))
        uniq[i] = len(a) < 2 or a[1] - a[0] > 1e-4 * a[0]
    return val, grad, uniq


ODIOU_C_VAL = 32.0
ODIOU_C_GRAD = 64.0


def odiou_bounds(gboxes, qboxes, grad_ref):
    """fp32 evaluation of odiou_pair (device kernel or host twin) vs odiou_ref, per pair: (value bound [n], gradient bound [n]; the
    gradient bound applies to each of the 7 components).

    The template works in absolute coordinates.  With R = the largest |x|, |y| of the two centres plus half the larger BEV diagonal and
    S = the smallest BEV side of the two boxes, every corner, clip vertex and rotated hull point carries an absolute error of order u R
    (sin / cos 4u on terms <= R, two adds), and the shoelace sum over <= 8 clip vertices forms 16 products of size <= R^2 that cancel to
    an area of size >= S^2 when the boxes overlap: <= 16 product roundings + 16 additions = 32 u R^2.  The mbr diagonal and the centre
    term are ratios of the same coordinate differences, the IoU a ratio of the area to a union >= S^2 h; every term of odiou is O(1), so
        |d odiou| <= ODIOU_C_VAL u (R / S)^2.
    The forward-mode partials run the same operation sequence on the partials of the same coordinates: each picks up the value's
    relative (R / S)^2 cancellation on its own magnitude, and a differentiated length 1 / S more,
        |d g_j| <= ODIOU_C_GRAD u (R / S)^2 (max_j |g_j| + 1 / S),
    the constant doubled over the value's for the clip's intersection points (u = cs / (cs - ct) divides by the crossing's sine).
    Where the hull's minimising edge is not unique within rounding (odiou_ref's `unique`), fp32 may take another edge: value only."""
    g = np.asarray(gboxes, np.float64)
    q = np.asarray(qboxes, np.float64)
    gc, qc = np.clip(g, -200, 200), np.clip(q, -200, 200)
    R = np.maximum(np.abs(gc[:, :2]).max(1), np.abs(qc[:, :2]).max(1)) \
        + 0.5 * np.hypot(np.maximum(gc[:, 3], qc[:, 3]), np.maximum(gc[:, 4], qc[:, 4]))
    S = np.minimum(np.minimum(gc[:, 3], gc[:, 4]), np.minimum(qc[:, 3], qc[:, 4]))
    k = (R / S) ** 2
    return ODIOU_C_VAL * U * k, ODIOU_C_GRAD * U * k * (np.abs(grad_ref).max(1) + 1.0 / S)


# ------------------------------------------------------------------------------------------------ IoU prediction (iou_pred_loss_kernel)
IP_CTA_SPAN = 74 * 256                                            # anchors one grid-stride step of iou_pred_loss_kernel covers
IP_MARGIN = 1e-5                                                  # rb_inside's margin (rotbox.cuh)


def _ip_decode64(e, an):
    """second_box_decode in fp64 of fp32 encodings e [n, 7] against fp32 anchors an [n, 7]"""
    e, an = e.astype(np.float64), an.astype(np.float64)
    diag = np.sqrt(an[:, 4] ** 2 + an[:, 3] ** 2)
    return np.stack([e[:, 0] * diag + an[:, 0], e[:, 1] * diag + an[:, 1], e[:, 2] * an[:, 5] + an[:, 2], np.exp(e[:, 3]) * an[:, 3],
                     np.exp(e[:, 4]) * an[:, 4], np.exp(e[:, 5]) * an[:, 5], e[:, 6] + an[:, 6]], 1)


def _ip_corners(b):
    """the BEV rectangle [x -+ w/2, y -+ l/2] rotated clockwise by r about its centre (rb_spin), corners in rb_spin's order"""
    x, y, w, l, r = (np.float64(b[k]) for k in (0, 1, 3, 4, 6))
    c, s = np.cos(r), np.sin(r)
    out = []
    for px, py in ((-w / 2, -l / 2), (w / 2, -l / 2), (w / 2, l / 2), (-w / 2, l / 2)):
        out.append((px * c + py * s + x, -px * s + py * c + y))
    return out


def _ip_outside(p, b):
    """Chebyshev distance by which point p lies outside rectangle b in b's own frame (negative: inside), as rb_inside measures it"""
    c, s = np.cos(b[6]), np.sin(b[6])
    dx, dy = p[0] - b[0], p[1] - b[1]
    lx, ly = dx * c - dy * s, dx * s + dy * c                     # undo the clockwise rotation
    return max(abs(lx) - b[3] / 2, abs(ly) - b[4] / 2)


def iou3d_aligned_ref(q, g):
    """fp64 aligned 3-D IoU of box rows q, g [n, 7] (decoded): exact convex BEV intersection of the rb_spin rectangles, the height
    overlap about the z centres, the union clamped at 1e-7 (iou3d_utils.py:197-252).  Returns (iou [n], bev overlap [n], ih [n])."""
    n = len(q)
    iou, ov, ih = np.zeros(n), np.zeros(n), np.zeros(n)
    for i in range(n):
        cg = _ip_corners(g[i])[::-1]                               # rb_spin's order is counter-clockwise; the clip wants clockwise
        ov[i] = _od_inter_area(cg, _ip_corners(q[i]), np.float64(0))
        ih[i] = max(min(q[i, 2] + q[i, 5] / 2, g[i, 2] + g[i, 5] / 2) - max(q[i, 2] - q[i, 5] / 2, g[i, 2] - g[i, 5] / 2), 0.0)
        ov3 = ov[i] * ih[i]
        iou[i] = ov3 / max(q[i, 3] * q[i, 4] * q[i, 5] + g[i, 3] * g[i, 4] * g[i, 5] - ov3, 1e-7)
    return iou, ov, ih


def _ip_positives(head, labels):
    """(frame, anchor, slot) index arrays of the positives, in frame-major ascending-anchor order"""
    b, a = np.nonzero(labels > 0)
    return b, a, a % 2


def iou_pred_ref(head, anchors, labels, targets, sigma=3.0, w_iou=1.0):
    """fp64 reference of sessd_iou_pred_loss on the fp32 inputs: (sums [B], grad [B, P, S], per-positive details for iou_pred_bounds).
    grad holds d (w_iou * sum / B) / d head in the iou channels 20 + r of the positives and zero elsewhere."""
    B, P, S = head.shape
    bi, ai, ri = _ip_positives(head, labels)
    an = anchors[ai]
    e = np.stack([head[bi, ai // 2, 7 * ri + k] for k in range(7)], 1)
    q, g = _ip_decode64(e, an), _ip_decode64(targets[bi, ai], an)
    iou, ov, ih = iou3d_aligned_ref(q, g)
    h = head[bi, ai // 2, 20 + ri].astype(np.float64)
    t = 2.0 * iou - 1.0
    d = h - t
    k, s2 = 1.0 / sigma ** 2, sigma ** 2
    npos = np.maximum((labels > 0).sum(1), 1).astype(np.float64)
    rw = 1.0 / npos[bi]
    f = np.where(np.abs(d) <= k, 0.5 * s2 * d * d, np.abs(d) - 0.5 * k) * rw
    fp = np.where(np.abs(d) <= k, s2 * d, np.sign(d)) * rw * w_iou / B
    sums = np.zeros(B)
    np.add.at(sums, bi, f)
    grad = np.zeros((B, P, S))
    grad[bi, ai // 2, 20 + ri] = fp
    info = dict(b=bi, a=ai, r=ri, an=an.astype(np.float64), q=q, g=g, iou=iou, ov=ov, ih=ih, d=d, f=f, fp=fp, rw=rw, sigma=sigma,
                w_iou=w_iou, B=B, A=labels.shape[1], shape=head.shape)
    return sums, grad, info


def iou_pred_bounds(info):
    """(sum bound [B], gradient bound [B, P, S]) of the module docstring's IoU-prediction section, from iou_pred_ref's details"""
    u = U
    q, g, an = info["q"], info["g"], info["an"]
    n = len(q)
    R = np.maximum.reduce([np.abs(q[:, 0]), np.abs(q[:, 1]), np.abs(g[:, 0]), np.abs(g[:, 1]), np.abs(an[:, 0]), np.abs(an[:, 1])]) \
        + 0.5 * np.maximum(np.hypot(q[:, 3], q[:, 4]), np.hypot(g[:, 3], g[:, 4]))
    Ep = u * R * (24 + np.abs(q[:, 6]) + np.abs(g[:, 6]))
    Pmin = np.minimum(2 * (q[:, 3] + q[:, 4]), 2 * (g[:, 3] + g[:, 4]))
    D2 = np.minimum(q[:, 3] ** 2 + q[:, 4] ** 2, g[:, 3] ** 2 + g[:, 4] ** 2)
    near = np.zeros(n, bool)                                      # a corner within the margin (+ rounding) of the other rectangle
    for i in range(n):
        dist = [_ip_outside(p, g[i]) for p in _ip_corners(q[i])] + [_ip_outside(p, q[i]) for p in _ip_corners(g[i])]
        near[i] = min(abs(x) for x in dist) <= IP_MARGIN + 2 * Ep[i]
    EA = (2 * Ep + np.where(near, IP_MARGIN, 0.0)) * Pmin + 72 * u * D2
    Ezb = lambda b: u * (2 * np.abs(b[:, 2]) + np.abs(an[:, 2]) + 3 * b[:, 5])           # noqa: E731
    Eih = 2 * np.maximum(Ezb(q), Ezb(g)) + u * info["ih"]
    ov, ih, iou = info["ov"], info["ih"], info["iou"]
    Eov3 = EA * ih + ov * Eih + EA * Eih + u * ov * ih
    vq, vg = q[:, 3] * q[:, 4] * q[:, 5], g[:, 3] * g[:, 4] * g[:, 5]
    Un = vq + vg - ov * ih
    EUn = 19 * u * (vq + vg) + Eov3
    EI = (Eov3 + iou * EUn) / np.maximum(Un - EUn, 1e-7) + u * iou
    Et = 2 * EI + u
    sigma, d, rw = info["sigma"], info["d"], info["rw"]
    s2, k = sigma ** 2, 1.0 / sigma ** 2
    Ed = Et + u * np.abs(d)
    fb = rw * (np.minimum(s2 * np.abs(d), 1) * Ed + s2 * Ed ** 2 + u * k) + 4 * u * np.abs(info["f"])
    gb = rw * info["w_iou"] / info["B"] * s2 * (Ed + u * k) + 4 * u * np.abs(info["fp"])
    B, A = info["B"], info["A"]
    depth = -(-A // IP_CTA_SPAN) + 5 + 8 + 74
    sb = np.zeros(B)
    np.add.at(sb, info["b"], fb + depth * u * np.abs(info["f"]))
    grad_b = np.zeros(info["shape"])
    grad_b[info["b"], info["a"] // 2, 20 + info["r"]] = gb
    return sb, grad_b


IP_MUTANTS = ("angle_neg", "wl_swap", "z_bottom", "no_batch_div", "wrong_slot", "iou_target")


def iou_pred_emul(head, anchors, labels, targets, sigma=3.0, w_iou=1.0, mutant=None):
    """fp32 twin of iou_pred_loss_kernel: the C oracle's decode and rotated BEV overlap (oracle/csrc/oracle.c, the reference's iou3d_cpu
    arithmetic), the rest in numpy fp32 in the kernel's operation order.  `mutant` plants one of IP_MUTANTS, or "no_npos_clamp".
    Returns (sums [B] float32, grad [B, P, S] float32 with the iou channels of the positives, zero elsewhere)."""
    from oracle import cpu as ocpu
    f = np.float32
    B, P, S = head.shape
    bi, ai, ri = _ip_positives(head, labels)
    an = anchors[ai]
    e = np.stack([head[bi, ai // 2, 7 * ri + k] for k in range(7)], 1)
    q, g = ocpu.box_decode(e, an), ocpu.box_decode(targets[bi, ai], an)
    two = f(2)

    def rect(b):
        x = b.copy()
        if mutant == "wl_swap":
            x[:, [3, 4]] = x[:, [4, 3]]
        if mutant == "angle_neg":
            x[:, 6] = -x[:, 6]
        return ocpu.boxes3d_to_bev(x)
    rq, rg = rect(q), rect(g)
    ov = np.array([ocpu.boxes_overlap_bev(rq[i:i + 1], rg[i:i + 1])[0, 0] for i in range(len(q))], f)
    if mutant == "z_bottom":
        lo, hi = np.maximum(q[:, 2], g[:, 2]), np.minimum(q[:, 2] + q[:, 5], g[:, 2] + g[:, 5])
    else:
        lo = np.maximum(q[:, 2] - q[:, 5] / two, g[:, 2] - g[:, 5] / two)
        hi = np.minimum(q[:, 2] + q[:, 5] / two, g[:, 2] + g[:, 5] / two)
    ov3 = ov * np.maximum(hi - lo, f(0))
    iou = ov3 / np.maximum(q[:, 3] * q[:, 4] * q[:, 5] + g[:, 3] * g[:, 4] * g[:, 5] - ov3, f(1e-7))
    target = iou if mutant == "iou_target" else two * iou - f(1)
    slot = 1 - ri if mutant == "wrong_slot" else ri
    d = head[bi, ai // 2, 20 + slot] - target
    cnt = (labels > 0).sum(1).astype(f)
    with np.errstate(divide="ignore"):
        rw_frame = f(1) / (cnt if mutant == "no_npos_clamp" else np.maximum(cnt, f(1)))
    rw = rw_frame[bi]
    sig = f(sigma)
    inv_s2 = f(1) / (sig * sig)
    ad = np.abs(d)
    small = ad <= inv_s2
    sd = ad * sig
    term = np.where(small, f(0.5) * sd * sd, ad - f(0.5) * inv_s2) * rw
    inv_b = f(1) if mutant == "no_batch_div" else f(B)
    gv = np.where(small, sig * sig * d, np.sign(d).astype(f)) * rw * f(w_iou) / inv_b
    sums = np.zeros(B, f)
    for b in range(B):
        sums[b] = term[bi == b].sum(dtype=f)
    grad = np.zeros((B, P, S), f)
    grad[bi, ai // 2, 20 + ri] = gv
    return sums, grad


def iou_pred_violations(sums, grad, ref_sums, ref_grad, sb, gb, scale=1.0):
    """(worst |got - ref| / (scale * bound) over the sums, over the iou channels of the positives); non-finite counts as infinite"""
    def ratio(got, ref, bound):
        got = got.astype(np.float64)
        err = np.abs(got - ref)
        r = np.where(err == 0, 0.0, err / np.maximum(scale * bound, 1e-300))
        r[~np.isfinite(got)] = np.inf
        return float(r.max()) if r.size else 0.0
    return ratio(sums, ref_sums, sb), ratio(grad, ref_grad, gb)


# crafted (prediction, target) pairs in decoded form, centres relative to the anchor's: (name, q [7], g [7])
def iou_pred_pairs():
    pi = np.pi
    car = [0.15, -0.2, 0.05, 1.7, 4.1, 1.5, 0.3]
    out = []
    add = lambda name, q, g: out.append((name, np.float64(q), np.float64(g)))       # noqa: E731
    add("identical", car, car)
    add("yaw_plus_pi", car[:6] + [car[6] + pi], car)
    add("yaw_plus_half_pi_wl_swapped", car[:3] + [car[4], car[3], car[5], car[6] + pi / 2], car)
    add("disjoint_bev", [6.5] + car[1:], car)                                          # target exactly -1
    add("no_height_overlap", car[:2] + [car[2] + 1.6] + car[3:], car)                  # target exactly -1
    ax = [0.0, 0.0, 0.0, 1.6, 3.9, 1.56, 0.0]
    add("touching_faces", [1.6] + ax[1:], ax)                                          # x faces touch: zero area
    add("contained", [0.1, 0.3, 0.0, 0.8, 2.0, 1.0, 0.4], ax)
    s = 1.2                                                                            # a square rotated by pi/4: its corner on ax's x face
    add("corner_on_edge", [0.8 + s / np.sqrt(2), 0.5, 0.0, s, s, 1.5, pi / 4], ax)
    add("corner_poking_in", [0.8 + s / np.sqrt(2) - 0.1, 0.5, 0.0, s, s, 1.5, pi / 4], ax)
    add("pedestrian", [0.1, 0.05, 0.1, 0.6, 0.8, 1.73, 0.2], [0.0, 0.0, 0.0, 0.55, 0.9, 1.7, -0.1])
    add("enc_dims_plus5", car, car)                                                    # dims of q re-encoded below
    add("enc_dims_minus5", car, car)
    add("enc_dims_minus104", car, car)                                                 # expf underflows: zero-size box, target -1
    rng = np.random.default_rng(17)
    for i in range(6):                                                                 # generic: rotated, offset in x and y, heights differ
        gq = [rng.uniform(-0.5, 0.5), rng.uniform(-0.5, 0.5), rng.uniform(-0.3, 0.3), rng.uniform(1.4, 1.9), rng.uniform(3.4, 4.4),
              rng.uniform(1.3, 1.8), rng.uniform(-pi, pi)]
        gg = [rng.uniform(-0.5, 0.5), rng.uniform(-0.5, 0.5), rng.uniform(-0.3, 0.3), rng.uniform(1.4, 1.9), rng.uniform(3.4, 4.4),
              rng.uniform(1.3, 1.8), gq[6] + rng.uniform(-0.6, 0.6)]
        add("generic%d" % i, gq, gg)
    return out


IP_EXACT_MINUS_ONE = ("disjoint_bev", "no_height_overlap")          # pairs whose target is exactly -1 in fp32 and in fp64


def _ip_encode(box, anc):
    """second_box_encode in fp64 of a decoded box against one anchor, rounded to fp32"""
    diag = np.sqrt(np.float64(anc[4]) ** 2 + np.float64(anc[3]) ** 2)
    a = anc.astype(np.float64)
    return np.float32([(box[0] - a[0]) / diag, (box[1] - a[1]) / diag, (box[2] - a[2]) / a[5], np.log(box[3] / a[3]), np.log(box[4] / a[4]),
                       np.log(box[5] / a[5]), box[6] - a[6]])


def _ip_head_values(sigma):
    """iou head values around the exact target -1: target -+ knee, one ulp either side of each, and d = 0"""
    k = np.float32(1.0) / (np.float32(sigma) * np.float32(sigma))
    m1 = np.float32(-1)
    vals = [m1, m1 + k, m1 - k]
    for v in (m1 + k, m1 - k):
        vals += [np.nextafter(v, np.float32(2)), np.nextafter(v, np.float32(-2))]
    return np.float32(vals)


def make_iou_pred_case(B, A, stride, seed, sigma, frames):
    """head [B, A/2, stride], anchors [A, 7], labels [B, A], targets [B, A, 7].  frames: per frame "all", "empty", "edges" (only the
    positives at anchor 0, A - 1 and past the grid-stride wrap) or "shifted" (every placement, the pairs rotated by 5)."""
    rng = np.random.default_rng(seed)
    P = A // 2
    anc = _anchors(A)
    head = (rng.standard_normal((B, P, stride)) * 0.5).astype(np.float32)
    labels = rng.choice(np.int32([-1, 0]), (B, A), p=[0.2, 0.8]).astype(np.int32)
    targets = (rng.standard_normal((B, A, 7)) * 0.3).astype(np.float32)
    pairs = iou_pred_pairs()
    hv = _ip_head_values(sigma)
    jobs = [(i, None) for i in range(len(pairs))]
    jobs += [(i, v) for i, (n, _, _) in enumerate(pairs) if n in IP_EXACT_MINUS_ONE for v in hv]
    edges = [0, 1, A - 2, A - 1, IP_CTA_SPAN - 1, IP_CTA_SPAN, IP_CTA_SPAN + 1, 350, 351]          # 350 / 351: x = 70.2, y = -39.8
    edges += [x for x in (2 * IP_CTA_SPAN + 3, 3 * IP_CTA_SPAN + 8) if x < A]
    mid = [(100 * 176 + 40) * 2 + i for i in range(max(0, len(jobs) - len(edges)) + 4)]
    slots = edges + mid
    for b, kind in enumerate(frames):
        if kind == "empty":
            labels[b] = np.minimum(labels[b], 0)
            continue
        use = edges if kind == "edges" else slots
        rot = 5 if kind == "shifted" else 0
        for n, a in enumerate(use):
            i, v = jobs[(n + rot) % len(jobs)]
            name, qd, gd = pairs[i]
            labels[b, a] = 1
            qa, ga = qd.copy(), gd.copy()
            qa[:3] += anc[a, :3]
            ga[:3] += anc[a, :3]
            eq, eg = _ip_encode(qa, anc[a]), _ip_encode(ga, anc[a])
            if name == "enc_dims_plus5":
                eq[3:6] = 5
            elif name == "enc_dims_minus5":
                eq[3:6] = -5
            elif name == "enc_dims_minus104":
                eq[3] = -104
            r = a % 2
            head[b, a // 2, 7 * r:7 * r + 7] = eq
            targets[b, a] = eg
            head[b, a // 2, 20 + r] = v if v is not None else np.float32(rng.uniform(-1, 1))
    return head, anc, labels, targets


def iou_pred_cases():
    """(name, head, anchors, labels, targets, sigma, w_iou) of the crafted IoU-prediction cases"""
    A1, A2 = 37890, 70400
    return [
        ("a37890_s22_ragged5", *make_iou_pred_case(5, A1, 22, 31, 3.0, ["all", "empty", "edges", "shifted", "all"]), 3.0, 1.0),
        ("a70400_s24_sig1", *make_iou_pred_case(2, A2, 24, 32, 1.0, ["shifted", "all"]), 1.0, 0.5),
        ("a70400_s32_empty", *make_iou_pred_case(3, A2, 32, 33, 3.0, ["edges", "empty", "all"]), 3.0, 0.5),
    ]
