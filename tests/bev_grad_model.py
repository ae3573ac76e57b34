"""fp64 torch restatements of the BEV neck / head backward (csrc/bevgrad.cu, sessd_b200/bev_grad.py); shared by
tests/test_bev_grad_model.py (CPU) and tests/test_gpu_bev_grad.py.

* ``tap_conv``: the forward kernels' tap-list conv (sessd_conv_desc semantics) at the index level, NHWC;
* ``wgrad_index``: what sessd_bev_wgrad computes, gW[t][ci][co] = sum_{b,y,x} X[b, y s + dy_t, x s + dx_t, ci] G[b, y, x, co];
* ``bg_geometry``: its work-item decomposition (the item count is a function of the descriptor only);
* ``ssfa_train_ref`` / ``head_ref``: rpn_v1.py:220-235 written out with train-mode BatchNorm2d, and the four head convs, in fp64 torch."""
import torch
import torch.nn.functional as F

ITEMS_TARGET = 4 * 132
KC = 64


def shifted(x, dy, dx, stride, out_hw):
    """X[b, y s + dy, x s + dx, :] for every output pixel (y, x), zero outside the map: x NHWC -> [B, Ho, Wo, C]"""
    b, h, w, c = x.shape
    ho, wo = out_hw
    out = x.new_zeros((b, ho, wo, c))
    ys = torch.arange(ho) * stride + dy
    xs = torch.arange(wo) * stride + dx
    vy, vx = (ys >= 0) & (ys < h), (xs >= 0) & (xs < w)
    out[:, vy.nonzero()[:, 0][:, None], vx.nonzero()[:, 0][None, :]] = x[:, ys[vy][:, None], xs[vx][None, :]]
    return out


def tap_conv(x, wp, taps, stride, out_hw):
    """out[b, y, x] = sum_t X[b, y s + dy_t, x s + dx_t] @ wp[t]  (x NHWC, wp [taps, Cin, Cout])"""
    out = 0
    for t, (dy, dx) in enumerate(taps):
        out = out + shifted(x, dy, dx, stride, out_hw) @ wp[t]
    return out


def wgrad_index(x, g, taps, stride):
    """[taps, Cin, Cout]: gW[t][ci][co] = sum_{b, y, x} X[b, y s + dy_t, x s + dx_t, ci] G[b, y, x, co] (x, g NHWC)"""
    out_hw = tuple(g.shape[1:3])
    return torch.stack([torch.einsum("byxc,byxn->cn", shifted(x, dy, dx, stride, out_hw), g) for dy, dx in taps], 0)


def bg_geometry(batch, out_hw, cin, cout, ntaps):
    """(nc, groups, chunks, rounds per chunk) of csrc/bevgrad.cu bg_geometry"""
    nc = 128 if cout % 128 == 0 else 64
    groups = ntaps * (cin // 128) * (cout // nc)
    rounds = -(-batch * out_hw[0] * out_hw[1] // KC)
    c = min(max(ITEMS_TARGET // groups, 1), rounds)
    rpc = -(-rounds // c)
    return nc, groups, -(-rounds // rpc), rpc


def module_forward(L, x, w, bias=None):
    """launch L as the reference module computes it (torch, NCHW): Conv2d padded by k // 2 / ConvTranspose2d(k3, s2, p1, op1)"""
    if L.kind == "deconv":
        return F.conv_transpose2d(x, w, bias, 2, 1, output_padding=1)
    return F.conv2d(x, w, bias, L.stride, L.k // 2)


# the conv modules of SSFA (rpn_v1.py:135-210), each followed by its BatchNorm2d
SSFA_CONV_NAMES = ("bottom_up_block_0.1", "bottom_up_block_0.4", "bottom_up_block_0.7", "bottom_up_block_1.0", "bottom_up_block_1.3",
                   "bottom_up_block_1.6", "trans_0.0", "trans_1.0", "deconv_block_0.0", "deconv_block_1.0", "conv_0.0", "w_0.0", "conv_1.0",
                   "w_1.0")


class _DataGradNoise(torch.autograd.Function):
    """identity forward; backward adds u xi mag to the data gradient, mag = the conv's data gradient of |g_out| through |W| (box["mag"])"""

    @staticmethod
    def forward(ctx, v, u, gen, box):
        ctx.u, ctx.gen, ctx.box = u, gen, box
        return v.view_as(v)

    @staticmethod
    def backward(ctx, g):
        mag = ctx.box["mag"]()
        return g + ctx.u * (2 * torch.rand(g.shape, generator=ctx.gen, device=g.device, dtype=g.dtype) - 1) * mag, None, None, None


def perturbed_conv(op, v, w, perturb):
    """op(v, w), and with perturb = (u, torch.Generator on v's device) the rounding model of a kernel that computes it: every element
    of the output and of the data gradient off by u xi (xi uniform in [-1, 1]) times its magnitude -- the same product over |v|, |w|
    (forward) or |g_out|, |w| (backward), as the per-operator bounds of tests/test_gpu_bev_grad.py have it"""
    if perturb is None:
        return op(v, w)
    u, gen = perturb
    box = {}
    y = op(_DataGradNoise.apply(v, u, gen, box), w)
    with torch.no_grad():
        y_mag = op(v.abs(), w.abs())
    y = y + u * (2 * torch.rand(y.shape, generator=gen, device=y.device, dtype=y.dtype) - 1) * y_mag
    y.register_hook(lambda g: box.__setitem__("g", g.abs()))

    def mag():
        with torch.enable_grad():
            va = v.detach().abs().requires_grad_(True)
            return torch.autograd.grad(op(va, w.detach().abs()), va, box["g"])[0]

    box["mag"] = mag
    return y


def ssfa_train_ref(x, P, momentum=0.01, eps=1e-3, perturb=None):
    """rpn_v1.py:220-235 written out, in fp64 torch with train-mode BatchNorm2d (independent of the launch table the code under test
    walks).  x NCHW; P: {conv module name: dict(weight, gamma, beta, mean, var)} (running stats updated in place).  perturb: see
    ``perturbed_conv``, applied to every conv"""
    def cbr(name, v, stride=1, relu=True):
        p = P[name]
        k = p["weight"].shape[2]
        y = perturbed_conv(lambda a, b: F.conv2d(a, b, None, stride, k // 2), v, p["weight"], perturb)
        y = F.batch_norm(y, p["mean"], p["var"], p["gamma"], p["beta"], True, momentum, eps)
        return torch.relu(y) if relu else y

    def deconv(name, v):
        p = P[name]
        y = perturbed_conv(lambda a, b: F.conv_transpose2d(a, b, None, 2, 1, output_padding=1), v, p["weight"], perturb)
        return torch.relu(F.batch_norm(y, p["mean"], p["var"], p["gamma"], p["beta"], True, momentum, eps))

    x_0 = cbr("bottom_up_block_0.7", cbr("bottom_up_block_0.4", cbr("bottom_up_block_0.1", x)))
    x_1 = cbr("bottom_up_block_1.6", cbr("bottom_up_block_1.3", cbr("bottom_up_block_1.0", x_0, stride=2)))
    x_trans_0 = cbr("trans_0.0", x_0)
    x_trans_1 = cbr("trans_1.0", x_1)
    x_middle_0 = deconv("deconv_block_0.0", x_trans_1) + x_trans_0
    x_middle_1 = deconv("deconv_block_1.0", x_trans_1)
    x_output_0 = cbr("conv_0.0", x_middle_0)
    x_output_1 = cbr("conv_1.0", x_middle_1)
    x_weight_0 = cbr("w_0.0", x_output_0, relu=False)
    x_weight_1 = cbr("w_1.0", x_output_1, relu=False)
    x_weight = torch.softmax(torch.cat([x_weight_0, x_weight_1], dim=1), dim=1)
    return x_output_0 * x_weight[:, 0:1, :, :] + x_output_1 * x_weight[:, 1:, :, :]


def ssfa_params(neck, device="cpu", dtype=torch.float64):
    """fp64 copies of an SSFA module's conv weights (requiring grad), BN affine parameters (requiring grad) and running stats"""
    P = {}
    for name in SSFA_CONV_NAMES:
        blk, i = name.rsplit(".", 1)
        conv, bn = getattr(neck, blk)[int(i)], getattr(neck, blk)[int(i) + 1]
        c = lambda v, g: v.detach().to(device, dtype).clone().requires_grad_(g)      # noqa: E731
        P[name] = dict(weight=c(conv.weight, True), gamma=c(bn.weight, True), beta=c(bn.bias, True), mean=c(bn.running_mean, False),
                       var=c(bn.running_var, False))
    return P


HEAD_CONVS = ("conv_box", "conv_cls", "conv_dir", "conv_iou")


def head_params(head, device="cpu", dtype=torch.float64):
    return {n: dict(weight=getattr(head, n).weight.detach().to(device, dtype).clone().requires_grad_(True),
                    bias=getattr(head, n).bias.detach().to(device, dtype).clone().requires_grad_(True)) for n in HEAD_CONVS}


def head_ref(x, H, perturb=None):
    """packed NHWC [B, H, W, 24] = [box 14 | cls 2 | dir 4 | iou 2 | 0 0] of the four 1x1 convs (mg_head_sessd.py:202-230)"""
    outs = [perturbed_conv(F.conv2d, x, H[n]["weight"], perturb) + H[n]["bias"].view(1, -1, 1, 1) for n in HEAD_CONVS]
    outs.append(x.new_zeros((x.shape[0], 2) + tuple(x.shape[2:])))
    return torch.cat(outs, 1).permute(0, 2, 3, 1)
