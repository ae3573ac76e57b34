"""Autograd through the SSFA neck and the detection head (SSFA / Head in train mode, det3d/models/necks/rpn_v1.py:220-235 and
det3d/models/bbox_heads/mg_head_sessd.py:202-230).

One conv / deconv of the neck, and the head's four 1x1 convs taken together, is one ``BevConvFunction`` on the launch geometry of
``sessd_data.layers.SSFA_LAUNCHES`` / ``ssfa_extents``.  BatchNorm2d, ReLU, the deconv_0 + trans_0 residual add and the attention tail
(w_0 / w_1 1x1 128 -> 1 convs + BN, 2-way softmax, weighted sum) stay the torch modules and ops they are (batch statistics and running-stat
updates exactly as the reference).  Per conv:

* forward: the input is split into fp16 (hi, lo) planes (absmax + bev_split_planes) and the p2 kernel (csrc/bevconv_p2.cu) writes the fp32
  pre-BN output: scale = the weight packing's 2^-e, shift = the bias (head) or none, no ReLU;
* data gradient: the output gradient is split the same way and fed to the forward kernels with re-packed weights
  (oracle/bev_grad_ref.py): a stride-1 conv runs the stride-1 conv with taps flipped and Cin <-> Cout (train.conv2d_s1_dgrad_weight),
  the stride-2 conv runs the deconv with the same weight tensor, the deconv runs the stride-2 conv with the same weight tensor; the
  head's 24-channel gradient is zero-padded to 64 channels (whole 64-channel groups of the p2 kernel);
* weight gradient: sessd_bev_wgrad (csrc/bevgrad.cu) over the saved input planes and the gradient planes; a deconv's is the stride-2
  conv's with the roles swapped (input = its output gradient, gradient = its input), transposed.

Activations between the layers are NHWC tensors (channels-last memory); BatchNorm2d sees them through an NCHW view."""
import torch
import torch.nn.functional as F

from sessd_data.layers import SSFA_LAUNCHES, ssfa_extents

from . import ops
from .runners import _cout_pad, _pack_conv, conv_taps, head_weight, launch_desc, launch_weight
from .train import conv2d_s1_dgrad_weight

HEAD = SSFA_LAUNCHES[-1]
HEAD_PAD = 64          # the head's output gradient is zero-padded to this many channels: the p2 kernel reads whole 64-channel groups


def split(x):
    """fp32 NHWC tensor -> (planes [2, *x.shape] fp16, info {abs-max, scale})"""
    x = x.contiguous()
    info = torch.zeros((2,), dtype=torch.float32, device=x.device)
    planes = torch.empty((2,) + tuple(x.shape), dtype=torch.float16, device=x.device)
    ops.absmax(x, info[0:1])
    ops.bev_split_planes(x, info, planes)
    return planes, info


def conv_desc(batch, in_hw, cin, out_hw, cout, k, stride):
    """ConvDesc of a data- or weight-gradient launch, whose input and output swap roles against the forward launch's: the taps of
    runners.conv_taps, no ReLU"""
    return ops.conv_desc(batch, in_hw, cin, out_hw, cout, out_hw, conv_taps(k), in_stride=stride, relu=False)


def _run(kind, planes, info, wp, shift, out, desc=None):
    """one forward-kernel launch into the fp32 NHWC ``out``: wp [taps, Cin, Cout] (conv: the taps of desc; deconv: 9-tap packing of
    W[cin][cout][ky][kx]), no BN, no ReLU"""
    cout = int(wp.shape[2])
    w_h2, inv = ops.pack_weight_h2(wp.float().contiguous(), _cout_pad(cout))
    scale = inv[:cout].contiguous()
    if kind == "conv":
        ops.bev_conv_p2(planes, info, w_h2, scale, shift, None, None, 0.0, 0.0, out, None, None, desc)
    else:
        ops.bev_deconv_p2(planes, info, w_h2, scale, shift, None, None, 0.0, 0.0, out, None, None, relu=False)
    return out


def dgrad_launch(L, weight):
    """(kind, packed weight [taps, Cin', Cout'], stride) of the forward launch that maps the output gradient of launch L (weight in the
    module's layout) to its input gradient"""
    if L.kind == "deconv":                                  # conv 3x3 s2 p1, Cout' = the deconv's Cin, with the same weight tensor
        return "conv", _pack_conv(weight)[0], 2
    if L.stride == 2:                                       # deconv k3 s2 p1 op1 with the same weight tensor: W[co][ci] is W_d[cin][cout]
        return "deconv", _pack_conv(weight.transpose(0, 1))[0], 1
    return "conv", _pack_conv(conv2d_s1_dgrad_weight(weight))[0], 1


def wgrad_to_weight(gw, k):
    """[k k, Cin, Cout] of sessd_bev_wgrad -> a Conv2d weight gradient [Cout, Cin, k, k]; for a deconv (the stride-2 conv with the roles
    swapped: Cin = its Cout, Cout = its Cin) the same permutation yields its ConvTranspose2d weight layout [Cin, Cout, k, k]"""
    return gw.reshape(k, k, gw.shape[1], gw.shape[2]).permute(3, 2, 0, 1)


class BevConvFunction(torch.autograd.Function):
    """out NHWC [B, Ho, Wo, Cout] fp32 (pre-BN) = launch L of x NHWC [B, Hi, Wi, Cin] with ``weight`` in the module's layout (Conv2d
    [Cout, Cin, k, k], ConvTranspose2d [Cin, Cout, 3, 3]) and the optional ``bias`` [Cout]; in_hw / out_hw from ssfa_extents"""

    @staticmethod
    def forward(ctx, x, weight, bias, L, in_hw, out_hw):
        b = int(x.shape[0])
        planes, info = split(x.detach().float())
        wp, taps = launch_weight(L, weight.detach().float())
        out = torch.empty((b,) + tuple(out_hw) + (L.cout,), dtype=torch.float32, device=x.device)
        shift = None if bias is None else bias.detach().float().contiguous()
        _run(L.kind, planes, info, wp, shift, out, launch_desc(L, b, in_hw, out_hw, taps, relu=False) if L.kind == "conv" else None)
        # through save_for_backward: an in-place change of the weight or of the input planes between forward and backward raises
        ctx.save_for_backward(weight, planes, info)
        ctx.L, ctx.in_hw, ctx.out_hw, ctx.has_bias = L, tuple(in_hw), tuple(out_hw), bias is not None
        return out

    @staticmethod
    def backward(ctx, gout):
        L, in_hw, out_hw = ctx.L, ctx.in_hw, ctx.out_hw
        weight, planes, info = ctx.saved_tensors
        w = weight.detach().float()
        g = gout.detach().float().contiguous()
        b, dev = int(g.shape[0]), g.device
        want_x, want_w, want_b = ctx.needs_input_grad[0], ctx.needs_input_grad[1], ctx.needs_input_grad[2]
        cg = L.cout
        if L.name == HEAD.name:                             # zero-pad the gradient to whole 64-channel groups
            g = F.pad(g, (0, HEAD_PAD - L.cout))
            cg = HEAD_PAD
        g_planes, g_info = split(g)
        gx = gw = gb = None
        if want_x:
            kind, wd, stride = dgrad_launch(L, w)
            if cg != L.cout:
                wd = F.pad(wd, (0, 0, 0, cg - L.cout))     # [taps, Cout -> cg, Cin]
            gx = torch.empty((b,) + in_hw + (L.cin,), dtype=torch.float32, device=dev)
            desc = conv_desc(b, out_hw, cg, in_hw, L.cin, L.k, stride) if kind == "conv" else None
            _run(kind, g_planes, g_info, wd, None, gx, desc)
        if want_w:
            if L.kind == "conv":
                gw = ops.bev_wgrad(planes, info, g_planes, g_info, conv_desc(b, in_hw, L.cin, out_hw, cg, L.k, L.stride))[..., :L.cout]
            else:                                           # roles swapped: in = the output gradient, g = the deconv's input
                gw = ops.bev_wgrad(g_planes, g_info, planes, info, conv_desc(b, out_hw, L.cout, in_hw, L.cin, L.k, 2))
            gw = wgrad_to_weight(gw, L.k).contiguous()
        if want_b and ctx.has_bias:
            gb = gout.detach().float().sum(dim=(0, 1, 2))
        return gx, gw, gb, None, None, None


def _module(root, name):
    blk, idx = name.rsplit(".", 1)
    return getattr(root, blk)[int(idx)], getattr(root, blk), int(idx)


def ssfa_forward(neck, x):
    """rpn_v1.py:220-235 layer by layer on x [B, 128, H, W] (logical NCHW, any memory format): the convs through BevConvFunction,
    BatchNorm2d / ReLU / the residual add / the attention tail as the torch modules and ops.  Returns [B, 128, H, W] (channels-last)."""
    b, _c, h, w = x.shape
    t = {"x": x.permute(0, 2, 3, 1)}
    for L in SSFA_LAUNCHES[:-1]:
        conv, blk, i = _module(neck, L.name)
        in_hw, out_hw = ssfa_extents(L, h, w)
        y = BevConvFunction.apply(t[L.src], conv.weight, None, L, in_hw, out_hw).permute(0, 3, 1, 2)
        y = blk[i + 1](y)                                   # BatchNorm2d
        if L.relu:
            y = blk[i + 2](y)
        if L.residual:
            y = y + t[L.residual].permute(0, 3, 1, 2)
        t[L.dst] = y.permute(0, 2, 3, 1)
    o0, o1 = t["o0"].permute(0, 3, 1, 2), t["o1"].permute(0, 3, 1, 2)
    wgt = torch.softmax(torch.cat([_attention_logit(neck.w_0, o0), _attention_logit(neck.w_1, o1)], dim=1), dim=1)
    return o0 * wgt[:, 0:1] + o1 * wgt[:, 1:]


def _attention_logit(seq, o):
    """w_0 / w_1 (rpn_v1.py:229-230): 1x1 128 -> 1 conv + BatchNorm2d.  The conv is a product and a channel sum in fp32, forward and
    backward: a cuDNN conv would run in TF32 (torch's default for cuDNN convs), and its 10-bit rounding would pass through the BN, the
    softmax and every layer's backward below, unlike the eval path's fused fp32 kernel."""
    conv, bn = seq[0], seq[1]
    return bn((o * conv.weight.view(1, -1, 1, 1)).sum(dim=1, keepdim=True))


def head_forward(head, x):
    """the four 1x1 convs of a Head (mg_head_sessd.py:202-230) as one BevConvFunction on x [B, 128, H, W] -> packed NHWC [B, H, W, 24] =
    [box 14 | cls 2 | dir 4 | iou 2 | pad 2] (runners.head_weight's layout), with a graph to x and every conv's weight and bias"""
    w, bias = head_weight(head.get_parameter)
    hw = tuple(x.shape[2:])
    return BevConvFunction.apply(x.permute(0, 2, 3, 1), w, bias, HEAD, hw, hw)
