"""CPU: the re-packings behind the neck / head backward (sessd_b200/bev_grad.py) against torch autograd of F.conv2d /
F.conv_transpose2d in fp64, for every launch of SSFA_LAUNCHES: the data gradient as one forward launch of the kernels (tap-list conv or
the deconv's 9-tap packing) and the weight gradient as csrc/bevgrad.cu computes it (tap shifts, stride, zero padding, the deconv's role
swap + transpose, the head's zero-padded gradient).  Plus the kernel's work-item count."""
import pytest
import torch
import torch.nn.functional as F

from bev_grad_model import bg_geometry, module_forward, tap_conv, wgrad_index
from sessd_data.layers import SSFA_LAUNCHES, ssfa_extents


@pytest.mark.parametrize("L", SSFA_LAUNCHES, ids=[L.name for L in SSFA_LAUNCHES])
def test_dgrad_and_wgrad_restatements_equal_autograd(L):
    from sessd_b200 import bev_grad
    g = torch.Generator().manual_seed(3)
    h, w = 10, 14
    in_hw, out_hw = ssfa_extents(L, h, w)
    cin, cout = L.cin, L.cout
    wshape = (cin, cout, 3, 3) if L.kind == "deconv" else (cout, cin, L.k, L.k)
    W = torch.randn(wshape, generator=g, dtype=torch.float64).requires_grad_(True)
    bias = torch.randn(cout, generator=g, dtype=torch.float64).requires_grad_(True) if L.name == "head" else None
    x = torch.randn((2, cin) + in_hw, generator=g, dtype=torch.float64).requires_grad_(True)
    y = module_forward(L, x, W, bias)
    assert tuple(y.shape[2:]) == out_hw
    G = torch.randn(y.shape, generator=g, dtype=torch.float64)
    (y * G).sum().backward()
    xh, gh = x.detach().permute(0, 2, 3, 1), G.permute(0, 2, 3, 1)          # NHWC

    # data gradient: one forward launch with the re-packed weight
    kind, wd, stride = bev_grad.dgrad_launch(L, W.detach())
    gin = gh
    if L.name == "head":                                                     # zero-padded to whole 64-channel groups
        gin = F.pad(gh, (0, bev_grad.HEAD_PAD - cout))
        wd = F.pad(wd, (0, 0, 0, bev_grad.HEAD_PAD - cout))
    if kind == "conv":
        gx = tap_conv(gin, wd, bev_grad.conv_taps(L.k), stride, in_hw)
    else:                                                                    # the deconv kernel's 9-tap packing of W[cin][cout][ky][kx]
        wt = wd.reshape(3, 3, wd.shape[1], wd.shape[2]).permute(2, 3, 0, 1)
        gx = F.conv_transpose2d(gin.permute(0, 3, 1, 2), wt, None, 2, 1, output_padding=1).permute(0, 2, 3, 1)
    assert float((gx - x.grad.permute(0, 2, 3, 1)).abs().max()) <= 1e-12 * float(x.grad.abs().max())

    # weight gradient: what the kernel computes, then the layout change of BevConvFunction.backward
    taps = bev_grad.conv_taps(L.k)
    if L.kind == "conv":
        gw = wgrad_index(xh, gin, taps, L.stride)[..., :cout]
    else:                                                                    # roles swapped: in = the output gradient, g = the input
        gw = wgrad_index(gh, xh, taps, 2)
    gW = bev_grad.wgrad_to_weight(gw, L.k)
    assert gW.shape == W.shape
    assert float((gW - W.grad).abs().max()) <= 1e-12 * float(W.grad.abs().max())
    if bias is not None:
        assert float((G.sum(dim=(0, 2, 3)) - bias.grad).abs().max()) <= 1e-12 * float(bias.grad.abs().max())


def test_wgrad_item_count_is_a_function_of_the_descriptor():
    """sessd_bev_wgrad_items == the decomposition of tests/bev_grad_model.bg_geometry on every neck / head launch at two map sizes and
    batches 1 and 8, never more than four waves of one CTA per SM; invalid descriptors (channel counts, stride, output offset) are refused"""
    import ctypes as C
    from sessd_b200 import bev_grad
    from sessd_b200._lib import lib
    for b, (h, w) in ((1, (13, 21)), (8, (200, 176))):
        for L in SSFA_LAUNCHES:
            in_hw, out_hw = ssfa_extents(L, h, w)
            cg = bev_grad.HEAD_PAD if L.name == "head" else L.cout
            if L.kind == "conv":
                d = bev_grad.conv_desc(b, in_hw, L.cin, out_hw, cg, L.k, L.stride)
                hw, ci, co = out_hw, L.cin, cg
            else:
                d = bev_grad.conv_desc(b, out_hw, L.cout, in_hw, L.cin, 3, 2)
                hw, ci, co = in_hw, L.cout, L.cin
            nc, groups, chunks, rpc = bg_geometry(b, hw, ci, co, L.k * L.k)
            assert lib.sessd_bev_wgrad_items(C.byref(d)) == groups * chunks
            assert groups * chunks <= 4 * 132                  # no partial fifth wave at one CTA per SM
            assert lib.sessd_bev_wgrad_workspace_bytes(C.byref(d)) == 4 * groups * chunks * 128 * nc
            assert (chunks - 1) * rpc * 64 < b * hw[0] * hw[1] <= chunks * rpc * 64
    bad = [bev_grad.conv_desc(1, (8, 8), 64, (8, 8), 128, 3, 1), bev_grad.conv_desc(1, (8, 8), 128, (8, 8), 24, 1, 1),
           bev_grad.conv_desc(1, (8, 8), 128, (4, 4), 256, 3, 3)]
    off = bev_grad.conv_desc(1, (8, 8), 128, (8, 8), 128, 3, 1)
    off.out_off_x = 1
    for d in bad + [off]:
        assert lib.sessd_bev_wgrad_items(C.byref(d)) == -1 and lib.sessd_bev_wgrad_workspace_bytes(C.byref(d)) == 0
