"""BEV neck (SSFA) + head kernels vs the reference modules' golden output (small map) and the torch-CPU oracle."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = 1e-4   # north_star: <= 1e-4 rel on regressions / confidences


def _rel(a, b):
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


MODES = ["simt", "tf32x3", "fp16x2", "planes"]   # fp32 SIMT baseline | 3xTF32 weights | fp16 split of fp32 inputs | pre-split planes (default)


def _runner(batch, hw, mode):
    from sessd_b200.runners import SSFAPlanesRunner, SSFARunner
    if mode == "planes":
        return SSFAPlanesRunner(batch, hw, "cuda")
    return SSFARunner(batch, hw, "cuda", use_tc=mode != "simt", split="tf32" if mode == "tf32x3" else "fp16")


def _act(r, name):
    return r.activation(name) if hasattr(r, "activation") else r.buf[name]


def _to_planes(xd):
    """fp32 NHWC device tensor -> (planes [2,B,H,W,C], info [2])"""
    from sessd_b200 import ops
    info = torch.zeros(2, device="cuda")
    ops.absmax(xd, info[0:1])
    planes = ops.alloc_bev_planes(xd.shape[0], xd.shape[1], xd.shape[2], xd.shape[3], "cuda")
    ops.bev_split_planes(xd, info, planes)
    return planes, info


@pytest.mark.parametrize("mode", MODES)
def test_ssfa_and_head_match_reference_golden(golden_dir, mode):
    from oracle import bev_ref
    from sessd_b200.runners import SSFARunner
    g = np.load(os.path.join(golden_dir, "ssfa_head_case.npz"))
    sd = bev_ref.ssfa_random_state(7)
    hsd = bev_ref.head_random_state(9, prefix="tasks.0.")
    gen = torch.Generator().manual_seed(8)
    x = torch.relu(torch.randn(1, 128, 24, 16, generator=gen))
    r = _runner(1, (24, 16), mode)
    r.load_state(sd, hsd)
    out, head = r.forward(x.permute(0, 2, 3, 1).contiguous().cuda())
    torch.cuda.synchronize()
    got = out.permute(0, 3, 1, 2).cpu().numpy()
    assert _rel(got, g["ssfa_out"]) < TOL
    # the golden head used prefix "" weights drawn from the same seed
    hsd0 = bev_ref.head_random_state(9, prefix="")
    for k in hsd0:
        assert torch.equal(hsd0[k], hsd["tasks.0." + k])
    h = head.cpu().numpy()
    assert _rel(h[..., 0:14], g["box_preds"]) < TOL
    assert _rel(h[..., 14:16], g["cls_preds"]) < TOL
    assert _rel(h[..., 16:20], g["dir_cls_preds"]) < TOL
    assert _rel(h[..., 20:22], g["iou_preds"]) < TOL


@pytest.mark.parametrize("mode", MODES)
def test_ssfa_intermediates_match_oracle_fp64_batch2(mode):
    from oracle import bev_ref
    from sessd_b200.runners import SSFARunner
    sd = bev_ref.ssfa_random_state(17)
    hsd = bev_ref.head_random_state(19)
    gen = torch.Generator().manual_seed(18)
    x = torch.relu(torch.randn(2, 128, 40, 48, generator=gen))
    trace = {}
    ref = bev_ref.ssfa_forward(x.double(), {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}, trace)
    r = _runner(2, (40, 48), mode)
    r.load_state(sd, hsd)
    out, _ = r.forward(x.permute(0, 2, 3, 1).contiguous().cuda())
    torch.cuda.synchronize()
    for mine, theirs in (("x0", "x0"), ("x1", "x1"), ("t0", "t0"), ("t1", "t1"), ("m0", "m0"), ("m1", "m1"), ("o0", "o0"), ("o1", "o1")):
        got = _act(r, mine).permute(0, 3, 1, 2).cpu().numpy()
        assert _rel(got, trace[theirs].numpy()) < 2e-5, mine
    assert _rel(out.permute(0, 3, 1, 2).cpu().numpy(), ref.numpy()) < 2e-5


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("cin,cout,k,hw", [(128, 128, 3, (21, 37)), (256, 256, 3, (9, 50)), (128, 128, 1, (8, 16)), (256, 256, 1, (13, 17)),
                                           (128, 24, 1, (20, 33))])
def test_single_conv_vs_fp64(mode, cin, cout, k, hw):
    """One tap-list conv incl. partial 8x16 tiles, BN scale/shift, ReLU and residual, against an fp64 torch conv."""
    import torch.nn.functional as F
    from sessd_b200 import ops
    from sessd_b200.runners import _pack_conv
    g = torch.Generator().manual_seed(cin + cout + k)
    b = 2
    x = torch.randn(b, cin, hw[0], hw[1], generator=g)
    w = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5
    sc = 1.0 + 0.1 * torch.randn(cout, generator=g)
    sh = 0.1 * torch.randn(cout, generator=g)
    res = torch.randn(b, cout, hw[0], hw[1], generator=g)
    ref = F.relu(F.conv2d(x.double(), w.double(), None, 1, k // 2) * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1)) + res.double()
    wp, taps = _pack_conv(w)
    taps = [(dy - k // 2, dx - k // 2) for dy, dx in taps]
    xd = x.permute(0, 2, 3, 1).contiguous().cuda()
    rd = res.permute(0, 2, 3, 1).contiguous().cuda()
    out = torch.zeros((b, hw[0], hw[1], cout), device="cuda")
    d = ops.conv_desc(b, hw, cin, hw, cout, hw, taps, relu=True)
    cout_pad = 32 if cout <= 32 else -(-cout // 128) * 128
    if mode == "tf32x3":
        ops.bev_conv_tc(xd, ops.pack_weight_tc(wp.cuda(), cout_pad), sc.cuda(), sh.cuda(), rd, out, d)
    elif mode == "planes":
        planes, inv = ops.pack_weight_h2(wp.cuda(), cout_pad)
        xp, info = _to_planes(xd)
        rinfo = torch.zeros(2, device="cuda")
        ops.absmax(rd, rinfo[0:1])
        oinfo = torch.zeros(2, device="cuda")
        oplanes = ops.alloc_bev_planes(b, hw[0], hw[1], cout, "cuda")
        ops.bev_conv_p2(xp, info, planes, sc.cuda() * inv[:cout], sh.cuda(), rd, rinfo, ops.conv_gain(wp.cuda(), sc.cuda()), float(sh.abs().max()),
                        out, oplanes, oinfo, d)
        torch.cuda.synchronize()
        assert float(oinfo[0]) == float(out.abs().max())
        back = ops.planes_to_float(oplanes, oinfo)
        assert float((back - out).abs().max()) <= 4e-7 * float(out.abs().max()), "planes output differs from the fp32 output"
    elif mode == "fp16x2":
        planes, inv = ops.pack_weight_h2(wp.cuda(), cout_pad)
        amax = torch.zeros(2, device="cuda")
        ops.absmax(xd, amax[0:1])
        ops.bev_conv_h2(xd, planes, sc.cuda() * inv[:cout], sh.cuda(), rd, out, d, amax[0:1], amax[1:2])
        torch.cuda.synchronize()
        assert float(amax[0]) == float(xd.abs().max()) and float(amax[1]) == float(out.abs().max())
    else:
        ops.bev_conv(xd, wp.cuda(), sc.cuda(), sh.cuda(), rd, out, d)
    torch.cuda.synchronize()
    got = out.permute(0, 3, 1, 2).cpu().double()
    err = float((got - ref).abs().max() / ref.abs().max())
    assert err < 5e-6, err


def test_tf32_split_is_exact():
    from sessd_b200 import ops
    w = torch.randn(4096, generator=torch.Generator().manual_seed(1))
    hi, lo = ops.split_tf32(w)
    assert torch.equal(hi + lo, w)
    assert int((hi.view(torch.int32) & 8191).abs().max()) == 0


def test_fp16_split_range_and_precision():
    """Activations far outside fp16's range (1e7, 1e-7 scales) go through the exact power-of-two scaling: same relative accuracy."""
    import torch.nn.functional as F
    from sessd_b200 import ops
    from sessd_b200.runners import _pack_conv
    g = torch.Generator().manual_seed(5)
    cin, cout, hw = 128, 128, (16, 32)
    w = torch.randn(cout, cin, 3, 3, generator=g) * 0.03
    wp, taps = _pack_conv(w)
    taps = [(dy - 1, dx - 1) for dy, dx in taps]
    planes, inv = ops.pack_weight_h2(wp.cuda(), 128)
    d = ops.conv_desc(1, hw, cin, hw, cout, hw, taps, relu=False)
    for scale in (1.0, 1e7, 1e-7, 3e-30):
        x = torch.randn(1, cin, hw[0], hw[1], generator=g) * scale
        ref = F.conv2d(x.double(), w.double(), None, 1, 1)
        xd = x.permute(0, 2, 3, 1).contiguous().cuda()
        out = torch.zeros((1, hw[0], hw[1], cout), device="cuda")
        amax = torch.zeros(1, device="cuda")
        ops.absmax(xd, amax)
        ops.bev_conv_h2(xd, planes, inv[:cout].contiguous(), None, None, out, d, amax, None)
        torch.cuda.synchronize()
        got = out.permute(0, 3, 1, 2).cpu().double()
        err = float((got - ref).abs().max() / ref.abs().max())
        assert err < 5e-6, (scale, err)


@pytest.mark.parametrize("k,stride,hw", [(3, 2, (40, 48)), (3, 2, (200, 176)), (3, 1, (200, 176)), (3, 1, (100, 88))])
def test_planes_conv_full_shapes_vs_fp64(k, stride, hw):
    """bev_conv_p2 on the SSFA layer shapes incl. the stride-2 conv (128 -> 256) and both tile orientations."""
    import torch.nn.functional as F
    from sessd_b200 import ops
    from sessd_b200.runners import _pack_conv
    g = torch.Generator().manual_seed(k + stride + hw[0])
    b, cin = 1, (128 if hw[0] != 100 else 256)
    cout = 256 if (stride == 2 or cin == 256) else 128
    x = torch.randn(b, cin, hw[0], hw[1], generator=g)
    w = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5
    sc = 1.0 + 0.1 * torch.randn(cout, generator=g)
    sh = 0.1 * torch.randn(cout, generator=g)
    ref = F.relu(F.conv2d(x.double(), w.double(), None, stride, k // 2) * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1))
    ohw = (ref.shape[2], ref.shape[3])
    wp, taps = _pack_conv(w)
    taps = [(dy - k // 2, dx - k // 2) for dy, dx in taps]
    xd = x.permute(0, 2, 3, 1).contiguous().cuda()
    out = torch.zeros((b, ohw[0], ohw[1], cout), device="cuda")
    d = ops.conv_desc(b, hw, cin, ohw, cout, ohw, taps, in_stride=stride, relu=True)
    planes, inv = ops.pack_weight_h2(wp.cuda(), -(-cout // 128) * 128)
    xp, info = _to_planes(xd)
    oinfo = torch.zeros(2, device="cuda")
    ops.bev_conv_p2(xp, info, planes, sc.cuda() * inv[:cout], sh.cuda(), None, None, ops.conv_gain(wp.cuda(), sc.cuda()), float(sh.abs().max()),
                    out, None, oinfo, d)
    torch.cuda.synchronize()
    got = out.permute(0, 3, 1, 2).cpu().double()
    err = float((got - ref).abs().max() / ref.abs().max())
    assert err < 5e-6, err


@pytest.mark.parametrize("split", ["tf32", "fp16", "planes"])
@pytest.mark.parametrize("hw", [(13, 17), (100, 88)])
def test_deconv_single_launch_vs_fp64(hw, split):
    """ConvTranspose2d(k3,s2,p1,op1)+BN+ReLU+residual as one 4-class tensor-core launch."""
    import torch.nn.functional as F
    from sessd_b200 import ops
    g = torch.Generator().manual_seed(3)
    b, cin, cout = 2, 256, 128
    x = torch.randn(b, cin, hw[0], hw[1], generator=g)
    w = torch.randn(cin, cout, 3, 3, generator=g) * (2.0 / (cin * 2.25)) ** 0.5
    sc = 1.0 + 0.1 * torch.randn(cout, generator=g)
    sh = 0.1 * torch.randn(cout, generator=g)
    res = torch.randn(b, cout, 2 * hw[0], 2 * hw[1], generator=g)
    ref = F.relu(F.conv_transpose2d(x.double(), w.double(), None, 2, 1, output_padding=1) * sc.double().view(1, -1, 1, 1)
                 + sh.double().view(1, -1, 1, 1)) + res.double()
    w9 = w.permute(2, 3, 0, 1).reshape(9, cin, cout).contiguous().cuda()
    out = torch.zeros((b, 2 * hw[0], 2 * hw[1], cout), device="cuda")
    xd, rd = x.permute(0, 2, 3, 1).contiguous().cuda(), res.permute(0, 2, 3, 1).contiguous().cuda()
    if split == "tf32":
        ops.bev_deconv_tc(xd, ops.pack_weight_tc(w9, 128), sc.cuda(), sh.cuda(), rd, out)
    elif split == "planes":
        planes, inv = ops.pack_weight_h2(w9, 128)
        xp, info = _to_planes(xd)
        rinfo = torch.zeros(2, device="cuda")
        ops.absmax(rd, rinfo[0:1])
        oinfo = torch.zeros(2, device="cuda")
        ops.bev_deconv_p2(xp, info, planes, sc.cuda() * inv[:cout], sh.cuda(), rd, rinfo, ops.conv_gain(w9, sc.cuda()), float(sh.abs().max()),
                          out, None, oinfo, True)
    else:
        planes, inv = ops.pack_weight_h2(w9, 128)
        amax = torch.zeros(1, device="cuda")
        ops.absmax(xd, amax)
        ops.bev_deconv_h2(xd, planes, sc.cuda() * inv[:cout], sh.cuda(), rd, out, True, amax, None)
    torch.cuda.synchronize()
    got = out.permute(0, 3, 1, 2).cpu().double()
    assert float((got - ref).abs().max() / ref.abs().max()) < 5e-6
