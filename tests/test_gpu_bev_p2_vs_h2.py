"""The planes-chain BEV conv (`bev_conv_p2` / `bev_deconv_p2`) against the lab split-fp16 mode (`bev_conv_h2` / `bev_deconv_h2`), bit for bit.

Given the same fp32 input, the two modes feed the tensor cores the same fp16 (hi, lo) operands: h2 splits the input inside the kernel
with the power-of-two scale of its abs-max, p2 reads the planes `bev_split_planes` made with that same scale.  The p2 main loop issues
a_hi x [b_lo ; b_hi] as one wgmma over the whole weight stage, then a_lo x b_hi into the cross half; h2 keeps three separate products.
Each accumulator still sums the same products in the same order, and the epilogues apply the same fp32 operations per element, so the
fp32 outputs and the running abs-max must be equal bit for bit.  The p2 planes output must equal the split of the h2 fp32 output with
the scale p2 reports (hi = fp16(o S), lo = fp16(o S - hi)).  The cases are the neck's launch shapes the h2 mode accepts (its fp32
staging leaves no room for the stride-2 conv's weight ring), at batch 1 and 2, plus maps whose edges cut through tiles.
"""
import pytest
import torch

from sessd_b200 import ops

pytestmark = pytest.mark.gpu

TAPS3 = [(dy, dx) for dy in (-1, 0, 1) for dx in (-1, 0, 1)]
TAPS1 = [(0, 0)]
F16_SENTINEL = 0x5A5A

# (label, kind, batch, (h, w) of the input, cin, cout, taps, relu, residual)
CASES = [
    ("conv3x3_128_200x176", "conv", 1, (200, 176), 128, 128, TAPS3, True, False),
    ("conv1x1_128_200x176", "conv", 1, (200, 176), 128, 128, TAPS1, True, False),
    ("conv3x3_256_100x88", "conv", 1, (100, 88), 256, 256, TAPS3, True, False),
    ("conv1x1_256_100x88", "conv", 1, (100, 88), 256, 256, TAPS1, True, False),
    ("deconv_256_128_100x88_resid", "deconv", 1, (100, 88), 256, 128, None, True, True),
    ("deconv_256_128_100x88", "deconv", 1, (100, 88), 256, 128, None, True, False),
    ("head_128_24_200x176", "conv", 1, (200, 176), 128, 24, TAPS1, False, False),
    ("conv3x3_128_b2_37x21", "conv", 2, (37, 21), 128, 128, TAPS3, True, False),
    ("conv3x3_128_b2_21x37", "conv", 2, (21, 37), 128, 128, TAPS3, True, False),
    ("deconv_256_128_b2_13x11_resid", "deconv", 2, (13, 11), 256, 128, None, True, True),
    ("head_128_24_b2_19x27", "conv", 2, (19, 27), 128, 24, TAPS1, False, False),
]


def _input(batch, hw, c, gen):
    """NHWC fp32 with magnitudes spread over 2^-12 .. 4 and a third of the pixels exactly zero (post-ReLU maps)"""
    x = torch.randn((batch, hw[0], hw[1], c), generator=gen, device="cuda")
    x = x * torch.exp2(-torch.randint(0, 13, (batch, hw[0], hw[1], 1), generator=gen, device="cuda").float()) * 4.0
    return x * (torch.rand((batch, hw[0], hw[1], 1), generator=gen, device="cuda") > 0.33)


def _bits(t):
    return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t.contiguous().view(torch.int16)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_p2_equals_h2_bitwise(case):
    label, kind, batch, hw, cin, cout, taps, relu, with_resid = case
    gen = torch.Generator(device="cuda")
    gen.manual_seed(sum(map(ord, label)))
    ntaps = 9 if kind == "deconv" else len(taps)
    w = torch.randn((ntaps, cin, cout), generator=gen, device="cuda") / (cin * ntaps) ** 0.5
    sc = torch.rand((cout,), generator=gen, device="cuda") + 0.5
    sh = torch.randn((cout,), generator=gen, device="cuda") * 0.1
    cout_pad = 32 if cout <= 32 else -(-cout // 128) * 128
    planes_w, inv = ops.pack_weight_h2(w, cout_pad)
    scale = (sc * inv[:cout]).contiguous()
    x = _input(batch, hw, cin, gen)
    out_hw = (2 * hw[0], 2 * hw[1]) if kind == "deconv" else hw
    oshape = (batch, out_hw[0], out_hw[1], cout)
    resid = resid_info = None
    if with_resid:
        resid = torch.randn(oshape, generator=gen, device="cuda")
        resid_info = torch.zeros((2,), device="cuda")
        ops.absmax(resid, resid_info[0:1])

    # p2 operands: the input's abs-max and its planes with the scale of that abs-max
    info = torch.zeros((2,), device="cuda")
    ops.absmax(x, info[0:1])
    xp = ops.alloc_bev_planes(batch, hw[0], hw[1], cin, x.device)
    ops.bev_split_planes(x, info, xp)

    out_h2 = torch.full(oshape, float("nan"), device="cuda")
    amax_h2 = torch.zeros((1,), device="cuda")
    out_p2 = torch.full(oshape, float("nan"), device="cuda")
    planes_p2 = torch.full((2,) + oshape, 0, dtype=torch.int16, device="cuda").fill_(F16_SENTINEL).view(torch.float16)
    out_info = torch.zeros((2,), device="cuda")
    gain, shift_max = ops.conv_gain(w, sc), float(sh.abs().max())
    if kind == "deconv":
        ops.bev_deconv_h2(x, planes_w, scale, sh, resid, out_h2, relu, info[0:1], amax_h2)
        ops.bev_deconv_p2(xp, info, planes_w, scale, sh, resid, resid_info, gain, shift_max, out_p2, planes_p2, out_info, relu)
    else:
        d = ops.conv_desc(batch, hw, cin, hw, cout, hw, taps, relu=relu)
        ops.bev_conv_h2(x, planes_w, scale, sh, resid, out_h2, d, info[0:1], amax_h2)
        ops.bev_conv_p2(xp, info, planes_w, scale, sh, resid, resid_info, gain, shift_max, out_p2, planes_p2, out_info, d)
    torch.cuda.synchronize()

    assert not torch.isnan(out_h2).any(), label          # every output pixel written
    assert torch.equal(_bits(out_p2), _bits(out_h2)), label
    assert _bits(out_info[0:1]).item() == _bits(amax_h2).item(), label
    s = out_info[1]
    xs = out_h2 * s
    hi = xs.half()
    lo = (xs - hi.float()).half()
    assert torch.equal(_bits(planes_p2[0]), _bits(hi)), label
    assert torch.equal(_bits(planes_p2[1]), _bits(lo)), label
