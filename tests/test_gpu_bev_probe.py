"""The loader-only probe of the BEV conv kernel (sessd_bev_conv_p2_loads, lab library): its consumers wait on the full barriers and release
them without issuing wgmma or an epilogue.  Checked on a small 3x3 conv, with the single patch copy of the register-fed A and with the
copies shared-memory A descriptors would need: every work item and every tap step is walked (the counters say so), the launch ends, and
the output buffer is left alone."""
import ctypes as C

import pytest
import torch

gpu = pytest.mark.gpu

F32_SENTINEL = -1234.5
TAPS3 = [(dy, dx) for dy in (-1, 0, 1) for dx in (-1, 0, 1)]
ITEMS, STEPS = 1, 2          # P2Prof word order (csrc/bevconv_p2.cuh)


@gpu
@pytest.mark.parametrize("smem_a", [0, 1])
def test_loads_probe_walks_every_step_and_writes_nothing(smem_a):
    from sessd_b200 import _lib, ops
    h, w, cin, cout = 40, 24, 128, 64
    planes = torch.zeros((2, 1, h, w, cin), dtype=torch.float16, device="cuda")
    info = torch.tensor([1.0, 2.0 ** 14], device="cuda")
    weight = torch.zeros((2, len(TAPS3), 128, cin), dtype=torch.float16, device="cuda")
    scale = torch.ones(128, device="cuda")
    out = torch.full((1, h, w, cout), F32_SENTINEL, device="cuda")
    out_info = torch.zeros(2, device="cuda")
    num_sms = torch.cuda.get_device_properties(0).multi_processor_count
    prof = torch.zeros((num_sms, 16), dtype=torch.int64, device="cuda")
    d = ops.conv_desc(1, (h, w), cin, (h, w), cout, (h, w), TAPS3)
    _lib.check(_lib.lib.sessd_bev_conv_p2_loads(ops._p(planes), ops._p(info), ops._p(weight), 128, ops._p(scale), None, None, None, 1.0, 0.0,
                                                ops._p(out), None, ops._p(out_info), C.byref(d), None, smem_a, ops._p(prof), ops._st()),
               "sessd_bev_conv_p2_loads")
    torch.cuda.synchronize()
    # 8 x 16 pixel tiles in the orientation with fewer of them, one n-block; cin / 32 chunks of 9 tap steps per item
    tiles = min(-(-w // 8) * -(-h // 16), -(-h // 8) * -(-w // 16))
    rec = prof.cpu().numpy()
    assert rec[:, ITEMS].sum() == tiles and rec[:, STEPS].sum() == tiles * (cin // 32) * len(TAPS3)
    assert bool((out == F32_SENTINEL).all())
