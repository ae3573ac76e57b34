"""The pair-gather tensor-core conv (spconv_cg.cu) runs two persistent CTAs on each SM, so that one tile's chain of gathers overlaps the
other CTA's wgmmas and epilogue.  These tests pin that occupancy for the four default instantiations, and check that the deep pipeline
(one CTA per SM, twice the stages, several stages per producer warp) computes the same bits as the default on a whole frame."""
import numpy as np
import pytest
import torch

gpu = pytest.mark.gpu

CG_SHAPES = [(32, 32), (32, 64), (64, 32), (64, 64)]       # (cp, cout): layers 3-4, 5, the 32 -> 64 data gradient, layers 6-12


@gpu
@pytest.mark.parametrize("cp,cout", CG_SHAPES, ids=["%d-%d" % s for s in CG_SHAPES])
def test_cg_default_pipeline_fits_two_ctas_per_sm(cp, cout):
    from sessd_b200 import ops
    assert ops.spconv_cg_blocks_per_sm(cp, cout, 0) == 2
    assert ops.spconv_cg_blocks_per_sm(cp, cout, 1) >= 1


@gpu
def test_cg_blocks_per_sm_rejects_unknown_shapes():
    from sessd_b200 import ops
    from sessd_b200._lib import SessdError
    with pytest.raises(SessdError):
        ops.spconv_cg_blocks_per_sm(16, 32, 0)


def _encoder_outputs(feat, coors, deep):
    """every layer's output and the dense BEV tensor of one frame through SpMiddleRunner, with the cg kernels at `deep`"""
    from sessd_b200 import ops, weights
    from sessd_b200.runners import SpMiddleRunner
    n = len(coors)
    r = SpMiddleRunner(1, n, device="cuda")
    layers, _, _ = weights.split_detector_state(weights.random_detector_state(3))
    r.load_weights(layers)
    ops.set_sp_cg_deep(deep)
    try:
        dense = r.forward(torch.from_numpy(feat).cuda(), torch.from_numpy(coors).cuda(), torch.tensor([n], dtype=torch.int32, device="cuda"))
        torch.cuda.synchronize()
    finally:
        ops.set_sp_cg_deep(0)
    assert int(r.status.item()) == 0
    cg_layers = [li for li, p in enumerate(r.plan) if p["impl"] == "cg"]
    rows = [r.layer_output(li)[: int(r.levels[p["lout"]]["n"].item())].clone() for li, p in enumerate(r.plan)]
    return cg_layers, rows, dense.clone()


@gpu
def test_cg_deep_pipeline_matches_default_bitwise_on_a_uniform_frame():
    """uniform-20k frame (531-808 tiles per cg layer: on 132 SMs each CTA of the 264-CTA default grid runs 2 or 3 tiles and of the
    132-CTA deep grid 4 to 7, carrying its ring state between them): each layer's output and the dense BEV tensor bitwise equal at deep 0
    and deep 1.  The ring state at each tile boundary is checked on crafted tables in test_gpu_spconv_cg_grid."""
    from oracle import cpu as ocpu
    from sessd_b200 import synth
    v, c, num = ocpu.points_to_voxel(synth.uniform_cloud(0, 20000), synth.VOXEL_SIZE, synth.PC_RANGE, 5, 20000)
    coors = np.concatenate([np.zeros((len(c), 1), np.int32), c], 1).astype(np.int32)
    feat = (v.sum(1) / num[:, None]).astype(np.float32)
    cg0, out0, dense0 = _encoder_outputs(feat, coors, 0)
    cg1, out1, dense1 = _encoder_outputs(feat, coors, 1)
    assert cg0 == cg1 and len(cg0) == 11
    for li in cg0:
        assert out0[li].shape == out1[li].shape and out0[li].shape[0] > 0, li
        assert torch.equal(out0[li].view(torch.int32), out1[li].view(torch.int32)), "layer %d" % li
    assert torch.equal(dense0.view(torch.int32), dense1.view(torch.int32))
