"""Layer tables of the car model (shared by the runners, the weight generators and the tests)."""
from collections import namedtuple

# (kind, cout, ksize, stride, padding, indice_key)   det3d/models/backbones/scn.py:106-149
SPMIDDLE_LAYERS = [
    ("subm", 16, (3, 3, 3), (1, 1, 1), (1, 1, 1), "subm0"),
    ("subm", 16, (3, 3, 3), (1, 1, 1), (1, 1, 1), "subm0"),
    ("spconv", 32, (3, 3, 3), (2, 2, 2), (1, 1, 1), None),
    ("subm", 32, (3, 3, 3), (1, 1, 1), (1, 1, 1), "subm1"),
    ("subm", 32, (3, 3, 3), (1, 1, 1), (1, 1, 1), "subm1"),
    ("spconv", 64, (3, 3, 3), (2, 2, 2), (1, 1, 1), None),
    ("subm", 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), "subm2"),
    ("subm", 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), "subm2"),
    ("subm", 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), "subm2"),
    ("spconv", 64, (3, 3, 3), (2, 2, 2), (0, 1, 1), None),
    ("subm", 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), "subm3"),
    ("subm", 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), "subm3"),
    ("subm", 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), "subm3"),
    ("spconv", 64, (3, 1, 1), (2, 1, 1), (0, 0, 0), None),
]

# name, kind, cin, cout, k     det3d/models/necks/rpn_v1.py:135-210
SSFA_CONVS = [
    ("bottom_up_block_0.1", "conv", 128, 128, 3), ("bottom_up_block_0.4", "conv", 128, 128, 3),
    ("bottom_up_block_0.7", "conv", 128, 128, 3), ("bottom_up_block_1.0", "conv", 128, 256, 3),
    ("bottom_up_block_1.3", "conv", 256, 256, 3), ("bottom_up_block_1.6", "conv", 256, 256, 3),
    ("trans_0.0", "conv", 128, 128, 1), ("trans_1.0", "conv", 256, 256, 1),
    ("deconv_block_0.0", "deconv", 256, 128, 3), ("deconv_block_1.0", "deconv", 256, 128, 3),
    ("conv_0.0", "conv", 128, 128, 3), ("w_0.0", "conv", 128, 1, 1),
    ("conv_1.0", "conv", 128, 128, 3), ("w_1.0", "conv", 128, 1, 1),
]

# the four 1x1 head convs (mg_head_sessd.py:202-215) fused into one 128 -> 22 (+2 zero pad) GEMM
HEAD_CONV = ("head", "conv", 128, 24, 1)

# The neck + head launches of one SSFA forward (rpn_v1.py:220-235), in the record order of the skip plan (csrc/bevskip.cu).  kind, cin,
# cout and k come from SSFA_CONVS / HEAD_CONV; every conv pads by k // 2.  src / dst / residual name tensors; half: src is at half
# resolution; stride: the conv's input stride; f32: the planes runner writes dst in fp32 rather than as fp16 planes.
SSFALaunch = namedtuple("SSFALaunch", "name kind cin cout k src dst half stride residual relu f32")
_SPEC = {name: spec for name, *spec in SSFA_CONVS + [HEAD_CONV]}
SSFA_LAUNCHES = tuple(SSFALaunch(name, *_SPEC[name], *rest) for name, *rest in (
    # name                 src    dst    half   stride residual relu   f32
    ("bottom_up_block_0.1", "x", "b0a", False, 1, None, True, False),
    ("bottom_up_block_0.4", "b0a", "b0b", False, 1, None, True, False),
    ("bottom_up_block_0.7", "b0b", "x0", False, 1, None, True, False),
    ("bottom_up_block_1.0", "x0", "b1a", False, 2, None, True, False),
    ("bottom_up_block_1.3", "b1a", "b1b", True, 1, None, True, False),
    ("bottom_up_block_1.6", "b1b", "x1", True, 1, None, True, False),
    ("trans_0.0", "x0", "t0", False, 1, None, True, True),
    ("trans_1.0", "x1", "t1", True, 1, None, True, False),
    ("deconv_block_0.0", "t1", "m0", True, 1, "t0", True, False),
    ("deconv_block_1.0", "t1", "m1", True, 1, None, True, False),
    ("conv_0.0", "m0", "o0", False, 1, None, True, True),
    ("conv_1.0", "m1", "o1", False, 1, None, True, True),
    ("head", "out", "head", False, 1, None, False, True),
))


def ssfa_extents(launch, h, w):
    """(input, output) extent of a launch on an h x w neck: half resolution is (h // 2, w // 2); a deconv doubles its input"""
    full, half = (h, w), (h // 2, w // 2)
    src = half if launch.half else full
    return src, full if launch.kind == "deconv" else (half if launch.half or launch.stride == 2 else full)
