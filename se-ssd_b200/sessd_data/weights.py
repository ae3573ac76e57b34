"""Seeded random-initialised parameters of the SE-SSD car model (no checkpoint is available offline) and the
conversion of reference-style state dicts into the runner inputs.

State-dict key names follow the reference modules (``backbone.middle_conv.{0,3,..}``, ``neck.bottom_up_block_0.1`` ...,
``bbox_head.tasks.0.conv_box`` ...) so that a real SE-SSD checkpoint (det3d/torchie/trainer/checkpoint.py:117-171)
can be fed through ``split_detector_state``.
"""
import math
import os

import numpy as np
import torch

from .layers import SPMIDDLE_LAYERS, SSFA_CONVS


def _bn(g, c, prefix, sd):
    sd[prefix + ".weight"] = 1.0 + 0.1 * torch.randn(c, generator=g)
    sd[prefix + ".bias"] = 0.1 * torch.randn(c, generator=g)
    sd[prefix + ".running_mean"] = 0.1 * torch.randn(c, generator=g)
    sd[prefix + ".running_var"] = 1.0 + 0.2 * torch.rand(c, generator=g)
    sd[prefix + ".num_batches_tracked"] = torch.tensor(0)


def random_detector_state(seed=0, num_input_features=4, cls_bias=None):
    """Full VoxelNet state dict with kaiming-style conv weights and non-trivial BN statistics.
    ``cls_bias``: bias of the classification conv (e.g. -2.5 makes ~few % of anchors pass the 0.3 score threshold,
    resembling a trained detector's candidate counts instead of random init's ~50 %)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    cin = num_input_features
    for i, (_kind, cout, ks, _st, _pd, _key) in enumerate(SPMIDDLE_LAYERS):
        fan_in = cin * ks[0] * ks[1] * ks[2]
        sd["backbone.middle_conv.%d.weight" % (3 * i)] = torch.randn((*ks, cin, cout), generator=g) * math.sqrt(2.0 / fan_in)
        _bn(g, cout, "backbone.middle_conv.%d" % (3 * i + 1), sd)
        cin = cout
    for name, kind, ci, co, k in SSFA_CONVS:
        shape = (co, ci, k, k) if kind == "conv" else (ci, co, k, k)
        sd["neck." + name + ".weight"] = torch.randn(shape, generator=g) * math.sqrt(2.0 / (ci * k * k))
        blk, idx = name.rsplit(".", 1)
        _bn(g, co, "neck.%s.%d" % (blk, int(idx) + 1), sd)
    for nm, co in (("conv_box", 14), ("conv_cls", 2), ("conv_iou", 2), ("conv_dir", 4)):
        sd["bbox_head.tasks.0.%s.weight" % nm] = torch.randn((co, 128, 1, 1), generator=g) * math.sqrt(1.0 / 128)
        sd["bbox_head.tasks.0.%s.bias" % nm] = 0.1 * torch.randn(co, generator=g)
    if cls_bias is not None:
        sd["bbox_head.tasks.0.conv_cls.bias"] = torch.full((2,), float(cls_bias))
    return sd


def split_detector_state(sd):
    """-> (middle_layers for SpMiddleRunner.load_weights, ssfa_state, head_state) from a VoxelNet state dict."""
    layers = []
    for i in range(len(SPMIDDLE_LAYERS)):
        c, b = "backbone.middle_conv.%d" % (3 * i), "backbone.middle_conv.%d" % (3 * i + 1)
        layers.append(dict(weight=sd[c + ".weight"], gamma=sd[b + ".weight"], beta=sd[b + ".bias"],
                           mean=sd[b + ".running_mean"], var=sd[b + ".running_var"]))
    ssfa = {k[len("neck."):]: v for k, v in sd.items() if k.startswith("neck.")}
    head = {k[len("bbox_head."):]: v for k, v in sd.items() if k.startswith("bbox_head.")}
    return layers, ssfa, head


def kitti_car_anchors(feature_size=(1, 200, 176), anchor_range=(0, -40.0, -1.0, 70.4, 40.0, -1.0), sizes=(1.6, 3.9, 1.56),
                      rotations=(0, 1.57), dtype=np.float32):
    """Anchor grid of examples/second/configs/config.py:82-100 == create_anchors_3d_range (box_np_ops.py:780-833):
    [70400, 7] with anchor index (y*176 + x)*2 + rot."""
    ar = np.array(anchor_range, dtype)
    stride = (ar[3] - ar[0]) / feature_size[2]
    zc = np.linspace(ar[2], ar[5], feature_size[0], dtype=dtype)
    yc = np.linspace(ar[1], ar[4], feature_size[1], endpoint=False, dtype=dtype) + stride / 2
    xc = np.linspace(ar[0], ar[3], feature_size[2], endpoint=False, dtype=dtype) + stride / 2
    rot = np.array(rotations, dtype)
    sz = np.array(sizes, dtype).reshape(-1, 3)
    out = np.zeros((len(zc), len(yc), len(xc), sz.shape[0], len(rot), 7), dtype)
    out[..., 0] = xc[None, None, :, None, None]
    out[..., 1] = yc[None, :, None, None, None]
    out[..., 2] = zc[:, None, None, None, None]
    out[..., 3:6] = sz[None, None, None, :, None, :]
    out[..., 6] = rot[None, None, None, None, :]
    return out.reshape(-1, 7)


# ---------------------------------------------------------------------------------------------------------------- bench weights
_CALIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "bench_calib.json")
BOX_HEAD_SCALE = 0.1
IOU_HEAD_SCALE = 0.1
EMPTY_LOGIT = -6.0        # classification logit of every anchor over empty space (sigmoid = 2.5e-3, far below the 0.3 threshold)


def load_bench_calibration():
    import json
    with open(_CALIB_PATH) as f:
        return json.load(f)


NECK_GAIN_LAYERS = ("bottom_up_block_0.1", "bottom_up_block_0.4", "bottom_up_block_0.7", "bottom_up_block_1.0", "bottom_up_block_1.3",
                    "bottom_up_block_1.6", "trans_0.0", "trans_1.0", "deconv_block_0.0", "deconv_block_1.0", "conv_0.0", "conv_1.0")


def _bn_of(conv_name):
    blk, idx = conv_name.rsplit(".", 1)
    return "%s.%d" % (blk, int(idx) + 1)


def quiet_neck_state(ssfa_state, seed=0, gains=None):
    """Make the SSFA neck silent over empty space and keep the signal of the occupied regions alive, like a trained detector:
    * every BatchNorm gets running_mean = 0 and a slightly NEGATIVE beta, so that a zero input stays exactly zero through
      conv -> BN -> ReLU (and through the deconv / residual / attention fusion).  A plain random init answers empty space (and the
      zero padding at the map border) with a constant as large as the response to the points themselves: hundreds of anchors then
      share bit-identical logits around the score threshold and the kept set depends on tie-breaking;
    * `gains` (one scalar per conv layer, committed in bench_calib.json) multiplies the BatchNorm weight: kaiming init assumes dense
      inputs, the BEV map is ~12 % occupied, so without it the activations shrink below the negative betas within three layers
      (a trained BN has running_var matched to its input instead)."""
    g = torch.Generator().manual_seed(1000 + seed)
    out = dict(ssfa_state)
    for k in sorted(out):
        if k.endswith(".running_mean"):
            out[k] = torch.zeros_like(out[k])
            b = k[:-len("running_mean")] + "bias"
            out[b] = -(0.02 + 0.05 * torch.randn(out[b].shape, generator=g).abs())
    for name, gain in (gains or {}).items():
        out[_bn_of(name) + ".weight"] = out[_bn_of(name) + ".weight"] * float(gain)
    return out


def apply_cls_calibration(head_state, alpha, prefix="tasks.0."):
    """logit = alpha * (w . x) + EMPTY_LOGIT: x is exactly 0 over empty space (quiet neck), alpha puts ~400 anchors of the calibration
    frame over the 0.3 score threshold (what a trained SE-SSD produces on a KITTI frame)."""
    head = dict(head_state)
    head[prefix + "conv_cls.weight"] = head[prefix + "conv_cls.weight"].clone().float() * float(alpha)
    head[prefix + "conv_cls.bias"] = torch.full((2,), EMPTY_LOGIT)
    return head


def bench_detector_state(cloud="ring", seed=0, alpha=None, gains=None):
    """The bench / parity workload's parameters: seeded random init, quiet neck, and the COMMITTED classification scale of
    sessd_data/bench_calib.json (generated once with scripts/make_bench_calib.py from the CPU oracle), so that the CUDA arm and the
    CPU reference arm use bit-identical weights.  Returns (middle_layers, ssfa_state, head_state)."""
    sd = random_detector_state(seed)
    layers, ssfa, head = split_detector_state(sd)
    if alpha is None or gains is None:
        cal = load_bench_calibration()
        assert cal["seed"] == seed
        gains = cal["neck_gains"] if gains is None else gains
        alpha = cal[cloud]["alpha"] if alpha is None else alpha
    ssfa = quiet_neck_state(ssfa, seed, gains)
    # box regression head scaled to trained-like magnitudes (|residual| <~ 1): random-init residuals of +-10 put most decoded boxes
    # outside the post-processing range and give them sizes of e^10 m
    head = dict(head)
    for k in ("tasks.0.conv_box.weight", "tasks.0.conv_box.bias"):
        head[k] = head[k].float() * BOX_HEAD_SCALE
    # IoU head: predictions around 0.5 +- 0.3 like a trained head (random init gives iou in [-3, 3]: (iou + 1) / 2 near 0 makes the
    # rectified score x^4 ill-conditioned, relative differences of 1e-5 in the head become 3e-3 in the score)
    head["tasks.0.conv_iou.weight"] = head["tasks.0.conv_iou.weight"].float() * IOU_HEAD_SCALE
    head["tasks.0.conv_iou.bias"] = torch.full((2,), 0.5)
    return layers, ssfa, apply_cls_calibration(head, alpha)


def task_anchors(target_assigner, feature_size=(1, 200, 176), dtype=np.float32):
    """Per-task anchors [A, 7] of a config's ``target_assigner`` (its ``anchor_generators``, one per one-class task, in task order),
    by the grid arithmetic of kitti_car_anchors with each generator's sizes, anchor_ranges and rotations -- what
    AnchorGeneratorRange / TargetAssigner.generate_anchors_dict give.  The list FrameEngine.load_weights takes for a multi-class head."""
    gens = target_assigner["anchor_generators"]
    tasks = target_assigner.get("tasks") if hasattr(target_assigner, "get") else None
    if tasks is not None and any(int(t["num_class"]) != 1 for t in tasks):
        raise NotImplementedError("multi-class inference takes one class per task")
    out = []
    for g in gens:
        if g.get("type", "anchor_generator_range") != "anchor_generator_range":
            raise NotImplementedError("anchor generator %r: only anchor_generator_range is supported" % g.get("type"))
        out.append(kitti_car_anchors(feature_size, anchor_range=tuple(g["anchor_ranges"]), sizes=tuple(g["sizes"]),
                                     rotations=tuple(g["rotations"]), dtype=dtype))
    return out


def add_task_heads(sd, num_tasks, seed=1, cls_bias=None):
    """Adds seeded heads ``bbox_head.tasks.1.`` ... ``tasks.{num_tasks-1}.`` (same shapes and scales as random_detector_state's
    ``tasks.0.``) to a detector state dict, for a model with num_tasks one-class tasks; ``tasks.0.`` and everything else is kept."""
    g = torch.Generator().manual_seed(seed)
    for t in range(1, int(num_tasks)):
        for nm, co in (("conv_box", 14), ("conv_cls", 2), ("conv_iou", 2), ("conv_dir", 4)):
            sd["bbox_head.tasks.%d.%s.weight" % (t, nm)] = torch.randn((co, 128, 1, 1), generator=g) * math.sqrt(1.0 / 128)
            sd["bbox_head.tasks.%d.%s.bias" % (t, nm)] = 0.1 * torch.randn(co, generator=g)
        if cls_bias is not None:
            sd["bbox_head.tasks.%d.conv_cls.bias" % t] = torch.full((2,), float(cls_bias))
    return sd
