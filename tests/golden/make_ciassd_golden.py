"""Generate tests/golden/ciassd_loss_case.npz by running the reference's own CIA-SSD head loss in place on the CPU:
det3d/models/bbox_heads/mg_head_ciassd.py MultiGroupHead.loss (with its prepare_loss_weights, add_sin_difference, get_direction_target,
_get_pos_neg_loss) over the reference's loss classes (losses.py) and box coder (box_torch_ops.second_box_decode).  The aligned 3-D IoU
is the reference's own iou3d_utils.boxes_aligned_iou3d_gpu with its CUDA overlap kernel bound to the reference's CPU twin
(iou3d_cpu.cpp, compiled in place into oracle/_ref) and ``torch.cuda.FloatTensor`` to a CPU tensor; the other shims are make_golden.py's.

    python tests/golden/make_ciassd_golden.py

Inputs (stored): a crafted head output of 4 frames on a 16 x 22 grid (2 anchors per cell), its anchors, labels and regression targets --
frame 0 with many positives, frame 1 with none, frame 2 with ignored anchors (-1) among few positives, frame 3 with yaws across the
+-pi wrap; box residuals on both sides of the smooth-L1 knee 1/sigma^2 (never within 5e-3 of it), and IoU predictions away from it.
Stored outputs: every value of the returned dict and the autograd gradient of ``loss`` w.r.t. box_preds, cls_preds, dir_cls_preds and
iou_preds."""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "se-ssd_b200"), os.path.join(ROOT, "tests"), HERE]

import make_golden as mg  # noqa: E402
from oracle import build as obuild  # noqa: E402

B, H, W = 4, 16, 22
A = H * W * 2
SIGMA = 3.0
KNEE = 1.0 / SIGMA ** 2


def _away_from_knee(rs, n, lo=0.005):
    """|d| in [0.01, KNEE - lo] or [KNEE + lo, 0.8], random sign, half on each side"""
    small = rs.uniform(0.01, KNEE - lo, n)
    large = rs.uniform(KNEE + lo, 0.8, n)
    return np.where(rs.rand(n) < 0.5, small, large) * np.where(rs.rand(n) < 0.5, -1.0, 1.0)


def inputs(seed=17):
    rs = np.random.RandomState(seed)
    iy, ix = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    cx = (ix.reshape(-1) + 0.5) * (70.4 / W)
    cy = -40.0 + (iy.reshape(-1) + 0.5) * (80.0 / H)
    anchors = np.zeros((H * W, 2, 7), np.float32)
    anchors[..., 0], anchors[..., 1] = cx[:, None], cy[:, None]
    anchors[..., 2], anchors[..., 3:6] = -1.0, (1.6, 3.9, 1.56)
    anchors[:, 1, 6] = 1.57
    anchors = anchors.reshape(A, 7)
    labels = np.zeros((B, A), np.int64)
    labels[0] = np.where(rs.rand(A) < 0.4, 1, np.where(rs.rand(A) < 0.1, -1, 0))
    labels[2] = np.where(rs.rand(A) < 0.05, 1, np.where(rs.rand(A) < 0.3, -1, 0))
    labels[3] = np.where(rs.rand(A) < 0.1, 1, 0)
    targets = np.zeros((B, A, 7), np.float32)
    targets[..., :3] = rs.normal(0, 0.3, (B, A, 3))
    targets[..., 3:6] = rs.normal(0, 0.1, (B, A, 3))
    targets[..., 6] = rs.uniform(-1.2, 1.2, (B, A))
    # frame 3: ground-truth yaws near +pi or -pi (target residual = yaw - anchor yaw), predictions on the other side of the wrap
    yaw = np.where(rs.rand(A) < 0.5, np.pi - rs.uniform(0.01, 0.1, A), -np.pi + rs.uniform(0.01, 0.1, A))
    targets[3, :, 6] = yaw - anchors[:, 6]
    box = targets.astype(np.float64).copy()
    box[..., :6] += _away_from_knee(rs, B * A * 6).reshape(B, A, 6)
    box[..., 6] += _away_from_knee(rs, B * A).reshape(B, A)
    box[3, :, 6] = targets[3, :, 6] + _away_from_knee(rs, A) - 2 * np.pi * np.sign(yaw)       # across the wrap: a - b = delta -+ 2 pi
    box = box.astype(np.float32)
    cls = rs.normal(-2.0, 1.5, (B, A)).astype(np.float32)
    cls[labels > 0] += 2.5
    dirs = rs.normal(0, 1.0, (B, A, 2)).astype(np.float32)
    iou = rs.uniform(-1.0, 1.0, (B, A)).astype(np.float32)
    return anchors, labels, targets, box, cls, dirs, iou


def _reference_head():
    mg.install_det3d_shims()
    mg._stub("det3d.models.losses.utils", weight_reduce_loss=None)
    mg._stub("det3d.models.losses.gious", gious_3D=None)
    losses = mg._load("det3d.models.losses.losses", "det3d/models/losses/losses.py")
    bn = mg._load("det3d.core.bbox.box_np_ops", "det3d/core/bbox/box_np_ops.py")
    sys.modules["det3d.core.bbox"].box_np_ops = bn
    bt = mg._load("det3d.core.bbox.box_torch_ops", "det3d/core/bbox/box_torch_ops.py")
    sys.modules["det3d.core.bbox"].box_torch_ops = bt
    iu = mg._load("det3d.core.iou3d.utils", "det3d/core/iou3d/utils.py")
    sys.modules["det3d.core.iou3d"].utils = iu
    ref = obuild.load_ref() or (obuild.build_ref() and obuild.load_ref())

    def aligned_overlap(a, b, out):                     # the reference's CPU overlap kernel, pair i with pair i
        full = torch.zeros(a.shape[0], b.shape[0])
        ref.boxes_overlap_bev_cpu(a.contiguous(), b.contiguous(), full)
        out.copy_(torch.diagonal(full).reshape(-1, 1))
    mg._stub("iou3d_cuda", boxes_aligned_overlap_bev_gpu=aligned_overlap)
    torch.cuda.FloatTensor = lambda size: torch.FloatTensor(size)
    iou3d = mg._load("det3d.core.iou3d.iou3d_utils", "det3d/core/iou3d/iou3d_utils.py")
    ci = mg._load("det3d.models.bbox_heads.mg_head_ciassd", "det3d/models/bbox_heads/mg_head_ciassd.py")
    ci.iou3d_utils = iou3d
    head = types.SimpleNamespace(
        box_coder=types.SimpleNamespace(decode_torch=lambda enc, a: bt.second_box_decode(enc, a, False, False)),
        box_n_dim=7, num_classes=[1], encode_rad_error_by_sin=True, use_direction_classifier=True, direction_offset=0.0,
        loss_norm=dict(type="NormByNumPositives", pos_cls_weight=1.0, neg_cls_weight=1.0),
        loss_cls=losses.SigmoidFocalLoss(alpha=0.25, gamma=2.0, loss_weight=1.0),
        loss_reg=losses.WeightedSmoothL1Loss(sigma=SIGMA, code_weights=[1.0] * 7, codewise=True, loss_weight=2.0),
        loss_aux=losses.WeightedSoftmaxClassificationLoss(name="direction_classifier", loss_weight=0.2),
        loss_iou_pred=losses.WeightedSmoothL1Loss(sigma=SIGMA, code_weights=None, codewise=True, loss_weight=1.0))
    head.prepare_loss_weights = types.MethodType(ci.MultiGroupHead.prepare_loss_weights, head)
    return ci, head, iou3d, bt


def main():
    ci, head, iou3d, bt = _reference_head()
    anchors, labels, targets, box, cls, dirs, iou = inputs()
    preds = dict(box_preds=torch.from_numpy(box).reshape(B, H, W, 14), cls_preds=torch.from_numpy(cls).reshape(B, H, W, 2),
                 dir_cls_preds=torch.from_numpy(dirs).reshape(B, H, W, 4), iou_preds=torch.from_numpy(iou).reshape(B, H, W, 2))
    preds = {k: v.clone().requires_grad_(True) for k, v in preds.items()}
    anc = torch.from_numpy(anchors)[None].expand(B, -1, -1).contiguous()
    example = dict(anchors=[anc], labels=[torch.from_numpy(labels)], reg_targets=[torch.from_numpy(targets)])
    out = ci.MultiGroupHead.loss(head, example, [preds])
    # margins of the crafted cases, in the reference's own arithmetic
    pos = labels > 0
    assert pos[0].sum() > 200 and pos[1].sum() == 0 and (labels[2] < 0).sum() > 100 and 0 < pos[2].sum() < 60 and pos[3].sum() > 20
    d = np.abs(box.astype(np.float64) - targets)[pos][:, :6]
    assert (np.abs(d - KNEE) > 4e-3).all() and (d < KNEE).any() and (d > KNEE).any()
    sd = np.abs(np.sin(box[..., 6]) * np.cos(targets[..., 6]) - np.cos(box[..., 6]) * np.sin(targets[..., 6]))[pos]
    assert (np.abs(sd - KNEE) > 1e-3).all()
    assert (np.abs(box[3, :, 6] - targets[3, :, 6])[pos[3]] > 5.0).all()                      # the +-pi wrap
    pm = torch.from_numpy(pos)
    q = bt.second_box_decode(torch.from_numpy(box)[pm], anc[pm], False, False)
    g = bt.second_box_decode(torch.from_numpy(targets)[pm], anc[pm], False, False)
    t = 2 * iou3d.boxes_aligned_iou3d_gpu(q, g) - 1
    assert (np.abs(np.abs(iou[pos] - t.numpy().reshape(-1)) - KNEE) > 1e-3).all() and (t.numpy() > -1).any()
    out["loss"][0].backward()
    grads = {"grad_" + k: v.grad.numpy() for k, v in preds.items()}
    vals = {}
    for k, v in out.items():
        if k == "loss":
            vals[k] = np.float32(v[0].item())
        elif k == "loc_loss_elem":
            vals[k] = np.float32([float(e) for e in v[0]])
        else:
            vals[k] = np.asarray(v[0].detach().numpy() if hasattr(v[0], "detach") else v[0])
    np.savez_compressed(os.path.join(HERE, "ciassd_loss_case.npz"), anchors=anchors, labels=labels.astype(np.int8), reg_targets=targets,
                        box_preds=box, cls_preds=cls, dir_cls_preds=dirs, iou_preds=iou, **vals, **grads)
    print({k: (float(v) if np.ndim(v) == 0 else np.round(v, 5).tolist()) for k, v in vals.items()})
    print("positives per frame", pos.sum(1).tolist(), "grad abs sums", {k: float(np.abs(v).sum()) for k, v in grads.items()})


if __name__ == "__main__":
    main()
