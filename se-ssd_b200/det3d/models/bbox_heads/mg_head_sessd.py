"""MultiGroupHead (SE-SSD variant) -- inference half (reference: det3d/models/bbox_heads/mg_head_sessd.py:195-230, 379-523,
893-1057).  Same constructor signature / parameter names (``tasks.0.conv_box`` ...).

* ``forward``  : the four 1x1 convs are ONE 128 -> 22 tensor-core GEMM writing NHWC directly (the reference launches 4 convs + 4
  permute copies); the returned dict has the reference's keys and shapes.
* ``predict``  : decode -> sigmoid -> threshold -> IoU-rectified score -> top-k -> rotated NMS -> frustum filter -> direction fix
  -> range mask in five kernels with no host round trip (sessd_postprocess); the reference syncs to the host twice per frame
  (box_torch_ops.py:536, mg_head_sessd.py:1026) and clips polygons on one CPU thread.
* ``loss``     : the assembled SE-SSD head loss (supervised terms + ODIoU on the device, consistency loss against the teacher); value and
  gradient w.r.t. the packed head tensor.  In train mode the packed tensor carries a graph to the head's input and its convs' weights
  and biases (sessd_b200.bev_grad), so ``loss.backward()`` reaches the neck and the encoder below it."""
import logging
import math

import numpy as np
import torch
from torch import nn

from det3d.core.bbox.geometry import frustum_planes
from sessd_b200 import bev_grad, ops
from sessd_b200.runners import HeadRunner, RunnerCache

from ..builder import build_loss
from ..registry import HEADS


class _HeadLossFn(torch.autograd.Function):
    """Scalar loss whose value and gradient w.r.t. the packed head tensor were both produced by the device loss kernels."""

    @staticmethod
    def forward(ctx, packed, value, grad):
        ctx.save_for_backward(grad)
        return value.detach().reshape(()).clone()

    @staticmethod
    def backward(ctx, grad_out):
        (grad,) = ctx.saved_tensors
        return grad_out * grad, None, None


@HEADS.register_module
class Head(nn.Module):
    def __init__(self, num_input, num_pred, num_cls, use_dir=False, num_dir=0, header=True, name="", focal_loss_init=False, **kwargs):
        super().__init__(**kwargs)
        self.use_dir = use_dir
        self.conv_box = nn.Conv2d(num_input, num_pred, 1)
        self.conv_cls = nn.Conv2d(num_input, num_cls, 1)
        self.conv_iou = nn.Conv2d(num_input, 2, 1)
        self.trans_conv = None
        if self.use_dir:
            self.conv_dir = nn.Conv2d(num_input, num_dir, 1)
        self._runner = RunnerCache()

    def packed_forward(self, x):
        """x logical NCHW [B,128,H,W] -> packed NHWC [B,H,W,24] = [box 14 | cls 2 | dir 4 | iou 2 | pad 2]."""
        if not (self.use_dir and self.conv_box.out_channels == 14 and self.conv_cls.out_channels == 2 and self.conv_dir.out_channels == 4):
            raise NotImplementedError("the fused head kernel is built for the car head: 2 anchors x (7 box, 1 cls, 2 dir, 1 iou)")
        if self.training:       # differentiable w.r.t. x and the four convs' weights and biases (sessd_b200.bev_grad); a fresh tensor
            return bev_grad.head_forward(self, x)
        b, c, h, w = x.shape
        runner = self._runner.get(self, (b, h, w, str(x.device)), lambda: HeadRunner(b, (h, w), x.device),
                                  lambda r: r.load_state({k: v.detach() for k, v in self.state_dict().items()}, prefix=""))
        return runner.forward(x.detach().float().permute(0, 2, 3, 1).contiguous())

    def forward(self, x):
        # a fresh tensor per call (like the reference): the runner's output buffer is overwritten by the next forward, and the SE-SSD
        # teacher / student flow runs two forwards before either result is consumed
        packed = self.packed_forward(x)
        if not self.training:
            packed = packed.clone()
        ret = {"box_preds": packed[..., 0:14].contiguous(), "cls_preds": packed[..., 14:16].contiguous()}
        if self.use_dir:
            ret["dir_cls_preds"] = packed[..., 16:20].contiguous()
        ret["iou_preds"] = packed[..., 20:22].contiguous()
        ret["_packed"] = packed            # private: lets predict() skip re-packing
        return ret


@HEADS.register_module
class MultiGroupHead(nn.Module):
    def __init__(self, mode="3d", in_channels=[128, ], norm_cfg=None, tasks=[], weights=[], num_classes=[1, ], box_coder=None,
                 with_cls=True, with_reg=True, reg_class_agnostic=False, encode_background_as_zeros=True,
                 loss_norm=dict(type="NormByNumPositives", pos_cls_weight=1.0, neg_cls_weight=1.0, ),
                 loss_cls=dict(type="SigmoidFocalLoss", alpha=0.25, gamma=2.0, loss_weight=1.0, ), use_sigmoid_score=True,
                 loss_bbox=dict(type="WeightedSmoothL1Loss", sigma=3.0, code_weights=[1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0], codewise=True,
                                loss_weight=2.0, ),
                 encode_rad_error_by_sin=True,
                 loss_aux=dict(type="WeightedSoftmaxClassificationLoss", name="direction_classifier", loss_weight=0.2, ),
                 direction_offset=0.0, name="rpn", logger=None, ):
        super().__init__()
        assert with_cls or with_reg
        num_classes = [len(t["class_names"]) for t in tasks]
        self.class_names = [t["class_names"] for t in tasks]
        self.num_anchor_per_locs = [2 * n for n in num_classes]
        self.box_coder = box_coder
        self.with_cls, self.with_reg, self.in_channels, self.num_classes = with_cls, with_reg, in_channels, num_classes
        self.reg_class_agnostic, self.encode_rad_error_by_sin = reg_class_agnostic, encode_rad_error_by_sin
        self.encode_background_as_zeros, self.use_sigmoid_score = encode_background_as_zeros, use_sigmoid_score
        self.box_n_dim = self.box_coder.n_dim
        self.loss_cls = build_loss(loss_cls)
        self.loss_reg = build_loss(loss_bbox)
        if loss_aux is not None:
            self.loss_aux = build_loss(loss_aux)
        self.loss_norm = loss_norm
        self.logger = logger or logging.getLogger("MultiGroupHead")
        self.use_direction_classifier = loss_aux is not None
        if loss_aux:
            self.direction_offset = direction_offset
        self.bev_only = mode == "bev"
        self.tasks = nn.ModuleList()
        num_preds, num_dirs = [], []
        for num_c, num_a in zip(num_classes, self.num_anchor_per_locs):
            num_cls = num_a * num_c if encode_background_as_zeros else num_a * (num_c + 1)
            num_pred = num_a * (self.box_n_dim - 2 if self.bev_only else self.box_n_dim)
            num_dir = num_a * 2 if self.use_direction_classifier else None
            num_preds.append(num_pred)
            num_dirs.append(num_dir)
            self.tasks.append(Head(in_channels, num_pred, num_cls, use_dir=self.use_direction_classifier, num_dir=num_dir, header=False))
        self.logger.info("num_classes: %s, num_preds: %s, num_dirs: %s" % (num_classes, num_preds, num_dirs))
        self.logger.info("Finish MultiGroupHead Initialization")
        self.post_center_range = [0, -40.0, -5.0, 70.4, 40.0, 5.0]      # reference hard-codes this (:484)
        self.thresh = 0.3                                                # and this (:486)
        self._post = None
        self._post_key = None

    def init_weights(self, pretrained=None):
        if isinstance(pretrained, str):
            from det3d.torchie.trainer.checkpoint import load_checkpoint
            load_checkpoint(self, pretrained, strict=False)
            return
        if pretrained is not None:
            raise TypeError("pretrained must be a str or None")
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)

    def forward(self, x):
        return [task(x) for task in self.tasks]

    def _supervision_mask(self, example, batch, device):
        if "ssl_labeled" in example:
            return (torch.as_tensor(example["ssl_labeled"]) == 1).to(device)
        return torch.ones(batch, dtype=torch.bool, device=device)

    def _supervised_terms(self, example, preds_dict, keys, with_odiou):
        """One pass of the supervised terms over the supervised frames of ``preds_dict``: (values dict, loss scalar wired to the packed head
        tensor through ``_HeadLossFn``).  ``keys`` = the example entries to read (anchors, labels, reg_targets -- or their ``_raw`` twins for
        the teacher, mg_head_sessd.py:810-830)."""
        k_anc, k_lab, k_reg = keys
        packed = preds_dict["_packed"]
        mask = self._supervision_mask(example, packed.shape[0], packed.device)
        sel = packed if bool(mask.all()) else packed[mask]
        ex = dict(anchors=[example[k_anc][0][mask.to(example[k_anc][0].device)]], labels=[example[k_lab][0]], reg_targets=[example[k_reg][0]])
        out = self.loss_supervised(ex, [dict(_packed=sel.detach())], with_grad=True, with_odiou=with_odiou)
        b = sel.shape[0]
        labels = ex["labels"][0]
        head = sel.detach().reshape(b, -1, sel.shape[-1])
        box = head[..., :2 * self.box_n_dim].reshape(b, -1, self.box_n_dim)
        tgt = ex["reg_targets"][0].float()
        pos = labels > 0
        w = pos.float() / pos.sum(1, keepdim=True).clamp(min=1).float()
        d = torch.cat([box[..., :-1] - tgt[..., :-1], torch.sin(box[..., -1:]) * torch.cos(tgt[..., -1:]) - torch.cos(box[..., -1:]) * torch.sin(tgt[..., -1:])], -1)
        elem = (self._smooth_l1(d, float(self.loss_reg._sigma)) * w[..., None]).sum((0, 1)) / b      # analysis only (:752)
        value = out["cls_loss_reduced"] + out["dir_loss_reduced"] + out["iou_pred_loss"]
        if with_odiou:
            value = value + out["ious_loss"]
        grad = out["grad_head"]
        if sel is not packed:                                         # scatter the supervised frames' gradient back into the full batch
            full = torch.zeros_like(packed)
            full[mask] = grad
            grad = full
        out["loc_loss_elem"] = [e.cpu() for e in elem]
        out["num_pos"], out["num_neg"] = (labels > 0)[0].sum(), (labels == 0)[0].sum()
        return out, _HeadLossFn.apply(packed, value, grad)

    def loss(self, example, preds_dicts, preds_ema=None, **kwargs):
        """The SE-SSD head loss (reference mg_head_sessd.py:706-808), single-task car head: ``loss`` = focal cls + ODIoU box loss +
        direction CE + IoU-prediction smooth-L1 on the supervised frames (the smooth-L1 box term is reported, not summed, as in the
        reference :781), plus ``consistency_loss`` against the teacher's predictions (added by the trainer with the ramp-up weight,
        trainer_sessd.py:267) and the teacher's own supervised terms on the raw targets (``*_ema``, :810-884).  Values and the gradient
        w.r.t. the packed head tensor come from one device pass (csrc/headloss.cu, odiou.cu); ``loss`` is a torch scalar whose backward
        hands that gradient to ``preds_dicts[0]['_packed']``'s graph, and ``consistency_loss`` is differentiable through
        ``box_preds / cls_preds / iou_preds`` by torch autograd.  Returns the reference's key -> [per-task value] dict.  A head tensor
        produced by ``Head.forward`` in train mode carries the graph of the head, the neck and the encoder (in eval mode none)."""
        if len(preds_dicts) != 1:
            raise NotImplementedError("the fused loss kernels are built for the single-task (car) head")
        merged = {}
        if preds_ema is not None:
            merged["consistency_loss"] = [self.consistency_loss(preds_dicts, preds_ema, example)]
        out, loss = self._supervised_terms(example, preds_dicts[0], ("anchors", "labels", "reg_targets"), with_odiou=True)
        cpu = lambda v: v.detach().cpu()                                                     # noqa: E731
        merged.update(loss=[loss], cls_loss_reduced=[cpu(out["cls_loss_reduced"])], loc_loss_reduced=[cpu(out["loc_loss_reduced"])],
                      dir_loss_reduced=[cpu(out["dir_loss_reduced"])], iou_pred_loss=[cpu(out["iou_pred_loss"])],
                      loc_loss_elem=[out["loc_loss_elem"]], cls_pos_loss=[cpu(out["cls_pos_loss"])], cls_neg_loss=[cpu(out["cls_neg_loss"])],
                      ious_loss=[cpu(out["ious_loss"])], num_pos=[out["num_pos"]], num_neg=[out["num_neg"]])
        if preds_ema is not None:
            for k, v in self.get_model_ema_loss(example, preds_ema).items():
                merged[k] = [v[0]]
        return merged

    def get_model_ema_loss(self, example, preds_dicts):
        """The teacher's supervised terms on the un-augmented targets (``labels_raw`` / ``reg_targets_raw`` / ``anchors_raw``), reported only
        (reference mg_head_sessd.py:810-890; no ODIoU term there)."""
        out, loss = self._supervised_terms(example, preds_dicts[0], ("anchors_raw", "labels_raw", "reg_targets_raw"), with_odiou=False)
        cpu = lambda v: v.detach().cpu()                                                     # noqa: E731
        return dict(loss_ema=[cpu(loss)], cls_loss_reduced_ema=[cpu(out["cls_loss_reduced"])], loc_loss_reduced_ema=[cpu(out["loc_loss_reduced"])],
                    dir_loss_reduced_ema=[cpu(out["dir_loss_reduced"])], iou_pred_loss_ema=[cpu(out["iou_pred_loss"])],
                    loc_loss_elem_ema=[out["loc_loss_elem"]], cls_pos_loss_ema=[cpu(out["cls_pos_loss"])],
                    cls_neg_loss_ema=[cpu(out["cls_neg_loss"])], num_pos_ema=[out["num_pos"]], num_neg_ema=[out["num_neg"]])

    # ------------------------------------------------------------------------------------------------------------------ teacher / student
    @staticmethod
    def _smooth_l1(diff, sigma=3.0):
        """elementwise value of WeightedSmoothL1Loss (losses.py:180-191): 0.5 (sigma d)^2 below 1 / sigma^2, |d| - 0.5 / sigma^2 above"""
        a, cut = diff.abs(), 1.0 / (sigma * sigma)
        return torch.where(a <= cut, 0.5 * (a * sigma) ** 2, a - 0.5 * cut)

    def nn_distance(self, box1, box2, iou_thres=0.7, return_loss="10"):
        """Mutual nearest-neighbour matching of two box sets by rotated BEV IoU and the sin-difference smooth-L1 between matched boxes
        (reference mg_head_sessd.py:573-611).  box1 [N,7] (student, carries the gradient), box2 [M,7].  Returns (loss, idx1, idx2, mask1,
        mask2) with the reference's meaning, or five Nones when nothing overlaps by more than ``iou_thres``.  The IoU matrix is the device
        kernel behind det3d.core.iou3d.iou3d_utils.boxes_iou_bev_gpu; it only selects pairs (no gradient flows through it there either)."""
        from det3d.core.iou3d import iou3d_utils
        if return_loss not in ("10", "01", "11"):
            raise NotImplementedError
        iou = iou3d_utils.boxes_iou_bev_gpu(box1.detach().contiguous(), box2.detach().contiguous())
        mask1, mask2 = iou.max(dim=1).values > iou_thres, iou.max(dim=0).values > iou_thres
        sub = iou[mask1][:, mask2]
        if sub.shape[0] == 0 or sub.shape[1] == 0:
            return [None] * 5
        idx1, idx2 = sub.argmax(dim=1), sub.argmax(dim=0)            # partner of every kept box1 / of every kept box2
        kept1, kept2 = box1[mask1], box2[mask2]

        def pair_loss(a, b):                                         # add_sin_difference (:39-44) + smooth-L1, mean over the 7 codes
            d = torch.cat([a[:, :-1] - b[:, :-1], torch.sin(a[:, -1:]) * torch.cos(b[:, -1:]) - torch.cos(a[:, -1:]) * torch.sin(b[:, -1:])], -1)
            return self._smooth_l1(d, float(self.loss_reg._sigma)).sum(-1) / 7.0

        loss1 = pair_loss(kept1, kept2[idx1]) if return_loss[0] == "1" else None
        loss2 = pair_loss(kept2, kept1[idx2]) if return_loss[1] == "1" else None
        if return_loss == "10":
            val = loss1.sum() / loss1.shape[0]
        elif return_loss == "01":
            val = loss2.sum() / loss2.shape[0]
        else:
            val = (loss1.sum() + loss2.sum()) / (loss1.shape[0] + loss2.shape[0])
        return val, idx1, idx2, mask1, mask2

    def consistency_loss(self, preds_stu, preds_tea, example):
        """SE-SSD consistency loss between the student's and the teacher's predictions (reference mg_head_sessd.py:622-703): per frame,
        both heads' boxes are decoded, filtered (sigmoid score >= 0.3, centre inside the post-processing range), the teacher's boxes are
        carried into the student's augmentation frame (flip, global rotation, scale: ``example['transformation']``), matched by
        ``nn_distance`` and compared: box smooth-L1 + score smooth-L1 (sigmoid scores) + IoU-head smooth-L1 ((x+1)/2), summed over frames
        and divided by the batch size.  (The reference also evaluates a direction term and leaves it out of the sum; it is not computed
        here.)  Differentiable w.r.t. ``preds_stu`` through torch autograd; runs on the device (the matching uses the CUDA IoU kernel)."""
        from det3d.core.bbox import box_torch_ops
        stu, tea = preds_stu[0], preds_tea[0]
        batch = stu["box_preds"].shape[0]
        anchors = example["anchors"][0][0].reshape(-1, self.box_n_dim).to(stu["box_preds"].device).float()
        dev = stu["box_preds"].device
        lo = torch.tensor(self.post_center_range[:3], dtype=torch.float32, device=dev)
        hi = torch.tensor(self.post_center_range[3:], dtype=torch.float32, device=dev)

        def candidates(p, f):
            boxes = box_torch_ops.second_box_decode(p["box_preds"][f].reshape(-1, self.box_n_dim), anchors)
            cls = p["cls_preds"][f].reshape(-1, 1)
            keep = (torch.sigmoid(cls).squeeze(-1) >= 0.3) & (boxes[:, :3] >= lo).all(1) & (boxes[:, :3] <= hi).all(1)
            return boxes[keep], cls[keep], p["iou_preds"][f].reshape(-1, 1)[keep]

        total = torch.zeros(1, dtype=torch.float32, device=dev)
        sigma = 3.0                                                      # loss_score_consistency / loss_iou_consistency (:489-490)
        for f in range(batch):
            sb, scls, siou = candidates(stu, f)
            tb, tcls, tiou = candidates(tea, f)
            if sb.shape[0] == 0 or tb.shape[0] == 0:
                continue
            t = example["transformation"][f]
            tb = tb.detach().clone()
            if t["flipped"]:
                tb[:, 1] = -tb[:, 1]
                tb[:, 6] = math.pi - tb[:, 6]
            c, s = math.cos(t["noise_rotation"]), math.sin(t["noise_rotation"])
            x, y = tb[:, 0].clone(), tb[:, 1].clone()
            tb[:, 0], tb[:, 1] = x * c + y * s, y * c - x * s             # rotation_points_single_angle(axis=2) (box_torch_ops.py:331-345)
            tb[:, 6] += t["noise_rotation"]
            tb[:, :6] *= t["noise_scale"]
            box_loss, idx1, _idx2, mask1, mask2 = self.nn_distance(sb, tb)
            if box_loss is None:
                continue
            score_loss = self._smooth_l1(torch.sigmoid(scls[mask1]) - torch.sigmoid(tcls[mask2][idx1]).detach(), sigma).mean()
            iou_loss = self._smooth_l1((siou[mask1] + 1) * 0.5 - ((tiou[mask2][idx1] + 1) * 0.5).detach(), sigma).mean()
            total = total + box_loss + score_loss + iou_loss
        return total / batch

    def loss_supervised(self, example, preds_dicts, with_grad=True, with_odiou=False):
        """Supervised terms of ``loss`` (reference mg_head_sessd.py:706-768 without the teacher / ODIoU parts) for the
        single-task car head, value and gradient w.r.t. the fused head tensor in one device pass (csrc/headloss.cu).
        ``example``: ``anchors`` [[B,A,7]], ``labels`` [[B,A]], ``reg_targets`` [[B,A,7]] (device tensors, e.g. from
        TargetAssigner.assign_batch_gpu).  Returns the reference's reduced values (loss_weight * batch total / batch_size) and the gradient
        of ``cls_loss_reduced + dir_loss_reduced + iou_pred_loss`` (the reference's total does not include the smooth-L1 term)."""
        from sessd_b200 import ops
        packed = preds_dicts[0]["_packed"]
        b = packed.shape[0]
        head = packed.reshape(b, -1, packed.shape[-1]).contiguous()
        anchors = example["anchors"][0][0].reshape(-1, self.box_n_dim).contiguous().float()
        labels = example["labels"][0].to(torch.int32).contiguous()
        reg_targets = example["reg_targets"][0].float().contiguous()
        w_cls, w_dir = float(self.loss_cls._loss_weight), float(self.loss_aux._loss_weight)
        losses, grad = ops.head_loss(head, anchors, labels, reg_targets, alpha=float(self.loss_cls._alpha), sigma=float(self.loss_reg._sigma),
                                     dir_offset=float(self.direction_offset), pos_cls_weight=float(self.loss_norm["pos_cls_weight"]),
                                     neg_cls_weight=float(self.loss_norm["neg_cls_weight"]), w_cls=w_cls, w_loc=0.0, w_dir=w_dir,
                                     w_iou=1.0, with_grad=with_grad)
        tot = losses.sum(0) / b
        ious_loss = None
        if with_odiou:          # ODIoU box loss (odious.py:845-900): 2.0 * batch total / batch_size, gradient added to the box channels
            ious_loss = 2.0 * ops.odiou_loss(head, anchors, labels, reg_targets, losses, grad, w_odiou=2.0).sum() / b
        return dict(cls_loss_reduced=w_cls * tot[0], loc_loss_reduced=float(self.loss_reg._loss_weight) * tot[1], dir_loss_reduced=w_dir * tot[2],
                    cls_pos_loss=tot[3] / float(self.loss_norm["pos_cls_weight"]), cls_neg_loss=tot[4] / float(self.loss_norm["neg_cls_weight"]),
                    iou_pred_loss=tot[5], ious_loss=ious_loss, num_pos=losses[0, 6], num_neg=losses[0, 7], grad_head=None if grad is None else grad.view_as(packed))

    # ------------------------------------------------------------------------------------------------------------------
    def predict(self, example, preds_dicts, test_cfg, **kwargs):
        if len(preds_dicts) != 1:
            raise NotImplementedError("the fused post-processing is built for the single-task (car) head")
        preds = preds_dicts[0]
        anchors = example["anchors"][0]
        batch = int(anchors.shape[0])
        anc = anchors[0].reshape(-1, self.box_n_dim).float().contiguous()
        if not anc.is_cuda:
            anc = anc.cuda()
        packed = preds.get("_packed")
        if packed is None:
            b, h, w, _ = preds["box_preds"].shape
            packed = torch.zeros((b, h, w, 24), dtype=torch.float32, device=preds["box_preds"].device)
            packed[..., 0:14], packed[..., 14:16] = preds["box_preds"], preds["cls_preds"]
            packed[..., 16:20], packed[..., 20:22] = preds["dir_cls_preds"], preds["iou_preds"]
        nms = test_cfg.nms if hasattr(test_cfg, "nms") else test_cfg["nms"]
        if test_cfg["score_threshold"] <= 0.0:
            raise NotImplementedError("score_threshold must be positive (the reference path thresholds before NMS)")
        frustum = None
        calib = example.get("calib") if isinstance(example, dict) else None
        if calib is not None and "frustum" in calib:
            fr = calib["frustum"]
            fr = fr.cpu().numpy() if isinstance(fr, torch.Tensor) else np.asarray(fr)
            planes = np.stack([frustum_planes(fr[i])[0] for i in range(batch)], 0)          # [B, 6, 4]
            frustum = torch.from_numpy(np.ascontiguousarray(planes, np.float32)).to(packed.device)
        # "rotate_weighted_nms" selects DI-NMS with the head's constants (mg_head_sessd.py:999-1018 of the reference, where the choice is
        # a local variable); a config without the key keeps rotate_nms
        nms_type = nms.get("nms_type", "rotate_nms") if hasattr(nms, "get") else getattr(nms, "nms_type", "rotate_nms")
        key = (batch, int(anc.shape[0]), float(self.thresh), int(nms["nms_pre_max_size"]), int(nms["nms_post_max_size"]),
               float(nms["nms_iou_threshold"]), frustum is not None, str(packed.device), nms_type)
        if self._post is None or self._post_key != key:
            cfg = ops.make_post_cfg(batch=batch, num_anchors=int(anc.shape[0]), anchors_per_loc=self.num_anchor_per_locs[0],
                                    head_stride=24, score_thresh=self.thresh, nms_pre_max=nms["nms_pre_max_size"],
                                    nms_post_max=nms["nms_post_max_size"], nms_iou_thresh=nms["nms_iou_threshold"], nms_ge=True,
                                    post_range=self.post_center_range, direction_offset=getattr(self, "direction_offset", 0.0),
                                    use_frustum=frustum is not None, nms_type=nms_type)
            self._post, self._post_key = ops.PostBuffers(cfg, packed.device), key
        buf = ops.postprocess(packed.contiguous(), anc, frustum, self._post)
        counts = buf.count.cpu().tolist()                       # the one host sync of the frame
        meta = example.get("metadata", [None] * batch)
        out = []
        for i in range(batch):
            k = counts[i]
            out.append({"box3d_lidar": buf.boxes[i, :k].clone(), "scores": buf.scores[i, :k].clone(),
                        "label_preds": buf.labels[i, :k].long(), "metadata": meta[i]})
        return out
