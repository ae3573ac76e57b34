"""Torch box ops on the hot path (reference: det3d/core/bbox/box_torch_ops.py:23-147, 527-621).

``rotate_nms`` keeps the reference signature but runs top-k + rotated IoU mask + greedy reduction ON THE GPU
(sessd_rotate_nms) instead of ``dets.cpu().numpy()`` -> boost::geometry on one CPU thread (nms_cpu.h:72-168).
``rotate_weighted_nms`` (DI-NMS) likewise runs top-k, centerness, the IoU matrix and the cluster loop on the GPU
(sessd_rotate_weighted_nms) instead of nms_cpu.h:173-384 on the host."""
import torch

from sessd_b200 import ops


def second_box_encode(boxes, anchors, encode_angle_to_vector=False, smooth_dim=False, norm_velo=False):
    if anchors.shape[-1] != 7 or encode_angle_to_vector or smooth_dim:
        raise NotImplementedError("only the 7-dim log-size encoding of the SE-SSD config is supported")
    xa, ya, za, wa, la, ha, ra = torch.split(anchors, 1, dim=-1)
    xg, yg, zg, wg, lg, hg, rg = torch.split(boxes, 1, dim=-1)
    diag = torch.sqrt(la ** 2 + wa ** 2)
    return torch.cat([(xg - xa) / diag, (yg - ya) / diag, (zg - za) / ha, torch.log(wg / wa), torch.log(lg / la),
                      torch.log(hg / ha), rg - ra], dim=-1)


def second_box_decode(box_encodings, anchors, encode_angle_to_vector=False, bin_loss=False, smooth_dim=False, norm_velo=False):
    if anchors.shape[-1] != 7 or encode_angle_to_vector or smooth_dim:
        raise NotImplementedError("only the 7-dim log-size encoding of the SE-SSD config is supported")
    xa, ya, za, wa, la, ha, ra = torch.split(anchors, 1, dim=-1)
    xt, yt, zt, wt, lt, ht, rt = torch.split(box_encodings, 1, dim=-1)
    diag = torch.sqrt(la ** 2 + wa ** 2)
    return torch.cat([xt * diag + xa, yt * diag + ya, zt * ha + za, torch.exp(wt) * wa, torch.exp(lt) * la,
                      torch.exp(ht) * ha, rt + ra], dim=-1)


def rotate_nms(rbboxes, scores, pre_max_size=None, post_max_size=None, iou_threshold=0.5):
    """rbboxes [n,5] (x,y,w,l,r), scores [n] (CUDA) -> LongTensor of kept indices (<= post_max_size, best first)."""
    n = int(scores.shape[0])
    if n == 0:
        return torch.zeros([0], dtype=torch.long, device=rbboxes.device)
    pre = n if pre_max_size is None else min(n, int(pre_max_size))
    post = pre if post_max_size is None else int(post_max_size)
    b = rbboxes.detach().float().contiguous()
    s = scores.detach().float().contiguous()
    if not b.is_cuda:
        raise RuntimeError("rotate_nms expects CUDA tensors (there is no CPU fallback)")
    cnt = torch.tensor([n], dtype=torch.int32, device=b.device)
    keep, num = ops.rotate_nms(b, s, cnt, n, pre, min(post, pre), float(iou_threshold), ge=True)
    return keep[: int(num.item())].long()


def rotate_weighted_nms(box_preds, rbboxes, dir_labels, labels_preds, scores, iou_preds, anchors, enable_centerness=True, centerness_pow=1,
                        centerness_c=False, pre_max_size=None, post_max_size=None, iou_threshold=0.5, nms_cnt_thresh=2.6,
                        nms_sigma_dist_interval=(0, 20, 40, 60), nms_sigma_square=(0.0009, 0.009, 0.1, 1), suppressed_thresh=0.3):
    """DI-NMS, the reference's signature and 5-tuple: (boxes [K,7] float64, dir labels [K] int64, labels [K] int64, scores [K] float64,
    selected [K] int64 = input index of each cluster's pick), clusters in pick order.  box_preds [n,7], rbboxes [n,5] (x,y,w,l,r),
    scores [n] >= 0, iou_preds [n] (the rectified q), anchors [n,7] (CUDA tensors).
    As in the reference, post_max_size and iou_threshold are not used (DI-NMS may return up to pre_max_size clusters).  Differences:
    n == 0 returns empty tensors (the reference returns None); pre_max_size=None means all n (the reference raises NameError);
    equal scores keep the lower index first in the top-k.  centerness_c=True (the C core's own centerness) is not built."""
    if centerness_c:
        raise NotImplementedError("centerness_c (the C core's centerness) is not built; the reference head passes centerness_c=False")
    dev = box_preds.device
    n = int(scores.shape[0])
    if n == 0:
        return (torch.zeros([0, 7], dtype=torch.float64, device=dev), torch.zeros([0], dtype=torch.long, device=dev),
                torch.zeros([0], dtype=torch.long, device=dev), torch.zeros([0], dtype=torch.float64, device=dev),
                torch.zeros([0], dtype=torch.long, device=dev))
    if not box_preds.is_cuda:
        raise RuntimeError("rotate_weighted_nms expects CUDA tensors (there is no CPU fallback)")
    pre = n if pre_max_size is None else min(n, int(pre_max_size))
    if pre > ops.DINMS_MAX_PRE:
        raise ValueError("DI-NMS keeps at most %d boxes before the loop (pre_max_size)" % ops.DINMS_MAX_PRE)
    cfg = ops.make_dinms_cfg(nms_cnt_thresh, nms_sigma_dist_interval, nms_sigma_square, suppressed_thresh, centerness_pow, enable_centerness)
    f32 = lambda t: t.detach().to(torch.float32).contiguous()
    i32 = lambda t: t.detach().to(torch.int32).contiguous()
    cnt = torch.tensor([n], dtype=torch.int32, device=dev)
    out = ops.rotate_weighted_nms(f32(box_preds), f32(rbboxes), f32(scores), f32(iou_preds), i32(labels_preds), i32(dir_labels),
                                  f32(anchors) if enable_centerness else None, cnt, n, pre, cfg)
    k = int(out["count"][0].item())
    return (out["boxes"][:k].double(), out["dirs"][:k].long(), out["labels"][:k].long(), out["scores"][:k].double(),
            out["selected"][:k].long())
