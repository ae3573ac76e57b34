"""det3d/datasets/utils/sa_da_v2.py: shape-aware data augmentation (SA-DA) with the reference's signature, run on the device.

``pyramid_augment_v0`` takes and returns numpy and draws from ``np.random`` with the reference's calls in the reference's order; the
dropout, the farthest-point sparsify and the swap run as the kernels of csrc/sada.cu (sessd_b200.sada).  It waits on the device to read
the swap counts back (when a box is swap-selected) and to return the points.  The sparsify step is exact farthest-point sampling, the
contract DESIGN §7 pins for the reference's external ``ifp_sample``.
"""
import numpy as np
import torch

from sessd_b200.sada import SadaConfig, sada_frame


def pyramid_augment_v0(gt_boxes, points, enable_sa_dropout=0.1, enable_sa_sparsity=[0.05, 50], enable_sa_swap=[0.05, 50]):
    """gt_boxes [K, 7] float32, points [N, 4] float32 (numpy) -> the augmented [N', 4] float32 points"""
    gt_boxes, points = np.asarray(gt_boxes), np.asarray(points)
    if points.ndim != 2 or points.shape[1] != 4:
        raise ValueError("pyramid_augment_v0 takes [N, 4] points")
    if gt_boxes.dtype != np.float32 or points.dtype != np.float32:
        raise ValueError("pyramid_augment_v0 runs in float32: gt_boxes and points must be float32 arrays")
    gt_boxes = gt_boxes.reshape(-1, 7)
    cfg = SadaConfig(dropout=enable_sa_dropout, sparsity=None if enable_sa_sparsity is None else tuple(enable_sa_sparsity),
                     swap=None if enable_sa_swap is None else tuple(enable_sa_swap))
    d_pts = torch.from_numpy(np.ascontiguousarray(points)).cuda()
    d_boxes = torch.from_numpy(np.ascontiguousarray(gt_boxes)).cuda()
    out, num = sada_frame(d_pts if len(points) else torch.empty((0, 4), dtype=torch.float32, device="cuda"), d_boxes, len(gt_boxes),
                          np.random.mtrand._rand, cfg)
    n = int(num.item())
    return out[:n].cpu().numpy()
