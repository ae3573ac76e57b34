"""``spconv.utils`` names that det3d/core/bbox/box_np_ops.py:9 imports at module import time (rbbox_iou / rbbox_intersection:
boost-based CPU helpers of spconv 1.x).  They are not on the SE-SSD hot path; use ``det3d.core.iou3d.iou3d_utils`` instead."""


def rbbox_iou(*args, **kwargs):
    raise NotImplementedError("spconv.utils.rbbox_iou is not part of the CUDA hot path; use det3d.core.iou3d.iou3d_utils.boxes_iou_bev_gpu")


def rbbox_intersection(*args, **kwargs):
    raise NotImplementedError("spconv.utils.rbbox_intersection is not part of the CUDA hot path")
