"""Result-annotation constructors of the KITTI mirror (reference det3d/datasets/kitti/kitti_common.py:879-913)."""
from sessd_b200.kitti_eval import empty_anno


def get_start_result_anno():
    """Empty per-key lists that a frame's detections are appended to."""
    return {k: [] for k in ("name", "truncated", "occluded", "alpha", "bbox", "dimensions", "location", "rotation_y", "score")}


def empty_result_anno():
    """The annotation of a frame without detections: zero-length arrays, [0, 4] / [0, 3] for the box fields."""
    return empty_anno()
