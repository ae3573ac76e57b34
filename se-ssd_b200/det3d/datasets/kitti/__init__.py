from .eval import get_coco_eval_result, get_official_eval_result, get_official_eval_result_v2
from .kitti import KittiDataset

__all__ = ["KittiDataset", "get_official_eval_result", "get_official_eval_result_v2", "get_coco_eval_result"]
