from . import pipelines  # noqa: F401
from .registry import DATASETS, PIPELINES
from .kitti import KittiDataset  # noqa: F401  (registers itself in DATASETS)

__all__ = ["DATASETS", "PIPELINES", "KittiDataset"]
