from . import pipelines  # noqa: F401
from .registry import DATASETS, PIPELINES
from .kitti import KittiDataset  # noqa: F401  (registers itself in DATASETS)
from .builder import build_dataset
from .loader import build_dataloader

__all__ = ["DATASETS", "PIPELINES", "KittiDataset", "build_dataset", "build_dataloader"]
