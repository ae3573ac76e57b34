"""``build_dataloader`` (reference: det3d/datasets/loader/build_loader.py): batches whose tensors are built on the device
(sessd_b200.kitti_loader)."""
from sessd_b200.kitti_loader import build_dataloader

__all__ = ["build_dataloader"]
