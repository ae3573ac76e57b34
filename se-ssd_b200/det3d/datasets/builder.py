"""``build_dataset`` (reference: det3d/datasets/builder.py:33-46): the registry lookup of a ``data.<split>`` config entry."""
from det3d.utils import build_from_cfg

from .registry import DATASETS


def build_dataset(cfg, default_args=None):
    if isinstance(cfg, (list, tuple)) or cfg["type"] == "RepeatDataset":
        raise NotImplementedError("concatenated and repeated datasets are not supported (the SE-SSD configs use neither)")
    return build_from_cfg(cfg, DATASETS, default_args)
