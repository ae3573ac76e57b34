"""Dataset-side registries: ``DATASETS`` (build_dataset) and ``PIPELINES`` (the per-frame transforms)."""
from det3d.utils import Registry

DATASETS, PIPELINES = (Registry(kind) for kind in ("dataset", "pipeline"))
__all__ = ["DATASETS", "PIPELINES"]
