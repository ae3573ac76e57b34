"""det3d -- the Det3D / SE-SSD registry + operator API surface for the per-frame LiDAR hot path, backed by the
GPU-native (sm_90a) kernels of ``sessd_b200`` (libsessd_b200.so).

This package mirrors the names, signatures and error behaviour of the reference interfaces that
``examples/second/configs/config.py`` and ``tools/test.py`` bind (SURVEY.md 8b), so that the config loads unchanged and
``VoxelNet.forward(example, return_loss=False)`` is a drop-in.  It *owns* its registries (the reference's
``Registry._register_module`` raises on duplicates, det3d/utils/registry.py:36-39).  Everything outside the hot path
(dataset I/O, augmentation, trainer, evaluation, unused ops) is intentionally absent.
"""
__version__ = "sessd_b200-0.1"
