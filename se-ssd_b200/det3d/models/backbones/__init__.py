"""Sparse 3-D middle encoders on the hot path: SpMiddleFHD (rulebooks + sparse convs + dense() on the sessd_b200 CUDA kernels)."""
from .scn import SpMiddleFHD

__all__ = ["SpMiddleFHD"]
