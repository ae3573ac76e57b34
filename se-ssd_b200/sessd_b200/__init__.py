"""sessd_b200 -- GPU-native (H100, sm_90a) implementation of the SE-SSD per-frame LiDAR hot path.

Importing the package loads libsessd_b200.so through ctypes; there is no CPU or eager-PyTorch fallback: if the CUDA
library has not been built the import fails."""
from . import _lib  # noqa: F401  (fails loudly when the library is missing)

__version__ = "0.1"
