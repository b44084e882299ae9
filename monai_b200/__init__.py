"""monai_b200 -- H100-native (sm_90a) sliding-window inference and spatial-transform hot path behind MONAI's API.

Python host code keeps the reference's call signatures; all arithmetic on the path runs in hand-written CUDA kernels
reached through the C ABI declared in include/monai_b200.h (ctypes, raw device pointers).
"""
__version__ = "0.1.0"

from . import _lib  # noqa: F401

__all__ = ["__version__"]
