"""xapiand_b200 — H100-native (sm_90a) inverted-index matcher behind the Xapian Enquire/MSet surface.

Only what the hot path needs lives here: csrc/ (CUDA kernels + the C-ABI of include/xgm.h, built
in-tree into libxgm.so) and xgm.py (ctypes bindings + Enquire/MSet-shaped host layer).
"""
from . import xgm  # noqa: F401

__all__ = ["xgm"]
