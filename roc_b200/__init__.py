"""roc_b200 — H100-native (sm_90a) engine for ROC's GCN-training hot path.

The compute lives in roc_b200/lib/libroc_b200.so (CUDA kernels + C ABI + C++ host);
this package is the ctypes mirror of the reference's Model/op-builder API plus
dataset helpers.  Importing it without the built library raises ImportError;
using it without a CUDA device raises RocError — there is no CPU fallback.
"""
from . import _lib
from ._lib import RocError, device_count

__all__ = ["_lib", "RocError", "device_count"]
