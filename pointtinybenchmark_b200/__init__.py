"""pointtinybenchmark_b200 — H100 (sm_90a) native CPR / P2P point-localization head path.

Python host layer that mirrors the reference's mmdet dense-head interface (CPRHead / P2PHead, HEADS registry,
same ctor kwargs and state_dict keys) over the C-ABI CUDA library libptb_b200.so (include/ptb_b200.h).
"""
from . import _lib, ops  # noqa: F401

__all__ = ['_lib', 'ops']
