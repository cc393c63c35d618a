"""opengemini_b200 — H100-native scan/aggregate path behind openGemini's cursor seam (the package keeps its original name).

Product = libogpu.so (hand-written sm_90a CUDA behind the C ABI in include/ogpu.h).
This package only holds the host-side bindings; aggregation and decoding never run on the CPU
(the bindings only slice the records the library returns).
"""
from . import _lib  # noqa: F401
from .cursor import AggQuery, Comm, ScanCursor, Shard, write_tssp  # noqa: F401

__all__ = ["Shard", "AggQuery", "ScanCursor", "Comm", "write_tssp", "_lib"]
