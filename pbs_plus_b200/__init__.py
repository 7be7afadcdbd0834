"""pbs_plus_b200 -- H100-native chunk + digest + probe engine behind pbs-plus's chunker surface.

Only the ONE hot path of SURVEY.md section 8: buzhash boundary scan, per-chunk SHA-256,
known-digest probe.  The product is libpbsgpu.so (csrc/, C ABI in include/pbsgpu.h);
this package is the Python host mirror used by tests and bench.py.
"""
from ._lib import CHUNK_DTYPE, CHUNK_KNOWN, LIB_PATH, PbsGpuError  # noqa: F401
from .engine import DigestSet, Engine, Job, NcclComm, Stream, corpus, default_table, make_config  # noqa: F401
from . import buzhash, transfer  # noqa: F401

__all__ = ["Engine", "DigestSet", "Job", "Stream", "NcclComm", "make_config", "default_table", "corpus", "buzhash", "transfer",
           "CHUNK_DTYPE", "CHUNK_KNOWN", "PbsGpuError", "LIB_PATH"]
