"""pcodec_b200 — B200-native implementation of Pcodec's per-chunk encode/decode hot path.

Host-side mirror of the reference's Python surface (`pcodec.standalone`, pco_python/src/standalone.rs:44-135)
over libcpcodec.so, the C-ABI library that holds the sm_90a kernels.  This package contains no CPU
implementation of the codec: if the shared library (or a CUDA device) is missing, calls raise.
"""
from . import _lib, standalone, wrapped  # noqa: F401  (inspect and benchfmt load on demand: `from pcodec_b200 import inspect`)
from ._lib import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec, PcoError, Progress  # noqa: F401

__all__ = ["standalone", "wrapped", "inspect", "benchfmt", "ChunkConfig", "DeltaSpec", "ModeSpec", "PagingSpec", "PcoError", "Progress"]
