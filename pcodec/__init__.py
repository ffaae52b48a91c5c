"""`pcodec` — the import name of the reference's Python package (pco_python/src/lib.rs:17-54), served by the GPU library.

`import pcodec` / `from pcodec import standalone, wrapped, ChunkConfig, ...` resolves to pcodec_b200 (ctypes over libcpcodec.so: the
sm_90a kernels behind the C-ABI), so code and tests written against the reference's module run against the GPU path without edits.
Nothing here computes: there is no CPU codec in this repository's product tree."""
from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec, PcoError, Progress, standalone, wrapped  # noqa: F401

__all__ = ["standalone", "wrapped", "ChunkConfig", "DeltaSpec", "ModeSpec", "PagingSpec", "PcoError", "Progress"]
