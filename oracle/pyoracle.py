"""ORACLE — TEST INFRASTRUCTURE ONLY.

ctypes binding for oracle/liboracle.so (the CPU restatement of pco 1.0.3).
Imported only by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
``--impl reference`` legs; the product package (pcodec_b200/) never imports it.
"""
import ctypes as C
import json
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle.so")

# dtype bytes: pco_c/include/cpcodec.h:10-20
DTYPE_BYTES = {
    "u32": 1, "u64": 2, "i32": 3, "i64": 4, "f32": 5, "f64": 6,
    "u16": 7, "i16": 8, "f16": 9, "u8": 10, "i8": 11,
}
NP_DTYPES = {
    1: np.uint32, 2: np.uint64, 3: np.int32, 4: np.int64, 5: np.float32, 6: np.float64,
    7: np.uint16, 8: np.int16, 9: np.float16, 10: np.uint8, 11: np.int8,
}
NP_TO_BYTE = {np.dtype(v): k for k, v in NP_DTYPES.items()}

MODE_AUTO, MODE_CLASSIC, MODE_FLOAT_MULT, MODE_FLOAT_QUANT, MODE_INT_MULT, MODE_DICT = range(6)
DELTA_AUTO, DELTA_NOOP, DELTA_CONSECUTIVE, DELTA_LOOKBACK, DELTA_CONV1 = range(5)
PAGING_EQUAL_UP_TO, PAGING_EXACT = range(2)

ERROR_KINDS = {0: None, 1: "Corruption", 2: "InsufficientData", 3: "InvalidArgument", 4: "Io"}


class OracleError(Exception):
    def __init__(self, kind, msg):
        super().__init__(f"pco {kind} error: {msg}")
        self.kind = kind
        self.message = msg


class Config(C.Structure):
    """Same layout as PcoB200ChunkConfig (include/pco_b200.h)."""

    _fields_ = [
        ("compression_level", C.c_uint32),
        ("mode_spec", C.c_uint32),
        ("float_mult_base", C.c_double),
        ("int_mult_base", C.c_uint64),
        ("float_quant_k", C.c_uint32),
        ("delta_spec", C.c_uint32),
        ("delta_order", C.c_uint32),
        ("paging_spec", C.c_uint32),
        ("max_page_n", C.c_uint64),
        ("exact_page_ns", C.POINTER(C.c_uint64)),
        ("n_exact_pages", C.c_uint64),
        ("enable_8_bit", C.c_uint32),
        ("reserved", C.c_uint32),
    ]


def make_config(level=8, mode=MODE_CLASSIC, delta=DELTA_NOOP, delta_order=0, float_mult_base=0.0, int_mult_base=0,
                float_quant_k=0, max_page_n=0, exact_pages=None, enable_8_bit=True):
    cfg = Config()
    cfg.compression_level = level
    cfg.mode_spec = mode
    cfg.float_mult_base = float_mult_base
    cfg.int_mult_base = int_mult_base
    cfg.float_quant_k = float_quant_k
    cfg.delta_spec = delta
    cfg.delta_order = delta_order
    cfg.max_page_n = max_page_n
    cfg.enable_8_bit = 1 if enable_8_bit else 0
    if exact_pages is not None:
        arr = (C.c_uint64 * len(exact_pages))(*exact_pages)
        cfg._keepalive = arr
        cfg.exact_page_ns = C.cast(arr, C.POINTER(C.c_uint64))
        cfg.n_exact_pages = len(exact_pages)
        cfg.paging_spec = PAGING_EXACT
    else:
        cfg.paging_spec = PAGING_EQUAL_UP_TO
    return cfg


def build(force=False):
    """Compile oracle/liboracle.so with the committed Makefile."""
    if force or not os.path.exists(_LIB_PATH) or any(
        os.path.getmtime(os.path.join(_HERE, f)) > os.path.getmtime(_LIB_PATH)
        for f in os.listdir(_HERE) if f.endswith((".hpp", ".cpp", "Makefile"))
    ):
        subprocess.run(["make", "-C", _HERE, "-s"], check=True)
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.pco_oracle_last_error.restype = C.c_char_p
        _lib.pco_oracle_file_size_guarantee.restype = C.c_size_t
        _lib.pco_oracle_file_size_guarantee.argtypes = [C.c_size_t, C.c_uint8]
        _lib.pco_oracle_free.argtypes = [C.c_void_p]
        _lib.pco_oracle_kat_log2_approx.restype = C.c_float
        _lib.pco_oracle_kat_log2_approx.argtypes = [C.c_float]
        _lib.pco_oracle_chunk_compressor_n_pages.restype = C.c_size_t
        _lib.pco_oracle_chunk_compressor_page_n.restype = C.c_size_t
        _lib.pco_oracle_chunk_compressor_n_pages.argtypes = [C.c_void_p]
        _lib.pco_oracle_chunk_compressor_page_n.argtypes = [C.c_void_p, C.c_size_t]
        _lib.pco_oracle_chunk_compressor_free.argtypes = [C.c_void_p]
    return _lib


def _check(rc):
    if rc != 0:
        raise OracleError(ERROR_KINDS.get(rc, f"code {rc}"), lib().pco_oracle_last_error().decode())


def _take_bytes(ptr, n):
    data = C.string_at(ptr, n.value)
    lib().pco_oracle_free(ptr)
    return data


def _as_array(nums):
    arr = np.ascontiguousarray(nums)
    if arr.dtype not in NP_TO_BYTE:
        raise TypeError(f"unsupported dtype {arr.dtype}")
    return arr, NP_TO_BYTE[arr.dtype]


def simple_compress(nums, config=None, uniform_type=False):
    """pco::standalone::simple_compress (uniform_type=False) / simple_compress_into (True)."""
    arr, dt = _as_array(nums)
    out = C.c_void_p()
    n = C.c_size_t()
    rc = lib().pco_oracle_simple_compress(
        arr.ctypes.data_as(C.c_void_p), C.c_size_t(arr.size), C.c_uint8(dt),
        C.byref(config) if config is not None else None, C.c_int(1 if uniform_type else 0), C.byref(out), C.byref(n))
    _check(rc)
    return _take_bytes(out, n)


def simple_decompress(data, dtype):
    dt = NP_TO_BYTE[np.dtype(dtype)]
    out = C.c_void_p()
    n = C.c_size_t()
    buf = (C.c_uint8 * max(len(data), 1)).from_buffer_copy(data if len(data) else b"\0")
    rc = lib().pco_oracle_simple_decompress(buf, C.c_size_t(len(data)), C.c_uint8(dt), C.byref(out), C.byref(n))
    _check(rc)
    res = np.frombuffer(C.string_at(out, n.value * np.dtype(dtype).itemsize), dtype=dtype).copy()
    lib().pco_oracle_free(out)
    return res


def simple_decompress_into(data, dst):
    """Returns (n_processed, finished) — pco::standalone::simple_decompress_into."""
    dt = NP_TO_BYTE[dst.dtype]
    n = C.c_size_t()
    fin = C.c_int()
    buf = (C.c_uint8 * max(len(data), 1)).from_buffer_copy(data if len(data) else b"\0")
    rc = lib().pco_oracle_simple_decompress_into(buf, C.c_size_t(len(data)), C.c_uint8(dt), dst.ctypes.data_as(C.c_void_p),
                                                 C.c_size_t(dst.size), C.byref(n), C.byref(fin))
    _check(rc)
    return n.value, bool(fin.value)


def file_size_guarantee(n, dtype):
    return lib().pco_oracle_file_size_guarantee(n, NP_TO_BYTE[np.dtype(dtype)])


def last_fallback_margins():
    """[(worst_case_size, baseline)] in bytes for each chunk of this thread's last simple_compress or ChunkCompressor, in chunk
    order (chunk_compressor.rs:502-541): the chunk fell back to Classic / NoOp where worst_case_size > baseline."""
    f = lib().pco_oracle_last_fallback_margins
    f.restype = C.c_size_t
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    n = f(None, None, 0)
    worst, base = np.zeros(n, dtype=np.uint64), np.zeros(n, dtype=np.uint64)
    f(worst.ctypes.data_as(C.c_void_p), base.ctypes.data_as(C.c_void_p), n)
    return [(int(w), int(b)) for w, b in zip(worst, base)]


def inspect(data, dtype):
    dt = NP_TO_BYTE[np.dtype(dtype)]
    out = C.c_void_p()
    buf = (C.c_uint8 * max(len(data), 1)).from_buffer_copy(data if len(data) else b"\0")
    rc = lib().pco_oracle_inspect(buf, C.c_size_t(len(data)), C.c_uint8(dt), C.byref(out))
    _check(rc)
    s = C.string_at(out).decode()
    lib().pco_oracle_free(out)
    return json.loads(s)


class ChunkCompressor:
    """pco::wrapped::ChunkCompressor (pco/src/wrapped/chunk_compressor.rs:543-705)."""

    def __init__(self, nums, config):
        arr, dt = _as_array(nums)
        self._h = C.c_void_p()
        rc = lib().pco_oracle_chunk_compressor_new(arr.ctypes.data_as(C.c_void_p), C.c_size_t(arr.size), C.c_uint8(dt),
                                                   C.byref(config) if config is not None else None, C.byref(self._h))
        _check(rc)

    def __del__(self):
        if getattr(self, "_h", None):
            lib().pco_oracle_chunk_compressor_free(self._h)
            self._h = None

    def n_per_page(self):
        n = lib().pco_oracle_chunk_compressor_n_pages(self._h)
        return [lib().pco_oracle_chunk_compressor_page_n(self._h, i) for i in range(n)]

    def write_meta(self):
        out, n = C.c_void_p(), C.c_size_t()
        _check(lib().pco_oracle_chunk_compressor_write_meta(self._h, C.byref(out), C.byref(n)))
        return _take_bytes(out, n)

    def write_page(self, i):
        out, n = C.c_void_p(), C.c_size_t()
        _check(lib().pco_oracle_chunk_compressor_write_page(self._h, C.c_size_t(i), C.byref(out), C.byref(n)))
        return _take_bytes(out, n)


def wrapped_decompress_page(meta, page, dtype, page_n):
    """Decode one wrapped page; returns (nums, meta_bytes_consumed, page_bytes_consumed)."""
    dt = NP_TO_BYTE[np.dtype(dtype)]
    dst = np.empty(page_n, dtype=dtype)
    mc, pc = C.c_size_t(), C.c_size_t()
    mb = (C.c_uint8 * max(len(meta), 1)).from_buffer_copy(meta if len(meta) else b"\0")
    pb = (C.c_uint8 * max(len(page), 1)).from_buffer_copy(page if len(page) else b"\0")
    rc = lib().pco_oracle_wrapped_decompress_page(mb, C.c_size_t(len(meta)), pb, C.c_size_t(len(page)), C.c_uint8(dt),
                                                  C.c_size_t(page_n), dst.ctypes.data_as(C.c_void_p), C.byref(mc), C.byref(pc))
    _check(rc)
    return dst, mc.value, pc.value


class _ExplicitVar(C.Structure):  # pco_oracle_explicit_var (c_api.cpp)
    _fields_ = [("ans_size_log", C.c_uint32), ("n_bins", C.c_uint32), ("weights", C.c_void_p), ("lowers", C.c_void_p), ("offset_bits", C.c_void_p),
                ("n_stored", C.c_uint64), ("symbols", C.c_void_p), ("offsets", C.c_void_p), ("moments", C.c_void_p)]


class _ExplicitChunk(C.Structure):  # pco_oracle_explicit_chunk (c_api.cpp)
    _fields_ = [("n", C.c_uint64), ("mode", C.c_uint32), ("float_quant_k", C.c_uint32), ("mode_base_latent", C.c_uint64), ("delta_order", C.c_uint32),
                ("secondary_uses_delta", C.c_uint32), ("vars", _ExplicitVar * 2)]


EXPLICIT_MODES = {"classic": 0, "int_mult": 1, "float_mult": 2, "float_quant": 3}


def write_explicit_file(dtype, chunks):
    """A standalone file of chunks with explicit bins and stored latents (pco_oracle_write_explicit_file).  Each chunk is a dict:
    n; mode ("classic", "int_mult", "float_mult", "float_quant") with `base` (IntMult base, or FloatMult base as latent-ordered bits)
    or `k`; `order` (consecutive delta, 0 = none) and `secondary_uses_delta`; `vars`: one dict per latent var (primary, then secondary)
    with ans_size_log, bins [(weight, lower, offset_bits), ...], symbols and offsets (the stored latents), and moments (the delta
    state) when the var uses the delta.  Returns (file, [(meta, page) per chunk])."""
    dt = NP_TO_BYTE[np.dtype(dtype)]
    arr = (_ExplicitChunk * max(len(chunks), 1))()
    keep = []

    def buf(values, ctype):
        a = np.ascontiguousarray(np.asarray(values, dtype=np.uint64).astype(ctype).reshape(-1))
        keep.append(a)
        return a.ctypes.data_as(C.c_void_p) if a.size else None

    for c, spec in zip(arr, chunks):
        c.n = spec["n"]
        c.mode = EXPLICIT_MODES[spec.get("mode", "classic")]
        c.mode_base_latent = spec.get("base", 0)
        c.float_quant_k = spec.get("k", 0)
        c.delta_order = spec.get("order", 0)
        c.secondary_uses_delta = 1 if spec.get("secondary_uses_delta") else 0
        for v, var in zip(c.vars, spec["vars"]):
            bins = np.asarray(var["bins"], dtype=np.uint64).reshape(-1, 3)
            v.ans_size_log = var["ans_size_log"]
            v.n_bins = bins.shape[0]
            v.weights, v.lowers, v.offset_bits = buf(bins[:, 0], np.uint32), buf(bins[:, 1], np.uint64), buf(bins[:, 2], np.uint32)
            v.n_stored = len(var["symbols"])
            v.symbols, v.offsets = buf(var["symbols"], np.uint32), buf(var["offsets"], np.uint64)
            v.moments = buf(var.get("moments", []), np.uint64)
    out, n = C.c_void_p(), C.c_size_t()
    metas, pages = C.c_void_p(), C.c_void_p()
    mlens, plens = (C.c_size_t * max(len(chunks), 1))(), (C.c_size_t * max(len(chunks), 1))()
    f = lib().pco_oracle_write_explicit_file
    f.argtypes = [C.c_uint8, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    _check(f(dt, C.cast(arr, C.c_void_p), len(chunks), C.byref(out), C.byref(n), C.byref(metas), mlens, C.byref(pages), plens))
    data = _take_bytes(out, n)
    mall = _take_bytes(metas, C.c_size_t(sum(mlens[:len(chunks)])))
    pall = _take_bytes(pages, C.c_size_t(sum(plens[:len(chunks)])))
    parts, mo, po = [], 0, 0
    for i in range(len(chunks)):
        parts.append((mall[mo:mo + mlens[i]], pall[po:po + plens[i]]))
        mo, po = mo + mlens[i], po + plens[i]
    return data, parts


def bench_roundtrip(nums, n_chunks, chunk_n, config, threads):
    """Compress + decompress `n_chunks` chunks of `chunk_n` numbers (contiguous in `nums`) on `threads` native threads, one chunk
    per task, verifying the round trip.  Returns (compress seconds, decompress seconds, compressed bytes).  bench.py's CPU arm."""
    arr = np.ascontiguousarray(nums)
    assert arr.size == n_chunks * chunk_n
    cs, ds, cb = C.c_double(), C.c_double(), C.c_uint64()
    f = lib().pco_oracle_bench_roundtrip
    f.restype = C.c_int
    rc = f(arr.ctypes.data_as(C.c_void_p), C.c_size_t(n_chunks), C.c_size_t(chunk_n), C.c_uint8(NP_TO_BYTE[arr.dtype]), C.byref(config), C.c_int(threads),
           C.byref(cs), C.byref(ds), C.byref(cb))
    _check(rc)
    return cs.value, ds.value, cb.value
