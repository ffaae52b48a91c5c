"""Host side of the asynchronous compress (pco_b200_compress_async_plan / _result) without a GPU: the plan's refusals and their kinds, its
workspace and index sizes, and how a status written by the device becomes a kind, a message and sizes."""
import ctypes as C

import numpy as np
import pytest

U8, U16, U32, U64, I64, F16, F32, F64 = 10, 7, 1, 2, 4, 9, 5, 6  # number type bytes (cpcodec.h)


@pytest.fixture(scope="module")
def L():
    from pcodec_b200 import standalone

    return standalone._lib_async_compress()


def _cfg(order=1, level=8, mode=None, delta=None, page=1 << 18, paging=None, enable_8_bit=True):
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec

    return ChunkConfig(compression_level=level, mode_spec=mode or ModeSpec.classic(), delta_spec=delta or DeltaSpec.try_consecutive(order),
                       paging_spec=paging or PagingSpec.equal_pages_up_to(page), enable_8_bit=enable_8_bit)


def _plan(L, n=1 << 20, dtype=U64, cfg="default", uniform=0, dst_cap=1 << 24, index_cap=0):
    from pcodec_b200 import standalone

    p = standalone._CAsyncCompressPlan()
    c = _cfg() if cfg == "default" else cfg
    cc = c._to_c() if c is not None else None
    rc = L.pco_b200_compress_async_plan(C.c_size_t(n), C.c_ubyte(dtype), C.byref(cc) if cc is not None else None, C.c_int(uniform),
                                        C.c_size_t(dst_cap), C.c_size_t(index_cap), C.byref(p))
    return rc, p, L.pco_b200_last_error_message().decode()


@pytest.fixture(scope="module")
def ok(L):
    """What an accepted plan returns here: OK with a device, Cuda (after the plan is filled) without one."""
    return 0 if L.pco_b200_device_available() else 6


def test_refusals_and_their_kinds(L):
    from pcodec_b200 import DeltaSpec, ModeSpec, PagingSpec

    cases = [
        (dict(dtype=99), 5, "type"),
        (dict(cfg=None), 7, "Auto"),  # the default config: Auto mode and delta
        (dict(cfg=_cfg(mode=ModeSpec.auto())), 7, "Auto"),
        (dict(cfg=_cfg(delta=DeltaSpec.auto())), 7, "Auto"),
        (dict(cfg=_cfg(level=9)), 7, "256 unoptimized bins"),
        (dict(cfg=_cfg(level=12)), 7, "256 unoptimized bins"),
        (dict(n=100, cfg=_cfg(paging=PagingSpec.exact_page_sizes([50, 50]))), 7, "Exact"),
        # chunks of 4096 and 4095 numbers: unoptimized_bins_log 8 and 7 at level 8
        (dict(n=8191, cfg=_cfg(page=4096)), 7, "several runs"),
        # what compress_ex refuses, with its kinds
        (dict(cfg=_cfg(level=13)), 3, "compression level"),
        (dict(cfg=_cfg(order=8)), 3, "delta order"),
        (dict(dtype=U8, cfg=_cfg(enable_8_bit=False)), 3, "8-bit"),
        (dict(dtype=F64, cfg=_cfg(mode=ModeSpec.try_int_mult(7))), 3, "int mult"),
        (dict(dtype=U64, cfg=_cfg(mode=ModeSpec.try_float_quant(3))), 3, "float mode"),
        (dict(dtype=F16, cfg=_cfg(mode=ModeSpec.try_float_mult(0.5))), 7, "f16 FloatMult"),
        (dict(cfg=_cfg(mode=ModeSpec.try_dict())), 7, "TryDict"),
        (dict(cfg=_cfg(delta=DeltaSpec.try_lookback())), 7, "Lookback"),
        (dict(cfg=_cfg(delta=DeltaSpec.try_conv1(1))), 7, "Conv1"),
        (dict(n=(1 << 24) + 1, cfg=_cfg(page=1 << 25)), 3, "16777216"),
    ]
    for kw, kind, words in cases:
        rc, _, msg = _plan(L, **kw)
        assert rc == kind and words in msg, (kw, rc, msg)


def test_accepted_plans(L, ok):
    from pcodec_b200 import ModeSpec

    for kw in [dict(), dict(n=0), dict(n=1), dict(n=8192, cfg=_cfg(page=4096)), dict(cfg=_cfg(level=9, page=1000), n=5000),
               dict(dtype=F32, cfg=_cfg(mode=ModeSpec.try_float_mult(0.1))), dict(dtype=F16, cfg=_cfg(mode=ModeSpec.try_float_quant(3))),
               dict(dtype=I64, cfg=_cfg(mode=ModeSpec.try_int_mult(10), order=7)), dict(uniform=1)]:
        rc, p, msg = _plan(L, **kw)
        assert rc == ok, (kw, msg)


def test_plan_fields(L, ok):
    from pcodec_b200 import ModeSpec

    rc, p, _ = _plan(L, n=1000, dtype=F32, cfg=_cfg(order=2, level=5, mode=ModeSpec.try_float_quant(4), page=300), uniform=1, dst_cap=777)
    assert rc == ok
    assert (p.dtype, p.uniform_type_header, p.mode, p.order, p.n_vars, p.mode_k) == (F32, 1, 3, 2, 2, 4)
    assert (p.n, p.max_page_n, p.dst_cap, p.index_cap) == (1000, 300, 777, 0)
    # 4 chunks of 250 numbers: header, 4 records, then per chunk 2 vars x 1 batch x 12 bytes rounded up to 16
    assert p.index_bytes == 64 + 4 * 32 + 4 * 32


def _index_bytes(n, page, n_vars):
    if n == 0:
        return 64
    k = -(-n // page)
    low, rem = divmod(n, k)
    ent = lambda m: (n_vars * -(-m // 256) * 12 + 15) // 16 * 16  # noqa: E731
    return (64 + 32 * k + 15) // 16 * 16 + rem * ent(low + 1) + (k - rem) * ent(low)


@pytest.mark.parametrize("n,page", [(0, 1 << 18), (1, 1 << 18), (255, 256), (257, 256), (1 << 20, 1 << 18), ((1 << 20) + 1, 1 << 18), (10**6, 1000)])
def test_index_size_and_index_cap_one_byte_short(L, ok, n, page):
    from pcodec_b200 import ModeSpec

    for cfg, n_vars in [(_cfg(page=page), 1), (_cfg(page=page, mode=ModeSpec.try_int_mult(3)), 2)]:
        need = _index_bytes(n, page, n_vars)
        rc, p, msg = _plan(L, n=n, cfg=cfg, index_cap=need)
        assert rc == ok and p.index_bytes == need, msg
        rc, p, msg = _plan(L, n=n, cfg=cfg, index_cap=need - 1)
        assert rc == 4 and str(need) in msg, msg  # Io


def test_workspace_grows_with_n_and_the_var_count(L):
    from pcodec_b200 import ModeSpec

    sizes = [_plan(L, n=n)[1].workspace_bytes for n in (1, 1 << 16, 1 << 20, 1 << 24)]
    assert sizes == sorted(sizes) and len(set(sizes)) == 4
    # Classic u64: 3 x 8 + 5 bytes per number, plus a per-chunk share
    per_n = (sizes[3] - sizes[2]) / ((1 << 24) - (1 << 20))
    assert 29 <= per_n <= 29.5, per_n
    two = _plan(L, n=1 << 20, cfg=_cfg(mode=ModeSpec.try_int_mult(3)))[1].workspace_bytes
    assert two > sizes[2]
    assert _plan(L, n=1 << 20, dtype=U16)[1].workspace_bytes < _plan(L, n=1 << 20, dtype=U32)[1].workspace_bytes < sizes[2]
    assert _plan(L, n=0)[1].workspace_bytes < sizes[0]


def _result(L, **fields):
    from pcodec_b200 import standalone

    s = standalone._CAsyncCompressStatus(**fields)
    nw, il = C.c_size_t(111), C.c_size_t(222)
    rc = L.pco_b200_compress_async_result(C.byref(s), C.byref(nw), C.byref(il))
    return rc, L.pco_b200_last_error_message().decode(), (nw.value, il.value)


def test_result_maps_statuses_to_kinds_messages_and_sizes(L):
    rc, _, sizes = _result(L, kind=0, file_bytes=1000, n_written=1000, index_bytes=96)
    assert (rc, sizes) == (0, (1000, 96))
    rc, msg, sizes = _result(L, kind=4, device_status=0x106, file_bytes=12345, n_written=0)
    assert rc == 4 and "12345" in msg and "whole buffer" in msg, msg
    assert sizes == (111, 222)  # left alone on an error
    rc, _, _ = _result(L, kind=99, device_status=5)
    assert rc == 1  # a kind the library does not know reads as Corruption
    assert L.pco_b200_compress_async_result(None, None, None) == 3
    from pcodec_b200 import standalone

    s = standalone._CAsyncCompressStatus(kind=0, n_written=5, index_bytes=0)
    assert L.pco_b200_compress_async_result(C.byref(s), None, None) == 0


def test_call_refuses_bad_arguments_before_the_device(L):
    from pcodec_b200 import standalone

    _, p, _ = _plan(L, n=1000, cfg=_cfg(page=300))
    s = standalone._CAsyncCompressStatus()
    nz = C.c_void_p(256)  # never dereferenced: the call refuses first
    call = L.pco_b200_compress_async
    assert call(None, nz, nz, None, nz, C.byref(s), None) == 3
    assert call(C.byref(p), None, nz, None, nz, C.byref(s), None) == 3  # no numbers
    assert call(C.byref(p), nz, None, None, nz, C.byref(s), None) == 3  # no dst
    assert call(C.byref(p), nz, nz, None, None, C.byref(s), None) == 3  # no workspace
    assert call(C.byref(p), nz, nz, None, nz, None, None) == 3  # no status
    assert call(C.byref(p), nz, nz, nz, nz, C.byref(s), None) == 3  # an index with a plan made without one
    assert call(C.byref(p), nz, nz, None, C.c_void_p(257), C.byref(s), None) == 3  # unaligned workspace
    for field, delta in [("workspace_bytes", 1), ("index_bytes", 16), ("n_vars", 1), ("mode", 9), ("bins_log", 9), ("dtype", 90)]:
        bad = standalone._CAsyncCompressPlan.from_buffer_copy(bytes(p))
        setattr(bad, field, getattr(bad, field) + delta)
        assert call(C.byref(bad), nz, nz, None, nz, C.byref(s), None) == 3, field
    _, pi, _ = _plan(L, n=1000, cfg=_cfg(page=300), index_cap=1 << 12)
    assert call(C.byref(pi), nz, nz, C.c_void_p(264), nz, C.byref(s), None) == 3  # index not 16-byte aligned


def test_no_device_is_cuda_after_the_checks(L):
    if L.pco_b200_device_available():
        pytest.skip("a device is present")
    rc, p, msg = _plan(L, n=4096)
    assert rc == 6 and "CUDA" in msg, msg
    assert p.workspace_bytes > 0 and p.n == 4096  # filled before the device is touched


def test_the_library_exports_the_async_compress_symbols():
    import subprocess

    from pcodec_b200 import _lib

    path = _lib.lib()._name
    out = subprocess.run(["nm", "-D", "--defined-only", path], capture_output=True, text=True, check=True).stdout
    names = {line.split()[-1] for line in out.splitlines() if line.strip()}
    for sym in ("pco_b200_compress_async_plan", "pco_b200_compress_async", "pco_b200_compress_async_result"):
        assert sym in names, sym
