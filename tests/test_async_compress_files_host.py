"""Host side of the asynchronous batch compress (pco_b200_compress_files_async_plan / _async / _result) without a GPU: the plan's refusals
and their kinds, its chunk bound, dst and index bounds and workspace formula, how a status written by the device becomes a kind and a
message, and the call's argument checks."""
import ctypes as C

import numpy as np
import pytest

U8, U16, U32, U64, I64, F16, F32, F64 = 10, 7, 1, 2, 4, 9, 5, 6  # number type bytes (cpcodec.h)
BITS = {U8: 8, U16: 16, U32: 32, U64: 64, I64: 64, F16: 16, F32: 32, F64: 64}


@pytest.fixture(scope="module")
def L():
    from pcodec_b200 import standalone

    return standalone._lib_async_compress_files()


@pytest.fixture(scope="module")
def ok(L):
    """What an accepted plan returns here: OK with a device, Cuda (after the plan is filled) without one."""
    return 0 if L.pco_b200_device_available() else 6


def _cfg(order=1, level=8, mode=None, delta=None, page=1 << 18, paging=None, enable_8_bit=True):
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec

    return ChunkConfig(compression_level=level, mode_spec=mode or ModeSpec.classic(), delta_spec=delta or DeltaSpec.try_consecutive(order),
                       paging_spec=paging or PagingSpec.equal_pages_up_to(page), enable_8_bit=enable_8_bit)


def _plan(L, dtype=U64, cfg="default", uniform=0, max_files=64, nums_cap=1 << 20, max_file_n=1 << 16, dst_cap=1 << 24, index_cap=0):
    from pcodec_b200 import standalone

    p = standalone._CAsyncCompressFilesPlan()
    c = _cfg() if cfg == "default" else cfg
    cc = c._to_c() if c is not None else None
    rc = L.pco_b200_compress_files_async_plan(C.c_ubyte(dtype), C.byref(cc) if cc is not None else None, C.c_int(uniform), C.c_size_t(max_files),
                                              C.c_size_t(nums_cap), C.c_size_t(max_file_n), C.c_size_t(dst_cap), C.c_size_t(index_cap), C.byref(p))
    return rc, p, L.pco_b200_last_error_message().decode()


def test_refusals_and_their_kinds(L):
    from pcodec_b200 import DeltaSpec, ModeSpec, PagingSpec

    cases = [
        (dict(dtype=99), 5, "type"),
        (dict(cfg=None), 7, "Auto"),  # the default config: Auto mode and delta
        (dict(cfg=_cfg(mode=ModeSpec.auto())), 7, "Auto"),
        (dict(cfg=_cfg(delta=DeltaSpec.auto())), 7, "Auto"),
        # level 9 at the largest chunk (2^16 numbers: unoptimized_bins_log 9)
        (dict(cfg=_cfg(level=9)), 7, "256 unoptimized bins"),
        (dict(cfg=_cfg(level=12)), 7, "256 unoptimized bins"),
        (dict(cfg=_cfg(paging=PagingSpec.exact_page_sizes([50, 50]))), 7, "Exact"),
        (dict(cfg=_cfg(level=13)), 3, "compression level"),
        (dict(cfg=_cfg(order=8)), 3, "delta order"),
        (dict(dtype=U8, cfg=_cfg(enable_8_bit=False)), 3, "8-bit"),
        (dict(dtype=F64, cfg=_cfg(mode=ModeSpec.try_int_mult(7))), 3, "int mult"),
        (dict(dtype=U64, cfg=_cfg(mode=ModeSpec.try_float_quant(3))), 3, "float mode"),
        (dict(cfg=_cfg(mode=ModeSpec.try_dict())), 7, "TryDict"),
        (dict(cfg=_cfg(delta=DeltaSpec.try_lookback())), 7, "Lookback"),
        (dict(cfg=_cfg(delta=DeltaSpec.try_conv1(1))), 7, "Conv1"),
        (dict(cfg=_cfg(page=1 << 25), max_file_n=(1 << 24) + 1, nums_cap=1 << 25), 3, "16777216"),
        # capacities
        (dict(max_files=0), 3, "max_files"),
        (dict(max_files=1 << 31), 3, "max_files"),
        (dict(max_file_n=0), 3, "max_file_n"),
        (dict(nums_cap=(1 << 56) + 1), 3, "nums_cap"),
        (dict(nums_cap=1 << 40, max_file_n=1), 3, "chunk slots"),
    ]
    for kw, kind, words in cases:
        rc, _, msg = _plan(L, **kw)
        assert rc == kind and words in msg, (kw, rc, msg)


def test_accepted_plans(L, ok):
    from pcodec_b200 import ModeSpec

    for kw in [dict(), dict(nums_cap=0), dict(max_files=1, nums_cap=1, max_file_n=1), dict(nums_cap=1 << 30, max_file_n=1 << 18),
               # chunk sizes that imply different unoptimized_bins_log in one batch are fine
               dict(cfg=_cfg(page=4096)), dict(cfg=_cfg(level=9), max_file_n=1 << 12),
               dict(dtype=F32, cfg=_cfg(mode=ModeSpec.try_float_mult(0.1))), dict(dtype=F16, cfg=_cfg(mode=ModeSpec.try_float_quant(3))),
               dict(dtype=I64, cfg=_cfg(mode=ModeSpec.try_int_mult(10), order=7)), dict(uniform=1), dict(max_files=(1 << 30) - 1, nums_cap=0)]:
        rc, p, msg = _plan(L, **kw)
        assert rc == ok, (kw, msg)


def _baseline_meta(bits):
    obb = {8: 4, 16: 5, 32: 6, 64: 7}[bits]  # bits of the offset width
    return (4 + (4 + 5 + 5 + 64 + 32 * 32) + 4 + 15 + bits + obb + 7) // 8


@pytest.mark.parametrize("dtype,max_files,nums_cap,max_file_n,page,mode", [
    (U64, 64, 1 << 20, 1 << 16, 1 << 18, "classic"), (U32, 1, 1, 1, 1 << 18, "classic"), (F32, 4096, 1 << 28, 1 << 16, 1 << 18, "fq"),
    (U16, 1706, (1 << 28) + 5, 1 << 20, 1 << 18, "classic"), (I64, 7, 1000, 5000, 300, "im"), (U8, 3, 0, 10, 1 << 18, "classic"),
])
def test_bounds_and_plan_fields(L, ok, dtype, max_files, nums_cap, max_file_n, page, mode):
    from pcodec_b200 import ModeSpec

    ms = {"classic": ModeSpec.classic(), "fq": ModeSpec.try_float_quant(3), "im": ModeSpec.try_int_mult(3)}[mode]
    rc, p, msg = _plan(L, dtype=dtype, cfg=_cfg(mode=ms, page=page), max_files=max_files, nums_cap=nums_cap, max_file_n=max_file_n,
                       dst_cap=12345, index_cap=777)
    assert rc == ok, msg
    m = max(1, min(page, max_file_n, nums_cap))
    n_vars = 1 if mode == "classic" else 2
    bits = BITS[dtype]
    assert p.max_chunks == nums_cap // m + max_files
    assert (p.dtype, p.n_vars, p.level, p.max_files, p.nums_cap, p.max_file_n, p.dst_cap, p.index_cap) == (
        dtype, n_vars, 8, max_files, nums_cap, max_file_n, 12345, 777)
    assert p.dst_bound == max_files * 18 + p.max_chunks * (5 + _baseline_meta(bits)) + (nums_cap * bits + 7) // 8
    assert p.index_bound == max_files * 64 + p.max_chunks * (32 + 12 * n_vars + 15) + 12 * n_vars * (-(-nums_cap // 256))


def _files_bytes(ns, page, bits, n_vars):
    """What a batch of these sizes can take at most, from the guarantees; and what its indexes take exactly."""
    dst = idx = 0
    for n in ns:
        k = -(-n // page) if n else 0
        idx += 64 + 32 * k
        dst += 18
        if k:
            low, rem = divmod(n, k)
            for size in [low + 1] * rem + [low] * (k - rem):
                dst += 4 + _baseline_meta(bits) + (size * bits + 7) // 8
                idx += (n_vars * -(-size // 256) * 12 + 15) // 16 * 16
    return dst, idx


def test_bounds_hold_for_extreme_batches(L, ok):
    rng = np.random.default_rng(5)
    for max_files, nums_cap, max_file_n, page in [(64, 1 << 20, 1 << 16, 1 << 18), (10, 5000, 5000, 300), (100, 100, 7, 1 << 18)]:
        rc, p, msg = _plan(L, max_files=max_files, nums_cap=nums_cap, max_file_n=max_file_n, cfg=_cfg(page=page))
        assert rc == ok, msg
        batches = [[max_file_n] * (nums_cap // max_file_n) + [nums_cap % max_file_n] + [1] * max_files, [1] * max_files, [0] * max_files]
        for _ in range(20):
            left, ns = nums_cap, []
            for _ in range(max_files):
                ns.append(int(min(left, rng.integers(0, max_file_n + 1))))
                left -= ns[-1]
            batches.append(ns)
        for ns in batches:
            ns = [min(n, max_file_n) for n in ns[:max_files]]
            while sum(ns) > nums_cap:
                ns[ns.index(max(ns))] -= 1
            d, i = _files_bytes(ns, page, 64, 1)
            assert sum(-(-n // page) for n in ns) <= p.max_chunks
            assert d <= p.dst_bound and i <= p.index_bound, (ns, d, p.dst_bound, i, p.index_bound)


def test_workspace_formula(L, ok):
    from pcodec_b200 import ModeSpec

    def ws(**kw):
        rc, p, msg = _plan(L, **kw)
        assert rc == ok, msg
        return p.workspace_bytes

    # per number of nums_cap (with the chunk slots fixed: nums_cap / max_file_n constant): 3 x 8 + 5 bytes for Classic u64, 4 x 8 + 10 for
    # two vars, in each of the six (or ten) per-number regions
    base = ws(nums_cap=1 << 20, max_file_n=1 << 20, max_files=64)
    more = ws(nums_cap=(1 << 20) + 256 * 64, max_file_n=1 << 20, max_files=64)
    assert more - base == 256 * 64 * (3 * 8 + 5)
    two = ws(nums_cap=(1 << 20) + 256 * 64, max_file_n=1 << 20, max_files=64, cfg=_cfg(mode=ModeSpec.try_int_mult(3))) - \
        ws(nums_cap=1 << 20, max_file_n=1 << 20, max_files=64, cfg=_cfg(mode=ModeSpec.try_int_mult(3)))
    assert two == 256 * 64 * (4 * 8 + 10)
    # more files: more chunk slots and file rows, so more workspace
    assert ws(max_files=1 << 12) > ws(max_files=64)
    assert ws(dtype=U16) < ws(dtype=U32) < ws(dtype=U64)


def _result(L, **fields):
    from pcodec_b200 import standalone

    s = standalone._CAsyncCompressFilesStatus(**fields)
    dl, il = C.c_size_t(111), C.c_size_t(222)
    rc = L.pco_b200_compress_files_async_result(C.byref(s), C.byref(dl), C.byref(il))
    return rc, L.pco_b200_last_error_message().decode(), (dl.value, il.value)


def test_result_maps_statuses_to_kinds_and_messages(L):
    rc, _, sizes = _result(L, kind=0, dst_bytes=1000, index_bytes=96, dst_written=1000, index_written=96)
    assert (rc, sizes) == (0, (1000, 96))
    rc, msg, sizes = _result(L, kind=3, device_status=0x10e, file=(1 << 64) - 1, n_files=99)
    assert rc == 3 and "99 files" in msg and "max_files" in msg, msg
    assert sizes == (111, 222)  # left alone on an error
    rc, msg, _ = _result(L, kind=3, device_status=0x116, file=17)
    assert rc == 3 and msg.startswith("file 17: ") and "max_file_n" in msg, msg
    rc, msg, _ = _result(L, kind=3, device_status=0x117, file=5)
    assert rc == 3 and msg.startswith("file 5: ") and "nums_cap" in msg, msg
    for code in (0x118, 0x119):
        rc, msg, _ = _result(L, kind=4, device_status=code, dst_bytes=12345, index_bytes=678)
        assert rc == 4 and "need 12345 file bytes and 678 index bytes" in msg, msg
    rc, _, _ = _result(L, kind=99, device_status=5)
    assert rc == 1  # a kind the library does not know reads as Corruption
    assert L.pco_b200_compress_files_async_result(None, None, None) == 3
    from pcodec_b200 import standalone

    s = standalone._CAsyncCompressFilesStatus(kind=0, dst_written=5)
    assert L.pco_b200_compress_files_async_result(C.byref(s), None, None) == 0


def test_call_refuses_bad_arguments_before_the_device(L):
    from pcodec_b200 import standalone

    _, p, _ = _plan(L)
    s = standalone._CAsyncCompressFilesStatus()
    nz = C.c_void_p(256)  # never dereferenced: the call refuses first
    call = L.pco_b200_compress_files_async

    def run(plan=C.byref(p), nums=nz, file_ns=nz, n_files=nz, dst=nz, index=None, files=nz, ws=nz, status=C.byref(s)):
        return call(plan, nums, file_ns, n_files, dst, index, files, ws, status, None)

    assert run(plan=None) == 3
    for name in ("nums", "file_ns", "n_files", "dst", "files", "ws", "status"):
        assert run(**{name: None}) == 3, name
    assert run(index=nz) == 3  # an index with a plan made without one
    assert run(ws=C.c_void_p(257)) == 3  # unaligned workspace
    for field, delta in [("workspace_bytes", 1), ("max_chunks", 1), ("n_vars", 1), ("mode", 9), ("level", 13), ("dtype", 90), ("max_files", -64),
                         ("max_file_n", -(1 << 16))]:
        bad = standalone._CAsyncCompressFilesPlan.from_buffer_copy(bytes(p))
        setattr(bad, field, getattr(bad, field) + delta)
        assert run(plan=C.byref(bad)) == 3, field
    unfilled = standalone._CAsyncCompressFilesPlan()
    assert run(plan=C.byref(unfilled)) == 3
    _, pi, _ = _plan(L, index_cap=1 << 20)
    assert run(plan=C.byref(pi), index=C.c_void_p(264)) == 3  # index not 16-byte aligned


def test_no_device_is_cuda_after_the_checks(L):
    if L.pco_b200_device_available():
        pytest.skip("a device is present")
    rc, p, msg = _plan(L)
    assert rc == 6 and "CUDA" in msg, msg
    assert p.workspace_bytes > 0 and p.max_chunks == 16 + 64  # filled before the device is touched


def test_device_header_writer_matches_the_host_header():
    """standalone_header_into serves the host and acf_frame_kernel alike; its bytes must not change: they are the reference's (varint size
    hint of 6 bits power - 1, then `power` bits of n), for n across every varint length and both flavours."""
    for uniform in (False, True):
        for power in range(0, 65):
            for n in {max(0, (1 << power) - 1), 1 << min(power, 63), (1 << min(power, 63)) + 1}:
                if n >= 1 << 64:
                    continue
                # the header of an empty file written by the library is header + terminator; compare with the format's bytes
                p = 1
                while p < 64 and (n >> p) != 0:
                    p += 1
                nbytes = (6 + p + 7) // 8
                val = (p - 1) | (n << 6)
                want = bytes([112, 99, 111, 33, 3, 2 if uniform else 0]) + val.to_bytes(nbytes + 1, "little")[:nbytes] + bytes([4, 1])
                assert len(want) == 8 + nbytes <= 17
                got = _header_bytes(n, uniform)
                assert got == want, (n, uniform, got, want)


def _header_bytes(n, uniform):
    """The library's standalone header for a size hint of n (pco_b200_debug_standalone_header, the function acf_frame_kernel calls)."""
    from pcodec_b200 import _lib

    L = _lib.lib()
    L.pco_b200_debug_standalone_header.restype = C.c_size_t
    L.pco_b200_debug_standalone_header.argtypes = [C.c_uint64, C.c_ubyte, C.c_void_p]
    buf = (C.c_ubyte * 32)()
    k = L.pco_b200_debug_standalone_header(C.c_uint64(n), C.c_ubyte(2 if uniform else 0), buf)
    return bytes(buf[:k])
