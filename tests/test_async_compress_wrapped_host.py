"""Host side of the asynchronous batch compress into wrapped chunks (pco_b200_compress_wrapped_async_plan / _async / _result) without a
GPU: the plan's refusals and their kinds, its fields, its metas, pages and workspace formulas, the bounds against extreme batches, how a
status written by the device becomes a kind and a message, and the call's argument checks."""
import ctypes as C

import pytest

U8, U16, U32, U64, I64, F16, F32, F64 = 10, 7, 1, 2, 4, 9, 5, 6  # number type bytes (cpcodec.h)
BITS = {U8: 8, U16: 16, U32: 32, U64: 64, I64: 64, F16: 16, F32: 32, F64: 64}
OBB = {8: 4, 16: 5, 32: 6, 64: 7}  # bits of the offset width: log2(L) + 1


@pytest.fixture(scope="module")
def L():
    from pcodec_b200 import wrapped

    return wrapped._lib_async_compress_wrapped()


@pytest.fixture(scope="module")
def LF():
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


def _plan(L, dtype=U64, cfg="default", max_arrays=64, nums_cap=1 << 20, max_array_n=1 << 16, metas_cap=1 << 20, pages_cap=1 << 24):
    from pcodec_b200 import wrapped

    p = wrapped._CAsyncCompressWrappedPlan()
    c = _cfg() if cfg == "default" else cfg
    cc = c._to_c() if c is not None else None
    rc = L.pco_b200_compress_wrapped_async_plan(C.c_ubyte(dtype), C.byref(cc) if cc is not None else None, C.c_size_t(max_arrays),
                                                C.c_size_t(nums_cap), C.c_size_t(max_array_n), C.c_size_t(metas_cap), C.c_size_t(pages_cap),
                                                C.byref(p))
    return rc, p, L.pco_b200_last_error_message().decode()


def _files_plan(LF, dtype=U64, cfg="default", max_arrays=64, nums_cap=1 << 20, max_array_n=1 << 16, **_):
    from pcodec_b200 import standalone

    p = standalone._CAsyncCompressFilesPlan()
    c = _cfg() if cfg == "default" else cfg
    cc = c._to_c() if c is not None else None
    rc = LF.pco_b200_compress_files_async_plan(C.c_ubyte(dtype), C.byref(cc) if cc is not None else None, C.c_int(0), C.c_size_t(max_arrays),
                                               C.c_size_t(nums_cap), C.c_size_t(max_array_n), C.c_size_t(0), C.c_size_t(0), C.byref(p))
    return rc, p, LF.pco_b200_last_error_message().decode()


def _refusals():
    from pcodec_b200 import DeltaSpec, ModeSpec, PagingSpec

    return [
        ("dtype", dict(dtype=99), 5, "type"),
        ("default_config", dict(cfg=None), 7, "Auto"),  # the default config: Auto mode and delta
        ("auto_mode", dict(cfg=_cfg(mode=ModeSpec.auto())), 7, "Auto"),
        ("auto_delta", dict(cfg=_cfg(delta=DeltaSpec.auto())), 7, "Auto"),
        ("level9", dict(cfg=_cfg(level=9)), 7, "256 unoptimized bins"),  # 2^16 numbers at the largest chunk: unoptimized_bins_log 9
        ("level12", dict(cfg=_cfg(level=12)), 7, "256 unoptimized bins"),
        ("exact", dict(cfg=_cfg(paging=PagingSpec.exact_page_sizes([50, 50]))), 7, "Exact"),
        ("level13", dict(cfg=_cfg(level=13)), 3, "compression level"),
        ("order8", dict(cfg=_cfg(order=8)), 3, "delta order"),
        ("u8_without_8_bit", dict(dtype=U8, cfg=_cfg(enable_8_bit=False)), 3, "8-bit"),
        ("f16_float_mult", dict(dtype=F16, cfg=_cfg(mode=ModeSpec.try_float_mult(0.5))), None, None),  # whatever compress_files_async_plan says
        ("int_mult_on_floats", dict(dtype=F64, cfg=_cfg(mode=ModeSpec.try_int_mult(7))), 3, "int mult"),
        ("dict", dict(cfg=_cfg(mode=ModeSpec.try_dict())), 7, "TryDict"),
        ("lookback", dict(cfg=_cfg(delta=DeltaSpec.try_lookback())), 7, "Lookback"),
        ("conv1", dict(cfg=_cfg(delta=DeltaSpec.try_conv1(1))), 7, "Conv1"),
        ("page_above_2_24", dict(cfg=_cfg(page=1 << 25), max_array_n=(1 << 24) + 1, nums_cap=1 << 25), 3, "16777216"),
        ("max_arrays_0", dict(max_arrays=0), 3, "max_arrays"),
        ("max_arrays_2_31", dict(max_arrays=1 << 31), 3, "max_arrays"),
        ("max_array_n_0", dict(max_array_n=0), 3, "max_array_n"),
        ("nums_cap_above_2_56", dict(nums_cap=(1 << 56) + 1), 3, "nums_cap"),
        ("too_many_ctas", dict(nums_cap=1 << 40, max_array_n=1), 3, "chunk slots"),
    ]


@pytest.mark.parametrize("name,kw,kind,words", _refusals(), ids=[r[0] for r in _refusals()])
def test_plan_refusals_and_their_kinds(L, LF, name, kw, kind, words):
    rc, _, msg = _plan(L, **kw)
    frc, _, fmsg = _files_plan(LF, **kw)
    assert rc == frc, (name, rc, msg, frc, fmsg)  # the kinds of pco_b200_compress_files_async_plan, refusal for refusal
    assert rc not in (0, 6), (name, msg)
    if kind is not None:
        assert rc == kind and words in msg, (name, rc, msg)
    if "files" not in fmsg and "file_n" not in fmsg:
        assert msg == fmsg, (name, msg, fmsg)


def test_refusal_order_matches_the_files_plan(L, LF):
    from pcodec_b200 import DeltaSpec, PagingSpec

    # several defects at once: the first one the files plan reports is the one reported here
    for kw in [dict(max_arrays=0, cfg=_cfg(paging=PagingSpec.exact_page_sizes([5]))), dict(cfg=_cfg(paging=PagingSpec.exact_page_sizes([5]), level=13)),
               dict(cfg=_cfg(level=13, delta=DeltaSpec.auto())), dict(cfg=_cfg(delta=DeltaSpec.auto(), level=12)),
               dict(cfg=_cfg(level=12), nums_cap=1 << 40, max_array_n=1 << 16, max_arrays=1 << 30), dict(nums_cap=(1 << 56) + 1, max_array_n=0)]:
        rc, _, msg = _plan(L, **kw)
        frc, _, fmsg = _files_plan(LF, **kw)
        assert rc == frc and msg.replace("array", "file") == fmsg, (kw, msg, fmsg)


def test_accepted_plans(L, ok):
    from pcodec_b200 import ModeSpec

    for kw in [dict(), dict(nums_cap=0), dict(max_arrays=1, nums_cap=1, max_array_n=1), dict(nums_cap=1 << 30, max_array_n=1 << 18),
               dict(cfg=_cfg(page=4096)), dict(cfg=_cfg(level=9), max_array_n=1 << 12), dict(metas_cap=0, pages_cap=0),
               dict(dtype=F32, cfg=_cfg(mode=ModeSpec.try_float_mult(0.1))), dict(dtype=F16, cfg=_cfg(mode=ModeSpec.try_float_quant(3))),
               dict(dtype=I64, cfg=_cfg(mode=ModeSpec.try_int_mult(10), order=7)), dict(max_arrays=(1 << 30) - 1, nums_cap=0)]:
        rc, p, msg = _plan(L, **kw)
        assert rc == ok, (kw, msg)


def _baseline_meta(bits):
    return (4 + (4 + 5 + 5 + 64 + 32 * 32) + 4 + 15 + bits + OBB[bits] + 7) // 8


def _meta_max(bits, mode):
    n_vars = 1 if mode == "classic" else 2
    mode_bits = {"classic": 0, "fq": 8, "im": bits, "fm": bits}[mode]
    return (4 + mode_bits + 1102 + n_vars * (19 + 256 * (15 + bits + OBB[bits])) + 7) // 8


def _bounds(dtype, mode, max_chunks, nums_cap):
    bits = BITS[dtype]
    pages = max_chunks * (1 + _baseline_meta(bits)) + (nums_cap * bits + 7) // 8
    return min(max_chunks * _meta_max(bits, mode), pages), pages


@pytest.mark.parametrize("dtype,max_arrays,nums_cap,max_array_n,page,mode", [
    (U64, 64, 1 << 20, 1 << 16, 1 << 18, "classic"), (U32, 1, 1, 1, 1 << 18, "classic"), (F32, 4096, 1 << 28, 1 << 16, 1 << 18, "fq"),
    (U16, 1706, (1 << 28) + 5, 1 << 20, 1 << 18, "classic"), (I64, 7, 1000, 5000, 300, "im"), (U8, 3, 0, 10, 1 << 18, "classic"),
    (F64, 1024, 1 << 28, 1 << 18, 1 << 18, "fm"), (U64, 1, 1 << 28, 1 << 28, 1 << 18, "classic"),
])
def test_plan_fields_and_formulas(L, LF, ok, dtype, max_arrays, nums_cap, max_array_n, page, mode):
    from pcodec_b200 import ModeSpec

    ms = {"classic": ModeSpec.classic(), "fq": ModeSpec.try_float_quant(3), "im": ModeSpec.try_int_mult(3), "fm": ModeSpec.try_float_mult(0.5)}[mode]
    cfg = _cfg(mode=ms, page=page)
    rc, p, msg = _plan(L, dtype=dtype, cfg=cfg, max_arrays=max_arrays, nums_cap=nums_cap, max_array_n=max_array_n, metas_cap=12345, pages_cap=777)
    assert rc == ok, msg
    m = max(1, min(page, max_array_n, nums_cap))
    n_vars = 1 if mode == "classic" else 2
    bits = BITS[dtype]
    assert p.max_chunks == nums_cap // m + max_arrays
    assert (p.dtype, p.n_vars, p.level, p.order, p.max_arrays, p.nums_cap, p.max_array_n, p.max_page_n, p.metas_cap, p.pages_cap) == (
        dtype, n_vars, 8, 1, max_arrays, nums_cap, max_array_n, page, 12345, 777)
    assert (p.metas_bound, p.pages_bound) == _bounds(dtype, mode, p.max_chunks, nums_cap)
    # the workspace: pco_b200_compress_files_async_plan's for the same capacities, then the staging region, the state, the meta lengths and
    # the CTA sums, each rounded up to 256 bytes
    frc, fp, fmsg = _files_plan(LF, dtype=dtype, cfg=cfg, max_arrays=max_arrays, nums_cap=nums_cap, max_array_n=max_array_n)
    assert frc == ok, fmsg
    assert fp.max_chunks == p.max_chunks

    def al(x):
        return (x + 255) // 256 * 256

    stage = p.max_chunks * (5 + _baseline_meta(bits)) + (nums_cap * bits + 7) // 8
    assert stage == fp.dst_bound - max_arrays * 18  # a headerless dst_bound
    assert p.workspace_bytes == fp.workspace_bytes + al(stage) + al(32) + al(4 * p.max_chunks) + al(48 * -(-(p.max_chunks + 1) // 256))


def _chunk_ns(n, page):
    if n == 0:
        return []
    k = -(-n // page)
    low, rem = divmod(n, k)
    return [low + 1] * rem + [low] * (k - rem)


def _need(ns, page, bits, mode):
    """What a batch of these sizes can take at most: per chunk, its meta and its page each at most B + ceil(n L / 8) bytes, its meta also at
    most the largest meta."""
    metas = pages = 0
    for n in ns:
        for c in _chunk_ns(n, page):
            body = _baseline_meta(bits) + (c * bits + 7) // 8
            metas += min(_meta_max(bits, mode), body)
            pages += body
    return metas, pages


def test_bounds_hold_for_extreme_batches(L, ok):
    for dtype, mode in [(U64, "classic"), (U8, "classic"), (F32, "fm"), (F16, "fq")]:
        from pcodec_b200 import ModeSpec

        ms = {"classic": ModeSpec.classic(), "fq": ModeSpec.try_float_quant(3), "fm": ModeSpec.try_float_mult(0.5)}[mode]
        for max_arrays, nums_cap, max_array_n, page in [(64, 1 << 20, 1 << 16, 1 << 18), (10, 5000, 5000, 300), (100, 100, 7, 1 << 18),
                                                         (4, 1 << 20, 1 << 20, 1 << 18), (3, (1 << 18) * 2 + 2, (1 << 18) + 1, 1 << 18)]:
            rc, p, msg = _plan(L, dtype=dtype, cfg=_cfg(mode=ms, page=page), max_arrays=max_arrays, nums_cap=nums_cap, max_array_n=max_array_n)
            assert rc == ok, msg
            m = min(page, max_array_n)
            batches = [[1] * max_arrays,                                        # every array of 1 number
                       [min(nums_cap, max_array_n)],                            # one full array
                       [max_array_n] * (nums_cap // max_array_n) + [nums_cap % max_array_n] + [1] * max_arrays,
                       [m] * max_arrays, [m + 1] * max_arrays, [m - 1] * max_arrays, [2 * m + 1] * max_arrays]  # at page boundaries
            for ns in batches:
                ns = [max(0, min(n, max_array_n)) for n in ns[:max_arrays]]
                while sum(ns) > nums_cap:
                    ns[ns.index(max(ns))] -= 1
                assert sum(len(_chunk_ns(n, page)) for n in ns) <= p.max_chunks
                metas, pages = _need(ns, page, BITS[dtype], mode)
                assert metas <= p.metas_bound and pages <= p.pages_bound, (dtype, ns[:4], metas, p.metas_bound, pages, p.pages_bound)


def _result(L, **fields):
    from pcodec_b200 import wrapped

    s = wrapped._CAsyncCompressWrappedStatus(**fields)
    ml, pl, nc = C.c_size_t(111), C.c_size_t(222), C.c_size_t(333)
    rc = L.pco_b200_compress_wrapped_async_result(C.byref(s), C.byref(ml), C.byref(pl), C.byref(nc))
    return rc, L.pco_b200_last_error_message().decode(), (ml.value, pl.value, nc.value)


def test_result_maps_statuses_to_kinds_and_messages(L):
    rc, _, sizes = _result(L, kind=0, n_chunks=9, metas_bytes=1000, pages_bytes=96, metas_written=1000, pages_written=96)
    assert (rc, sizes) == (0, (1000, 96, 9))
    rc, msg, sizes = _result(L, kind=3, device_status=0x10e, array=(1 << 64) - 1, n_arrays=99)
    assert rc == 3 and "99 arrays" in msg and "max_arrays" in msg, msg
    assert sizes == (111, 222, 333)  # left alone on an error
    rc, msg, _ = _result(L, kind=3, device_status=0x116, array=17)
    assert rc == 3 and msg.startswith("array 17: ") and "max_array_n" in msg, msg
    rc, msg, _ = _result(L, kind=3, device_status=0x117, array=5)
    assert rc == 3 and msg.startswith("array 5: ") and "nums_cap" in msg, msg
    rc, msg, _ = _result(L, kind=4, device_status=0x118, metas_bytes=12345, pages_bytes=678)
    assert rc == 4 and "need 12345 meta bytes and 678 page bytes" in msg, msg
    rc, msg, _ = _result(L, kind=1, device_status=1)
    assert rc == 1 and "split" in msg, msg
    rc, _, _ = _result(L, kind=99, device_status=5)
    assert rc == 1  # a kind the library does not know reads as Corruption
    assert L.pco_b200_compress_wrapped_async_result(None, None, None, None) == 3
    from pcodec_b200 import wrapped

    s = wrapped._CAsyncCompressWrappedStatus(kind=0, metas_written=5)
    assert L.pco_b200_compress_wrapped_async_result(C.byref(s), None, None, None) == 0


def test_status_codes_map_to_the_documented_kinds(L):
    kind = L.pco_b200_debug_async_kind
    assert [kind(c) for c in (0x10e, 0x116, 0x117, 0x118)] == [3, 3, 3, 4]


def test_call_refuses_bad_arguments_before_the_device(L):
    from pcodec_b200 import wrapped

    _, p, _ = _plan(L)
    s = wrapped._CAsyncCompressWrappedStatus()
    nz = C.c_void_p(256)  # never dereferenced: the call refuses first
    call = L.pco_b200_compress_wrapped_async

    def run(plan=C.byref(p), nums=nz, array_ns=nz, n_arrays=nz, metas=nz, pages=nz, refs=nz, first_chunk=nz, ws=nz, status=C.byref(s)):
        return call(plan, nums, array_ns, n_arrays, metas, pages, refs, first_chunk, ws, status, None)

    assert run(plan=None) == 3
    for name in ("nums", "array_ns", "n_arrays", "metas", "pages", "refs", "first_chunk", "ws", "status"):
        assert run(**{name: None}) == 3, name
    assert run(ws=C.c_void_p(257)) == 3  # unaligned workspace
    assert run(refs=C.c_void_p(260)) == 3 and run(first_chunk=C.c_void_p(257)) == 3  # unaligned refs, first_chunk
    for field, delta in [("workspace_bytes", 1), ("max_chunks", 1), ("n_vars", 1), ("mode", 9), ("level", 13), ("dtype", 90), ("max_arrays", -64),
                         ("max_array_n", -(1 << 16)), ("nums_cap", 1 << 57)]:
        bad = wrapped._CAsyncCompressWrappedPlan.from_buffer_copy(bytes(p))
        setattr(bad, field, getattr(bad, field) + delta)
        assert run(plan=C.byref(bad)) == 3, field
        assert "pco_b200_compress_wrapped_async_plan" in L.pco_b200_last_error_message().decode()
    unfilled = wrapped._CAsyncCompressWrappedPlan()
    assert run(plan=C.byref(unfilled)) == 3


def test_no_device_is_cuda_after_the_checks(L):
    if L.pco_b200_device_available():
        pytest.skip("a device is present")
    rc, p, msg = _plan(L)
    assert rc == 6 and "CUDA" in msg, msg
    assert p.workspace_bytes > 0 and p.max_chunks == 16 + 64  # filled before the device is touched
    # the call passes its checks, then fails on the missing device
    from pcodec_b200 import wrapped

    s = wrapped._CAsyncCompressWrappedStatus()
    nz = C.c_void_p(256)
    rc = L.pco_b200_compress_wrapped_async(C.byref(p), nz, nz, nz, nz, nz, nz, nz, nz, C.byref(s), None)
    assert rc == 6, L.pco_b200_last_error_message().decode()
