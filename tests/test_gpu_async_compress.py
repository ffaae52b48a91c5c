"""Asynchronous compress (pco_b200_compress_async, standalone.AsyncCompressor): the file bytes and the side index bytes equal what
pco_b200_compress_ex writes for the same numbers and config with every buffer on the device, the file decodes back to the input, and nothing
is written outside dst_cap bytes of dst or outside the index - on every front-end route, inside a CUDA graph replayed over different inputs,
and on concurrent streams.  A capture that contained a synchronising or allocating call would fail, so the graph tests also check that the
call makes none."""
import ctypes as C

import numpy as np
import pytest

from tests.golden_generators import bits_view

pytestmark = pytest.mark.gpu

DTYPES = [np.uint8, np.int8, np.uint16, np.int16, np.float16, np.uint32, np.int32, np.float32, np.uint64, np.int64, np.float64]
GUARD = 4096  # bytes of sentinel before and behind dst and index
SENT = 0xA5


@pytest.fixture(scope="module")
def sa():
    from pcodec_b200 import standalone

    return standalone


def _walk(dtype, n, seed, scale=0.05):
    rng = np.random.default_rng(seed)
    if np.dtype(dtype).kind == "f":
        x = np.cumsum(rng.normal(size=n)).astype(dtype)
        if n > 5:
            x[3], x[4], x[5] = np.nan, -np.inf, -0.0
        return x
    steps = rng.geometric(scale, size=n).astype(np.int64) - int(1 / scale) // 2
    return np.cumsum(steps).astype(np.uint64).astype(np.dtype(dtype).str.replace("i", "u")).view(dtype)


def _cfg(order=1, page=1 << 14, level=8, mode="classic", base=0.01, ibase=8, k=13):
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec

    ms = {"classic": ModeSpec.classic(), "float_mult": ModeSpec.try_float_mult(base), "int_mult": ModeSpec.try_int_mult(ibase),
          "float_quant": ModeSpec.try_float_quant(k)}[mode]
    ds = DeltaSpec.try_consecutive(order) if order else DeltaSpec.no_op()
    return ChunkConfig(compression_level=level, mode_spec=ms, delta_spec=ds, paging_spec=PagingSpec.equal_pages_up_to(page), enable_8_bit=True)


def _device_numbers(a):
    import torch

    from pcodec_b200.wrapped import _torch_dtypes

    if a.size == 0:
        return torch.empty(0, dtype=_torch_dtypes()[np.dtype(a.dtype)], device="cuda")
    return torch.as_tensor(np.ascontiguousarray(a).view(np.uint8).copy(), device="cuda").view(_torch_dtypes()[np.dtype(a.dtype)])


def _cap(L, x, cfg):
    c = cfg._to_c()
    return L.pco_standalone_guarantee_file_size(x.size, _dtb(x.dtype)) + 160 * max(-(-x.size // (c.max_page_n or (1 << 18))), 1)


def _dtb(dtype):
    from pcodec_b200 import _lib

    return _lib.dtype_byte(np.dtype(dtype))


def _ex(x, cfg, uniform=False):
    """pco_b200_compress_ex with nums, dst and index on the device (n == 0: host buffers, the same bytes): (file, index)."""
    import torch

    from pcodec_b200 import _lib

    L = _lib.lib()
    n = x.size
    cap = _cap(L, x, cfg)
    icap = L.pco_b200_index_size_bound(n, max(n >> 8, 64)) + 64 * max(-(-n // (cfg._to_c().max_page_n or (1 << 18))), 1)
    c = cfg._to_c()
    written, ilen = C.c_size_t(), C.c_size_t()
    if n == 0:
        dst, idx = np.zeros(cap, np.uint8), np.zeros(icap, np.uint8)
        _lib.check(L.pco_b200_compress_ex(None, C.c_size_t(0), C.c_ubyte(_dtb(x.dtype)), C.byref(c), C.c_int(int(uniform)), dst.ctypes.data_as(C.c_void_p),
                                          C.c_size_t(cap), C.byref(written), idx.ctypes.data_as(C.c_void_p), C.c_size_t(icap), C.byref(ilen), C.c_uint32(0), None))
        return dst[: written.value].tobytes(), idx[: ilen.value].tobytes()
    d_x = _device_numbers(x)
    dst = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    idx = torch.zeros(icap, dtype=torch.uint8, device="cuda")
    _lib.check(L.pco_b200_compress_ex(C.c_void_p(d_x.data_ptr()), C.c_size_t(n), C.c_ubyte(_dtb(x.dtype)), C.byref(c), C.c_int(int(uniform)),
                                      C.c_void_p(dst.data_ptr()), C.c_size_t(cap), C.byref(written), C.c_void_p(idx.data_ptr()), C.c_size_t(icap),
                                      C.byref(ilen), C.c_uint32(7), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    return dst[: written.value].cpu().numpy().tobytes(), idx[: ilen.value].cpu().numpy().tobytes()


def _buffers(comp, with_index):
    import torch

    dbuf = torch.full((GUARD + comp.dst_cap + GUARD,), SENT, dtype=torch.uint8, device="cuda")
    ibuf = torch.full((GUARD + comp.index_bytes + GUARD,), SENT, dtype=torch.uint8, device="cuda") if with_index else None
    return dbuf, ibuf


def _views(comp, dbuf, ibuf):
    return dbuf[GUARD:GUARD + comp.dst_cap], (ibuf[GUARD:GUARD + comp.index_bytes] if ibuf is not None else None)


def _read(comp, dbuf, ibuf, fits=True):
    """The call's outcome, the file and the index; checks the guard zones and that nothing lies behind the file."""
    from pcodec_b200 import PcoError

    d = dbuf.cpu().numpy()
    assert (d[:GUARD] == SENT).all() and (d[GUARD + comp.dst_cap:] == SENT).all(), "a write outside dst"
    if ibuf is not None:
        ix = ibuf.cpu().numpy()
        assert (ix[:GUARD] == SENT).all() and (ix[GUARD + comp.index_bytes:] == SENT).all(), "a write outside the index"
    if not fits:
        with pytest.raises(PcoError) as e:
            comp.result()
        assert e.value.kind == "Io"
        return None, None
    fb, ib = comp.result()
    assert (d[GUARD + fb:GUARD + comp.dst_cap] == SENT).all(), "a write behind the file"
    return d[GUARD:GUARD + fb].tobytes(), (ix[GUARD:GUARD + ib].tobytes() if ibuf is not None else b"")


def _async(sa, x, cfg, uniform=False, with_index=True, dst_cap=None):
    comp = sa.AsyncCompressor(x.size, x.dtype, cfg, dst_cap=dst_cap, index=with_index, uniform_type_header=uniform)
    dbuf, ibuf = _buffers(comp, with_index)
    dst, idx = _views(comp, dbuf, ibuf)
    comp(_device_numbers(x), dst, idx)
    return comp, dbuf, ibuf


def _check(sa, x, cfg, uniform=False, with_index=True, oracle=None):
    from pcodec_b200 import _lib

    ref_file, ref_index = _ex(x, cfg, uniform)
    comp, dbuf, ibuf = _async(sa, x, cfg, uniform, with_index, dst_cap=_cap(_lib.lib(), x, cfg))
    data, index = _read(comp, dbuf, ibuf)
    assert data == ref_file
    if with_index:
        assert index == ref_index
    back = sa.simple_decompress(data, x.dtype, index=index if with_index else None)
    np.testing.assert_array_equal(bits_view(back), bits_view(x))
    if oracle is not None:
        np.testing.assert_array_equal(bits_view(oracle.simple_decompress(data, x.dtype)), bits_view(x))
    return data, index


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("order", [0, 1, 2, 7])
def test_types_and_orders(sa, oracle, dtype, order):
    x = _walk(dtype, 3 * (1 << 14) + 77, seed=order)
    _check(sa, x, _cfg(order=order), oracle=oracle if order in (0, 7) else None)


@pytest.mark.parametrize("dtype,mode,kw", [(np.int64, "int_mult", dict(ibase=7)), (np.uint32, "int_mult", dict(ibase=1000)),
                                           (np.float32, "float_quant", dict(k=10)), (np.float64, "float_quant", dict(k=30)),
                                           (np.float16, "float_quant", dict(k=3)), (np.float32, "float_mult", dict(base=0.1)),
                                           (np.float64, "float_mult", dict(base=0.01))])
@pytest.mark.parametrize("order", [0, 1])
def test_two_var_modes(sa, oracle, dtype, mode, kw, order):
    rng = np.random.default_rng(11)
    n = 2 * (1 << 14) + 5
    if mode == "int_mult":
        x = (np.cumsum(rng.integers(0, 9, size=n)) * kw["ibase"] + rng.integers(0, 3, size=n)).astype(dtype)
    elif mode == "float_mult":
        x = (np.round(np.cumsum(rng.normal(size=n)) * 50) * kw["base"]).astype(dtype)
    else:
        x = np.cumsum(rng.normal(size=n)).astype(dtype)
    _check(sa, x, _cfg(order=order, mode=mode, **kw), oracle=oracle if order == 1 else None)


def _spans(n, wide_from, seed):
    """u64 walk whose chunks of 2^14 from chunk `wide_from` on have latents spanning more than 2^15 (2^20 steps)."""
    rng = np.random.default_rng(seed)
    steps = rng.integers(0, 50, size=n).astype(np.uint64)
    steps[wide_from * (1 << 14):] = rng.integers(0, 1 << 20, size=n - wide_from * (1 << 14)).astype(np.uint64)
    return np.cumsum(steps)


@pytest.mark.parametrize("case", ["all_wide", "some_wide", "sort_path", "narrow_order0"])
def test_front_end_routes(sa, oracle, case):
    """The two-kernel fallback (a chunk's latents span 2^15 or more), with the sort path when the range needs more than 15 bits, and a
    call where only some chunks overflow."""
    n = 4 * (1 << 14)
    if case == "all_wide":
        x, cfg = _spans(n, 0, 1), _cfg(order=1)
    elif case == "some_wide":
        x, cfg = _spans(n, 3, 2), _cfg(order=1)
    elif case == "sort_path":
        x, cfg = np.random.default_rng(3).integers(0, 1 << 40, size=n).astype(np.uint64), _cfg(order=0)
    else:
        x, cfg = np.random.default_rng(4).integers(0, 1 << 12, size=n).astype(np.uint32), _cfg(order=0)
    _check(sa, x, cfg, oracle=oracle)


@pytest.mark.parametrize("n,page", [(1, 1 << 18), (255, 1 << 18), (256, 1 << 18), (257, 1 << 18), (1 << 18, 1 << 18), ((1 << 20) + 1, 1 << 21),
                                    (2, 1), (2 * 300, 300), (1024 * 64, 64), (0, 1 << 18)])
def test_chunk_sizes_and_counts(sa, n, page):
    x = _walk(np.int32, n, seed=n)
    _check(sa, x, _cfg(order=1, page=page))


def test_one_chunk_of_2_24(sa, oracle):
    x = _walk(np.uint32, 1 << 24, seed=24)
    _check(sa, x, _cfg(order=1, page=1 << 24), oracle=oracle)


@pytest.mark.parametrize("uniform", [False, True])
@pytest.mark.parametrize("with_index", [False, True])
def test_header_flavours_with_and_without_index(sa, uniform, with_index):
    x = _walk(np.float32, 70000, seed=9)
    data, _ = _check(sa, x, _cfg(order=2, page=30000), uniform=uniform, with_index=with_index)
    assert data[5] == (5 if uniform else 0)  # the header's uniform type byte


def test_dst_cap_exact_slack_and_one_byte_short(sa):
    x = _walk(np.uint64, 50000, seed=12)
    cfg = _cfg(order=1, page=20000)
    ref, ref_index = _ex(x, cfg)
    for cap in (len(ref), len(ref) + 1000):
        comp, dbuf, ibuf = _async(sa, x, cfg, dst_cap=cap)
        assert _read(comp, dbuf, ibuf) == (ref, ref_index)
    comp, dbuf, ibuf = _async(sa, x, cfg, dst_cap=len(ref) - 1)
    _read(comp, dbuf, ibuf, fits=False)
    st = sa._CAsyncCompressStatus.from_buffer_copy(comp.status.cpu().numpy().tobytes())
    assert (st.kind, st.device_status, st.file_bytes, st.n_written) == (4, 0x106, len(ref), 0)
    comp, dbuf, ibuf = _async(sa, np.zeros(0, np.uint64), cfg, dst_cap=9)  # an empty file needs header + terminator
    _read(comp, dbuf, ibuf, fits=False)


def _graph_inputs(dtype, n):
    return [_walk(dtype, n, seed=s) for s in (1, 2, 3)]


def test_one_graph_over_three_inputs_and_after_thread_release(sa):
    import torch

    from pcodec_b200 import _lib

    n, cfg = 100000, _cfg(order=1, page=30000)
    xs = _graph_inputs(np.int64, n)
    xs[1] = _spans(n, 2, 5).view(np.int64)  # the second input takes the two-kernel fallback
    refs = [_ex(x, cfg) for x in xs]
    comp = sa.AsyncCompressor(n, np.int64, cfg, dst_cap=_cap(_lib.lib(), xs[0], cfg))
    dbuf, ibuf = _buffers(comp, True)
    dst, idx = _views(comp, dbuf, ibuf)
    d_nums = _device_numbers(xs[0])
    comp(d_nums, dst, idx)  # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        comp(d_nums, dst, idx)
    for rnd in range(3):
        if rnd == 1:
            _lib.lib().pco_b200_thread_release()
        if rnd == 2:  # a larger blocking compress on the same thread grows and reuses its scratch
            _ex(_walk(np.int64, 3 * n, seed=8), cfg)
        for x, ref in zip(xs, refs):
            d_nums.copy_(_device_numbers(x))
            dbuf.fill_(SENT)  # the files differ in size: nothing of an earlier one may stay behind
            ibuf.fill_(SENT)
            g.replay()
            torch.cuda.synchronize()
            assert _read(comp, dbuf, ibuf) == ref


def test_two_streams_two_workspaces(sa):
    import torch

    from pcodec_b200 import _lib

    cfg = _cfg(order=2, page=1 << 15)
    xa, xb = _walk(np.uint32, 200000, seed=21), _walk(np.uint32, 200000, seed=22)
    ra, rb = _ex(xa, cfg), _ex(xb, cfg)
    comps = [sa.AsyncCompressor(x.size, x.dtype, cfg, dst_cap=_cap(_lib.lib(), x, cfg)) for x in (xa, xb)]
    bufs = [_buffers(c, True) for c in comps]
    nums = [_device_numbers(x) for x in (xa, xb)]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for _ in range(3):
        for c, (d, i), t, s in zip(comps, bufs, nums, streams):
            with torch.cuda.stream(s):
                c(t, *_views(c, d, i))
    torch.cuda.synchronize()
    assert _read(comps[0], *bufs[0]) == ra
    assert _read(comps[1], *bufs[1]) == rb


def test_compress_and_decompress_round_trip_in_one_graph(sa):
    import torch

    from pcodec_b200 import _lib

    n, cfg = 1 << 17, _cfg(order=1, page=1 << 15)
    xs = _graph_inputs(np.uint64, n)
    ref_file, _ = _ex(xs[0], cfg)
    comp = sa.AsyncCompressor(n, np.uint64, cfg, dst_cap=_cap(_lib.lib(), xs[0], cfg))
    dst = torch.zeros(comp.dst_cap, dtype=torch.uint8, device="cuda")
    idx = torch.zeros(comp.index_bytes, dtype=torch.uint8, device="cuda")
    # the decompressor's plan takes its head from any file of the same flavour
    dec = sa.AsyncDecompressor(ref_file[:32], np.uint64, comp.dst_cap, comp.index_bytes, n, -(-n // (1 << 15)))
    d_nums = _device_numbers(xs[0])
    out = torch.zeros(n, dtype=torch.int64, device="cuda").view(torch.uint64)
    comp(d_nums, dst, idx)
    dec(dst, idx, out)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        comp(d_nums, dst, idx)
        dec(dst, idx, out)
    for x in xs:
        d_nums.copy_(_device_numbers(x))
        out.view(torch.int64).zero_()
        g.replay()
        torch.cuda.synchronize()
        fb, _ = comp.result()
        assert dst[:fb].cpu().numpy().tobytes() == _ex(x, cfg)[0]
        prog = dec.result()
        assert (prog.n_processed, prog.finished) == (n, True)
        np.testing.assert_array_equal(out.view(torch.int64).cpu().numpy().view(np.uint64), x)


def test_profiled_call_records_its_kernel_spans(sa):
    import torch

    from pcodec_b200 import _lib

    L = _lib.lib()
    x = _walk(np.uint64, 1 << 16, seed=31)
    cfg = _cfg(order=1)
    comp = sa.AsyncCompressor(x.size, x.dtype, cfg, dst_cap=_cap(L, x, cfg))
    dbuf, ibuf = _buffers(comp, True)
    L.pco_b200_profile_enable(1)
    try:
        comp(_device_numbers(x), *_views(comp, dbuf, ibuf))
        torch.cuda.synchronize()
        buf = C.create_string_buffer(1 << 16)
        L.pco_b200_profile_last(buf, C.c_size_t(1 << 16))
        spans = dict(kv.split("=") for kv in buf.value.decode().split(";") if "=" in kv)
    finally:
        L.pco_b200_profile_enable(0)
    for name in ("acomp_init_kernel", "split_count_kernel", "plan_solve_kernel", "bin_lut_kernel", "ans_encode_kernel", "pack_kernel", "acomp_finish_kernel"):
        assert name in spans and float(spans[name]) >= 0, (name, spans)
    assert _read(comp, dbuf, ibuf) == _ex(x, cfg)
