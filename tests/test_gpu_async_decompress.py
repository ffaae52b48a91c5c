"""Asynchronous decompress of indexed standalone files (pco_b200_decompress_async, standalone.AsyncDecompressor): every output equals
pco_b200_decompress_ex on the same file and index, and the input, bit for bit - whatever the spare capacity, inside a CUDA graph replayed
over different files, and on concurrent streams."""
import ctypes as C
import re

import numpy as np
import pytest

from tests.golden_generators import bits_view

pytestmark = pytest.mark.gpu

DTYPES = [np.uint8, np.int8, np.uint16, np.int16, np.float16, np.uint32, np.int32, np.float32, np.uint64, np.int64, np.float64]
GUARD = 4096  # numbers of sentinel before and behind every destination


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


def _cfg(order=0, page=1 << 14, level=8, mode="classic", base=0.01, ibase=8, k=13, exact=None):
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec

    ms = {"classic": ModeSpec.classic(), "float_mult": ModeSpec.try_float_mult(base), "int_mult": ModeSpec.try_int_mult(ibase),
          "float_quant": ModeSpec.try_float_quant(k)}[mode]
    ds = DeltaSpec.try_consecutive(order) if order else DeltaSpec.no_op()
    ps = PagingSpec.exact_page_sizes(exact) if exact else PagingSpec.equal_pages_up_to(page)
    return ChunkConfig(compression_level=level, mode_spec=ms, delta_spec=ds, paging_spec=ps, enable_8_bit=True)


def _n_chunks(index):
    return int(np.frombuffer(index[8:16], np.uint64)[0])


def _tdtype(dtype):
    from pcodec_b200.wrapped import _torch_dtypes

    return _torch_dtypes()[np.dtype(dtype)]


def _sentinel(dtype):
    return np.frombuffer(b"\xa5" * 8, np.uint8)[: np.dtype(dtype).itemsize].view(dtype)[0]


def _ex(sa, data, index, dtype, dst_cap):
    """pco_b200_decompress_ex on the same file and index: (numbers, Progress) or (None, (kind, chunk named in the message))."""
    from pcodec_b200 import PcoError

    dst = np.zeros(max(dst_cap, 1), dtype=dtype)
    try:
        prog = sa.decompress_into_with_index(data, dst[:dst_cap], index)
    except PcoError as e:
        m = re.search(r"chunk (\d+)", e.message)
        return None, (e.kind, int(m.group(1)) if m else None)
    return dst[: prog.n_processed], (prog.n_processed, prog.finished)


def _async(sa, data, index, dtype, src_cap=None, index_cap=None, dst_cap=None, max_chunks=None, stale=0):
    """One AsyncDecompressor call on device buffers of the given capacities (default: the file's own sizes), with sentinel guard zones
    around dst.  Bytes behind the file and the index are random when stale != 0.  Returns (numbers or None, Progress or (kind, chunk))."""
    import torch

    from pcodec_b200 import PcoError

    n = int(np.frombuffer(index[16:24], np.uint64)[0]) if len(index) >= 24 else 0
    src_cap = len(data) if src_cap is None else src_cap
    index_cap = len(index) if index_cap is None else index_cap
    dst_cap = n if dst_cap is None else dst_cap
    max_chunks = max(_n_chunks(index), 1) if max_chunks is None else max_chunks
    rng = np.random.default_rng(stale)
    srcb = rng.integers(0, 256, size=max(src_cap, 1), dtype=np.uint8) if stale else np.zeros(max(src_cap, 1), np.uint8)
    srcb[: len(data)] = np.frombuffer(data, np.uint8)[:src_cap]
    idxb = rng.integers(0, 256, size=max(index_cap, 1), dtype=np.uint8) if stale else np.zeros(max(index_cap, 1), np.uint8)
    idxb[: len(index)] = np.frombuffer(index, np.uint8)[:index_cap]
    d_src, d_idx = torch.as_tensor(srcb, device="cuda"), torch.as_tensor(idxb, device="cuda")
    d_buf = _device_numbers(np.full(GUARD + dst_cap + GUARD, _sentinel(dtype), dtype=dtype))
    dec = sa.AsyncDecompressor(data[:32], dtype, src_cap, index_cap, dst_cap, max_chunks)
    dec(d_src, d_idx, d_buf[GUARD:GUARD + dst_cap])
    err = None
    try:
        prog = dec.result()
        out = (prog.n_processed, prog.finished)
    except PcoError as e:
        st = sa._CAsyncStatus.from_buffer_copy(dec.status.cpu().numpy().tobytes())
        err = (e.kind, int(st.chunk) if st.chunk != (1 << 64) - 1 else None)
    back = _host_numbers(d_buf, dtype)
    g = bits_view(back)
    s = bits_view(np.array([_sentinel(dtype)], dtype=dtype))[0]
    assert (g[:GUARD] == s).all() and (g[GUARD + dst_cap:] == s).all(), "a write outside dst"
    if err is not None:
        if err[1] is None:
            assert (g[GUARD:GUARD + dst_cap] == s).all(), "a refused file wrote to dst"
        return None, err
    assert (g[GUARD + out[0]:GUARD + dst_cap] == s).all(), "a write behind n_processed"
    return back[GUARD:GUARD + out[0]], out


def _device_numbers(a):
    """A CUDA tensor of a's dtype holding a's bytes (through uint8: torch has few kernels for its unsigned types)."""
    import torch

    return torch.as_tensor(np.ascontiguousarray(a).view(np.uint8), device="cuda").view(_tdtype(a.dtype))


def _host_numbers(t, dtype):
    import torch

    return t.view(torch.uint8).cpu().numpy().view(dtype)


def _check(sa, data, index, x, **caps):
    """The async decode equals decompress_ex and the input, for the file's own capacities and for 4x spare ones with stale bytes."""
    n = x.size
    want, prog = _ex(sa, data, index, x.dtype, n)
    assert prog == (n, True)
    np.testing.assert_array_equal(bits_view(want), bits_view(x))
    got, p = _async(sa, data, index, x.dtype, **caps)
    assert p == (n, True), p
    np.testing.assert_array_equal(bits_view(got), bits_view(x))
    nc = max(_n_chunks(index), 1)
    got, p = _async(sa, data, index, x.dtype, src_cap=4 * len(data) + 5, index_cap=4 * len(index) + 3, dst_cap=4 * n + 7, max_chunks=4 * nc, stale=7)
    assert p == (n, True), p
    np.testing.assert_array_equal(bits_view(got), bits_view(x))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("order", [0, 1, 2, 7])
def test_every_type_and_order(sa, dtype, order):
    n = 3 * (1 << 14) + 777
    x = _walk(dtype, n, seed=order + 31)
    data, index = sa.simple_compress_with_index(x, _cfg(order))
    _check(sa, data, index, x)


@pytest.mark.parametrize("mode,dtype", [("float_mult", np.float32), ("float_mult", np.float64), ("int_mult", np.uint32), ("int_mult", np.int64),
                                        ("float_quant", np.float32), ("float_quant", np.float64)])
@pytest.mark.parametrize("order", [0, 1])
def test_two_var_modes_take_the_general_pair(sa, mode, dtype, order):
    n = 2 * (1 << 14) + 301
    rng = np.random.default_rng(order)
    if mode == "float_mult":
        x = (np.round(np.cumsum(rng.normal(size=n)) * 100) * 0.01).astype(dtype)
    elif mode == "float_quant":
        x = np.cumsum(rng.normal(size=n)).astype(dtype)
    else:
        x = (_walk(dtype, n, seed=order).astype(np.uint64) // 8 * 8 + 3).astype(dtype)
    data, index = sa.simple_compress_with_index(x, _cfg(order, mode=mode))
    _check(sa, data, index, x)


@pytest.mark.parametrize("dtype", [np.uint64, np.uint32, np.int16])
def test_wide_offsets_at_order_0(sa, dtype):
    """One bin of wide offsets: the fused kernel hands every chunk to the general pair."""
    rng = np.random.default_rng(3)
    bits = np.dtype(dtype).itemsize * 8
    x = rng.integers(0, 1 << min(bits, 63), size=2 * (1 << 14) + 9, dtype=np.uint64).astype(dtype)
    data, index = sa.simple_compress_with_index(x, _cfg(0))
    _check(sa, data, index, x)


@pytest.mark.parametrize("level", [9, 12])
def test_high_levels_take_the_catch_all_decoder(sa, oracle, level):
    rng = np.random.default_rng(level)
    n = 3 * (1 << 16) + 5
    x = rng.lognormal(10, 2, size=n).astype(np.uint64)
    data, index = sa.simple_compress_with_index(x, _cfg(0, page=1 << 16, level=level))
    if level == 12:
        info = oracle.inspect(data, np.uint64)["chunks"][0]
        assert max(len(v["bins"]) for v in info["vars"]) > 256 or max(v["ans_size_log"] for v in info["vars"]) > 10
    _check(sa, data, index, x)


def test_f16_float_mult_from_the_oracle(sa, oracle):
    n = 4000
    x = (np.round(np.random.default_rng(4).normal(size=n) * 40) * 0.25).astype(np.float16)
    cfg = oracle.make_config(mode=oracle.MODE_FLOAT_MULT, float_mult_base=0.25, delta=oracle.DELTA_CONSECUTIVE, delta_order=1, max_page_n=1500)
    data = oracle.simple_compress(x, cfg)
    index = sa.build_index(data, np.float16)
    _check(sa, data, index, x)
    np.testing.assert_array_equal(bits_view(oracle.simple_decompress(data, np.float16)), bits_view(x))


def _splice(sa, parts):
    """One standalone file whose chunks are the chunks of several files of one flavour, in order."""
    first = sa._header(parts[0])[3]
    body = b"".join(p[sa._header(p)[3]:-1] for p in parts)
    return parts[0][:first] + body + b"\0"


def test_one_file_takes_all_three_routes(sa, oracle):
    """Chunks for the fused kernel, the general pair and the catch-all decoder in one file."""
    rng = np.random.default_rng(5)
    a = _walk(np.uint64, (1 << 14) + 3, seed=1)
    b = (_walk(np.uint64, (1 << 14) + 100, seed=2) // 8 * 8 + 3).astype(np.uint64)
    c = rng.lognormal(10, 2, size=(1 << 16) + 1).astype(np.uint64)
    parts = [sa.simple_compress(a, _cfg(1, page=1 << 17)), sa.simple_compress(b, _cfg(0, page=1 << 17, mode="int_mult")),
             sa.simple_compress(c, _cfg(0, page=1 << 17, level=12)), sa.simple_compress(a[:1000], _cfg(0))]
    data = _splice(sa, parts)
    x = np.concatenate([a, b, c, a[:1000]])
    np.testing.assert_array_equal(oracle.simple_decompress(data, np.uint64), x)
    chunks = oracle.inspect(data, np.uint64)["chunks"]
    assert len(chunks) == 4 and len(chunks[1]["vars"]) == 2
    assert max(len(v["bins"]) for v in chunks[2]["vars"]) > 256 or max(v["ans_size_log"] for v in chunks[2]["vars"]) > 10
    index = sa.build_index(data, np.uint64)
    _check(sa, data, index, x)


@pytest.mark.parametrize("n", [0, 1, 256, 1024 * 256])
def test_chunk_counts(sa, n):
    x = _walk(np.uint32, n, seed=n)
    data, index = sa.simple_compress_with_index(x, _cfg(1, page=256))
    assert _n_chunks(index) == -(-n // 256)
    _check(sa, data, index, x)


@pytest.mark.parametrize("size", [1, 255, 256, 257, 1 << 18, (1 << 20) + 1])
def test_chunk_sizes(sa, size):
    x = _walk(np.int64, 2 * size + 5, seed=size)
    data, index = sa.simple_compress_with_index(x, _cfg(1, exact=[size, 5, size]))
    assert _n_chunks(index) == 3
    _check(sa, data, index, x)


@pytest.mark.parametrize("uniform", [False, True])
@pytest.mark.parametrize("dtype", [np.uint16, np.float32])
def test_both_header_flavours(sa, uniform, dtype):
    x = _walk(dtype, 2 * (1 << 14) + 17, seed=8)
    data, index = sa.simple_compress_with_index(x, _cfg(1), uniform_type=uniform)
    _check(sa, data, index, x)
    # a plan of the other flavour refuses the file before writing anything
    other, _ = sa.simple_compress_with_index(x[:10], _cfg(1), uniform_type=not uniform)
    dec = sa.AsyncDecompressor(other[:32], dtype, len(data), len(index), x.size, 4)
    got, err = _async_with(sa, dec, data, index, x.dtype, x.size)
    assert got is None and err[0] == "InvalidArgument" and "differs from the plan" in err[2] and not err[3], err


def _async_with(sa, dec, data, index, dtype, dst_cap):
    import torch

    from pcodec_b200 import PcoError

    d_src = torch.as_tensor(np.frombuffer(data, np.uint8).copy(), device="cuda")
    d_idx = torch.as_tensor(np.frombuffer(index, np.uint8).copy(), device="cuda")
    dst = _device_numbers(np.zeros(max(dst_cap, 1), dtype=dtype))
    dec(d_src, d_idx, dst)
    try:
        prog = dec.result()
    except PcoError as e:
        return None, (e.kind, None, e.message, bool(dst.view(torch.uint8).any()))
    return _host_numbers(dst, dtype)[: prog.n_processed], (prog.n_processed, prog.finished)


@pytest.mark.parametrize("level", [8, 12])
def test_short_destinations(sa, level):
    n = 3 * (1 << 14) + 5
    rng = np.random.default_rng(level)
    x = rng.lognormal(10, 2, size=n).astype(np.uint64) if level == 12 else _walk(np.uint64, n, seed=4)
    data, index = sa.simple_compress_with_index(x, _cfg(1 if level == 8 else 0, level=level))
    for cap in (0, 1, 255, 256, (1 << 14) - 1, 1 << 14, (1 << 14) + 1, n - 1, n, n + 1):
        want, wp = _ex(sa, data, index, np.uint64, cap)
        got, p = _async(sa, data, index, np.uint64, dst_cap=cap)
        assert p == wp, (cap, p, wp)
        np.testing.assert_array_equal(got, want)
        got, p = _async(sa, data, index, np.uint64, src_cap=len(data) + 1000, dst_cap=cap, max_chunks=9, stale=3)
        assert p == wp, (cap, p, wp)
        np.testing.assert_array_equal(got, want)


def test_more_chunks_than_max_chunks(sa):
    x = _walk(np.uint32, 5 * 1000, seed=6)
    data, index = sa.simple_compress_with_index(x, _cfg(1, page=1000))
    assert _n_chunks(index) == 5
    got, err = _async(sa, data, index, np.uint32, max_chunks=4)  # _async checks that dst stays untouched
    assert got is None and err == ("InvalidArgument", None), err
    got, p = _async(sa, data, index, np.uint32, max_chunks=5)
    assert p == (x.size, True)


def test_errors_match_decompress_ex(sa):
    n = 4 * (1 << 14)
    x = _walk(np.uint64, n, seed=10)
    data, index = sa.simple_compress_with_index(x, _cfg(1))
    other_x = _walk(np.uint64, n + 999, seed=11)
    _, other_index = sa.simple_compress_with_index(other_x, _cfg(1))
    # an index from another file
    _, want = _ex(sa, data, other_index, np.uint64, n + 999)
    got, err = _async(sa, data, other_index, np.uint64, dst_cap=n + 999, max_chunks=8)
    assert got is None and err[0] == want[0] == "InvalidArgument", (err, want)
    # one damaged chunk: the type byte of chunk 2 - on the fused route and on the catch-all route
    for level in (8, 12):
        y = x if level == 8 else np.random.default_rng(1).lognormal(10, 2, size=n).astype(np.uint64)
        d, ix = sa.simple_compress_with_index(y, _cfg(1 if level == 8 else 0, level=level))
        table_off = int(np.frombuffer(ix[32:40], np.uint64)[0])
        c2 = int(np.frombuffer(ix[table_off + 64:table_off + 72], np.uint64)[0])
        bad = bytearray(d)
        bad[c2] = 5  # f32
        _, want = _ex(sa, bytes(bad), ix, np.uint64, n)
        got, err = _async(sa, bytes(bad), ix, np.uint64)
        assert got is None and err == want == ("Corruption", 2), (level, err, want)


def test_bit_flips_fail_cleanly(sa):
    """30 seeded bit flips, half of them in a chunk's first bytes (its meta): every call succeeds or fails with a kind of damaged data.  A
    flip anywhere gives decompress_ex's outcome - the same kind and chunk, or the same numbers (with a side index, a flip inside a batch's
    tANS section changes numbers without failing a check).  A flip in a meta can send the chunk to the catch-all decoder, which
    decompress_ex runs over the whole file from its start and this call over that chunk alone, so there only the clean failure is checked."""
    n = 3 * (1 << 14)
    x = _walk(np.uint64, n, seed=12)
    data, index = sa.simple_compress_with_index(x, _cfg(1))
    first = sa._header(data)[3]
    table_off = int(np.frombuffer(index[32:40], np.uint64)[0])
    starts = [int(np.frombuffer(index[table_off + 32 * c:table_off + 32 * c + 8], np.uint64)[0]) for c in range(_n_chunks(index))]
    rng = np.random.default_rng(9)
    for i in range(30):
        bad = bytearray(data)
        pos = starts[int(rng.integers(0, len(starts)))] + int(rng.integers(0, 48)) if i % 2 else int(rng.integers(first, len(bad) - 1))
        bad[pos] ^= 1 << int(rng.integers(0, 8))
        got, p = _async(sa, bytes(bad), index, np.uint64)  # checks the guard zones
        if got is None:
            assert p[0] in ("InsufficientData", "Corruption", "InvalidArgument", "Unsupported"), p
        if i % 2 == 0:
            want, wp = _ex(sa, bytes(bad), index, np.uint64, n)
            assert p == wp, (pos, p, wp)
            if want is not None:
                np.testing.assert_array_equal(got, want)
    _check(sa, data, index, x)  # the library still works


def _graph_files(sa):
    """Three u64 files of different lengths, chunk counts and decode routes: fused, general pair, catch-all."""
    rng = np.random.default_rng(13)
    xs = [_walk(np.uint64, 5 * (1 << 14) + 3, seed=13), (_walk(np.uint64, 2 * (1 << 14) + 1, seed=14) // 8 * 8 + 3).astype(np.uint64),
          rng.lognormal(10, 2, size=(1 << 16) + 5).astype(np.uint64)]
    cfgs = [_cfg(1), _cfg(0, mode="int_mult"), _cfg(0, page=1 << 16, level=12)]
    return [(x,) + sa.simple_compress_with_index(x, c) for x, c in zip(xs, cfgs)]


def test_cuda_graph_replays_over_different_files(sa):
    import torch

    from pcodec_b200 import _lib

    files = _graph_files(sa)
    src_cap = max(len(d) for _, d, _ in files) + 100
    index_cap = max(len(i) for _, _, i in files) + 100
    dst_cap = max(x.size for x, _, _ in files) + 100
    d_src = torch.zeros(src_cap, dtype=torch.uint8, device="cuda")
    d_idx = torch.zeros(index_cap, dtype=torch.uint8, device="cuda")
    d_dst = _device_numbers(np.zeros(dst_cap, dtype=np.uint64))
    dec = sa.AsyncDecompressor(files[0][1][:32], np.uint64, src_cap, index_cap, dst_cap, 64)

    def load(k):
        _, d, ix = files[k]
        d_src[: len(d)].copy_(torch.as_tensor(np.frombuffer(d, np.uint8).copy(), device="cuda"))
        d_idx[: len(ix)].copy_(torch.as_tensor(np.frombuffer(ix, np.uint8).copy(), device="cuda"))

    def check(k):
        x = files[k][0]
        prog = dec.result()
        assert (prog.n_processed, prog.finished) == (x.size, True), (k, prog)
        np.testing.assert_array_equal(_host_numbers(d_dst, np.uint64)[: x.size], x)

    load(0)
    L = _lib.lib()
    g = torch.cuda.CUDAGraph()
    L.pco_b200_profile_enable(1)  # a call inside a capture records no spans
    try:
        with torch.cuda.graph(g):  # fails if the call synchronises or allocates
            dec(d_src, d_idx, d_dst)
    finally:
        L.pco_b200_profile_enable(0)
    for k in (0, 1, 2, 1, 0):
        load(k)
        g.replay()
        check(k)
    # the library's per-thread scratch is released and then regrown by a larger call: the replay does not depend on it
    L.pco_b200_thread_release()
    big = _walk(np.uint64, 4 * dst_cap, seed=15)
    bdata, bindex = sa.simple_compress_with_index(big, _cfg(1))
    want, prog = _ex(sa, bdata, bindex, np.uint64, big.size)
    assert prog == (big.size, True)
    for k in (2, 0):
        load(k)
        g.replay()
        check(k)


def test_two_streams_two_workspaces(sa):
    import torch

    files = _graph_files(sa)[:2]
    decs, bufs = [], []
    for x, d, ix in files:
        decs.append(sa.AsyncDecompressor(d[:32], np.uint64, len(d), len(ix), x.size, 8))
        bufs.append((torch.as_tensor(np.frombuffer(d, np.uint8).copy(), device="cuda"), torch.as_tensor(np.frombuffer(ix, np.uint8).copy(), device="cuda"),
                     _device_numbers(np.zeros(x.size, dtype=np.uint64))))
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for dec, (s, i, o), st in zip(decs, bufs, streams):
        with torch.cuda.stream(st):
            dec(s, i, o)
    for dec, (x, _, _), (_, _, o), st in zip(decs, files, bufs, streams):
        with torch.cuda.stream(st):
            prog = dec.result()
        assert (prog.n_processed, prog.finished) == (x.size, True)
        np.testing.assert_array_equal(_host_numbers(o, np.uint64), x)


def test_profiled_call_records_its_kernels(sa):
    import torch

    from pcodec_b200 import _lib

    x = _walk(np.uint32, 3 * (1 << 14), seed=16)
    data, index = sa.simple_compress_with_index(x, _cfg(1))
    dec = sa.AsyncDecompressor(data[:32], np.uint32, len(data), len(index), x.size, 4)
    L = _lib.lib()
    L.pco_b200_profile_enable(1)
    try:
        got, p = _async_with(sa, dec, data, index, np.uint32, x.size)
        torch.cuda.synchronize()
        buf = C.create_string_buffer(4096)
        n = L.pco_b200_profile_last(buf, C.c_size_t(len(buf)))
    finally:
        L.pco_b200_profile_enable(0)
    assert p == (x.size, True)
    np.testing.assert_array_equal(got, x)
    names = [kv.split("=")[0] for kv in buf.value.decode().split(";") if kv]
    # one span per launch; "decode_kernel" covers both instantiations
    assert n == 6 and names == ["async_check_kernel", "fused_narrow_kernel", "symwalk_kernel", "decode_kernel", "cold_chunks_kernel",
                                "async_finish_kernel"], names
