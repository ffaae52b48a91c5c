"""Asynchronous ranges of indexed standalone files (pco_b200_decompress_ranges_async, standalone.AsyncRangeDecompressor): every output
equals pco_b200_decompress_ranges on the same file, index and ranges, and the input, bit for bit - with sentinel guard zones around dst,
inside a CUDA graph replayed over different ranges, counts and files, and on concurrent streams.  Refusals give the sync call's kind and
leave dst untouched."""
import ctypes as C
import re
import struct

import numpy as np
import pytest

from tests.golden_generators import GENERATORS, bits_view, load_assets

pytestmark = pytest.mark.gpu

DTYPES = [np.uint8, np.int8, np.uint16, np.int16, np.float16, np.uint32, np.int32, np.float32, np.uint64, np.int64, np.float64]
INDEXED_ASSETS = ["v0_0_0_classic", "v0_0_0_delta_float_mult", "v0_1_0_delta_int_mult", "v0_1_1_standalone_versioned", "v0_3_0_f16",
                  "v0_3_0_float_quant", "v0_4_5_uniform_type", "v0_4_8_minor_version", "v1_0_0_u8", "v1_0_0_i8"]
GUARD = 4096
NONE = (1 << 64) - 1
KERNELS = ["async_check_kernel", "ar_chunks_kernel", "ar_count_kernel", "ar_scan_kernel", "ar_mark_kernel", "ar_window_kernel", "ar_gate_kernel",
           "ar_tasks_kernel", "fused_narrow_kernel", "symwalk_kernel", "decode_kernel", "ar_cold_kernel", "ar_gather_kernel", "ar_finish_kernel"]


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


def _cfg(order=0, page=1 << 14, level=8, mode="classic", base=0.01, ibase=8, k=13):
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec

    ms = {"classic": ModeSpec.classic(), "float_mult": ModeSpec.try_float_mult(base), "int_mult": ModeSpec.try_int_mult(ibase),
          "float_quant": ModeSpec.try_float_quant(k)}[mode]
    ds = DeltaSpec.try_consecutive(order) if order else DeltaSpec.no_op()
    return ChunkConfig(compression_level=level, mode_spec=ms, delta_spec=ds, paging_spec=PagingSpec.equal_pages_up_to(page), enable_8_bit=True)


def _chunk_table(index):
    n_chunks, chunks_offset = struct.unpack_from("<Q", index, 8)[0], struct.unpack_from("<Q", index, 32)[0]
    return [struct.unpack_from("<QIIQQ", index, chunks_offset + 32 * c) for c in range(n_chunks)]


def window_needed(index, pairs):
    """The documented rule: over the chunks the ranges touch, the chunk-relative end of the last number wanted, rounded up to 256."""
    hi = {}
    for rec in _chunk_table(index):
        n, off = int(rec[1]), int(rec[4])
        for s, c in pairs:
            a, b = max(s, off), min(s + c, off + n)
            if c and a < b:
                hi[off] = max(hi.get(off, 0), b - off)
    return sum((h + 255) // 256 * 256 for h in hi.values())


def _edges(index, n):
    out = [(0, 1), (3, 5), (250, 12), (255, 2), (n - 1, 1), (0, n)]
    for c in _chunk_table(index)[1:]:
        e = int(c[4])
        out += [(e - 1, 1), (e, 1), (e + 1, 1), (e - 3, 7), (max(e - 300, 0), 600)]
    return [(s, min(cnt, n - s)) for s, cnt in out if s < n]


def _random(n, m, seed, max_len=5000):
    rng = np.random.default_rng(seed)
    s = rng.integers(0, n, m)
    return [(int(a), int(min(b, n - a))) for a, b in zip(s, rng.integers(0, max_len, m))]


def _expect(x, pairs):
    parts = [x[s:s + c] for s, c in pairs]
    return np.concatenate(parts) if parts else x[:0]


def _tdtype(dtype):
    from pcodec_b200.wrapped import _torch_dtypes

    return _torch_dtypes()[np.dtype(dtype)]


def _sentinel(dtype):
    return np.frombuffer(b"\xa5" * 8, np.uint8)[: np.dtype(dtype).itemsize].view(dtype)[0]


def _device_numbers(a):
    import torch

    return torch.as_tensor(np.ascontiguousarray(a).view(np.uint8), device="cuda").view(_tdtype(a.dtype))


def _host_numbers(t, dtype):
    import torch

    return t.view(torch.uint8).cpu().numpy().view(dtype)


def _sync(sa, data, index, dtype, pairs):
    """pco_b200_decompress_ranges: (numbers, None) or (None, (kind, range named in the message))."""
    from pcodec_b200 import PcoError

    try:
        return sa.decompress_ranges(data, dtype, index, np.array(pairs, dtype=np.uint64).reshape(-1, 2)), None
    except PcoError as e:
        m = re.match(r"range (\d+): ", e.message)
        return None, (e.kind, int(m.group(1)) if m else None)


def _ranges_tensor(pairs, max_ranges):
    import torch

    r = np.zeros((max_ranges, 2), np.uint64)
    if pairs:
        r[: len(pairs)] = np.array(pairs, np.uint64).reshape(-1, 2)
    return torch.as_tensor(r.view(np.int64), device="cuda"), torch.tensor([len(pairs)], dtype=torch.int64, device="cuda")


class Bufs:
    """Device buffers of one decompressor, with sentinel guard zones around dst."""

    def __init__(self, sa, head, dtype, src_cap, index_cap, max_chunks, max_ranges, dst_cap, window_cap, stream=None):
        import torch

        self.dtype, self.dst_cap = np.dtype(dtype), dst_cap
        self.dec = sa.AsyncRangeDecompressor(head, dtype, src_cap, index_cap, max_chunks, max_ranges, dst_cap, window_cap)
        self.src = torch.zeros(max(src_cap, 1), dtype=torch.uint8, device="cuda")
        self.index = torch.zeros(max(index_cap, 1), dtype=torch.uint8, device="cuda")
        self.ranges, self.n = _ranges_tensor([], max_ranges)
        self.buf = _device_numbers(np.full(GUARD + dst_cap + GUARD, _sentinel(dtype), dtype=dtype))

    def load(self, data, index, pairs):
        import torch

        self.src.zero_()
        self.index.zero_()
        self.src[: len(data)] = torch.as_tensor(np.frombuffer(data, np.uint8).copy())
        self.index[: len(index)] = torch.as_tensor(np.frombuffer(index, np.uint8).copy())
        r, n = _ranges_tensor(pairs, self.ranges.shape[0])
        self.ranges.copy_(r)
        self.n.copy_(n)
        self.buf.copy_(_device_numbers(np.full(GUARD + self.dst_cap + GUARD, _sentinel(self.dtype), dtype=self.dtype)))

    def call(self):
        self.dec(self.src, self.index, self.ranges, self.n, self.buf[GUARD:GUARD + self.dst_cap])

    def outcome(self, total_hint=None):
        """(numbers or None, (kind, range) or None, status record); asserts the guard zones and, for refusals, an untouched dst."""
        from pcodec_b200 import PcoError

        st = self.dec.status_record()
        err = None
        nw = 0
        try:
            nw = self.dec.result()
        except PcoError as e:
            err = (e.kind, int(st.range) if st.range != NONE else None)
        back = _host_numbers(self.buf, self.dtype)
        g = bits_view(back)
        s = bits_view(np.array([_sentinel(self.dtype)], dtype=self.dtype))[0]
        assert (g[:GUARD] == s).all() and (g[GUARD + self.dst_cap:] == s).all(), "a write outside dst"
        if err is not None:
            limit = 0 if st.device_status >= 0x100 else (total_hint or 0)
            assert (g[GUARD + limit:GUARD + self.dst_cap] == s).all(), "a refused call wrote to dst"
            return None, err, st
        assert (g[GUARD + nw:GUARD + self.dst_cap] == s).all(), "a write behind n_written"
        return back[GUARD:GUARD + nw], None, st


def _run(sa, data, index, dtype, pairs, max_chunks=None, max_ranges=None, dst_cap=None, window_cap=None, src_cap=None, index_cap=None):
    total = sum(c for _, c in pairs)
    nc = max(len(_chunk_table(index)), 1)
    b = Bufs(sa, data[:32], dtype, src_cap or len(data), index_cap or len(index), max_chunks or nc, max_ranges or max(len(pairs), 1),
             total if dst_cap is None else dst_cap, window_needed(index, pairs) if window_cap is None else window_cap)
    b.load(data, index, pairs)
    b.call()
    return b.outcome(total)


def _check(sa, data, index, x, pairs, spare=True):
    """The async call equals decompress_ranges and the input, for exact capacities and for spare ones."""
    want = bits_view(_expect(x, pairs))
    got_sync, err = _sync(sa, data, index, x.dtype, pairs)
    assert err is None, err
    np.testing.assert_array_equal(bits_view(got_sync), want)
    got, err, st = _run(sa, data, index, x.dtype, pairs)
    assert err is None, err
    np.testing.assert_array_equal(bits_view(got), want)
    assert st.window_needed == window_needed(index, pairs)
    if spare:
        nc = len(_chunk_table(index))
        got, err, _ = _run(sa, data, index, x.dtype, pairs, max_chunks=2 * nc + 3, max_ranges=len(pairs) + 300, dst_cap=len(want) + 999,
                           window_cap=window_needed(index, pairs) + 777, src_cap=len(data) + 100, index_cap=len(index) + 64)
        assert err is None, err
        np.testing.assert_array_equal(bits_view(got), want)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("order", [0, 1, 2, 7])
def test_every_type_and_order(sa, dtype, order):
    n = 3 * (1 << 14) + 777
    x = _walk(dtype, n, seed=order + 11)
    data, index = sa.simple_compress_with_index(x, _cfg(order))
    pairs = _edges(index, n) + _random(n, 40, seed=order)
    _check(sa, data, index, x, pairs, spare=(order == 1))
    _check(sa, data, index, x, pairs[::-1], spare=False)


@pytest.mark.parametrize("mode,dtype", [("float_mult", np.float32), ("float_mult", np.float64), ("int_mult", np.uint32), ("int_mult", np.int64),
                                        ("float_quant", np.float32), ("float_quant", np.float64)])
def test_two_var_modes_take_the_general_pair(sa, mode, dtype):
    n = 2 * (1 << 14) + 301
    rng = np.random.default_rng(3)
    if mode == "float_mult":
        x = (np.round(np.cumsum(rng.normal(size=n)) * 100) * 0.01).astype(dtype)
    elif mode == "float_quant":
        x = np.cumsum(rng.normal(size=n)).astype(dtype)
    else:
        x = (_walk(dtype, n, seed=1).astype(np.uint64) // 8 * 8 + 3).astype(dtype)
    data, index = sa.simple_compress_with_index(x, _cfg(1, mode=mode))
    _check(sa, data, index, x, _edges(index, n) + _random(n, 30, seed=5))


def test_level_12_and_f16_float_mult_take_the_catch_all_decoder(sa, oracle):
    rng = np.random.default_rng(12)
    n = 3 * (1 << 16) + 5
    x = rng.lognormal(10, 2, size=n).astype(np.uint64)
    data, index = sa.simple_compress_with_index(x, _cfg(0, page=1 << 16, level=12))
    _check(sa, data, index, x, _edges(index, n) + [(100, 3), (101, 1), (20000, 5)])
    _check(sa, data, index, x, [((1 << 16) + 7, 10)], spare=False)  # a lone piece on the catch-all decoder goes through its slot
    n = 4000
    x = (np.round(np.random.default_rng(4).normal(size=n) * 40) * 0.25).astype(np.float16)
    cfg = oracle.make_config(mode=oracle.MODE_FLOAT_MULT, float_mult_base=0.25, delta=oracle.DELTA_CONSECUTIVE, delta_order=1, max_page_n=1500)
    data = oracle.simple_compress(x, cfg)
    index = sa.build_index(data, np.float16)
    _check(sa, data, index, x, [(5, 10), (1490, 300), (2000, 3), (n - 1, 1)])


def test_one_file_whose_ranges_take_all_three_routes(sa):
    n = 4 * (1 << 14)
    x = _walk(np.uint32, n, seed=31)
    data, index = sa.simple_compress_with_index(x, _cfg(1))
    c = 1 << 14
    pairs = [(5, 10),                       # chunk 0: one piece, straight into dst
             (c + 3, 100), (c + 50, 7000),  # chunk 1: two pieces, staged
             (2 * c - 1, 2),                # chunks 1 and 2
             (3 * c + 9, 1), (3 * c + 9, 1)]  # chunk 3: a repeated lookup
    _check(sa, data, index, x, pairs)


@pytest.mark.parametrize("order", [0, 1])
def test_chunks_of_2_20(sa, order):
    n = (1 << 20) + (1 << 18) + 3
    x = _walk(np.uint32, n, seed=20)
    data, index = sa.simple_compress_with_index(x, _cfg(order, page=1 << 20))
    c = 1 << 20
    pairs = [(c - 1, 1), (c, 2), (c - 100000, 200000), (c // 2 + 17, 1), (12345, 1 << 20), (n - 1, 1)] + _random(n, 50, seed=20, max_len=1 << 16)
    _check(sa, data, index, x, pairs, spare=False)


@pytest.mark.parametrize("uniform", [False, True])
def test_both_header_flavours(sa, uniform):
    n = 2 * (1 << 14) + 999
    x = _walk(np.float64, n, seed=9)
    data, index = sa.simple_compress_with_index(x, _cfg(1), uniform_type=uniform)
    _check(sa, data, index, x, _edges(index, n) + _random(n, 20, seed=1))
    _check(sa, data, sa.build_index(data, np.float64), x, _random(n, 20, seed=2), spare=False)


@pytest.mark.parametrize("name", INDEXED_ASSETS)
def test_golden_assets(sa, name):
    x = GENERATORS[name]()
    data = load_assets()[name]
    index = sa.build_index(data, x.dtype)
    n = x.size
    if n == 0:
        got, err, st = _run(sa, data, index, x.dtype, [(0, 0), (0, 0)], dst_cap=0)
        assert err is None and got.size == 0 and st.n_written == 0
        return
    pairs = [(0, n), (n - 1, 1), (n // 2, n - n // 2), (1, max(n - 2, 0))] + _random(n, 10, seed=4, max_len=max(n // 3, 1))
    _check(sa, data, index, x, [(s, c) for s, c in pairs if s < n], spare=False)


def test_range_shapes(sa):
    n = 8 * (1 << 12) + 5
    x = _walk(np.int64, n, seed=41)
    data, index = sa.simple_compress_with_index(x, _cfg(1, page=1 << 12))
    rng = np.random.default_rng(41)
    _check(sa, data, index, x, [(int(s), 1) for s in rng.integers(0, n, 300)])  # point lookups
    _check(sa, data, index, x, [(100, 50), (120, 50), (100, 50), (n - 10, 10), (0, 3), (110, 1)])  # overlapping, repeated, unordered
    _check(sa, data, index, x, [(5, 0), (7, 3), (n, 0), (0, 0), (9, 2)])  # count 0, also at the end
    _check(sa, data, index, x, [(17, n - 40)])  # one range across every chunk
    _check(sa, data, index, x, [(0, n)])  # the whole file
    got, err, st = _run(sa, data, index, np.int64, [], max_ranges=4, dst_cap=10, window_cap=0)  # n_ranges = 0
    assert err is None and got.size == 0 and st.n_written == 0


def test_one_range_across_many_chunks(sa):
    n = 1500 * 256 + 7
    x = _walk(np.uint16, n, seed=5)
    data, index = sa.simple_compress_with_index(x, _cfg(0, page=256))
    assert len(_chunk_table(index)) > 1000
    _check(sa, data, index, x, [(100, n - 200), (3, 1)], spare=False)


def test_graph_replays_with_different_ranges_counts_and_files(sa):
    import torch

    n = 6 * (1 << 14)
    xs = [_walk(np.uint32, n, seed=s) for s in (1, 2)]
    files = [sa.simple_compress_with_index(x, _cfg(o)) for x, o in zip(xs, (1, 0))]
    max_ranges, dst_cap, window_cap = 64, 1 << 16, 1 << 18
    b = Bufs(sa, files[0][0][:32], np.uint32, max(len(f[0]) for f in files) + 64, max(len(f[1]) for f in files) + 64, 16, max_ranges,
             dst_cap, window_cap)
    rng = np.random.default_rng(0)
    plans = [(0, [(int(s), 1) for s in rng.integers(0, n, 64)]), (0, _random(n, 10, seed=3, max_len=3000)), (1, [(7, 40000)]),
             (1, []), (0, _random(n, 33, seed=4, max_len=1000))]
    b.load(files[0][0], files[0][1], plans[0][1])
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        b.call()  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        b.call()
    for f, pairs in plans:
        data, index = files[f]
        b.load(data, index, pairs)
        g.replay()
        torch.cuda.synchronize()
        got, err, st = b.outcome()
        assert err is None, err
        np.testing.assert_array_equal(bits_view(got), bits_view(_expect(xs[f], pairs)))
        assert st.window_needed == window_needed(index, pairs)


def _refusal(sa, data, index, dtype, pairs, **kw):
    got, err, st = _run(sa, data, index, dtype, pairs, **kw)
    assert got is None
    return err, st


def test_refusals(sa):
    n = 3 * (1 << 14)
    x = _walk(np.uint32, n, seed=8)
    data, index = sa.simple_compress_with_index(x, _cfg(1))
    u = np.uint32
    # too many ranges: *n_ranges above max_ranges
    b = Bufs(sa, data[:32], u, len(data), len(index), 3, 2, 100, 1 << 16)
    b.load(data, index, [(0, 1), (1, 1)])
    b.n.fill_(3)
    b.call()
    _, err, st = b.outcome()
    assert err == ("InvalidArgument", None) and st.device_status == 0x109
    # a range past the file, and the sync call's kind and range
    for pairs in ([(0, 5), (n - 3, 4)], [(0, 5), (3, 4), (n, 1)], [(0, 5), (n + 5, 0)]):
        err, _ = _refusal(sa, data, index, u, pairs, dst_cap=100, window_cap=1 << 16)
        assert err == _sync(sa, data, index, u, pairs)[1] and err[1] == len(pairs) - 1, err
    # start + count overflowing 64 bits
    for pairs in ([(0, n), (0, (1 << 64) - 1)], [(3, 1), ((1 << 64) - 5, 10)], [(3, 1), (5, 1), (1, (1 << 64) - 1)]):
        err, st = _refusal(sa, data, index, u, pairs, dst_cap=n + 100, window_cap=1 << 16)
        assert err == _sync(sa, data, index, u, pairs)[1] and err[1] == len(pairs) - 1 and st.device_status == 0x10a, err
    # total above dst_cap
    err, st = _refusal(sa, data, index, u, [(0, 5), (5, 100)], dst_cap=104)
    assert err == ("InvalidArgument", None) and st.device_status == 0x10c and st.n_written == 105
    # window_needed above window_cap, reporting the documented rule
    pairs = [(10, 3), ((1 << 14) + 5000, 1), (2 * (1 << 14) + 300, 2)]
    need = window_needed(index, pairs)
    assert need == 256 + 5120 + 512
    err, st = _refusal(sa, data, index, u, pairs, window_cap=need - 1)
    assert err == ("Io", None) and st.window_needed == need
    # a non-tiling index, a foreign index, too many chunks
    bad = bytearray(index)
    co = struct.unpack_from("<Q", bad, 32)[0]
    struct.pack_into("<Q", bad, co + 32 + 24, struct.unpack_from("<Q", bad, co + 32 + 24)[0] + 1)
    err, st = _refusal(sa, data, bytes(bad), u, [(0, 5)])
    assert err[0] == _sync(sa, data, bytes(bad), u, [(0, 5)])[1][0] == "InvalidArgument" and st.device_status == 0x107 and st.chunk == 1
    other = sa.simple_compress_with_index(_walk(np.uint32, n + 1000, seed=9), _cfg(1))
    err, st = _refusal(sa, data, other[1], u, [(0, 5)], index_cap=len(other[1]))
    assert err[0] == "InvalidArgument" and st.device_status == 0x104
    err, st = _refusal(sa, data, index, u, [(0, 5)], max_chunks=2)
    assert err[0] == "InvalidArgument" and st.device_status == 0x105


@pytest.mark.parametrize("order", [0, 1])
def test_bit_flips_in_a_touched_chunk(sa, order):
    n = 3 * (1 << 14)
    x = _walk(np.uint64, n, seed=order)
    data, index = sa.simple_compress_with_index(x, _cfg(order))
    table = _chunk_table(index)
    c1, c2 = int(table[1][0]), int(table[2][0])
    rng = np.random.default_rng(order)
    pairs = [(0, 3), (n - 2, 2), (1 << 14, 1 << 14), ((1 << 14) + 5, 1000)]
    for pos in rng.integers((c1 + c2) // 2, c2, 24):
        bad = bytearray(data)
        bad[int(pos)] ^= 1 << int(rng.integers(0, 8))
        bad = bytes(bad)
        want, werr = _sync(sa, bad, index, np.uint64, pairs)
        got, err, _ = _run(sa, bad, index, np.uint64, pairs)
        assert err == werr, (err, werr)
        if err is None:
            np.testing.assert_array_equal(bits_view(got), bits_view(want))
    _check(sa, data, index, x, pairs, spare=False)


def test_two_streams_with_two_workspaces(sa):
    import torch

    n = 5 * (1 << 14) + 3
    xs = [_walk(np.int64, n, seed=s) for s in (21, 22)]
    files = [sa.simple_compress_with_index(x, _cfg(o)) for x, o in zip(xs, (1, 0))]
    pairs = [_random(n, 100, seed=3), _random(n, 70, seed=4)]
    bufs = []
    for (data, index), p in zip(files, pairs):
        b = Bufs(sa, data[:32], np.int64, len(data), len(index), 8, 128, sum(c for _, c in p), window_needed(index, p))
        b.load(data, index, p)
        bufs.append(b)
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for _ in range(3):
        for b, s in zip(bufs, streams):
            with torch.cuda.stream(s):
                b.call()
    torch.cuda.synchronize()
    for b, x, p in zip(bufs, xs, pairs):
        got, err, _ = b.outcome()
        assert err is None, err
        np.testing.assert_array_equal(bits_view(got), bits_view(_expect(x, p)))


def test_profiled_call_records_its_kernels_in_order(sa):
    from pcodec_b200 import _lib

    n = 3 * (1 << 14)
    x = _walk(np.float32, n, seed=6)
    data, index = sa.simple_compress_with_index(x, _cfg(1))
    L = _lib.lib()
    L.pco_b200_profile_enable(1)
    try:
        got, err, _ = _run(sa, data, index, np.float32, [(3, 10), (1 << 14, 5)])
        buf = C.create_string_buffer(1 << 16)
        L.pco_b200_profile_last(buf, C.c_size_t(len(buf)))
    finally:
        L.pco_b200_profile_enable(0)
    assert err is None
    prof = buf.value.decode()
    at = [prof.find(k) for k in KERNELS]
    assert all(a >= 0 for a in at) and at == sorted(at), prof
