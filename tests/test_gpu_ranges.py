"""Ranges of an indexed standalone file on the GPU (pco_b200_decompress_ranges): every range equals the same slice of
pco_b200_decompress_ex on the whole file, of the input and of the oracle's decode, bit for bit."""
import ctypes as C

import numpy as np
import pytest

from tests.golden_generators import GENERATORS, bits_view, load_assets

pytestmark = pytest.mark.gpu

DTYPES = [np.uint8, np.int8, np.uint16, np.int16, np.float16, np.uint32, np.int32, np.float32, np.uint64, np.int64, np.float64]
# reference assets whose chunks the side index covers (the Lookback, Dict and Conv1 assets have no index: build_index declines them)
INDEXED_ASSETS = ["v0_0_0_classic", "v0_0_0_delta_float_mult", "v0_1_0_delta_int_mult", "v0_1_1_standalone_versioned", "v0_3_0_f16",
                  "v0_3_0_float_quant", "v0_4_5_uniform_type", "v0_4_8_minor_version", "v1_0_0_u8", "v1_0_0_i8"]


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


def _whole(sa, data, dtype, index):
    n = sum(int(c[1]) for c in _chunk_table(index))
    dst = np.zeros(max(n, 1), dtype=dtype)
    prog = sa.decompress_into_with_index(data, dst, index)
    assert prog.finished and prog.n_processed == n
    return dst[:n]


def _chunk_table(index):
    import struct

    n_chunks, chunks_offset = struct.unpack_from("<Q", index, 8)[0], struct.unpack_from("<Q", index, 32)[0]
    return [struct.unpack_from("<QIIQQ", index, chunks_offset + 32 * c) for c in range(n_chunks)]


def _edges(index, n):
    """Ranges inside one batch, across batch and chunk edges, the last number and the whole file."""
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


def _check(sa, data, index, x, pairs, oracle=None, whole=None, profile=False):
    """Checks the ranges against the input, the whole-file decode and the oracle; returns the ranges' values, and with profile=True
    also the kernels of the range call."""
    dtype = x.dtype
    call = lambda: sa.decompress_ranges(data, dtype, index, np.array(pairs, dtype=np.uint64).reshape(-1, 2))  # noqa: E731
    got, prof = _profile(call) if profile else (call(), None)
    want = bits_view(_expect(x, pairs))
    np.testing.assert_array_equal(bits_view(got), want)
    whole = _whole(sa, data, dtype, index) if whole is None else whole
    np.testing.assert_array_equal(bits_view(_expect(whole, pairs)), want)
    if oracle is not None:
        np.testing.assert_array_equal(bits_view(_expect(oracle.simple_decompress(data, dtype), pairs)), want)
    return (got, prof) if profile else got


def _profile(fn):
    from pcodec_b200 import _lib

    L = _lib.lib()
    L.pco_b200_profile_enable(1)
    try:
        out = fn()
        buf = C.create_string_buffer(1 << 16)
        L.pco_b200_profile_last(buf, C.c_size_t(len(buf)))
    finally:
        L.pco_b200_profile_enable(0)
    return out, buf.value.decode()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("order", [0, 1, 2, 7])
def test_every_type_and_order(sa, oracle, dtype, order):
    n = 3 * (1 << 14) + 777
    x = _walk(dtype, n, seed=order + 11)
    data, index = sa.simple_compress_with_index(x, _cfg(order))
    pairs = _edges(index, n) + _random(n, 40, seed=order)
    _check(sa, data, index, x, pairs, oracle)
    _check(sa, data, index, x, pairs[::-1])  # descending


@pytest.mark.parametrize("mode,dtype", [("float_mult", np.float32), ("float_mult", np.float64), ("int_mult", np.uint32), ("int_mult", np.int64),
                                        ("float_quant", np.float32), ("float_quant", np.float64)])
@pytest.mark.parametrize("order", [0, 1])
def test_two_var_modes_take_the_general_pair(sa, oracle, mode, dtype, order):
    n = 2 * (1 << 14) + 301
    rng = np.random.default_rng(order)
    if mode == "float_mult":
        x = (np.round(np.cumsum(rng.normal(size=n)) * 100) * 0.01).astype(dtype)
    elif mode == "float_quant":
        x = np.cumsum(rng.normal(size=n)).astype(dtype)
    else:
        x = (_walk(dtype, n, seed=order).astype(np.uint64) // 8 * 8 + 3).astype(dtype)
    data, index = sa.simple_compress_with_index(x, _cfg(order, mode=mode))
    pairs = _edges(index, n) + _random(n, 30, seed=5)
    got, prof = _check(sa, data, index, x, pairs, oracle, profile=True)
    assert "decode_kernel" in prof and "symwalk_kernel" in prof, prof


def test_level_12_chunks_take_the_catch_all_decoder(sa, oracle):
    rng = np.random.default_rng(12)
    n = 3 * (1 << 16) + 5
    x = rng.lognormal(10, 2, size=n).astype(np.uint64)
    data, index = sa.simple_compress_with_index(x, _cfg(0, page=1 << 16, level=12))
    info = oracle.inspect(data, np.uint64)["chunks"][0]
    assert max(len(v["bins"]) for v in info["vars"]) > 256 or max(v["ans_size_log"] for v in info["vars"]) > 10
    pairs = _edges(index, n) + [(100, 3), (101, 1), (20000, 5)]
    _, prof = _check(sa, data, index, x, pairs, oracle, profile=True)
    assert "cold_decode_kernel" in prof and "gather_ranges_kernel" in prof, prof
    # one range in one chunk: no staging needed by the fast kernels, but the catch-all decoder's slot is copied
    _check(sa, data, index, x, [((1 << 16) + 7, 10)])


def test_f16_float_mult_takes_the_catch_all_decoder(sa, oracle):
    n = 4000
    x = (np.round(np.random.default_rng(4).normal(size=n) * 40) * 0.25).astype(np.float16)
    cfg = oracle.make_config(mode=oracle.MODE_FLOAT_MULT, float_mult_base=0.25, delta=oracle.DELTA_CONSECUTIVE, delta_order=1, max_page_n=1500)
    data = oracle.simple_compress(x, cfg)
    index = sa.build_index(data, np.float16)
    _, prof = _check(sa, data, index, x, [(5, 10), (1490, 300), (2000, 3), (n - 1, 1)], oracle, profile=True)
    assert "cold_decode_kernel" in prof, prof


def test_many_overlapping_ranges_in_one_chunk_are_gathered(sa, oracle):
    n = 4 * (1 << 14)
    for order in (0, 1):
        x = _walk(np.uint64, n, seed=3 + order)
        data, index = sa.simple_compress_with_index(x, _cfg(order))
        rng = np.random.default_rng(order)
        starts = rng.integers(1 << 14, 2 * (1 << 14) - 100, 300)
        pairs = [(int(s), int(c)) for s, c in zip(starts, rng.integers(1, 100, 300))]
        pairs += [(int(s), 1) for s in rng.integers(0, n, 200)]  # point lookups
        pairs = sorted(pairs, reverse=True)
        _, prof = _check(sa, data, index, x, pairs, oracle, profile=True)
        assert "gather_ranges_kernel" in prof and "fused_narrow_kernel" in prof, prof


@pytest.mark.parametrize("chunk_log", [20, 24])
@pytest.mark.parametrize("order", [0, 1])
def test_large_chunks(sa, chunk_log, order):
    n = (1 << chunk_log) + (1 << 18) + 3
    x = _walk(np.uint32, n, seed=chunk_log)
    data, index = sa.simple_compress_with_index(x, _cfg(order, page=1 << chunk_log))
    c = 1 << chunk_log
    pairs = [(c - 1, 1), (c, 2), (c - 100000, 200000), (c // 2 + 17, 1), (12345, 1 << 20), (n - 1, 1)] + _random(n, 50, seed=chunk_log, max_len=1 << 16)
    _check(sa, data, index, x, pairs)


@pytest.mark.parametrize("dtype", [np.uint32, np.float64, np.int16])
@pytest.mark.parametrize("uniform", [False, True])
def test_index_from_build_index_matches_compress(sa, oracle, dtype, uniform):
    n = 2 * (1 << 14) + 999
    x = _walk(dtype, n, seed=9)
    data, index = sa.simple_compress_with_index(x, _cfg(1), uniform_type=uniform)
    walked = sa.build_index(data, dtype)
    pairs = _edges(index, n) + _random(n, 20, seed=1)
    a = _check(sa, data, index, x, pairs, oracle)
    b = _check(sa, data, walked, x, pairs)
    np.testing.assert_array_equal(bits_view(a), bits_view(b))
    # index=None builds it on the way
    np.testing.assert_array_equal(bits_view(sa.decompress_ranges(data, dtype, None, pairs)), bits_view(a))


@pytest.mark.parametrize("name", INDEXED_ASSETS)
def test_golden_assets(sa, name):
    x = GENERATORS[name]()
    data = load_assets()[name]
    index = sa.build_index(data, x.dtype)
    n = x.size
    if n == 0:
        assert sa.decompress_ranges(data, x.dtype, index, [[0, 0], [0, 0]]).size == 0
        return
    pairs = [(0, n), (n - 1, 1), (n // 2, n - n // 2), (1, max(n - 2, 0))] + _random(n, 10, seed=4, max_len=max(n // 3, 1))
    _check(sa, data, index, x, [(s, c) for s, c in pairs if s < n])


def test_device_buffers_on_a_side_stream(sa, oracle):
    import torch

    n = 5 * (1 << 14) + 3
    x = _walk(np.int64, n, seed=21)
    data, index = sa.simple_compress_with_index(x, _cfg(1))
    pairs = _edges(index, n) + _random(n, 100, seed=3)
    want = bits_view(_expect(x, pairs))
    d = torch.as_tensor(np.frombuffer(data, np.uint8).copy(), device="cuda")
    ix = torch.as_tensor(np.frombuffer(index, np.uint8).copy(), device="cuda")
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        got = sa.decompress_ranges(d, np.int64, ix, pairs)
    side.synchronize()
    assert got.is_cuda
    np.testing.assert_array_equal(got.cpu().numpy().view(np.uint64), want)
    # host index with a device file
    got = sa.decompress_ranges(d, np.int64, index, pairs)
    np.testing.assert_array_equal(got.cpu().numpy().view(np.uint64), want)


def _raw(sa, data, index, dtype, ranges, dst, dst_len=None, flags=0, stream=None):
    from pcodec_b200 import _lib

    L = _lib.lib()
    r = sa._ranges_array(ranges)
    nw = C.c_size_t(777)
    ptr = lambda a: C.c_void_p(a.data_ptr()) if hasattr(a, "data_ptr") else a.ctypes.data_as(C.c_void_p)  # noqa: E731
    size = lambda a: a.numel() if hasattr(a, "numel") else a.size  # noqa: E731
    rc = L.pco_b200_decompress_ranges(ptr(data), C.c_size_t(size(data)), C.c_ubyte(_lib.dtype_byte(dtype)), ptr(index), C.c_size_t(size(index)),
                                      r.ctypes.data_as(C.c_void_p), C.c_size_t(r.size), ptr(dst), C.c_size_t(size(dst) if dst_len is None else dst_len),
                                      C.byref(nw), C.c_uint32(flags), stream)
    return rc, nw.value, L.pco_b200_last_error_message().decode()


def test_sentinel_past_n_written_stays(sa):
    import torch

    n = 3 * (1 << 14)
    x = _walk(np.uint16, n, seed=2)
    data, index = sa.simple_compress_with_index(x, _cfg(0))
    pairs = [(7, 1), (1 << 14, 300), (100, 5), (100, 5)]
    total = sum(c for _, c in pairs)
    dbuf, ibuf = np.frombuffer(data, np.uint8).copy(), np.frombuffer(index, np.uint8).copy()
    dst = np.full(total + 1000, 0xBEEF, dtype=np.uint16)
    rc, nw, msg = _raw(sa, dbuf, ibuf, np.uint16, pairs, dst)
    assert (rc, nw) == (0, total), msg
    np.testing.assert_array_equal(dst[:total], _expect(x, pairs))
    assert (dst[total:] == 0xBEEF).all()
    # the same into device memory, at an odd element offset
    ddst = torch.full((total + 1001,), 0x5A5A, dtype=torch.int16, device="cuda")
    rc, nw, msg = _raw(sa, torch.as_tensor(dbuf, device="cuda"), torch.as_tensor(ibuf, device="cuda"), np.uint16, pairs, ddst[1:], flags=7)
    assert (rc, nw) == (0, total), msg
    back = ddst.cpu().numpy().view(np.uint16)
    np.testing.assert_array_equal(back[1:total + 1], _expect(x, pairs))
    assert back[0] == 0x5A5A and (back[total + 1:] == 0x5A5A).all()


def test_refusals(sa):
    n = 3 * (1 << 14)
    x = _walk(np.uint32, n, seed=8)
    data, index = sa.simple_compress_with_index(x, _cfg(1))
    dbuf, ibuf = np.frombuffer(data, np.uint8).copy(), np.frombuffer(index, np.uint8).copy()
    dst = np.zeros(1 << 16, dtype=np.uint32)
    rc, _, msg = _raw(sa, dbuf, ibuf, np.uint32, [(0, 5), (n - 3, 4)], dst)
    assert rc == 3 and msg.startswith("range 1: "), msg
    rc, _, msg = _raw(sa, dbuf, ibuf, np.uint32, [(0, 5), (5, 100)], dst, dst_len=104)
    assert rc == 3 and "dst holds 104 numbers, the ranges 105" in msg, msg
    rc, _, msg = _raw(sa, dbuf[:-1], ibuf, np.uint32, [(0, 5)], dst)
    assert rc == 3 and "does not belong" in msg, msg
    rc, nw, msg = _raw(sa, dbuf, ibuf, np.uint32, [(0, 5)], dst)
    assert (rc, nw) == (0, 5), msg
    # chunk records that do not tile the numbers
    bad = ibuf.copy()
    co = int(np.frombuffer(bad[32:40].tobytes(), np.uint64)[0])
    out1 = bad[co + 32 + 24:co + 32 + 32].view(np.uint64)
    out1[0] += 1
    rc, _, msg = _raw(sa, dbuf, bad, np.uint32, [(0, 5)], dst)
    assert rc == 3 and "side index" in msg, msg
    # the same refusals with every buffer on the device
    import torch

    dd, di = torch.as_tensor(dbuf, device="cuda"), torch.as_tensor(ibuf, device="cuda")
    ddst = torch.zeros(1 << 16, dtype=torch.int32, device="cuda")
    rc, _, msg = _raw(sa, dd, di, np.uint32, [(0, 5), (3, 4), (n, 1)], ddst, flags=7)
    assert rc == 3 and msg.startswith("range 2: "), msg
    rc, _, msg = _raw(sa, dd, torch.as_tensor(bad, device="cuda"), np.uint32, [(0, 5)], ddst, flags=7)
    assert rc == 3 and "side index" in msg, msg


@pytest.mark.parametrize("order", [0, 1])
def test_bit_flips_in_a_touched_chunk(sa, order):
    from pcodec_b200 import PcoError

    n = 3 * (1 << 14)
    x = _walk(np.uint64, n, seed=order)
    data, index = sa.simple_compress_with_index(x, _cfg(order))
    table = _chunk_table(index)
    c1, c2 = int(table[1][0]), int(table[2][0])
    rng = np.random.default_rng(order)
    pairs = [(0, 3), (n - 2, 2), (1 << 14, 1 << 14), ((1 << 14) + 5, 1000)]  # chunk 1 whole: its end-of-page checks run
    kinds = set()
    for pos in rng.integers((c1 + c2) // 2, c2, 40):  # in the second half of chunk 1's bytes
        bad = bytearray(data)
        bad[int(pos)] ^= 1 << int(rng.integers(0, 8))
        try:
            got = sa.decompress_ranges(bytes(bad), np.uint64, index, pairs)
            assert got.size == sum(c for _, c in pairs)
            kinds.add("ok")
        except PcoError as e:
            assert e.kind in ("Corruption", "InsufficientData"), e
            assert e.message.startswith("range 2: "), e.message
            kinds.add(e.kind)
    # the library still works after every flip
    _check(sa, data, index, x, pairs)
