"""Asynchronous side index of a standalone file (pco_b200_build_index_async, standalone.AsyncIndexBuilder): the index it builds is the
one pco_b200_compress_ex writes for the same file, byte for byte, and says what pco_b200_build_index says on every file, pco-written and
older formats included; bad files fail with build_index's kind and chunk; and the index decodes through every asynchronous decompress,
inside a CUDA graph replayed over files of different lengths."""
import re
import struct

import numpy as np
import pytest

from tests.golden_generators import GENERATORS, load_assets

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from oracle import pyoracle as oracle  # noqa: E402
from pcodec_b200 import PcoError, standalone as sa  # noqa: E402

DTYPES = [np.uint8, np.int8, np.uint16, np.int16, np.float16, np.uint32, np.int32, np.float32, np.uint64, np.int64, np.float64]
INDEXED_ASSETS = ["v0_0_0_classic", "v0_0_0_delta_float_mult", "v0_1_0_delta_int_mult", "v0_1_1_standalone_versioned", "v0_3_0_f16",
                  "v0_3_0_float_quant", "v0_4_5_uniform_type", "v0_4_8_minor_version", "v1_0_0_u8", "v1_0_0_i8"]
COLD_ASSETS = ["v0_4_0_lookback_delta", "v1_0_0_dict", "v1_0_0_conv1"]
SENT = 0xA5


def _walk(dtype, n, seed, scale=0.05):
    rng = np.random.default_rng(seed)
    if np.dtype(dtype).kind == "f":
        x = np.cumsum(rng.normal(size=n)).astype(dtype)
        if n > 5:
            x[3], x[4], x[5] = np.nan, -np.inf, -0.0
        return x
    steps = rng.geometric(scale, size=n).astype(np.int64) - int(1 / scale) // 2
    return np.cumsum(steps).astype(np.uint64).astype(np.dtype(dtype).str.replace("i", "u")).view(dtype)


def _cfg(order=0, page=1 << 14, level=8, mode="classic", exact=None):
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec

    ms = {"classic": ModeSpec.classic(), "float_mult": ModeSpec.try_float_mult(0.01), "int_mult": ModeSpec.try_int_mult(8)}[mode]
    ds = DeltaSpec.try_consecutive(order) if order else DeltaSpec.no_op()
    ps = PagingSpec.exact_page_sizes(exact) if exact else PagingSpec.equal_pages_up_to(page)
    return ChunkConfig(compression_level=level, mode_spec=ms, delta_spec=ds, paging_spec=ps, enable_8_bit=True)


def _u8(b):
    return torch.as_tensor(np.frombuffer(bytes(b), np.uint8).copy(), device="cuda")


def _build(data, dtype, src_cap=None, index_cap=1 << 22, max_chunks=4096):
    """One AsyncIndexBuilder call: the file at the front of a src_cap buffer with random bytes behind it, the index buffer full of
    sentinels.  Returns (index bytes, status) or (PcoError, status); nothing past the index (everything, on an error) is written."""
    src_cap = len(data) + 300 if src_cap is None else src_cap
    b = sa.AsyncIndexBuilder(data[:32], dtype, src_cap, index_cap, max_chunks)
    rng = np.random.default_rng(len(data))
    src = torch.as_tensor(rng.integers(0, 256, size=max(src_cap, 1), dtype=np.uint8), device="cuda")
    src[: len(data)].copy_(_u8(data))
    index = torch.full((index_cap + 64,), SENT, dtype=torch.uint8, device="cuda")
    b(src, torch.tensor([len(data)], dtype=torch.int64, device="cuda"), index)
    st = b.status_record()
    host = index.cpu().numpy()
    try:
        n = b.result()
    except PcoError as e:
        assert (host == SENT).all(), "a failed call wrote to the index"
        return e, st
    assert n == st.index_bytes and (host[n:] == SENT).all(), "the call wrote past its index"
    return host[:n].tobytes(), st


def _fields(index):
    """What a side index says - header fields, each record and its entries - without where the entries lie."""
    magic, version, n_chunks, n_total, file_len, chunks_offset, end_byte = struct.unpack_from("<IIQQQQQ", index, 0)
    chunks = []
    for c in range(n_chunks):
        chunk_offset, n, n_vars, entries_offset, out_offset = struct.unpack_from("<QIIQQ", index, chunks_offset + 32 * c)
        chunks.append((chunk_offset, n, n_vars, out_offset, index[entries_offset: entries_offset + 12 * n_vars * -(-n // 256)]))
    return magic, version, n_chunks, n_total, file_len, end_byte, chunks


def _blocking(data, dtype):
    """build_index's index, or (kind, chunk named in its message)."""
    try:
        return sa.build_index(data, dtype)
    except PcoError as e:
        m = re.search(r"chunk (\d+)", e.message)
        return e.kind, int(m.group(1)) if m else None


def _same_as_blocking(data, dtype, **kw):
    got, st = _build(data, dtype, **kw)
    want = _blocking(data, dtype)
    if isinstance(want, tuple):
        assert isinstance(got, PcoError), want
        assert (got.kind, None if st.chunk == (1 << 64) - 1 else st.chunk) == want, (got.message, want)
    else:
        assert not isinstance(got, PcoError), got.message
        assert _fields(got) == _fields(want)
    return got, st


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("uniform", [False, True])
def test_byte_parity_with_compress_every_type_and_flavour(dtype, uniform):
    n = 3 * (1 << 14) + 5  # EqualPagesUpTo(2^14): one chunk of 12290, three of 12289 - two runs
    x = _walk(dtype, n, seed=5)
    data, index = sa.simple_compress_with_index(x, _cfg(1), uniform_type=uniform)
    got, st = _build(data, dtype)
    assert got == index
    assert st.n_chunks == 4 and st.n_total == n and st.serial_chunks == 0


@pytest.mark.parametrize("level", [0, 8, 12])
@pytest.mark.parametrize("order", [0, 1, 7])
@pytest.mark.parametrize("dtype", [np.uint32, np.float64])
def test_byte_parity_with_compress_levels_and_orders(level, order, dtype):
    n = 3 * (1 << 16) + 5
    x = _walk(dtype, n, seed=level + order)
    data, index = sa.simple_compress_with_index(x, _cfg(order, page=1 << 16, level=level))
    got, st = _build(data, dtype)
    assert got == index
    assert st.serial_chunks == 0  # EqualPagesUpTo's two runs are the two rounds', level 12's tables included
    if level == 12 and not (dtype == np.uint32 and order == 0):  # (that walk at order 0 is one bin)
        # tables above 2^10 states: the CAP_LOG 10 walk declines every chunk, so the chains above come from the CAP_LOG 12 re-walk
        assert min(max(v["ans_size_log"] for v in c["vars"]) for c in oracle.inspect(data, dtype)["chunks"]) > 10


@pytest.mark.parametrize("case", ["one_chunk", "two_runs_2e18", "exact_pages"])
def test_byte_parity_with_compress_paging(case):
    if case == "one_chunk":
        x, cfg = _walk(np.int64, 1000, seed=1), _cfg(1)
    elif case == "two_runs_2e18":
        x, cfg = _walk(np.uint64, 3 * (1 << 18) + 5, seed=2), _cfg(1, page=1 << 18)
    else:
        sizes = [700, 700, 300, 700, 1, 300, 300, 2000, 700, 700, 5]
        x, cfg = _walk(np.uint32, sum(sizes), seed=3), _cfg(0, exact=sizes)
    data, index = sa.simple_compress_with_index(x, cfg)
    got, st = _build(data, x.dtype)
    assert got == index
    assert st.n_total == x.size


@pytest.mark.parametrize("mode,dtype", [("float_mult", np.float64), ("float_mult", np.float32), ("int_mult", np.uint32), ("int_mult", np.int64)])
def test_two_var_files_field_by_field(mode, dtype):
    """compress_ex reserves two vars of entries for a chunk that fell back to one: such files are compared field by field."""
    n = 2 * (1 << 14) + 301
    rng = np.random.default_rng(0)
    if mode == "float_mult":
        x = (np.round(np.cumsum(rng.normal(size=n)) * 100) * 0.01).astype(dtype)
    else:
        x = (_walk(dtype, n, seed=4).astype(np.uint64) // 8 * 8 + 3).astype(dtype)
    data, index = sa.simple_compress_with_index(x, _cfg(1, mode=mode))
    got, st = _build(data, dtype)
    assert _fields(got) == _fields(index)
    assert st.serial_chunks == 0


@pytest.mark.parametrize("name", INDEXED_ASSETS)
def test_golden_assets_match_build_index(name):
    x = GENERATORS[name]()
    data = load_assets()[name]
    _same_as_blocking(data, x.dtype)


@pytest.mark.parametrize("name", COLD_ASSETS)
def test_cold_assets_fail_like_build_index(name):
    x = GENERATORS[name]()
    got, _ = _same_as_blocking(load_assets()[name], x.dtype)
    assert isinstance(got, PcoError) and got.kind == "Unsupported"


@pytest.mark.parametrize("dtype,n,page,order,level", [(np.uint64, 10 * 4096 + 123, 4096, 1, 8), (np.uint32, 37 * 1000 + 1, 1000, 0, 8),
                                                      (np.int64, 3 * (1 << 16) + 5, 1 << 16, 2, 12), (np.float32, 20 * 512 + 7, 512, 0, 3),
                                                      (np.uint16, 9 * 3000 + 2999, 3000, 1, 8)])
def test_oracle_files_match_build_index(dtype, n, page, order, level):
    x = _walk(dtype, n, seed=n)
    cfg = oracle.make_config(level=level, mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_CONSECUTIVE if order else oracle.DELTA_NOOP, delta_order=order,
                             max_page_n=page)
    data = oracle.simple_compress(x, cfg)
    _, st = _same_as_blocking(data, dtype)
    assert st.serial_chunks == 0


def test_oracle_cold_files_fail_like_build_index():
    x = _walk(np.uint32, 5 * 2048 + 7, seed=9)
    for cfg in (oracle.make_config(delta=oracle.DELTA_LOOKBACK, max_page_n=2048), oracle.make_config(mode=oracle.MODE_DICT, max_page_n=2048),
                oracle.make_config(delta=oracle.DELTA_CONV1, delta_order=2, max_page_n=2048)):
        _same_as_blocking(oracle.simple_compress(x, cfg), np.uint32)


def test_bad_files_fail_like_build_index():
    x = _walk(np.uint64, 9 * 2048, seed=7)
    data = oracle.simple_compress(x, oracle.make_config(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_CONSECUTIVE, delta_order=1, max_page_n=2048))
    starts = [c["chunk_start"] for c in oracle.inspect(data, np.uint64)["chunks"]]
    bad_type = bytearray(data)
    bad_type[starts[4]] = 0x37
    bad_count = bytearray(data)
    bad_count[starts[4] + 1] ^= 0x10
    bad_body = bytearray(data)
    bad_body[(starts[6] + starts[7]) // 2] ^= 0xFF
    for bad in (bytes(bad_type), bytes(bad_count), bytes(bad_body), data[: (starts[6] + starts[7]) // 2], data[: starts[6]], data[:-1]):
        got, st = _same_as_blocking(bad, np.uint64)
    got, st = _build(data[: starts[6]], np.uint64)
    assert got.kind == "InsufficientData" and st.chunk == 6


def test_refusals_of_the_plan_and_the_call():
    x = _walk(np.uint32, 5000, seed=1)
    plain = oracle.simple_compress(x, oracle.make_config(max_page_n=1000))
    uniform = oracle.simple_compress(x, oracle.make_config(max_page_n=1000), uniform_type=True)
    with pytest.raises(PcoError) as e:  # a uniform type other than dtype: refused by the plan, as build_index refuses the file
        sa.AsyncIndexBuilder(uniform[:32], np.int32, 1 << 16, 1 << 16, 16)
    assert e.value.kind == "InvalidArgument"
    assert isinstance(_blocking(uniform, np.int32), tuple)
    # a plan of one flavour, a file of another
    b = sa.AsyncIndexBuilder(plain[:32], np.uint32, 1 << 16, 1 << 16, 16)
    src, index = _u8(uniform + bytes(1 << 16)), torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    b(src, torch.tensor([len(uniform)], dtype=torch.int64, device="cuda"), index)
    with pytest.raises(PcoError) as e:
        b.result()
    assert e.value.kind == "InvalidArgument" and b.status_record().device_status == 0x103
    # *src_len above src_cap
    b(src, torch.tensor([(1 << 16) + 1], dtype=torch.int64, device="cuda"), index)
    with pytest.raises(PcoError) as e:
        b.result()
    assert e.value.kind == "InvalidArgument" and b.status_record().device_status == 0x10F
    # too many chunks (5 in the file), and an index larger than index_cap
    got, st = _build(plain, np.uint32, max_chunks=4)
    assert got.kind == "InvalidArgument" and st.device_status == 0x105
    got, st = _build(plain, np.uint32, max_chunks=5)
    assert st.n_chunks == 5 and not isinstance(got, PcoError)
    got, st = _build(plain, np.uint32, index_cap=len(got) - 1)
    assert got.kind == "Io" and st.device_status == 0x119
    with pytest.raises(ValueError):
        b(src, torch.tensor([len(plain)], dtype=torch.int32, device="cuda"), index)


def _planted_file(n0=4096, k=6):
    """Incompressible u64 chunks whose numbers' low bytes spell this file's chunk start (type byte 2, count - 1) all over them."""
    rng = np.random.default_rng(1)
    x = rng.integers(0, 1 << 63, size=n0 * k, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=n0 * k, dtype=np.uint64)
    pat = np.uint64(((n0 - 1) << 8) | 2)
    for i in range(100, n0 * k, 997):
        x[i] = (x[i] & np.uint64(0xFFFFFFFF00000000)) | pat
    x[::n0] = 0
    data = oracle.simple_compress(x, oracle.make_config(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_NOOP, max_page_n=n0))
    needle = bytes([2]) + int(n0 - 1).to_bytes(3, "little")
    hits = len(re.findall(re.escape(needle), data))
    assert hits >= k + 10, "the fixture lost its false chunk starts"
    return x, data


@pytest.mark.parametrize("max_chunks", [6, 64])
def test_planted_patterns_and_more_candidates_than_the_cap(max_chunks):
    """Candidates inside chunk bodies are never taken for chunks; with max_chunks = 6 more than max_chunks + 8 positions carry the
    pattern, so the kept candidates are a prefix of them."""
    x, data = _planted_file()
    got, st = _same_as_blocking(data, np.uint64, max_chunks=max_chunks)
    assert st.n_chunks == 6 and st.serial_chunks == 0
    out = torch.zeros(x.size, dtype=torch.int64, device="cuda")
    dec = sa.AsyncDecompressor(data[:32], np.uint64, len(data), len(got), x.size, 8)
    dec(_u8(data), _u8(got), out.view(torch.uint64))
    assert dec.result().finished
    assert np.array_equal(out.cpu().numpy().view(np.uint64), x)


def test_planted_file_with_an_exact_index_cap():
    """The coincidences the rounds walk take room in the round arena that no chunk uses; the serial walker has its own, so an index_cap
    of exactly the index's length and a max_chunks of exactly the file's chunks still index the file, and one chunk fewer is refused as
    too many chunks."""
    x, data = _planted_file()
    want = sa.build_index(data, np.uint64)
    size = 64 + 32 * 6 + 6 * 16 * 12  # header, 6 records, 6 chunks x 16 batches of one var (1408 bytes)
    full, _ = _build(data, np.uint64)
    assert len(full) == size
    for max_chunks in (6, 4096):
        got, st = _build(data, np.uint64, index_cap=size, max_chunks=max_chunks)
        assert not isinstance(got, PcoError), got.message
        assert got == full and _fields(got) == _fields(want) and st.n_chunks == 6
    got, st = _build(data, np.uint64, index_cap=size - 1, max_chunks=6)
    assert got.kind == "Io" and st.device_status == 0x119
    got, st = _build(data, np.uint64, index_cap=size, max_chunks=5)
    assert got.kind == "InvalidArgument" and st.device_status == 0x105


def test_a_round_that_takes_nothing_ends_the_rounds():
    """A file cut inside its first chunk: the first round's chain takes nothing, so the second round stays idle rather than walk the same candidates
    again, and the serial walker reports the chunk as build_index does.  The call's state words at the front of the workspace
    (AiState, async_index_kernels.cuh: status, active, stalled) show which round ran last."""
    x = _walk(np.uint64, 9 * 2048, seed=7)
    data = oracle.simple_compress(x, oracle.make_config(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_CONSECUTIVE, delta_order=1, max_page_n=2048))
    starts = [c["chunk_start"] for c in oracle.inspect(data, np.uint64)["chunks"]]
    bad = data[: (starts[0] + starts[1]) // 2]
    got, st = _same_as_blocking(bad, np.uint64)
    assert isinstance(got, PcoError) and got.kind == "InsufficientData" and st.chunk == 0 and st.serial_chunks == 0
    b = sa.AsyncIndexBuilder(bad[:32], np.uint64, len(bad), 1 << 20, 64)
    b(_u8(bad), torch.tensor([len(bad)], dtype=torch.int64, device="cuda"), torch.zeros(1 << 20, dtype=torch.uint8, device="cuda"))
    status, active, stalled = b.workspace[:12].cpu().numpy().view(np.uint32)
    assert (status, active, stalled) == (st.device_status, 0, 1)


def test_three_sizes_leave_the_rest_to_the_serial_walker():
    sizes = [3000, 3000, 1000, 1000, 2000, 2000, 2000, 5]
    x = _walk(np.uint64, sum(sizes), seed=6)
    data, index = sa.simple_compress_with_index(x, _cfg(1, exact=sizes))
    got, st = _build(data, np.uint64)
    assert got == index
    assert st.serial_chunks == 4  # the rounds take the runs of 3000 and 1000


def test_end_to_end_through_every_async_decompress():
    x = _walk(np.int64, 5 * (1 << 14) + 77, seed=8)
    data = oracle.simple_compress(x, oracle.make_config(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_CONSECUTIVE, delta_order=1, max_page_n=1 << 14))
    index, _ = _build(data, np.int64)
    d_src, d_idx = _u8(data), _u8(index)
    out = torch.zeros(x.size, dtype=torch.int64, device="cuda")
    dec = sa.AsyncDecompressor(data[:32], np.int64, len(data), len(index), x.size, 16)
    dec(d_src, d_idx, out)
    assert dec.result().n_processed == x.size
    assert np.array_equal(out.cpu().numpy(), x)
    pairs = [(0, 10), (16383, 3), (40000, 20000), (x.size - 1, 1)]
    rd = sa.AsyncRangeDecompressor(data[:32], np.int64, len(data), len(index), 16, 8, 40000, 1 << 17)
    ranges = torch.zeros((8, 2), dtype=torch.int64, device="cuda")
    ranges[: len(pairs)] = torch.tensor(pairs, dtype=torch.int64)
    rout = torch.zeros(40000, dtype=torch.int64, device="cuda")
    rd(d_src, d_idx, ranges, torch.tensor([len(pairs)], dtype=torch.int64, device="cuda"), rout)
    nw = rd.result()
    want = np.concatenate([x[s:s + c] for s, c in pairs])
    assert nw == want.size and np.array_equal(rout.cpu().numpy()[:nw], want)
    fd = sa.AsyncFilesDecompressor(data[:32], np.int64, len(data), len(index), 2, 16, x.size)
    refs = torch.zeros((2, 4), dtype=torch.int64, device="cuda")
    refs[0] = torch.tensor([0, len(data), 0, len(index)], dtype=torch.int64)
    fout, fns = torch.zeros(x.size, dtype=torch.int64, device="cuda"), torch.zeros(2, dtype=torch.int64, device="cuda")
    fd(d_src, d_idx, refs, torch.tensor([1], dtype=torch.int64, device="cuda"), fout, fns)
    assert fd.result() == x.size and np.array_equal(fout.cpu().numpy(), x)


def test_graph_of_build_and_decompress_replayed_on_two_files():
    from pcodec_b200 import _lib

    files = []
    for k, n in enumerate((4 * (1 << 14) + 9, 7 * (1 << 14) + 4001)):
        x = _walk(np.uint64, n, seed=20 + k)
        files.append((x, oracle.simple_compress(x, oracle.make_config(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_CONSECUTIVE, delta_order=1,
                                                                      max_page_n=1 << 14))))
    src_cap, index_cap, dst_cap, max_chunks = max(len(d) for _, d in files) + 1000, 1 << 20, 8 << 14, 16
    d_src = torch.zeros(src_cap, dtype=torch.uint8, device="cuda")
    d_len = torch.zeros(1, dtype=torch.int64, device="cuda")
    d_idx = torch.zeros(index_cap, dtype=torch.uint8, device="cuda")
    d_dst = torch.zeros(dst_cap, dtype=torch.int64, device="cuda")
    b = sa.AsyncIndexBuilder(files[0][1][:32], np.uint64, src_cap, index_cap, max_chunks)
    dec = sa.AsyncDecompressor(files[0][1][:32], np.uint64, src_cap, index_cap, dst_cap, max_chunks)

    def load(k):
        d = files[k][1]
        d_src.zero_()
        d_src[: len(d)].copy_(_u8(d))
        d_len.fill_(len(d))

    load(0)
    g = torch.cuda.CUDAGraph()
    L = _lib.lib()
    L.pco_b200_profile_enable(1)  # a call inside a capture records no spans
    try:
        with torch.cuda.graph(g):  # fails if a call synchronises or allocates
            b(d_src, d_len, d_idx)
            dec(d_src, d_idx, d_dst.view(torch.uint64))
    finally:
        L.pco_b200_profile_enable(0)
    for k in (1, 0, 1):
        load(k)
        g.replay()
        x = files[k][0]
        n_ix = b.result()
        assert _fields(d_idx[:n_ix].cpu().numpy().tobytes()) == _fields(sa.build_index(files[k][1], np.uint64))
        prog = dec.result()
        assert (prog.n_processed, prog.finished) == (x.size, True)
        assert np.array_equal(d_dst[: x.size].cpu().numpy().view(np.uint64), x)
