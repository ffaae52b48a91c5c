"""Batches of standalone files on the GPU (pco_b200_compress_files, pco_b200_decompress_files): every file of a batch equals the oracle's
bytes and pco_b200_compress_ex's bytes and side index, and every batch decodes to the input and to what pco_b200_decompress_ex gives
file by file."""
import ctypes as C

import numpy as np
import pytest

from tests.golden_generators import GENERATORS, bits_view, load_assets
from tests.test_gpu_encode import _cfgs, _parse_index, _walk

pytestmark = pytest.mark.gpu

DTYPES = [np.uint8, np.int8, np.uint16, np.int16, np.float16, np.uint32, np.int32, np.float32, np.uint64, np.int64, np.float64]
SIZES = [0, 1, 255, 256, 257, 1 << 18, (1 << 18) + 1]


def _sa():
    from pcodec_b200 import standalone

    return standalone


def _split(x, ns):
    at = np.concatenate([[0], np.cumsum(ns)]).astype(np.int64)
    return [x[at[i]:at[i + 1]] for i in range(len(ns))]


def _pieces(data, files):
    return [bytes(data[int(f["offset"]):int(f["offset"] + f["len"])]) for f in files]


def _index_pieces(index, files):
    return [bytes(index[int(f["index_offset"]):int(f["index_offset"] + f["index_len"])]) for f in files]


def _decompress_ex(data, dtype, index=None, cap=None):
    sa = _sa()
    dst = np.zeros(max(cap if cap is not None else max(sa.n_hint(data), 1) + 1024, 1), dtype=dtype)
    prog = sa.decompress_into_with_index(data, dst, index)
    assert prog.finished
    return dst[: prog.n_processed]


def _check_batch(oracle, x, ns, cfg, ocfg, dtype, uniform=False):
    """compress_files against the oracle and compress_ex file by file; decompress_files with and without indexes against the input."""
    sa = _sa()
    data, files, index = sa.compress_files(x, ns, cfg, uniform_type=uniform)
    assert len(files) == len(ns)
    parts = _split(x, ns)
    for i, (got, idx, nums) in enumerate(zip(_pieces(data, files), _index_pieces(index, files), parts)):
        assert int(files[i]["index_offset"]) % 16 == 0
        ex, ex_idx = sa._compress(nums, cfg, uniform, True)
        assert got == ex, f"file {i} (n={len(nums)}) differs from compress_ex"
        assert idx == ex_idx, f"file {i}: side index differs from compress_ex's: {_parse_index(idx) == _parse_index(ex_idx)=}"
        if ocfg is not None:
            assert got == oracle.simple_compress(nums, ocfg, uniform_type=uniform), f"file {i} differs from the oracle"
    want = bits_view(np.concatenate(parts)) if len(parts) else np.zeros(0)
    for with_index in (True, False):
        refs = files.copy()
        if not with_index:
            refs["index_len"] = 0
        vals, got_ns = sa.decompress_files(data, refs, dtype, index if with_index else None)
        np.testing.assert_array_equal(got_ns, np.asarray(ns, dtype=np.uint64))
        np.testing.assert_array_equal(bits_view(vals), want)
    return data, files, index


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("uniform", [False, True])
def test_every_type_mixed_sizes(oracle, dtype, uniform):
    ns = SIZES[::-1] + SIZES
    x = np.concatenate([_walk(dtype, n, seed=i) for i, n in enumerate(ns)]) if sum(ns) else np.zeros(0, dtype)
    cfg, ocfg = _cfgs(oracle, mode="classic", order=1)
    _check_batch(oracle, x.astype(dtype), ns, cfg, ocfg, dtype, uniform)


def test_auto_over_files_of_different_bins_log(oracle):
    from pcodec_b200 import ChunkConfig

    ns = [600, 1024, 3000, 70000, 300000, 600, 0, 3000]
    x = np.concatenate([_walk(np.int64, n, seed=n + i) for i, n in enumerate(ns)])
    ocfg = oracle.make_config(mode=oracle.MODE_AUTO, delta=oracle.DELTA_AUTO)
    _check_batch(oracle, x, ns, ChunkConfig(), ocfg, np.int64)


@pytest.mark.parametrize("mode,dtype", [("int_mult", np.uint32), ("int_mult", np.int64), ("float_mult", np.float32), ("float_mult", np.float64),
                                        ("float_quant", np.float32), ("float_quant", np.float64)])
@pytest.mark.parametrize("level", [0, 8, 9, 12])
def test_modes_orders_levels(oracle, mode, dtype, level):
    ns = [3000, 257, 1 << 16, 5000, 1]
    for order in (range(0, 4) if level != 12 else [1]) if mode != "int_mult" else range(4, 8):
        rng = np.random.default_rng(order + level)
        if mode == "float_mult":
            x = (np.round(np.cumsum(rng.normal(size=sum(ns))) * 100) * 0.01).astype(dtype)
        elif mode == "float_quant":
            x = np.cumsum(rng.normal(size=sum(ns))).astype(dtype)
        else:
            x = (_walk(dtype, sum(ns), seed=order).astype(np.uint64) // 8 * 8 + 3).astype(dtype)
        cfg, ocfg = _cfgs(oracle, mode=mode, order=order, level=level, k=13 if dtype == np.float64 else 7)
        _check_batch(oracle, x, ns, cfg, ocfg, dtype)


def test_refused_file_is_named_with_compress_ex_kind():
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec, PcoError

    sa = _sa()
    cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.no_op(), paging_spec=PagingSpec.exact_page_sizes([1000, 1000]))
    ns = [2000, 2000, 1999, 2000]
    x = _walk(np.uint32, sum(ns), seed=1)
    with pytest.raises(PcoError) as single:
        sa.simple_compress(x[4000:5999], cfg)
    with pytest.raises(PcoError) as batch:
        sa.compress_files(x, ns, cfg)
    assert batch.value.kind == single.value.kind and batch.value.message.startswith("file 2: ")


def test_device_buffers_on_a_side_stream(oracle):
    import torch

    sa = _sa()
    ns = [70000, 0, 1, 300000, 257]
    x = _walk(np.float32, sum(ns), seed=9)
    cfg, ocfg = _cfgs(oracle, mode="classic", order=2)
    host_data, host_files, host_index = sa.compress_files(x, ns, cfg)
    s = torch.cuda.Stream()
    dx = torch.from_numpy(x).cuda()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        data, files, index = sa.compress_files(dx, ns, cfg)
        vals, got_ns = sa.decompress_files(data, files, np.float32, index)
        refs = files.copy()
        refs["index_len"] = 0
        vals2, _ = sa.decompress_files(data, refs, np.float32)
    s.synchronize()
    assert data.is_cuda and index.is_cuda and vals.is_cuda
    assert bytes(data.cpu().numpy()) == host_data
    np.testing.assert_array_equal(files, host_files)
    assert [_parse_index(p) for p in _index_pieces(index.cpu().numpy().tobytes(), files)] == [_parse_index(p) for p in _index_pieces(host_index, files)]
    np.testing.assert_array_equal(bits_view(vals.cpu().numpy()), bits_view(x))
    np.testing.assert_array_equal(bits_view(vals2.cpu().numpy()), bits_view(x))
    np.testing.assert_array_equal(got_ns, ns)


@pytest.mark.parametrize("shift", [1, 3, 8])
def test_device_index_at_any_byte_offset(oracle, shift):
    """The index buffer may start at any byte, as compress_ex's may; offsets inside it stay 16-byte aligned."""
    import torch

    sa = _sa()
    L = sa._lib_files()
    ns = np.array([70000, 0, 3000, 257], dtype=np.uint64)
    x = _walk(np.uint32, int(ns.sum()), seed=6)
    cfg, _ = _cfgs(oracle, mode="classic", order=1)
    host_data, host_files, host_index = sa.compress_files(x, ns, cfg)
    dx = torch.from_numpy(x.view(np.int32)).cuda()
    d_data = torch.zeros(len(host_data) + 64, dtype=torch.uint8, device="cuda")
    d_idx = torch.zeros(len(host_index) + 64, dtype=torch.uint8, device="cuda")
    files = np.zeros(len(ns), dtype=sa.FILE_REF)
    c = cfg._to_c()
    rc = L.pco_b200_compress_files(C.c_void_p(dx.data_ptr()), ns.ctypes.data_as(C.c_void_p), C.c_size_t(len(ns)), C.c_ubyte(1), C.byref(c), C.c_int(0),
                                   C.c_void_p(d_data.data_ptr() + shift), C.c_size_t(len(host_data)), C.c_void_p(d_idx.data_ptr() + shift),
                                   C.c_size_t(len(host_index)), files.ctypes.data_as(C.c_void_p), C.c_uint32(1 | 2 | 4),
                                   C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    torch.cuda.synchronize()
    np.testing.assert_array_equal(files, host_files)
    assert bytes(d_data[shift:shift + len(host_data)].cpu().numpy()) == host_data
    assert bytes(d_idx[shift:shift + len(host_index)].cpu().numpy()) == host_index


def _damaged_record(index, f, chunk, field, value):
    """A copy of `index` with one field of one IndexChunk record of file f replaced."""
    import struct

    b = bytearray(index)
    base = int(f["index_offset"])
    chunks_offset = struct.unpack_from("<Q", b, base + 32)[0]
    at = base + chunks_offset + 32 * chunk + {"chunk_offset": 0, "n": 8, "n_vars": 12, "entries_offset": 16, "out_offset": 24}[field]
    struct.pack_into("<Q" if field in ("chunk_offset", "entries_offset", "out_offset") else "<I", b, at, value)
    return bytes(b)


@pytest.mark.parametrize("field,value", [("chunk_offset", 10**6), ("out_offset", 3000), ("out_offset", 10**12), ("entries_offset", 10**9), ("n", 5)])
def test_damaged_index_record_stays_in_its_file(oracle, field, value):
    """A record of file 1 that points outside that file (its bytes, its index, its count) cannot reach another file: the batch gives what
    decompress_ex gives for file 1 with the same index, and every other file decodes to its numbers."""
    sa = _sa()
    ns = [3000, 9000, 5000, 3000]
    x = _walk(np.int64, sum(ns), seed=31)
    cfg, _ = _cfgs(oracle, mode="classic", order=1, max_page_n=2048)
    data, files, index = sa.compress_files(x, ns, cfg)
    bad = _damaged_record(index, files[1], 1, field, value)
    one_index = _index_pieces(bad, files)[1]
    want_kind, want_msg = _kind(lambda: _decompress_ex(_pieces(data, files)[1], np.int64, index=one_index, cap=ns[1]))
    got_kind, msg = _kind(lambda: sa.decompress_files(data, files, np.int64, bad))
    assert got_kind == want_kind, (msg, want_msg)
    if got_kind is not None:
        assert msg.startswith("file 1: ")
        return
    vals, got_ns = sa.decompress_files(data, files, np.int64, bad)
    parts = _split(x, ns)
    at = np.concatenate([[0], np.cumsum(got_ns)]).astype(np.int64)
    for i in (0, 2, 3):
        np.testing.assert_array_equal(vals[at[i]:at[i + 1]], parts[i])


def test_small_buffers_give_io_with_the_sizes():
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec

    sa = _sa()
    L = sa._lib_files()
    ns = np.array([1000, 0, 50000], dtype=np.uint64)
    x = _walk(np.uint64, int(ns.sum()), seed=4)
    cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(1))
    data, files, index = sa.compress_files(x, ns, cfg)
    c = cfg._to_c()
    for dcap, icap in [(len(data) - 1, len(index)), (len(data), len(index) - 1)]:
        dst = np.zeros(max(dcap, 1), np.uint8)
        idx = np.zeros(max(icap, 1), np.uint8)
        got = np.zeros(3, dtype=sa.FILE_REF)
        rc = L.pco_b200_compress_files(x.ctypes.data_as(C.c_void_p), ns.ctypes.data_as(C.c_void_p), C.c_size_t(3), C.c_ubyte(2), C.byref(c), C.c_int(0),
                                       dst.ctypes.data_as(C.c_void_p), C.c_size_t(dcap), idx.ctypes.data_as(C.c_void_p), C.c_size_t(icap),
                                       got.ctypes.data_as(C.c_void_p), C.c_uint32(0), None)
        assert rc == 4
        np.testing.assert_array_equal(got, files)


def _oracle_files(oracle, dtype):
    """Oracle-written files of `dtype` (cold ones among them: Lookback, Dict, Conv1) plus the golden assets of that type."""
    x = _walk(dtype, 9000, seed=2)
    out = []
    for k, (mode, delta, order) in enumerate([(oracle.MODE_CLASSIC, oracle.DELTA_CONSECUTIVE, 1), (oracle.MODE_CLASSIC, oracle.DELTA_LOOKBACK, 0),
                                              (oracle.MODE_DICT, oracle.DELTA_NOOP, 0), (oracle.MODE_CLASSIC, oracle.DELTA_CONV1, 2),
                                              (oracle.MODE_CLASSIC, oracle.DELTA_NOOP, 0)]):
        nums = x[: 3000 + 1000 * k]
        try:
            out.append((oracle.simple_compress(nums, oracle.make_config(mode=mode, delta=delta, delta_order=order, max_page_n=2048)), nums))
        except Exception:  # a spec the oracle does not take for this type
            continue
    assets = load_assets()
    for name, gen in GENERATORS.items():
        want = gen()
        if want.dtype == np.dtype(dtype):
            out.append((assets[name], want))
    return out


@pytest.mark.parametrize("dtype", [np.uint32, np.int64, np.float32, np.float64, np.uint8, np.float16])
def test_mixed_decompress_batch(oracle, dtype):
    """Files with and without an index, oracle-written and golden ones, cold ones between fast ones, shuffled and repeated."""
    sa = _sa()
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec

    items = _oracle_files(oracle, dtype)
    ours = _walk(dtype, 50000, seed=3)
    for level in (8, 12):
        d, ix = sa.simple_compress_with_index(ours[: 20000 + level], ChunkConfig(compression_level=level, mode_spec=ModeSpec.classic(),
                                                                                  delta_spec=DeltaSpec.try_consecutive(1), enable_8_bit=True))
        items.append((d, ours[: 20000 + level], ix))
    data, index, refs, want = bytearray(), bytearray(), [], []
    rng = np.random.default_rng(int(np.dtype(dtype).num))
    order = list(rng.permutation(len(items))) + [0, len(items) - 1]
    for j, k in enumerate(order):
        item = items[k]
        blob, nums = item[0], item[1]
        ix = item[2] if len(item) > 2 else None
        if ix is None and j % 2:
            try:  # the serial walker indexes what the fast kernels take
                ix = sa.build_index(blob, dtype)
            except Exception:
                ix = None
        io, il = 0, 0
        if ix is not None:
            index += b"\0" * (-len(index) % 16)
            io, il = len(index), len(ix)
            index += ix
        refs.append((len(data), len(blob), io, il))
        data += blob + b"\x07" * (j % 3)  # bytes between files belong to no file
        want.append(nums)
    files = np.array(refs, dtype=sa.FILE_REF)
    vals, ns = sa.decompress_files(bytes(data), files, dtype, bytes(index))
    np.testing.assert_array_equal(ns, [len(w) for w in want])
    np.testing.assert_array_equal(bits_view(vals), bits_view(np.concatenate(want)))
    at = 0
    for f, w in zip(files, want):
        blob = bytes(data[int(f["offset"]):int(f["offset"] + f["len"])])
        one = _decompress_ex(blob, dtype, cap=len(w) + 16)
        np.testing.assert_array_equal(bits_view(vals[at:at + len(w)]), bits_view(one))
        at += len(w)


def _kind(fn):
    from pcodec_b200 import PcoError

    try:
        fn()
    except PcoError as e:
        return e.kind, e.message
    return None, None


@pytest.mark.parametrize("with_index", [False, True])
def test_corrupt_truncated_mislabelled(oracle, with_index):
    sa = _sa()
    ns = [3000, 70000, 5000, 3000]
    x = _walk(np.int32, sum(ns), seed=8)
    cfg, _ = _cfgs(oracle, mode="classic", order=1, max_page_n=2048)
    data, files, index = sa.compress_files(x, ns, cfg)
    data = bytearray(data)
    blobs = _pieces(data, files)
    cases = {
        "truncated": lambda b: b[: len(b) // 2],
        "magic": lambda b: b"xco!" + b[4:],
        "body": lambda b: b[:40] + bytes(v ^ 0x5a for v in b[40:200]) + b[200:],
        "no_terminator": lambda b: b[:-1],
    }
    for name, bad in cases.items():
        for victim in (1, 3):
            new = [bad(b) if i == victim else b for i, b in enumerate(blobs)]
            refs = files.copy()
            at = 0
            for i, b in enumerate(new):
                refs[i]["offset"], refs[i]["len"] = at, len(b)
                at += len(b)
            if not with_index:
                refs["index_len"] = 0
            want_kind, _ = _kind(lambda: _decompress_ex(new[victim], np.int32, index=_index_pieces(index, files)[victim] if with_index else None,
                                                        cap=ns[victim] + 16))
            got_kind, msg = _kind(lambda: sa.decompress_files(b"".join(new), refs, np.int32, index if with_index else None))
            assert got_kind == want_kind, (name, victim, msg)
            if want_kind is not None:
                assert msg.startswith(f"file {victim}: "), (name, msg)
    # mislabelled: another file's index
    refs = files.copy()
    refs[2]["index_offset"], refs[2]["index_len"] = files[0]["index_offset"], files[0]["index_len"]
    kind, msg = _kind(lambda: sa.decompress_files(bytes(data), refs, np.int32, index))
    assert kind == "InvalidArgument" and msg.startswith("file 2: ")
    # a destination one number short
    L = sa._lib_files()
    src = np.frombuffer(bytes(data), np.uint8)
    dst = np.zeros(sum(ns), np.int32)
    nsw = np.zeros(4, np.uint64)
    nw = C.c_size_t()
    refs = files.copy()
    refs["index_len"] = 0
    rc = L.pco_b200_decompress_files(src.ctypes.data_as(C.c_void_p), C.c_size_t(src.size), None, C.c_size_t(0), C.c_ubyte(3),
                                     refs.ctypes.data_as(C.c_void_p), C.c_size_t(4), dst.ctypes.data_as(C.c_void_p), C.c_size_t(sum(ns) - 1),
                                     nsw.ctypes.data_as(C.c_void_p), C.byref(nw), C.c_uint32(0), None)
    assert rc == 4 and sa._lib.lib().pco_b200_last_error_message().decode().startswith("file 3: ")


def _walk_launches(fn):
    from pcodec_b200 import _lib

    L = _lib.lib()
    L.pco_b200_profile_enable(1)
    try:
        fn()
        buf = C.create_string_buffer(1 << 16)
        L.pco_b200_profile_last(buf, C.c_size_t(len(buf)))
    finally:
        L.pco_b200_profile_enable(0)
    return buf.value.decode().count("walk_kernel=")


def test_walk_bound():
    """300 index-free files of 3 chunks each launch walk_kernel no more often than decompress_ex does on one of them, which launches it
    at most twice: the speculative round, and the serial walker if the round does not end at the terminator."""
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec

    sa = _sa()
    ns = [2 * 4096 + 1000] * 300
    x = _walk(np.uint64, sum(ns), seed=12)
    cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(1), paging_spec=PagingSpec.equal_pages_up_to(4096))
    data, files = sa.compress_files(x, ns, cfg, with_index=False)
    assert all(f["index_len"] == 0 for f in files)
    one = _pieces(data, files[:1])[0]
    single = _walk_launches(lambda: _decompress_ex(one, np.uint64, cap=ns[0]))
    got = {}
    batch = _walk_launches(lambda: got.update(v=sa.decompress_files(data, files, np.uint64)[0]))
    np.testing.assert_array_equal(got["v"], x)
    assert 0 < batch <= single <= 2, (batch, single)


@pytest.mark.parametrize("name", ["v0_0_0_classic", "v0_1_0_delta_int_mult", "v0_3_0_f16", "v0_4_5_uniform_type", "v1_0_0_u8"])
def test_walk_bound_older_formats(name):
    """Index-free files of an older format version (or the uniform-type header) are walked together too: 40 copies of a golden file
    launch walk_kernel no more often than decompress_ex does on one."""
    sa = _sa()
    blob, want = load_assets()[name], GENERATORS[name]()
    files = np.array([(k * len(blob), len(blob), 0, 0) for k in range(40)], dtype=sa.FILE_REF)
    single = _walk_launches(lambda: _decompress_ex(blob, want.dtype, cap=len(want) + 16))
    got = {}
    batch = _walk_launches(lambda: got.update(v=sa.decompress_files(blob * 40, files, want.dtype)[0]))
    np.testing.assert_array_equal(bits_view(got["v"]), bits_view(np.concatenate([want] * 40)))
    assert 0 < batch <= single, (batch, single)


def test_scale_round_trip():
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec

    sa = _sa()
    rng = np.random.default_rng(21)
    ns = np.clip(rng.lognormal(np.log(1 << 17), 1.0, size=500), 1, 1 << 20).astype(np.int64)
    ns = (ns * ((1 << 26) / ns.sum())).astype(np.int64)
    ns[-1] += (1 << 26) - ns.sum()
    x = np.cumsum(rng.geometric(0.01, size=1 << 26)).astype(np.uint64)
    cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(1))
    data, files, index = sa.compress_files(x, ns, cfg)
    for ix in (index, None):
        refs = files.copy()
        if ix is None:
            refs["index_len"] = 0
        vals, got_ns = sa.decompress_files(data, refs, np.uint64, ix)
        np.testing.assert_array_equal(got_ns, ns)
        assert np.array_equal(vals, x)
