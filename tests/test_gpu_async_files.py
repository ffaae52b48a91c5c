"""Asynchronous batches of indexed standalone files (pco_b200_decompress_files_async, standalone.AsyncFilesDecompressor): every output
equals pco_b200_decompress_files on the same buffers and refs, and the input, bit for bit - with sentinel guard zones around dst and
file_ns, inside a CUDA graph replayed over different refs, counts and files, and on concurrent streams.  Refusals give the sync call's
kind and file, and write nothing behind the files before the refused one."""
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
NS_SENTINEL = -0x5a5a5a5a5a5a5a5b
KERNELS = ["af_files_kernel", "check_index_kernel", "af_scan_kernel", "af_place_kernel", "af_table_kernel", "merge_index_kernel",
           "fused_narrow_kernel", "symwalk_kernel", "decode_kernel", "cold_chunks_kernel", "af_finish_kernel"]


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


def _batch(sa, xs, cfg, uniform=False):
    """compress_files over the arrays: (data, index, refs as an (n, 4) uint64 array)."""
    nums = np.concatenate(xs) if xs else np.zeros(0, np.uint32)
    data, files, index = sa.compress_files(nums, [len(x) for x in xs], cfg, uniform_type=uniform)
    refs = np.stack([files["offset"], files["len"], files["index_offset"], files["index_len"]], axis=1).astype(np.uint64)
    return data, index, refs


def _n_chunks(index, ref):
    return struct.unpack_from("<Q", index, int(ref[2]) + 8)[0] if ref[3] >= 64 else 0


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


def _sync(sa, data, index, dtype, refs, dst_cap):
    """pco_b200_decompress_files on host copies of the same buffers with dst_len = dst_cap: ((numbers, file_ns), None) or
    (None, (kind, file named in the message))."""
    from pcodec_b200 import _lib

    L = sa._lib_files()
    r = np.zeros(len(refs), dtype=sa.FILE_REF)
    if len(refs):
        rr = np.asarray(refs, np.uint64).reshape(-1, 4)
        r["offset"], r["len"], r["index_offset"], r["index_len"] = rr[:, 0], rr[:, 1], rr[:, 2], rr[:, 3]
    d = np.frombuffer(bytes(data) + b"\0", np.uint8)
    ix = np.frombuffer(bytes(index) + b"\0", np.uint8)
    dst = np.empty(max(dst_cap, 1), dtype=dtype)
    ns = np.zeros(max(len(refs), 1), np.uint64)
    nw = C.c_size_t()
    rc = L.pco_b200_decompress_files(d.ctypes.data_as(C.c_void_p), C.c_size_t(len(data)), ix.ctypes.data_as(C.c_void_p), C.c_size_t(len(index)),
                                     C.c_ubyte(_lib.dtype_byte(dtype)), r.ctypes.data_as(C.c_void_p), C.c_size_t(len(refs)), dst.ctypes.data_as(C.c_void_p),
                                     C.c_size_t(dst_cap), ns.ctypes.data_as(C.c_void_p), C.byref(nw), C.c_uint32(0), None)
    if rc != 0:
        msg = L.pco_b200_last_error_message().decode()
        m = re.match(r"file (\d+): ", msg)
        return None, (_lib.ERROR_KINDS[rc], int(m.group(1)) if m else None)
    return (dst[: nw.value], ns[: len(refs)]), None


class Bufs:
    """Device buffers of one decompressor, with sentinel guard zones around dst and file_ns."""

    def __init__(self, sa, head, dtype, src_cap, index_cap, max_files, max_chunks, dst_cap):
        import torch

        self.dtype, self.dst_cap, self.max_files = np.dtype(dtype), dst_cap, max_files
        self.dec = sa.AsyncFilesDecompressor(head, dtype, src_cap, index_cap, max_files, max_chunks, dst_cap)
        self.src = torch.zeros(max(src_cap, 1), dtype=torch.uint8, device="cuda")
        self.index = torch.zeros(max(index_cap, 1), dtype=torch.uint8, device="cuda")
        self.files = torch.zeros((max_files, 4), dtype=torch.int64, device="cuda")
        self.n = torch.zeros(1, dtype=torch.int64, device="cuda")
        self.buf = _device_numbers(np.full(GUARD + dst_cap + GUARD, _sentinel(dtype), dtype=dtype))
        self.ns = torch.full((GUARD + max_files + GUARD,), NS_SENTINEL, dtype=torch.int64, device="cuda")

    def load(self, data, index, refs):
        import torch

        self.src.zero_()
        self.index.zero_()
        self.src[: len(data)] = torch.as_tensor(np.frombuffer(data, np.uint8).copy())
        self.index[: len(index)] = torch.as_tensor(np.frombuffer(index, np.uint8).copy())
        self.set_refs(refs)
        self.reset_out()

    def set_refs(self, refs):
        import torch

        f = np.zeros((self.max_files, 4), np.uint64)
        if len(refs):
            f[: len(refs)] = np.asarray(refs, np.uint64).reshape(-1, 4)
        self.files.copy_(torch.as_tensor(f.view(np.int64)))
        self.n.fill_(len(refs))

    def reset_out(self):
        self.buf.copy_(_device_numbers(np.full(GUARD + self.dst_cap + GUARD, _sentinel(self.dtype), dtype=self.dtype)))
        self.ns.fill_(NS_SENTINEL)

    def call(self):
        self.dec(self.src, self.index, self.files, self.n, self.buf[GUARD:GUARD + self.dst_cap], self.ns[GUARD:GUARD + self.max_files])

    def outcome(self, counts=None):
        """((numbers, file_ns) or None, (kind, file) or None, status record); asserts the guard zones and, for a refusal before the
        decode, an untouched file_ns and nothing in dst behind the files before the refused one (`counts`: the files' index counts)."""
        from pcodec_b200 import PcoError

        st = self.dec.status_record()
        err = None
        nw = 0
        try:
            nw = self.dec.result()
        except PcoError as e:
            err = (e.kind, int(st.file) if st.file != NONE else None)
        back = _host_numbers(self.buf, self.dtype)
        g = bits_view(back)
        s = bits_view(np.array([_sentinel(self.dtype)], dtype=self.dtype))[0]
        ns = self.ns.cpu().numpy()
        assert (g[:GUARD] == s).all() and (g[GUARD + self.dst_cap:] == s).all(), "a write outside dst"
        assert (ns[:GUARD] == NS_SENTINEL).all() and (ns[GUARD + self.max_files:] == NS_SENTINEL).all(), "a write outside file_ns"
        if err is not None:
            assert (ns == NS_SENTINEL).all(), "a refused call wrote file_ns"
            if st.device_status >= 0x100:
                allowed = sum(counts[: int(st.file)]) if counts is not None and st.file != NONE else 0
                assert (g[GUARD + allowed:] == s).all(), "a call refused before its decode wrote behind the files before the refused one"
            return None, err, st
        n = int(st.n_files)
        assert (ns[GUARD + n:] == NS_SENTINEL).all(), "file_ns written behind n_files"
        return (back[GUARD:GUARD + nw], ns[GUARD:GUARD + n].view(np.uint64)), None, st


def _run(sa, data, index, dtype, refs, max_files=None, max_chunks=None, dst_cap=None, src_cap=None, index_cap=None, head=None):
    nc = sum(_n_chunks(index, r) for r in refs)
    if dst_cap is None:
        ok, err = _sync(sa, data, index, dtype, refs, 1 << 40)
        dst_cap = len(ok[0]) if ok else 0
    b = Bufs(sa, head if head is not None else data[int(refs[0][0]):int(refs[0][0]) + 32] if len(refs) else data[:32], dtype, src_cap or len(data),
             index_cap or len(index), max_files or max(len(refs), 1), max_chunks or max(nc, 1), dst_cap)
    b.load(data, index, refs)
    b.call()
    return b.outcome(_counts(index, refs))


def _counts(index, refs):
    """Each ref's index count (0 where its index is missing or outside the buffer)."""
    out = []
    for r in refs:
        at = int(r[2]) + 16
        out.append(struct.unpack_from("<Q", index, at)[0] if r[3] >= 64 and at + 8 <= len(index) else 0)
    return out


def _expect(xs, order):
    parts = [xs[i] for i in order]
    return np.concatenate(parts) if parts else np.zeros(0, xs[0].dtype if xs else np.uint8)


def _check(sa, data, index, xs, refs, order, spare=True):
    """The async call equals decompress_files and the input, for exact capacities and for spare ones."""
    want = bits_view(_expect(xs, order))
    sel = refs[order] if len(order) else refs[:0]
    dtype = xs[0].dtype
    ok, err = _sync(sa, data, index, dtype, sel, len(want))
    assert err is None, err
    np.testing.assert_array_equal(bits_view(ok[0]), want)
    got, err, st = _run(sa, data, index, dtype, sel, dst_cap=len(want))
    assert err is None, err
    np.testing.assert_array_equal(bits_view(got[0]), want)
    np.testing.assert_array_equal(got[1], ok[1])
    assert st.n_written == len(want) and st.n_files == len(sel)
    if spare:
        nc = sum(_n_chunks(index, r) for r in sel)
        got, err, _ = _run(sa, data, index, dtype, sel, max_files=len(sel) + 300, max_chunks=2 * nc + 3, dst_cap=len(want) + 999,
                           src_cap=len(data) + 100, index_cap=len(index) + 64)
        assert err is None, err
        np.testing.assert_array_equal(bits_view(got[0]), want)
        np.testing.assert_array_equal(got[1], ok[1])


def _sizes(n):
    return [n, 1, 0, 5000, 1 << 14, 257]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("order", [0, 1, 2, 7])
def test_every_type_and_order(sa, dtype, order):
    xs = [_walk(dtype, m, seed=order + 11 + i) for i, m in enumerate(_sizes(3 * (1 << 14) + 777))]
    data, index, refs = _batch(sa, xs, _cfg(order))
    k = len(xs)
    _check(sa, data, index, xs, refs, list(range(k)), spare=(order == 1))
    _check(sa, data, index, xs, refs, [4, 0, 0, 2, 5, 1, 3, 0], spare=False)  # out of order and repeated


@pytest.mark.parametrize("mode,dtype", [("float_mult", np.float32), ("float_mult", np.float64), ("int_mult", np.uint32), ("int_mult", np.int64),
                                        ("float_quant", np.float32), ("float_quant", np.float64)])
def test_two_var_modes(sa, mode, dtype):
    rng = np.random.default_rng(3)
    xs = []
    for m in (2 * (1 << 14) + 301, 999, 1):
        if mode == "float_mult":
            xs.append((np.round(np.cumsum(rng.normal(size=m)) * 100) * 0.01).astype(dtype))
        elif mode == "float_quant":
            xs.append(np.cumsum(rng.normal(size=m)).astype(dtype))
        else:
            xs.append((_walk(dtype, m, seed=m).astype(np.uint64) // 8 * 8 + 3).astype(dtype))
    data, index, refs = _batch(sa, xs, _cfg(1, mode=mode))
    _check(sa, data, index, xs, refs, [0, 1, 2, 0])


@pytest.mark.parametrize("uniform", [False, True])
def test_both_header_flavours(sa, uniform):
    xs = [_walk(np.float64, m, seed=m) for m in (2 * (1 << 14) + 999, 3, 7000)]
    data, index, refs = _batch(sa, xs, _cfg(1), uniform=uniform)
    assert (data[5] != 0) == uniform  # the uniform type byte of the first header
    _check(sa, data, index, xs, refs, [2, 1, 0])


@pytest.mark.parametrize("level", [9, 12])
def test_catch_all_chunks(sa, level):
    rng = np.random.default_rng(level)
    xs = [rng.lognormal(10, 2, size=m).astype(np.uint64) for m in (3 * (1 << 16) + 5, 1000, (1 << 16) + 1)]
    data, index, refs = _batch(sa, xs, _cfg(0, page=1 << 16, level=level))
    _check(sa, data, index, xs, refs, [0, 1, 2, 1], spare=False)


@pytest.mark.parametrize("page", [1 << 18, 1 << 20])
def test_large_chunks(sa, page):
    xs = [_walk(np.uint32, m, seed=m) for m in (page + (1 << 17) + 3, page, 17)]
    data, index, refs = _batch(sa, xs, _cfg(1, page=page))
    _check(sa, data, index, xs, refs, [0, 1, 2], spare=False)


def test_many_small_chunks(sa):
    xs = [_walk(np.uint16, m, seed=m) for m in (1500 * 256 + 7, 300 * 256, 5)]
    data, index, refs = _batch(sa, xs, _cfg(0, page=256))
    assert _n_chunks(index, refs[0]) > 1000
    _check(sa, data, index, xs, refs, [0, 1, 2, 1], spare=False)


@pytest.mark.parametrize("name", INDEXED_ASSETS)
def test_golden_assets(sa, name):
    x = GENERATORS[name]()
    one = load_assets()[name]
    idx = sa.build_index(one, x.dtype)
    # the asset twice, back to back, each with its index at a 16-byte aligned offset
    pad = (-len(idx)) % 16
    data, index = one + one, idx + b"\0" * pad + idx
    refs = np.array([[0, len(one), 0, len(idx)], [len(one), len(one), len(idx) + pad, len(idx)]], np.uint64)
    _check(sa, data, index, [x, x], refs, [0, 1, 1], spare=False)


def test_n_files_0_1_and_max(sa):
    xs = [_walk(np.int32, m, seed=m) for m in (5000, 20000, 1, 0)]
    data, index, refs = _batch(sa, xs, _cfg(1))
    got, err, st = _run(sa, data, index, np.int32, refs[:0], max_files=4, max_chunks=8, dst_cap=10)  # n_files = 0
    assert err is None and got[0].size == 0 and got[1].size == 0 and st.n_written == 0 and st.n_files == 0
    _check(sa, data, index, xs, refs, [1])
    got, err, _ = _run(sa, data, index, np.int32, refs, max_files=4)  # n_files = max_files
    assert err is None
    np.testing.assert_array_equal(bits_view(got[0]), bits_view(_expect(xs, [0, 1, 2, 3])))


def test_subset_chosen_on_the_device(sa):
    import torch

    xs = [_walk(np.float32, 300 + 97 * i, seed=i) for i in range(64)]
    data, index, refs = _batch(sa, xs, _cfg(1, page=256))
    all_refs = torch.as_tensor(refs.view(np.int64), device="cuda")
    nc = sum(_n_chunks(index, r) for r in refs)
    b = Bufs(sa, data[:32], np.float32, len(data), len(index), 16, nc, sum(x.size for x in xs))
    b.load(data, index, [])
    rng = np.random.default_rng(7)
    for m in (16, 1, 9):
        pick = torch.as_tensor(rng.integers(0, 64, m), device="cuda")
        b.files[:m].copy_(all_refs[pick])  # a gather on the device: no ref goes through the host
        b.n.fill_(m)
        b.reset_out()
        b.call()
        got, err, _ = b.outcome()
        assert err is None, err
        order = pick.cpu().tolist()
        np.testing.assert_array_equal(bits_view(got[0]), bits_view(_expect(xs, order)))
        np.testing.assert_array_equal(got[1], [xs[i].size for i in order])


def test_graph_replays_with_new_refs_counts_and_contents(sa):
    import torch

    from pcodec_b200 import _lib

    batches = []
    for s in (1, 2):
        xs = [_walk(np.uint32, 4000 * (i + 1) + s, seed=10 * s + i) for i in range(6)]
        batches.append((xs,) + _batch(sa, xs, _cfg(s - 1, page=4096)))
    src_cap = max(len(b[1]) for b in batches) + 64
    index_cap = max(len(b[2]) for b in batches) + 64
    b = Bufs(sa, batches[0][1][:32], np.uint32, src_cap, index_cap, 8, 64, 1 << 18)
    b.load(batches[0][1], batches[0][2], batches[0][3])
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        b.call()  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        b.call()
    plans = [(0, [0, 1, 2, 3, 4, 5]), (1, [5, 5, 0]), (0, []), (1, [3]), (0, [2, 0, 4, 1, 3, 5, 0, 0])]
    for step, (k, order) in enumerate(plans):
        xs, data, index, refs = batches[k]
        b.load(data, index, refs[order] if order else refs[:0])
        if step == 3:
            _lib.lib().pco_b200_thread_release()  # the library's per-thread scratch is gone; the graph refers to none of it
        if step == 4:
            big = _walk(np.uint32, 1 << 22, seed=5)
            d2, i2, r2 = _batch(sa, [big], _cfg(1))
            assert _sync(sa, d2, i2, np.uint32, r2, big.size)[1] is None  # a large blocking call in between
        g.replay()
        torch.cuda.synchronize()
        got, err, st = b.outcome()
        assert err is None, err
        np.testing.assert_array_equal(bits_view(got[0]), bits_view(_expect(xs, order)))
        assert st.n_files == len(order)


def test_two_streams_with_two_workspaces(sa):
    import torch

    runs = []
    for s in (21, 22):
        xs = [_walk(np.int64, 3000 * i + s, seed=s + i) for i in range(1, 9)]
        data, index, refs = _batch(sa, xs, _cfg(s % 2))
        order = list(range(8))[:: 1 if s % 2 else -1]
        b = Bufs(sa, data[:32], np.int64, len(data), len(index), 8, 64, sum(x.size for x in xs))
        b.load(data, index, refs[order])
        runs.append((b, xs, order))
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for _ in range(3):
        for (b, _, _), s in zip(runs, streams):
            with torch.cuda.stream(s):
                b.call()
    torch.cuda.synchronize()
    for b, xs, order in runs:
        got, err, _ = b.outcome()
        assert err is None, err
        np.testing.assert_array_equal(bits_view(got[0]), bits_view(_expect(xs, order)))


def test_async_compress_feeds_the_batch_in_one_graph(sa):
    import torch

    n = 3 * (1 << 14) + 11
    comp = sa.AsyncCompressor(n, np.float32, _cfg(1), index=True)
    xs = [_walk(np.float32, n, seed=s) for s in (1, 2)]
    nums = _device_numbers(xs[0])
    file_buf = torch.zeros(comp.dst_cap, dtype=torch.uint8, device="cuda")
    ix_cap = (comp.index_bytes + 15) // 16 * 16
    b = Bufs(sa, sa.simple_compress(xs[0][:10], _cfg(1))[:32], np.float32, comp.dst_cap, ix_cap, 2, 16, 2 * n)
    refs = np.array([[0, 0, 0, comp.index_bytes], [0, 0, 0, comp.index_bytes]], np.uint64)  # len filled on the device
    b.set_refs(refs)
    b.reset_out()

    def step():
        comp(nums, file_buf, b.index[: comp.index_bytes])
        b.src.copy_(file_buf)
        b.files[:, 1].copy_(comp.status.view(torch.int64)[1].expand(2))  # PcoB200AsyncCompressStatus.file_bytes
        b.call()

    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    for x in xs:
        nums.copy_(_device_numbers(x))
        b.reset_out()
        g.replay()
        torch.cuda.synchronize()
        got, err, _ = b.outcome()
        assert err is None, err
        np.testing.assert_array_equal(bits_view(got[0]), bits_view(np.concatenate([x, x])))


def _refusal(sa, data, index, dtype, refs, dst_cap=None, **kw):
    want, werr = _sync(sa, data, index, dtype, refs, (1 << 20) if dst_cap is None else dst_cap)
    got, err, st = _run(sa, data, index, dtype, refs, dst_cap=(1 << 20) if dst_cap is None else dst_cap, **kw)
    return got, err, werr, st


def test_refusals_match_the_sync_call(sa):
    u = np.uint32
    xs = [_walk(u, m, seed=m) for m in (3 * (1 << 14), 5000, 20000, 7)]
    data, index, refs = _batch(sa, xs, _cfg(1))
    kw = dict(src_cap=len(data), index_cap=len(index))

    def same(bad_refs, code, file, dst_cap=None, d=data, ix=index, **more):
        got, err, werr, st = _refusal(sa, d, ix, u, bad_refs, dst_cap=dst_cap, **{**kw, **more})
        assert got is None and err == werr and err[1] == file and st.device_status == code, (err, werr, hex(st.device_status))

    r = refs.copy()
    r[2, 0] = len(data) - 3  # file 2 outside src ...
    r[1, 2] += 16            # ... while file 1 (earlier) has a bad header (its index is not its own): the ref check comes first
    same(r, 0x10f, 2)
    r = refs.copy()
    r[3, 2] += 8  # misaligned index offset
    same(r, 0x110, 3)
    r = refs.copy()
    r[1, 3] = len(index)  # index outside index_cap
    same(r, 0x111, 1)
    # a corrupt header and a short one
    bad = bytearray(data)
    bad[int(refs[2, 0])] ^= 0xff
    same(refs, 0x101, 2, d=bytes(bad))
    r = refs.copy()
    r[1, 1] = 3
    got, err, werr, st = _refusal(sa, data, index, u, r, **kw)
    assert err == werr == ("InsufficientData", 1) and st.device_status == 0x102
    # a foreign index: file 1 with file 2's index
    r = refs.copy()
    r[1, 2:] = refs[2, 2:]
    same(r, 0x104, 1)
    # misaligned entries: shift file 0's entries by 2 bytes
    bad = bytearray(index)
    base, co = int(refs[0, 2]), struct.unpack_from("<Q", index, int(refs[0, 2]) + 32)[0]
    eo = struct.unpack_from("<Q", bad, base + co + 16)[0]
    struct.pack_into("<Q", bad, base + co + 16, eo + 2)
    same(refs, 0x113, 0, ix=bytes(bad))
    # dst too small: Io naming the first file that does not fit, dst untouched
    total = sum(x.size for x in xs)
    same(refs, 0x115, 2, dst_cap=xs[0].size + xs[1].size + 19999)
    same(refs, 0x115, 3, dst_cap=total - 1)
    # a decode failure in file 1 while file 3 is also bad: file 1, and the sync call's kind
    bad = None
    rec0 = int(refs[1, 2]) + struct.unpack_from("<Q", index, int(refs[1, 2]) + 32)[0]
    first = int(refs[1, 0]) + struct.unpack_from("<Q", index, rec0)[0] + 8  # inside file 1's first chunk, past its header
    for p in range(first, int(refs[1, 0] + refs[1, 1])):  # the first byte there whose flip the sync call fails on
        cand = bytearray(data)
        cand[p] ^= 0xff
        if _sync(sa, bytes(cand), index, u, refs, total)[1] is not None:
            bad = cand
            break
    assert bad is not None
    r = refs.copy()
    r[3, 1] -= 1  # file 3's index no longer matches it
    got, err, werr, st = _refusal(sa, bytes(bad), index, u, r, **kw)
    assert err == werr and err[1] == 1 and st.device_status < 0x100 and st.n_written == 0, (err, werr)
    # with file 3 fine, the decode failure is the outcome, and n_written is the total
    got, err, werr, st = _refusal(sa, bytes(bad), index, u, refs, **kw)
    assert err == werr and err[1] == 1 and st.device_status < 0x100 and st.n_written == total, (err, werr)


def test_refusals_of_the_async_call_only(sa):
    u = np.uint32
    xs = [_walk(u, m, seed=m) for m in (3 * (1 << 14), 5000, 20000)]
    data, index, refs = _batch(sa, xs, _cfg(1))
    kw = dict(src_cap=len(data), index_cap=len(index))
    # no index: the sync call walks the file, this one refuses it
    r = refs.copy()
    r[1, 3] = 0
    got, err, st = _run(sa, data, index, u, r, dst_cap=1 << 20, **kw)
    assert err == ("Unsupported", 1) and st.device_status == 0x112
    assert _sync(sa, data, index, u, r, 1 << 20)[1] is None
    # a flavour mismatch: a uniform-type file in a batch planned from a plain header
    d2, i2, r2 = _batch(sa, [xs[1]], _cfg(1), uniform=True)
    data3, pad = data + d2, (-len(index)) % 16
    index3 = index + b"\0" * pad + i2
    r = np.concatenate([refs, r2 + np.array([[len(data), 0, len(index) + pad, 0]], np.uint64)])
    got, err, st = _run(sa, data3, index3, u, r, dst_cap=1 << 20, head=data[:32])
    assert err == ("InvalidArgument", 3) and st.device_status == 0x103
    # records outside their file: file 2's index made to count fewer numbers than its records hold
    bad = bytearray(index)
    struct.pack_into("<Q", bad, int(refs[2, 2]) + 16, xs[2].size - 1)
    got, err, st = _run(sa, data, bytes(bad), u, refs, dst_cap=1 << 20, **kw)
    assert err == ("InvalidArgument", 2) and st.device_status == 0x114
    # too many chunks: the first file that takes the running count past max_chunks
    nc = [_n_chunks(index, rr) for rr in refs]
    got, err, st = _run(sa, data, index, u, refs, max_chunks=nc[0] + nc[1], dst_cap=1 << 20, **kw)
    assert err == ("InvalidArgument", 2) and st.device_status == 0x105
    # too many files
    b = Bufs(sa, data[:32], u, len(data), len(index), 2, 64, 1 << 20)
    b.load(data, index, refs[:2])
    b.n.fill_(3)
    b.call()
    _, err, st = b.outcome()
    assert err == ("InvalidArgument", None) and st.device_status == 0x10e and st.n_files == 3


@pytest.mark.parametrize("order", [0, 1])
def test_bit_flips_never_crash_and_match_the_sync_call(sa, order):
    xs = [_walk(np.uint64, m, seed=order + m) for m in (3 * (1 << 14), 9000, 4000)]
    data, index, refs = _batch(sa, xs, _cfg(order))
    rng = np.random.default_rng(order)
    lo, hi = int(refs[1, 0]), int(refs[2, 0] + refs[2, 1])
    total = sum(x.size for x in xs)
    for pos in rng.integers(lo, hi, 24):
        bad = bytearray(data)
        bad[int(pos)] ^= 1 << int(rng.integers(0, 8))
        bad = bytes(bad)
        want, werr = _sync(sa, bad, index, np.uint64, refs, total)
        got, err, _ = _run(sa, bad, index, np.uint64, refs, dst_cap=total)
        assert err == werr, (int(pos), err, werr)
        if err is None:
            np.testing.assert_array_equal(bits_view(got[0]), bits_view(want[0]))
    _check(sa, data, index, xs, refs, [0, 1, 2], spare=False)


def test_profiled_call_records_its_kernels_in_order(sa):
    from pcodec_b200 import _lib

    xs = [_walk(np.float32, m, seed=m) for m in (3 * (1 << 14), 700)]
    data, index, refs = _batch(sa, xs, _cfg(1))
    L = _lib.lib()
    L.pco_b200_profile_enable(1)
    try:
        got, err, _ = _run(sa, data, index, np.float32, refs)
        buf = C.create_string_buffer(1 << 16)
        L.pco_b200_profile_last(buf, C.c_size_t(len(buf)))
    finally:
        L.pco_b200_profile_enable(0)
    assert err is None
    prof = buf.value.decode()
    at = [prof.find(k) for k in KERNELS]
    assert all(a >= 0 for a in at) and at == sorted(at), prof
