"""The asynchronous filter of indexed standalone files on the GPU (pco_b200_filter_files_async, standalone.AsyncFilesFilter): every
selection is compared with numpy's (x >= lo) & (x <= hi) (NaN-aware) over the numbers AsyncFilesDecompressor returns for the same refs
with dst_cap = rows_cap, which are checked against the input; every refusal with that call's kind, file and chunk."""
import ctypes as C
import math
import struct

import numpy as np
import pytest

from tests.golden_generators import GENERATORS, bits_view, load_assets
from tests.test_gpu_async_files import INDEXED_ASSETS, _batch, _cfg, _expect, _n_chunks, _run, _walk
from tests.test_gpu_async_filter_pages import _intervals, _want

pytestmark = pytest.mark.gpu

DTYPES = [np.uint8, np.int8, np.uint16, np.int16, np.float16, np.uint32, np.int32, np.float32, np.uint64, np.int64, np.float64]
SENTINEL = 0x5A
NONE = (1 << 64) - 1


@pytest.fixture(scope="module")
def sa():
    from pcodec_b200 import standalone

    return standalone


class _Filter:
    """One AsyncFilesFilter with its device buffers; values and positions have 64 sentinel elements past out_cap."""

    def __init__(self, sa, head, dtype, src_cap, index_cap, max_files, max_chunks, rows_cap, out_cap):
        import torch

        from pcodec_b200.wrapped import _torch_dtypes

        self.dtype, self.max_files, self.out_cap = np.dtype(dtype), max_files, out_cap
        self.f = sa.AsyncFilesFilter(head, dtype, src_cap, index_cap, max_files, max_chunks, rows_cap, out_cap)
        self.src = torch.zeros(max(src_cap, 1), dtype=torch.uint8, device="cuda")
        self.index = torch.zeros(max(index_cap, 1), dtype=torch.uint8, device="cuda")
        self.files = torch.zeros((max_files, 4), dtype=torch.int64, device="cuda")
        self.n = torch.zeros(1, dtype=torch.int64, device="cuda")
        self.iv = torch.zeros(2, dtype=torch.int64, device="cuda")
        self.vals = torch.zeros(((out_cap + 64) * self.dtype.itemsize,), dtype=torch.uint8, device="cuda").view(_torch_dtypes()[self.dtype])
        self.pos = torch.zeros(out_cap + 64, dtype=torch.int64, device="cuda")
        self.nm = torch.zeros(1, dtype=torch.int64, device="cuda")
        self.ns = torch.zeros(max_files + 64, dtype=torch.int64, device="cuda")

    def load(self, data, index, refs):
        import torch

        self.src.zero_()
        self.index.zero_()
        self.src[: len(data)] = torch.as_tensor(np.frombuffer(data, np.uint8).copy())
        self.index[: len(index)] = torch.as_tensor(np.frombuffer(index, np.uint8).copy())
        f = np.zeros((self.max_files, 4), np.uint64)
        if len(refs):
            f[: len(refs)] = np.asarray(refs, np.uint64).reshape(-1, 4)
        self.files.copy_(torch.as_tensor(f.view(np.int64)))
        self.n.fill_(len(refs))

    def bounds(self, lo, hi):
        import torch

        from pcodec_b200 import wrapped

        self.iv.copy_(torch.from_numpy(wrapped.pack_interval(lo, hi, self.dtype)))
        self.vals.view(torch.uint8).fill_(SENTINEL)
        self.pos.fill_(-1)
        self.nm.fill_(-7)
        self.ns.fill_(-3)

    def call(self, file_ns=True):
        self.f(self.src, self.index, self.files, self.n, self.iv, self.vals, self.pos, self.nm, self.ns[: self.max_files] if file_ns else None)

    def outcome(self):
        """(values, positions, count tensor value, file_ns, PcoError or None, status); asserts nothing was written past the matches."""
        from pcodec_b200 import PcoError

        st = self.f.status_record()
        try:
            self.f.result()
            err = None
        except PcoError as e:
            err = e
        vals, pos, nm = self.vals.cpu().numpy(), self.pos.cpu().numpy(), int(self.nm.item())
        k = int(st.n_matches)
        assert nm == k, (nm, k)
        assert (pos[k:] == -1).all() and (vals.view(np.uint8)[k * vals.itemsize:] == SENTINEL).all(), "written past the matches"
        ns = self.ns.cpu().numpy()
        assert (ns[self.max_files:] == -3).all(), "written past file_ns"
        return vals[:k], pos[:k], nm, ns[: self.max_files], err, st


def _head(data, refs):
    return data[int(refs[0][0]):int(refs[0][0]) + 32] if len(refs) else data[:32]


def _filter(sa, data, index, dtype, refs, lo, hi, max_files=None, max_chunks=None, rows_cap=None, out_cap=None, src_cap=None, index_cap=None,
            profile=False, file_ns=True):
    from pcodec_b200 import _lib

    nc = sum(_n_chunks(index, r) for r in refs)
    if rows_cap is None:
        rows_cap = sum(int(struct.unpack_from("<Q", index, int(r[2]) + 16)[0]) for r in refs)
    fl = _Filter(sa, _head(data, refs), dtype, src_cap or len(data), index_cap or len(index), max_files or max(len(refs), 1), max_chunks or max(nc, 1),
                 rows_cap, rows_cap if out_cap is None else out_cap)
    fl.load(data, index, refs)
    fl.bounds(lo, hi)
    L = _lib.lib()
    spans = ""
    if profile:
        L.pco_b200_profile_enable(1)
    try:
        fl.call(file_ns)
        out = fl.outcome()
        if profile:
            buf = C.create_string_buffer(1 << 16)
            L.pco_b200_profile_last(buf, C.c_size_t(len(buf)))
            spans = buf.value.decode()
    finally:
        if profile:
            L.pco_b200_profile_enable(0)
    return out + (spans,)


def _check(sa, data, index, refs, dtype, intervals, x=None, **kw):
    """Each interval's selection equals numpy's over the files call's output (itself checked against x when given), with file_ns."""
    dec, err, _ = _run(sa, data, index, dtype, refs, dst_cap=kw.get("rows_cap"), max_files=kw.get("max_files"), max_chunks=kw.get("max_chunks"))
    assert err is None, err
    if x is not None:
        np.testing.assert_array_equal(bits_view(dec[0]), bits_view(np.asarray(x, dtype=dtype)))
    for lo, hi in intervals:
        vals, pos, k, ns, err, st, _ = _filter(sa, data, index, dtype, refs, lo, hi, **kw)
        assert err is None, (lo, hi, err)
        want = _want(dec[0], lo, hi)
        assert k == len(want) == st.matches_needed, (lo, hi, k, len(want))
        np.testing.assert_array_equal(pos, want)
        np.testing.assert_array_equal(bits_view(vals), bits_view(dec[0][want]))
        assert st.n_written == len(dec[0]) and st.n_files == len(refs)
        np.testing.assert_array_equal(ns[: len(refs)].view(np.uint64), dec[1])
    return dec[0]


@pytest.mark.parametrize("dtype", DTYPES)
def test_every_dtype_on_a_mixed_batch(sa, dtype):
    """several chunks per file, an empty file, files repeated and out of order, exact and spare capacities"""
    xs = [_walk(dtype, m, seed=int(np.dtype(dtype).num) + i) for i, m in enumerate([3 * (1 << 14) + 777, 1, 0, 5000, 1 << 14, 257])]
    data, index, refs = _batch(sa, xs, _cfg(1))
    order = [4, 0, 0, 2, 5, 1, 3, 0]
    x = _expect(xs, order)
    iv = _intervals(x, dtype)
    _check(sa, data, index, refs[order], dtype, iv, x=x)
    nc = sum(_n_chunks(index, r) for r in refs[order])
    _check(sa, data, index, refs[order], dtype, iv[:3], x=x, max_files=len(order) + 300, max_chunks=2 * nc + 3, rows_cap=len(x) + 999,
           out_cap=len(x) + 5, src_cap=len(data) + 100, index_cap=len(index) + 64)


@pytest.mark.parametrize("dtype", [np.float16, np.float32, np.float64])
def test_floats_with_nan_payloads_zeros_and_infinities(sa, dtype):
    dt = np.dtype(dtype)
    ut = np.dtype(f"u{dt.itemsize}")
    rng = np.random.default_rng(7)
    x = (rng.normal(size=20000) * 10).astype(dt)
    special = np.array([math.inf, -math.inf, 0.0, -0.0, math.nan], dtype=dt)
    x[rng.integers(0, x.size, size=800)] = special[rng.integers(0, special.size, size=800)]
    xb = x.view(ut).copy()
    nan_ix = rng.integers(0, x.size, size=100)
    exp = {2: 0x7C00, 4: 0x7F800000, 8: 0x7FF0000000000000}[dt.itemsize]
    xb[nan_ix] = (exp | rng.integers(1, 1 << 9, size=100)).astype(ut) | (rng.integers(0, 2, size=100).astype(ut) << (8 * dt.itemsize - 1))
    x = xb.view(dt)
    xs = [x[:7000], x[7000:]]
    for order in (0, 1):
        data, index, refs = _batch(sa, xs, _cfg(order, page=4096))
        _check(sa, data, index, refs, dtype, _intervals(x, dtype) + [(-1.0, 1.0), (-0.0, -0.0), (0.0, 0.0), (2.0, -2.0)], x=x)


ROUTE_CASES = {
    # name: (dtype, arrays, config, the kernel that decodes them)
    "fused_order0": (np.uint32, lambda: [_walk(np.uint32, m, seed=m) for m in (70000, 300)], lambda: _cfg(0, page=1 << 15), "fused_narrow_kernel"),
    "fused_order1": (np.int64, lambda: [_walk(np.int64, m, seed=m) for m in (70000, 300)], lambda: _cfg(1, page=1 << 15), "fused_narrow_kernel"),
    "fused_order3": (np.int16, lambda: [_walk(np.int16, m, seed=m) for m in (70000, 300)], lambda: _cfg(3, page=1 << 15), "fused_narrow_kernel"),
    "fused_order7": (np.float32, lambda: [_walk(np.float32, m, seed=m) for m in (70000, 300)], lambda: _cfg(7, page=1 << 15), "fused_narrow_kernel"),
    "general_one_var": (np.uint64, lambda: [np.random.default_rng(5).integers(0, 1 << 40, size=m).astype(np.uint64) for m in (70000, 999)],
                        lambda: _cfg(0, page=1 << 15), "decode_kernel"),
    "general_int_mult": (np.uint32, lambda: [(_walk(np.uint32, m, seed=m).astype(np.uint64) // 8 * 8 + 3).astype(np.uint32) for m in (40000, 999)],
                         lambda: _cfg(1, mode="int_mult"), "decode_kernel"),
    "general_float_mult": (np.float64, lambda: [(np.round(np.cumsum(np.random.default_rng(m).normal(size=m)) * 100) * 0.01) for m in (40000, 999)],
                           lambda: _cfg(1, mode="float_mult"), "decode_kernel"),
    "cold_level9": (np.uint64, lambda: [np.random.default_rng(9).lognormal(10, 2, size=m).astype(np.uint64) for m in (3 * (1 << 16) + 5, 1000)],
                    lambda: _cfg(0, page=1 << 16, level=9), "ff_cold_kernel"),
    "cold_level12": (np.uint64, lambda: [np.random.default_rng(12).lognormal(10, 2, size=m).astype(np.uint64) for m in ((1 << 16) + 1, 1000)],
                     lambda: _cfg(0, page=1 << 16, level=12), "ff_cold_kernel"),
}
ORDER = ["ff_map_kernel", "af_files_kernel", "merge_index_kernel", "fused_narrow_kernel", "symwalk_kernel", "decode_kernel", "ff_cold_list_kernel",
         "cold_chunks_kernel", "af_finish_kernel", "ff_cold_kernel", "fl_count_kernel", "ff_finish_kernel", "fl_gather_kernel"]


@pytest.mark.parametrize("name", sorted(ROUTE_CASES))
def test_every_route_with_spans(sa, name):
    dtype, arrays, cfg, _ = ROUTE_CASES[name]
    xs = [np.asarray(a, dtype=dtype) for a in arrays()]
    data, index, refs = _batch(sa, xs, cfg())
    order = [1, 0, 1]
    x = _expect(xs, order)
    dec = _check(sa, data, index, refs[order], dtype, _intervals(x, dtype), x=x)
    s = np.sort(dec[~np.isnan(dec)] if np.dtype(dtype).kind == "f" else dec)
    _, _, k, _, err, _, spans = _filter(sa, data, index, dtype, refs[order], s[len(s) // 3], s[2 * len(s) // 3], profile=True)
    assert err is None and k > 0
    at = [spans.find(kn) for kn in ORDER]
    assert all(a >= 0 for a in at) and at == sorted(at), spans


def test_cold_chunks_are_the_catch_all_decoders(sa):
    """level-12 chunks go through the catch-all decoder: the fused kernel reports them Unsupported, and the filter still selects them"""
    dtype, arrays, cfg, _ = ROUTE_CASES["cold_level12"]
    xs = [np.asarray(a, dtype=dtype) for a in arrays()]
    data, index, refs = _batch(sa, xs, cfg())
    x = _expect(xs, [0, 1, 0])
    lo, hi = np.quantile(x, 0.4).astype(np.uint64), np.quantile(x, 0.45).astype(np.uint64)
    vals, pos, k, _, err, _, _ = _filter(sa, data, index, dtype, refs[[0, 1, 0]], lo, hi)
    want = _want(x, lo, hi)
    assert err is None and k == len(want) > 0
    np.testing.assert_array_equal(pos, want)
    np.testing.assert_array_equal(vals, x[want])


@pytest.mark.parametrize("name", INDEXED_ASSETS)
def test_golden_assets(sa, name):
    x = GENERATORS[name]()
    one = load_assets()[name]
    idx = sa.build_index(one, x.dtype)
    pad = (-len(idx)) % 16
    data, index = one + one, idx + b"\0" * pad + idx
    refs = np.array([[0, len(one), 0, len(idx)], [len(one), len(one), len(idx) + pad, len(idx)]], np.uint64)
    want = np.concatenate([x, x, x])
    numbers = want[~np.isnan(want)] if want.dtype.kind == "f" else want
    iv = _intervals(want, x.dtype)[:4] if numbers.size else [(-math.inf, math.inf), (math.nan, 1.0), (0.0, -0.0)]  # an asset of NaNs only
    _check(sa, data, index, refs[[0, 1, 1]], x.dtype, iv, x=want)


def test_chunk_sizes_1_to_2_20(sa):
    sizes = [1, 255, 256, 257, 1 << 20]
    xs = [_walk(np.int64, m, seed=m) for m in sizes]
    data, index, refs = _batch(sa, xs, _cfg(1, page=1 << 20))
    order = [4, 0, 2, 2, 1, 3, 0]
    x = _expect(xs, order)
    _check(sa, data, index, refs[order], np.int64, _intervals(x, np.int64)[:4], x=x)


def test_more_than_1000_small_chunks(sa):
    xs = [_walk(np.uint16, m, seed=m) for m in (1500 * 256 + 7, 300 * 256, 5)]
    data, index, refs = _batch(sa, xs, _cfg(0, page=256))
    assert _n_chunks(index, refs[0]) > 1000
    x = _expect(xs, [0, 1, 2, 1])
    _check(sa, data, index, refs[[0, 1, 2, 1]], np.uint16, _intervals(x, np.uint16)[:4], x=x)


def test_out_cap_at_below_and_far_below(sa):
    xs = [_walk(np.uint64, m, seed=m) for m in (3 * (1 << 14) + 7, 9000, 4000)]
    data, index, refs = _batch(sa, xs, _cfg(1))
    x = _expect(xs, [0, 1, 2])
    lo, hi = np.quantile(x, 0.2).astype(np.uint64), np.quantile(x, 0.7).astype(np.uint64)
    want = _want(x, lo, hi)
    k = len(want)
    for cap in (k, k - 1, k // 10, 1, 0):
        vals, pos, nm, ns, err, st, _ = _filter(sa, data, index, np.uint64, refs, lo, hi, out_cap=cap)
        assert st.matches_needed == k and st.n_matches == min(cap, k) == nm
        if cap >= k:
            assert err is None
        else:
            assert err is not None and err.kind == "Io" and str(k) in err.message and st.device_status == 0x201, err
        np.testing.assert_array_equal(pos, want[:cap])
        np.testing.assert_array_equal(vals, x[want[:cap]])
        np.testing.assert_array_equal(ns[:3], [a.size for a in xs])


def _same_failure(sa, data, index, refs, dtype=np.uint32, rows_cap=1 << 20, **kw):
    """The filter fails as pco_b200_decompress_files_async does with dst_cap = rows_cap (kind, device status, file and chunk) and writes
    no match and no file count."""
    _, werr, wst = _run(sa, data, index, dtype, refs, dst_cap=rows_cap, **kw)
    assert werr is not None
    _, _, k, ns, err, st, _ = _filter(sa, data, index, dtype, refs, 0, np.iinfo(dtype).max, rows_cap=rows_cap, out_cap=1 << 10, **kw)
    assert err is not None and err.kind == werr[0], (err, werr)
    assert (st.device_status, st.file, st.chunk, st.n_files, st.n_written) == (wst.device_status, wst.file, wst.chunk, wst.n_files, wst.n_written)
    assert k == 0 and st.matches_needed == 0 and (ns == -3).all()
    return st, err


def test_refusals_match_the_files_call(sa):
    u = np.uint32
    xs = [_walk(u, m, seed=m) for m in (3 * (1 << 14), 5000, 20000, 7)]
    data, index, refs = _batch(sa, xs, _cfg(1))
    kw = dict(src_cap=len(data), index_cap=len(index))
    r = refs.copy()
    r[2, 0] = len(data) - 3
    r[1, 2] += 16
    assert _same_failure(sa, data, index, r, **kw)[0].device_status == 0x10f
    r = refs.copy()
    r[3, 2] += 8
    assert _same_failure(sa, data, index, r, **kw)[0].device_status == 0x110
    r = refs.copy()
    r[1, 3] = len(index)
    assert _same_failure(sa, data, index, r, **kw)[0].device_status == 0x111
    bad = bytearray(data)
    bad[int(refs[2, 0])] ^= 0xff
    assert _same_failure(sa, bytes(bad), index, refs, **kw)[0].device_status == 0x101
    r = refs.copy()
    r[1, 1] = 3
    assert _same_failure(sa, data, index, r, **kw)[0].device_status == 0x102
    r = refs.copy()
    r[1, 2:] = refs[2, 2:]
    assert _same_failure(sa, data, index, r, **kw)[0].device_status == 0x104
    bad = bytearray(index)
    base, co = int(refs[0, 2]), struct.unpack_from("<Q", index, int(refs[0, 2]) + 32)[0]
    eo = struct.unpack_from("<Q", bad, base + co + 16)[0]
    struct.pack_into("<Q", bad, base + co + 16, eo + 2)
    assert _same_failure(sa, data, bytes(bad), refs, **kw)[0].device_status == 0x113
    r = refs.copy()
    r[1, 3] = 0
    assert _same_failure(sa, data, index, r, **kw)[0].device_status == 0x112
    bad = bytearray(index)
    struct.pack_into("<Q", bad, int(refs[2, 2]) + 16, xs[2].size - 1)
    assert _same_failure(sa, data, bytes(bad), refs, **kw)[0].device_status == 0x114
    nc = [_n_chunks(index, rr) for rr in refs]
    assert _same_failure(sa, data, index, refs, max_chunks=nc[0] + nc[1], **kw)[0].device_status == 0x105
    total = sum(x.size for x in xs)
    for cap, file in ((xs[0].size + xs[1].size + 19999, 2), (total - 1, 3)):
        st, err = _same_failure(sa, data, index, refs, rows_cap=cap, **kw)
        assert st.device_status == 0x115 and st.file == file and "rows_cap" in err.message, err
    # a uniform-type file in a batch planned from a plain header
    d2, i2, r2 = _batch(sa, [xs[1]], _cfg(1), uniform=True)
    pad = (-len(index)) % 16
    r = np.concatenate([refs, r2 + np.array([[len(data), 0, len(index) + pad, 0]], np.uint64)])
    assert _same_failure(sa, data + d2, index + b"\0" * pad + i2, r)[0].device_status == 0x103


def test_too_many_files(sa):
    xs = [_walk(np.uint32, m, seed=m) for m in (5000, 700, 20)]
    data, index, refs = _batch(sa, xs, _cfg(1))
    fl = _Filter(sa, data[:32], np.uint32, len(data), len(index), 2, 64, 1 << 16, 1 << 16)
    fl.load(data, index, refs[:2])
    fl.n.fill_(3)
    fl.bounds(0, 1 << 31)
    fl.call()
    _, _, k, ns, err, st = fl.outcome()
    assert err.kind == "InvalidArgument" and st.device_status == 0x10e and st.n_files == 3 and st.file == NONE and k == 0 and (ns == -3).all()


@pytest.mark.parametrize("order", [0, 1])
def test_bit_flips_match_the_files_call(sa, order):
    xs = [_walk(np.uint64, m, seed=order + m) for m in (3 * (1 << 14), 9000, 4000)]
    data, index, refs = _batch(sa, xs, _cfg(order))
    rng = np.random.default_rng(order)
    lo, hi = int(refs[1, 0]), int(refs[2, 0] + refs[2, 1])
    total = sum(x.size for x in xs)
    for p in rng.integers(lo, hi, 16):
        bad = bytearray(data)
        bad[int(p)] ^= 1 << int(rng.integers(0, 8))
        bad = bytes(bad)
        dec, werr, wst = _run(sa, bad, index, np.uint64, refs, dst_cap=total)
        qlo, qhi = np.uint64(1 << 20), np.uint64(1 << 62)
        vals, pos, k, _, err, st, _ = _filter(sa, bad, index, np.uint64, refs, qlo, qhi, rows_cap=total)
        if werr is None:
            assert err is None, (int(p), err)
            want = _want(dec[0], qlo, qhi)
            np.testing.assert_array_equal(pos, want)
            np.testing.assert_array_equal(vals, dec[0][want])
        else:
            assert err is not None and err.kind == werr[0] and (st.device_status, st.file, st.chunk) == (wst.device_status, wst.file, wst.chunk)
            assert k == 0


def test_file_ns_may_be_null(sa):
    xs = [_walk(np.int32, m, seed=m) for m in (5000, 20000, 1)]
    data, index, refs = _batch(sa, xs, _cfg(1))
    x = _expect(xs, [0, 1, 2])
    vals, pos, k, ns, err, _, _ = _filter(sa, data, index, np.int32, refs, -(1 << 20), 1 << 20, file_ns=False)
    want = _want(x, -(1 << 20), 1 << 20)
    assert err is None and k == len(want) and (ns == -3).all()
    np.testing.assert_array_equal(pos, want)


def test_graph_replays_new_refs_counts_and_bounds(sa):
    import torch

    from pcodec_b200 import _lib

    batches = []
    for s in (1, 2):
        xs = [_walk(np.uint32, 4000 * (i + 1) + s, seed=10 * s + i) for i in range(6)]
        batches.append((xs,) + _batch(sa, xs, _cfg(s - 1, page=4096)))
    src_cap = max(len(b[1]) for b in batches) + 64
    index_cap = max(len(b[2]) for b in batches) + 64
    fl = _Filter(sa, batches[0][1][:32], np.uint32, src_cap, index_cap, 8, 64, 1 << 18, 1 << 18)
    fl.load(*batches[0][1:])
    fl.bounds(0, 1)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fl.call()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fl.call()
    plans = [(0, [0, 1, 2, 3, 4, 5], 0.1, 0.9), (1, [5, 5, 0], 0.0, 0.5), (0, [], 0.0, 1.0), (1, [3], 0.5, 0.5), (0, [2, 0, 4, 1, 3, 5, 0], 0.9, 0.1)]
    for step, (k, order, qlo, qhi) in enumerate(plans):
        xs, data, index, refs = batches[k]
        fl.load(data, index, refs[order] if order else refs[:0])
        x = _expect(xs, order) if order else np.zeros(0, np.uint32)
        lo, hi = (np.quantile(x, qlo).astype(np.uint32), np.quantile(x, qhi).astype(np.uint32)) if order else (0, 5)
        fl.bounds(lo, hi)
        if step == 3:
            _lib.lib().pco_b200_thread_release()
        g.replay()
        torch.cuda.synchronize()
        vals, pos, nm, ns, err, st = fl.outcome()
        assert err is None, err
        want = _want(x, lo, hi)
        assert nm == len(want) and st.n_files == len(order)
        np.testing.assert_array_equal(pos, want)
        np.testing.assert_array_equal(vals, x[want])
        np.testing.assert_array_equal(ns[: len(order)], [xs[i].size for i in order])


def test_graph_of_compress_on_a_device_chosen_subset_then_filter(sa):
    """AsyncFilesCompressor writes the files of a subset a device gather picked, and AsyncFilesFilter filters them, in one graph."""
    import torch

    cfg = _cfg(1, page=4096)
    n_files, max_n = 8, 6000
    comp = sa.AsyncFilesCompressor(np.int32, cfg, n_files, n_files * max_n, max_n, index=True)
    fl = _Filter(sa, sa.simple_compress(np.zeros(10, np.int32), cfg)[:32], np.int32, comp.dst_cap, comp.index_cap, n_files, 64,
                 n_files * max_n, n_files * max_n)
    pool = [_walk(np.int32, max_n, seed=s) for s in range(16)]
    pool_dev = torch.as_tensor(np.stack(pool), device="cuda")
    sizes = torch.zeros(16, dtype=torch.int64, device="cuda")
    pick = torch.zeros(n_files, dtype=torch.int64, device="cuda")
    nums = torch.zeros(n_files * max_n, dtype=torch.int32, device="cuda")
    file_ns = torch.zeros(n_files, dtype=torch.int64, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")

    def step():
        chosen = pool_dev[pick]                                 # the subset, gathered on the device
        nums.copy_(chosen.reshape(-1))
        file_ns.copy_(sizes[pick])
        comp(nums, file_ns, cnt, fl.src[: comp.dst_cap], fl.index[: comp.index_cap], fl.files)
        fl.n.copy_(cnt)
        fl.call()

    fl.bounds(0, 1)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    rng = np.random.default_rng(4)
    for m in (8, 3, 1):
        p = rng.integers(0, 16, n_files)
        sz = rng.integers(1, max_n + 1, 16)
        pick.copy_(torch.as_tensor(p))
        sizes.copy_(torch.as_tensor(sz))
        cnt.fill_(m)
        # compress reads the files back to back from nums: file i is the first sz[p[i]] numbers behind files 0 .. i - 1
        packed = np.stack([pool[j] for j in p]).reshape(-1)
        offs = np.concatenate([[0], np.cumsum([sz[p[i]] for i in range(m)])])
        x = np.concatenate([packed[offs[i]:offs[i + 1]] for i in range(m)])
        lo, hi = int(np.quantile(x, 0.3)), int(np.quantile(x, 0.6))
        fl.bounds(lo, hi)
        g.replay()
        torch.cuda.synchronize()
        comp.result()
        vals, pos, k, ns, err, st = fl.outcome()
        assert err is None, err
        want = _want(x, lo, hi)
        assert k == len(want) > 0
        np.testing.assert_array_equal(pos, want)
        np.testing.assert_array_equal(vals, x[want])
        np.testing.assert_array_equal(ns[:m], [sz[p[i]] for i in range(m)])
