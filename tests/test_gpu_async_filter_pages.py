"""The asynchronous page filter on the GPU (pco_b200_filter_pages_async, wrapped.AsyncPagesFilter): every selection is compared with numpy's
(x >= lo) & (x <= hi) (NaN-aware) over the numbers AsyncPagesDecompressor returns for the same refs, which are the input; every refusal
with that call's kind and page."""
import ctypes as C
import math

import numpy as np
import pytest

from tests.golden_generators import bits_view
from tests.test_gpu_async_pages import _cold_batch, _dev, _refs_dev, _run as _pages_run
from tests.test_gpu_encode import _walk
from tests.test_gpu_wrapped_batch import _container, _mixed_chunks, _shuffled, _six_pages

pytestmark = pytest.mark.gpu

DTYPES = [np.uint8, np.int8, np.uint16, np.int16, np.float16, np.uint32, np.int32, np.float32, np.uint64, np.int64, np.float64]
SENTINEL = 0x5A


def _want(x, lo, hi):
    """numpy's selection: IEEE comparisons for floats (NaN never matches; -0.0 == +0.0)."""
    x = np.asarray(x)
    with np.errstate(invalid="ignore"):
        m = (x >= x.dtype.type(lo)) & (x <= x.dtype.type(hi))
    return np.nonzero(m)[0]


def _filter(metas, pages, refs, dtype, lo, hi, out_cap=None, max_pages=None, rows_cap=None, frame_cap=-1, n=None, profile=False):
    """The filter over host bytes copied to the device; returns (values, positions, n_matches tensor value, PcoError or None, status, spans)."""
    import torch

    from pcodec_b200 import PcoError, _lib, wrapped
    from pcodec_b200.wrapped import _torch_dtypes

    total = int(np.asarray(refs)["page_n"].sum()) if len(refs) else 0
    max_pages = max_pages or max(len(refs), 1)
    rows_cap = total if rows_cap is None else rows_cap
    out_cap = total if out_cap is None else out_cap
    if frame_cap == -1:
        frame_cap = 2 * (len(metas) + len(pages)) + 32 * max_pages
    f = wrapped.AsyncPagesFilter(dtype, len(metas), len(pages), max_pages, rows_cap, out_cap, frame_cap)
    tdt = _torch_dtypes()[np.dtype(dtype)]
    vals = torch.full(((out_cap + 64) * np.dtype(dtype).itemsize,), SENTINEL, dtype=torch.uint8, device="cuda").view(tdt)
    pos = torch.full((out_cap + 64,), -1, dtype=torch.int64, device="cuda")
    nm = torch.full((1,), -7, dtype=torch.int64, device="cuda")
    iv = torch.from_numpy(wrapped.pack_interval(lo, hi, dtype)).cuda()
    nt = torch.tensor([len(refs) if n is None else n], dtype=torch.int64).cuda()
    L = _lib.lib()
    if profile:
        L.pco_b200_profile_enable(1)
    try:
        f(_dev(metas), _dev(pages), _refs_dev(refs, max_pages), nt, iv, vals, pos, nm)
        st = f.status_record()
        spans = ""
        if profile:
            buf = C.create_string_buffer(16384)
            L.pco_b200_profile_last(buf, C.c_size_t(len(buf)))
            spans = buf.value.decode()
    finally:
        if profile:
            L.pco_b200_profile_enable(0)
    try:
        k, err = f.result(), None
    except PcoError as e:
        k, err = None, e
    return vals.cpu().numpy(), pos.cpu().numpy(), int(nm.item()), err, st, spans


def _check(metas, pages, refs, dtype, intervals, x=None, **kw):
    """Each interval's selection equals numpy's over the pages call's output (itself checked against x when given)."""
    got_all, nw, err, _ = _pages_run(metas, pages, refs, dtype)
    assert err is None, err
    dec = got_all[:nw]
    if x is not None:
        np.testing.assert_array_equal(bits_view(dec), bits_view(np.asarray(x, dtype=dtype)))
    for lo, hi in intervals:
        vals, pos, k, err, st, _ = _filter(metas, pages, refs, dtype, lo, hi, **kw)
        assert err is None, (lo, hi, err)
        want = _want(dec, lo, hi)
        assert k == len(want) == st.n_matches == st.matches_needed, (lo, hi, k, len(want))
        np.testing.assert_array_equal(pos[:k], want)
        np.testing.assert_array_equal(bits_view(vals[:k]), bits_view(dec[want]))
        assert (pos[k:] == -1).all() and (vals.view(np.uint8)[k * vals.itemsize:] == SENTINEL).all(), "written past the matches"
        assert st.n_written == nw
    return dec


def _intervals(x, dtype):
    dt = np.dtype(dtype)
    s = np.sort(x[~np.isnan(x)] if dt.kind == "f" else x)
    q = lambda f: s[min(int(f * (len(s) - 1)), len(s) - 1)]  # noqa: E731
    lim = np.finfo(dt) if dt.kind == "f" else np.iinfo(dt)
    out = [(q(0.3), q(0.6)), (q(0.5), q(0.5)), (lim.min, lim.max), (lim.min, lim.min), (lim.max, lim.max), (q(0.7), q(0.2)),
           (s[0], s[0]), (s[-1], s[-1])]
    if dt.kind == "f":
        out += [(-math.inf, math.inf), (math.nan, 1.0), (0.0, math.nan), (-0.0, 0.0), (0.0, -0.0), (math.inf, math.inf), (-math.inf, -math.inf),
                (-0.0, q(0.9))]
    return out


@pytest.mark.parametrize("dtype", DTYPES)
def test_every_dtype_on_a_mixed_batch(oracle, dtype):
    metas, pages, refs, pieces = _container(_mixed_chunks(oracle, dtype))
    refs, pieces = _shuffled(refs, pieces, seed=int(np.dtype(dtype).num))
    frames = int(sum((4 + r["meta_len"] + r["page_len"] + 15) // 16 * 16 for r in refs))
    x = np.concatenate(pieces)
    _check(metas, pages, refs, dtype, _intervals(x, dtype), x=x, frame_cap=frames)


@pytest.mark.parametrize("dtype", [np.float16, np.float32, np.float64])
def test_floats_with_nan_payloads_zeros_and_infinities(oracle, dtype):
    dt = np.dtype(dtype)
    ut = np.dtype(f"u{dt.itemsize}")
    rng = np.random.default_rng(7)
    x = (rng.normal(size=5000) * 10).astype(dt)
    special = np.array([math.inf, -math.inf, 0.0, -0.0, math.nan], dtype=dt)
    x[rng.integers(0, x.size, size=200)] = special[rng.integers(0, special.size, size=200)]
    xb = x.view(ut).copy()
    nan_ix = rng.integers(0, x.size, size=50)
    exp = {2: 0x7C00, 4: 0x7F800000, 8: 0x7FF0000000000000}[dt.itemsize]
    xb[nan_ix] = (exp | rng.integers(1, 1 << 9, size=50)).astype(ut) | (rng.integers(0, 2, size=50).astype(ut) << (8 * dt.itemsize - 1))
    x = xb.view(dt)
    O = oracle
    chunks = [(x[:3000], O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_NOOP)), (x[3000:], O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=1))]
    metas, pages, refs, pieces = _container(chunks)
    _check(metas, pages, refs, dtype, _intervals(x, dtype) + [(-1.0, 1.0), (-0.0, -0.0), (0.0, 0.0)], x=x)


def _routes(oracle):
    """Pages on every route: fused (order 1), the general pair (order 0 in one bin of wide offsets), level 12, cold Lookback / Dict / Conv1."""
    metas, pages, refs, pieces = _cold_batch(oracle)
    return metas, pages, refs, np.concatenate(pieces)


def test_every_route_with_spans(oracle):
    metas, pages, refs, x = _routes(oracle)
    refs2, _ = _shuffled(refs, [None] * len(refs), seed=3)
    for r in (refs, refs2):
        dec = _check(metas, pages, r, np.int32, _intervals(np.sort(x), np.int32))
    _, _, _, err, _, spans = _filter(metas, pages, refs, np.int32, int(np.median(dec)), int(np.max(dec)), profile=True)
    assert err is None
    order = ["ap_pages_kernel", "walk_kernel", "fused_narrow_kernel", "symwalk_kernel", "decode_kernel", "ap_cold_kernel", "ap_finish_kernel",
             "fl_cold_kernel", "fl_count_kernel", "fl_finish_kernel", "fl_gather_kernel"]
    at = [spans.find(k) for k in order]
    assert all(a >= 0 for a in at) and at == sorted(at), spans


def test_general_pair_and_fused_alone(oracle):
    """order 0 with wide offsets takes decode_kernel; order 1 takes fused_narrow_kernel (the class bytes decide, as in the pages call)."""
    O = oracle
    rng = np.random.default_rng(5)
    wide = rng.integers(0, 1 << 40, size=70000).astype(np.uint64)
    walk = np.cumsum(rng.geometric(0.01, size=70000)).astype(np.uint64)
    for x, cfg in [(wide, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_NOOP, max_page_n=1 << 15)),
                   (walk, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=1, max_page_n=1 << 15))]:
        metas, pages, refs, _ = _container([(x, cfg)])
        _check(metas, pages, refs, np.uint64, _intervals(x, np.uint64), x=x)


def test_page_sizes_repeats_and_shared_metas(oracle):
    O = oracle
    x = _walk(np.int64, (1 << 20) + 256 + 257 + 255 + 1, seed=12)
    sizes = [1, 255, 256, 257, 1 << 20]
    chunks, at = [], 0
    for s in sizes:
        chunks.append((x[at:at + s], O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=1, max_page_n=1 << 20)))
        at += s
    metas, pages, refs, pieces = _container(chunks)
    order = [4, 0, 2, 2, 1, 3, 0]  # repeats, out of order
    sel = refs[order]
    want = np.concatenate([pieces[i] for i in order])
    _check(metas, pages, sel, np.int64, _intervals(want, np.int64), x=want)
    # pages that share a meta: a classic chunk cut into several pages
    y = _walk(np.uint32, 9000, seed=2)
    m2, p2, r2, pc2 = _container([(y, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=1, max_page_n=1000))])
    assert len(set(r2["meta_offset"])) < len(r2)
    _check(m2, p2, r2[::-1], np.uint32, _intervals(y, np.uint32), x=np.concatenate(pc2[::-1]))


def test_out_cap_at_below_and_far_below(oracle):
    metas, pages, refs, pieces = _six_pages(oracle)
    x = np.concatenate(pieces)
    lo, hi = np.quantile(x, 0.2).astype(np.uint64), np.quantile(x, 0.7).astype(np.uint64)
    want = _want(x, lo, hi)
    k = len(want)
    for cap in (k, k - 1, k // 10, 1, 0):
        vals, pos, nm, err, st, _ = _filter(metas, pages, refs, np.uint64, lo, hi, out_cap=cap)
        assert st.matches_needed == k and st.n_matches == min(cap, k) and nm == min(cap, k)
        if cap >= k:
            assert err is None
        else:
            assert err is not None and err.kind == "Io" and str(k) in err.message and st.device_status == 0x201, err
        np.testing.assert_array_equal(pos[:min(cap, k)], want[:cap])
        np.testing.assert_array_equal(vals[:min(cap, k)], x[want[:cap]])
        assert (pos[min(cap, k):] == -1).all(), "written beyond out_cap"


def _same_failure(metas, pages, refs, dtype=np.uint64, **kw):
    """The filter fails as pco_b200_decompress_pages_async does (kind, device status and page) and writes no match."""
    _, _, perr, pst = _pages_run(metas, pages, refs, dtype, **{k: v for k, v in kw.items() if k in ("max_pages", "n", "frame_cap")},
                                 dst_cap=kw.get("rows_cap"))
    vals, pos, nm, err, st, _ = _filter(metas, pages, refs, dtype, 0, (1 << 64) - 1, **kw)
    assert perr is not None and err is not None, (perr, err)
    assert (err.kind, st.device_status, st.page) == (perr.kind, pst.device_status, pst.page), (err, perr)
    assert err.message.split(":")[0] == perr.message.split(":")[0], (err, perr)
    assert nm == 0 and st.n_matches == 0 and (pos == -1).all()
    return err, st


def test_refusals_match_the_pages_call(oracle):
    metas, pages, refs, pieces = _six_pages(oracle)
    total = sum(len(p) for p in pieces)
    _same_failure(metas, pages, refs, max_pages=len(refs), n=len(refs) + 1, rows_cap=total)
    for field, value in [("meta_offset", len(metas)), ("page_len", len(pages) + 1), ("page_n", 0), ("page_n", (1 << 24) + 1)]:
        bad = refs.copy()
        bad[4][field] = value
        bad[6]["page_offset"] = len(pages)
        err, st = _same_failure(metas, pages, bad, rows_cap=total + (1 << 25))
        assert st.page == 4
    err, st = _same_failure(metas, pages, refs, rows_cap=int(refs["page_n"][:3].sum()) + 1)
    assert st.page == 3 and "rows_cap" in err.message
    frames = int(sum((4 + r["meta_len"] + r["page_len"] + 15) // 16 * 16 for r in refs))
    err, st = _same_failure(metas, pages, refs, frame_cap=frames - 1, rows_cap=total)
    assert st.frames_needed == frames
    for cut in (1, int(refs[3]["page_len"]) // 2):
        bad = refs.copy()
        bad[3]["page_len"] -= cut
        _same_failure(metas, pages, bad, rows_cap=total)
    bad = refs.copy()
    bad[2]["meta_len"] = int(bad[2]["meta_len"]) + 1
    _same_failure(metas, pages, bad, rows_cap=total)
    buf = bytearray(metas)
    buf[int(refs[1]["meta_offset"])] = (buf[int(refs[1]["meta_offset"])] & 0xF0) | 0xE
    _same_failure(bytes(buf), pages, refs, rows_cap=total)


def test_bit_flips_match_the_pages_call(oracle):
    metas, pages, refs, pieces = _six_pages(oracle)
    rng = np.random.default_rng(1)
    for trial in range(16):
        k = int(rng.integers(0, len(refs)))
        buf = bytearray(pages)
        buf[int(refs[k]["page_offset"] + rng.integers(0, refs[k]["page_len"]))] ^= 1 << int(rng.integers(0, 8))
        got, nw, perr, pst = _pages_run(metas, bytes(buf), refs, np.uint64)
        vals, pos, nm, err, st, _ = _filter(metas, bytes(buf), refs, np.uint64, 0, (1 << 63))
        if perr is None:
            assert err is None, err
            np.testing.assert_array_equal(pos[:nm], _want(got[:nw], 0, 1 << 63))
        else:
            assert err is not None and (err.kind, st.page) == (perr.kind, pst.page), (trial, err, perr)


class _Batch:
    def __init__(self, dtype, metas_cap, pages_cap, max_pages, rows_cap, out_cap):
        import torch

        from pcodec_b200 import wrapped
        from pcodec_b200.wrapped import _torch_dtypes

        self.f = wrapped.AsyncPagesFilter(dtype, metas_cap, pages_cap, max_pages, rows_cap, out_cap, 2 * (metas_cap + pages_cap) + 32 * max_pages)
        self.dtype = dtype
        self.metas = torch.zeros(metas_cap, dtype=torch.uint8, device="cuda")
        self.pages = torch.zeros(pages_cap, dtype=torch.uint8, device="cuda")
        self.refs = torch.zeros((max_pages, 5), dtype=torch.int64, device="cuda")
        self.n = torch.zeros(1, dtype=torch.int64, device="cuda")
        self.iv = torch.zeros(2, dtype=torch.int64, device="cuda")
        self.vals = torch.zeros(out_cap, dtype=_torch_dtypes()[np.dtype(dtype)], device="cuda")
        self.pos = torch.zeros(out_cap, dtype=torch.int64, device="cuda")
        self.nm = torch.zeros(1, dtype=torch.int64, device="cuda")
        self.max_pages = max_pages

    def load(self, metas, pages, refs, lo, hi):
        import torch

        from pcodec_b200 import wrapped

        self.metas[: len(metas)].copy_(torch.frombuffer(bytearray(metas) + bytearray(1), dtype=torch.uint8)[: len(metas)])
        self.pages[: len(pages)].copy_(torch.frombuffer(bytearray(pages) + bytearray(1), dtype=torch.uint8)[: len(pages)])
        self.refs.copy_(_refs_dev(refs, self.max_pages))
        self.n.fill_(len(refs))
        self.iv.copy_(torch.from_numpy(wrapped.pack_interval(lo, hi, self.dtype)))

    def call(self):
        self.f(self.metas, self.pages, self.refs, self.n, self.iv, self.vals, self.pos, self.nm)


def test_graph_replays_new_refs_counts_and_bounds(oracle):
    import torch

    from pcodec_b200 import _lib

    batches = [_six_pages(oracle), _container(_mixed_chunks(oracle, np.uint64))]
    b = _Batch(np.uint64, 1 << 14, 1 << 22, 32, 1 << 20, 1 << 20)
    b.load(*batches[0][:3], 0, 1)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        b.call()
    plans = [(0, [0, 1, 2, 3, 4, 5, 6, 7], 0.1, 0.9), (1, [5, 5, 0], 0.0, 0.5), (0, [], 0.0, 1.0), (1, [3, 9, 1], 0.5, 0.5), (0, [7, 0, 4], 0.9, 0.1)]
    for step, (k, order, qlo, qhi) in enumerate(plans):
        metas, pages, refs, pieces = batches[k]
        sel = refs[order] if order else refs[:0]
        x = np.concatenate([pieces[i] for i in order]) if order else np.zeros(0, np.uint64)
        lo, hi = (np.quantile(x, qlo).astype(np.uint64), np.quantile(x, qhi).astype(np.uint64)) if order else (0, 5)
        b.load(metas, pages, sel, lo, hi)
        if step == 2:
            _lib.lib().pco_b200_thread_release()
        g.replay()
        torch.cuda.synchronize()
        nm = b.f.result()
        want = _want(x, lo, hi)
        assert nm == len(want) == int(b.nm.item())
        np.testing.assert_array_equal(b.pos[:nm].cpu().numpy(), want)
        np.testing.assert_array_equal(b.vals[:nm].cpu().numpy(), x[want])


def test_graph_of_compress_then_filter():
    """AsyncChunksCompressor writes the pages a following AsyncPagesFilter reads, both captured in one graph."""
    import torch

    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec, wrapped

    cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(1), paging_spec=PagingSpec.equal_pages_up_to(1 << 14))
    n_cap = 1 << 17
    comp = wrapped.AsyncChunksCompressor(np.int32, cfg, 4, n_cap, n_cap)
    f = wrapped.AsyncPagesFilter(np.int32, comp.metas_cap, comp.pages_cap, comp.max_chunks, n_cap, n_cap)
    nums = torch.zeros(n_cap, dtype=torch.int32, device="cuda")
    array_ns = torch.zeros(4, dtype=torch.int64, device="cuda")
    n_arrays = torch.ones(1, dtype=torch.int64, device="cuda")
    metas = torch.zeros(comp.metas_cap, dtype=torch.uint8, device="cuda")
    pages = torch.zeros(comp.pages_cap, dtype=torch.uint8, device="cuda")
    refs = torch.zeros((comp.max_chunks, 5), dtype=torch.int64, device="cuda")
    first = torch.zeros(5, dtype=torch.int64, device="cuda")
    iv = torch.zeros(2, dtype=torch.int64, device="cuda")
    vals = torch.zeros(n_cap, dtype=torch.int32, device="cuda")
    pos = torch.zeros(n_cap, dtype=torch.int64, device="cuda")
    nm = torch.zeros(1, dtype=torch.int64, device="cuda")
    n_chunks = first[1:2]  # one array: its chunks are refs[0 : first[1]]
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        comp(nums, array_ns, n_arrays, metas, pages, refs, first)
        f(metas, pages, refs, n_chunks, iv, vals, pos, nm)
    for seed, n in [(1, 100000), (2, 5000), (3, n_cap)]:
        x = _walk(np.int32, n, seed=seed)
        nums[:n].copy_(torch.from_numpy(x))
        array_ns[0] = n
        lo, hi = int(np.quantile(x, 0.25)), int(np.quantile(x, 0.3))
        iv.copy_(torch.from_numpy(wrapped.pack_interval(lo, hi, np.int32)))
        g.replay()
        torch.cuda.synchronize()
        comp.result()
        k = f.result()
        want = _want(x, lo, hi)
        assert k == len(want)
        np.testing.assert_array_equal(pos[:k].cpu().numpy(), want)
        np.testing.assert_array_equal(vals[:k].cpu().numpy(), x[want])
