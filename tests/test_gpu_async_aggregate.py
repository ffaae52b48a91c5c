"""The asynchronous aggregates on the GPU (pco_b200_aggregate_pages_async / _files_async, wrapped.AsyncPagesAggregate,
standalone.AsyncFilesAggregate): every record is compared with tests/aggregate_reference.py over the numbers the matching decompress call
returns for the same refs: counts, min and max bits and integer sums exactly, float sums bit for bit in the specified order; every refusal
with that call's kind and page / file."""
import ctypes as C
import math
import struct

import numpy as np
import pytest

from tests import aggregate_reference as ref
from tests.test_gpu_async_files import _batch, _cfg, _n_chunks, _run as _files_run, _walk as _files_walk
from tests.test_gpu_async_filter_files import sa  # noqa: F401  (fixture)
from tests.test_gpu_async_filter_pages import _intervals
from tests.test_gpu_async_pages import _cold_batch, _dev, _refs_dev, _run as _pages_run
from tests.test_gpu_encode import _walk
from tests.test_gpu_wrapped_batch import _container, _mixed_chunks, _shuffled, _six_pages

pytestmark = pytest.mark.gpu

DTYPES = [np.uint8, np.int8, np.uint16, np.int16, np.float16, np.uint32, np.int32, np.float32, np.uint64, np.int64, np.float64]
UNTOUCHED = 0x5A5A5A5A5A5A5A5A


def _spans(L):
    buf = C.create_string_buffer(1 << 16)
    L.pco_b200_profile_last(buf, C.c_size_t(len(buf)))
    return buf.value.decode()


def _outcome(call, agg, max_groups, profile):
    import torch

    from pcodec_b200 import PcoError, _lib

    aggs = torch.full((max_groups, 6), UNTOUCHED, dtype=torch.int64, device="cuda")
    tot = torch.full((6,), UNTOUCHED, dtype=torch.int64, device="cuda")
    L = _lib.lib()
    if profile:
        L.pco_b200_profile_enable(1)
    try:
        call(aggs, tot)
        st = agg.status_record()
        spans = _spans(L) if profile else ""
    finally:
        if profile:
            L.pco_b200_profile_enable(0)
    try:
        k, err = agg.result(), None
    except PcoError as e:
        k, err = None, e
    return aggs.cpu().numpy(), tot.cpu().numpy(), k, err, st, spans


def _frames(metas, pages, refs, max_pages):
    """Room for every framed page (pages that share a meta each frame a copy of it) and the pad frame."""
    return int(sum((4 + int(r["meta_len"]) + int(r["page_len"]) + 15) // 16 * 16 for r in refs)) + 2 * (len(metas) + len(pages)) + 32 * max_pages


def _agg_pages(metas, pages, refs, dtype, lo, hi, max_pages=None, rows_cap=None, frame_cap=-1, n=None, profile=False):
    import torch

    from pcodec_b200 import wrapped

    total = int(np.asarray(refs)["page_n"].sum()) if len(refs) else 0
    max_pages = max_pages or max(len(refs), 1)
    rows_cap = total if rows_cap is None else rows_cap
    if frame_cap == -1:
        frame_cap = _frames(metas, pages, refs, max_pages)
    a = wrapped.AsyncPagesAggregate(dtype, len(metas), len(pages), max_pages, rows_cap, frame_cap)
    iv = torch.from_numpy(wrapped.pack_interval(lo, hi, dtype)).cuda()
    nt = torch.tensor([len(refs) if n is None else n], dtype=torch.int64).cuda()
    m, p, r = _dev(metas), _dev(pages), _refs_dev(refs, max_pages)
    return _outcome(lambda aggs, tot: a(m, p, r, nt, iv, aggs, tot), a, max_pages, profile)


def _check_records(aggs, tot, k, groups, dtype, lo, hi):
    """groups: per group, (its numbers, its pages' / chunks' lengths)."""
    floats = np.dtype(dtype).kind == "f"
    want = [ref.record(x, pieces, lo, hi) for x, pieces in groups]
    for g, (w, _) in enumerate(want):
        assert ref.same(aggs[g], w, floats), (g, lo, hi, [int(v) & ref.MASK64 for v in aggs[g]], w)
    assert (aggs[len(groups):].view(np.uint64) == UNTOUCHED).all(), "records past the count written"
    wt = ref.total(want, dtype)
    assert ref.same(tot, wt, floats), (lo, hi, [int(v) & ref.MASK64 for v in tot], wt)
    assert k == wt[1]


def _check_pages(metas, pages, refs, dtype, intervals, **kw):
    got, nw, err, _ = _pages_run(metas, pages, refs, dtype, frame_cap=_frames(metas, pages, refs, max(len(refs), 1)))
    assert err is None, err
    dec = got[:nw]
    groups, at = [], 0
    for n in np.asarray(refs)["page_n"].tolist():
        groups.append((dec[at:at + n], [n]))
        at += n
    for lo, hi in intervals:
        aggs, tot, k, err, st, _ = _agg_pages(metas, pages, refs, dtype, lo, hi, **kw)
        assert err is None, (lo, hi, err)
        _check_records(aggs, tot, k, groups, dtype, lo, hi)
        assert st.n_written == nw and st.n_matches == k
    return dec


@pytest.mark.parametrize("dtype", DTYPES)
def test_every_dtype_on_a_mixed_batch_of_pages(oracle, dtype):
    metas, pages, refs, pieces = _container(_mixed_chunks(oracle, dtype))
    refs, pieces = _shuffled(refs, pieces, seed=int(np.dtype(dtype).num))
    frames = int(sum((4 + r["meta_len"] + r["page_len"] + 15) // 16 * 16 for r in refs))
    _check_pages(metas, pages, refs, dtype, _intervals(np.concatenate(pieces), dtype), frame_cap=frames)


@pytest.mark.parametrize("dtype", [np.float16, np.float32, np.float64])
def test_floats_with_nan_payloads_zeros_infinities_and_nan_sums(oracle, dtype):
    dt = np.dtype(dtype)
    ut = np.dtype(f"u{dt.itemsize}")
    rng = np.random.default_rng(7)
    x = (rng.normal(size=5000) * 10).astype(dt)
    special = np.array([math.inf, -math.inf, 0.0, -0.0, math.nan], dtype=dt)
    x[rng.integers(0, x.size, size=200)] = special[rng.integers(0, special.size, size=200)]
    xb = x.view(ut).copy()
    exp = {2: 0x7C00, 4: 0x7F800000, 8: 0x7FF0000000000000}[dt.itemsize]
    xb[rng.integers(0, x.size, size=50)] = (exp | rng.integers(1, 1 << 9, size=50)).astype(ut)
    x = xb.view(dt)
    O = oracle
    chunks = [(x[:3000], O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_NOOP)), (x[3000:], O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=1))]
    metas, pages, refs, _ = _container(chunks)
    # (-inf, inf) sums +inf and -inf to NaN; (-0.0, -0.0) selects only zeros, whose sum is +0.0
    _check_pages(metas, pages, refs, dtype, _intervals(x, dtype) + [(-1.0, 1.0), (-0.0, -0.0), (0.0, 0.0), (-math.inf, math.inf), (1.0, math.inf)])


@pytest.mark.parametrize("dtype", [np.uint64, np.int64])
def test_sums_that_need_the_high_word(oracle, dtype):
    O = oracle
    rng = np.random.default_rng(3)
    if dtype == np.uint64:
        x = rng.integers(1 << 62, (1 << 64) - 1, size=20000, dtype=np.uint64)
    else:
        x = rng.integers(-(1 << 63), -(1 << 61), size=20000, dtype=np.int64)
    metas, pages, refs, _ = _container([(x, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_NOOP, max_page_n=6000))])
    lim = np.iinfo(dtype)
    _check_pages(metas, pages, refs, dtype, [(lim.min, lim.max), (x.min(), np.sort(x)[15000])])


def test_every_route_with_spans(oracle):
    metas, pages, refs, pieces = _cold_batch(oracle)
    x = np.concatenate(pieces)
    dec = _check_pages(metas, pages, refs, np.int32, _intervals(np.sort(x), np.int32))
    *_, err, _, spans = _agg_pages(metas, pages, refs, np.int32, int(np.median(dec)), int(np.max(dec)), profile=True)
    assert err is None
    order = ["ap_pages_kernel", "walk_kernel", "fused_narrow_kernel", "symwalk_kernel", "decode_kernel", "ap_cold_kernel", "ap_finish_kernel",
             "fl_cold_kernel", "ag_pages_kernel", "ag_finish_kernel"]
    at = [spans.find(k) for k in order]
    assert all(a >= 0 for a in at) and at == sorted(at), spans


def test_a_page_of_2_24_and_many_small_pages(oracle):
    O = oracle
    x = _walk(np.uint32, 1 << 24, seed=4)
    metas, pages, refs, _ = _container([(x, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=1, max_page_n=1 << 24))])
    assert len(refs) == 1
    _check_pages(metas, pages, refs, np.uint32, [(np.uint32(0), np.uint32((1 << 32) - 1)), (x[1000], x[(1 << 24) - 1000])])
    y = _walk(np.float32, 1100 * 37, seed=5)
    m2, p2, r2, _ = _container([(y, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=1, max_page_n=37))])
    assert len(r2) >= 1000
    _check_pages(m2, p2, r2, np.float32, [(-math.inf, math.inf), (float(np.median(y)), math.inf)])


def _same_failure(metas, pages, refs, **kw):
    _, _, perr, pst = _pages_run(metas, pages, refs, np.uint64, **{k: v for k, v in kw.items() if k in ("max_pages", "n", "frame_cap")},
                                 dst_cap=kw.get("rows_cap"))
    aggs, tot, _, err, st, _ = _agg_pages(metas, pages, refs, np.uint64, 0, (1 << 64) - 1, **kw)
    assert perr is not None and err is not None, (perr, err)
    assert (err.kind, st.device_status, st.page) == (perr.kind, pst.device_status, pst.page), (err, perr)
    assert err.message.split(":")[0] == perr.message.split(":")[0], (err, perr)
    assert (tot == 0).all() and (aggs.view(np.uint64) == UNTOUCHED).all() and st.n_matches == 0
    return err, st


def test_refusals_and_bit_flips_match_the_pages_call(oracle):
    metas, pages, refs, pieces = _six_pages(oracle)
    total = sum(len(p) for p in pieces)
    _same_failure(metas, pages, refs, max_pages=len(refs), n=len(refs) + 1, rows_cap=total)
    bad = refs.copy()
    bad[4]["page_n"] = 0
    assert _same_failure(metas, pages, bad, rows_cap=total)[1].page == 4
    err, st = _same_failure(metas, pages, refs, rows_cap=int(refs["page_n"][:3].sum()) + 1)
    assert st.page == 3 and "rows_cap" in err.message
    bad = refs.copy()
    bad[3]["page_len"] -= 1
    _same_failure(metas, pages, bad, rows_cap=total)
    rng = np.random.default_rng(1)
    for trial in range(8):
        k = int(rng.integers(0, len(refs)))
        buf = bytearray(pages)
        buf[int(refs[k]["page_offset"] + rng.integers(0, refs[k]["page_len"]))] ^= 1 << int(rng.integers(0, 8))
        _, _, perr, pst = _pages_run(metas, bytes(buf), refs, np.uint64)
        _, tot, _, err, st, _ = _agg_pages(metas, bytes(buf), refs, np.uint64, 0, 1 << 63)
        assert (perr is None) == (err is None), (trial, err, perr)
        if perr is not None:
            assert (err.kind, st.page) == (perr.kind, pst.page) and (tot == 0).all(), (trial, err, perr)


def test_identical_calls_give_identical_records(oracle):
    metas, pages, refs, pieces = _container(_mixed_chunks(oracle, np.float32))
    x = np.concatenate(pieces)
    a = _agg_pages(metas, pages, refs, np.float32, float(np.nanmin(x)), float(np.nanmax(x)))
    b = _agg_pages(metas, pages, refs, np.float32, float(np.nanmin(x)), float(np.nanmax(x)))
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_graph_replays_new_refs_counts_and_bounds(oracle):
    import torch

    from pcodec_b200 import wrapped

    metas, pages, refs, pieces = _six_pages(oracle)
    mp, total = len(refs), sum(len(p) for p in pieces)
    a = wrapped.AsyncPagesAggregate(np.uint64, len(metas), len(pages), mp, total)
    d_m, d_p, d_r = _dev(metas), _dev(pages), _refs_dev(refs, mp)
    nt = torch.tensor([mp], dtype=torch.int64, device="cuda")
    iv = torch.zeros(2, dtype=torch.int64, device="cuda")
    aggs = torch.zeros((mp, 6), dtype=torch.int64, device="cuda")
    tot = torch.zeros(6, dtype=torch.int64, device="cuda")
    a(d_m, d_p, d_r, nt, iv, aggs, tot)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        a(d_m, d_p, d_r, nt, iv, aggs, tot)
    rng = np.random.default_rng(2)
    for trial in range(4):
        order = rng.permutation(mp)[: int(rng.integers(1, mp + 1))]
        sel = refs[order]
        xs = [pieces[i] for i in order]
        x = np.concatenate(xs)
        lo, hi = np.sort(x)[len(x) // 5], np.sort(x)[len(x) * 3 // 4]
        d_r.copy_(_refs_dev(sel, mp))
        nt.fill_(len(sel))
        iv.copy_(torch.from_numpy(wrapped.pack_interval(lo, hi, np.uint64)))
        g.replay()
        k = a.result()
        _check_records(aggs.cpu().numpy()[: len(sel)], tot.cpu().numpy(), k, [(p, [len(p)]) for p in xs], np.uint64, lo, hi)


# ---- files


def _agg_files(sa, data, index, dtype, refs, lo, hi, max_files=None, max_chunks=None, rows_cap=None, profile=False):
    import torch

    from pcodec_b200 import wrapped

    nc = sum(_n_chunks(index, r) for r in refs)
    if rows_cap is None:
        rows_cap = sum(int(struct.unpack_from("<Q", index, int(r[2]) + 16)[0]) for r in refs)
    mf = max_files or max(len(refs), 1)
    head = data[int(refs[0][0]):int(refs[0][0]) + 32] if len(refs) else data[:32]
    a = sa.AsyncFilesAggregate(head, dtype, len(data), len(index), mf, max_chunks or max(nc, 1), rows_cap)
    d_data = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    d_index = torch.frombuffer(bytearray(index), dtype=torch.uint8).cuda()
    fr = np.zeros((mf, 4), np.uint64)
    fr[: len(refs)] = refs
    d_files = torch.from_numpy(fr.view(np.int64)).cuda()
    nt = torch.tensor([len(refs)], dtype=torch.int64, device="cuda")
    iv = torch.from_numpy(wrapped.pack_interval(lo, hi, dtype)).cuda()
    return _outcome(lambda aggs, tot: a(d_data, d_index, d_files, nt, iv, aggs, tot), a, mf, profile)


def _chunk_ns(index, r):
    """The numbers of each chunk of one file, from its side index's records."""
    nc = _n_chunks(index, r)
    base = int(r[2]) + struct.unpack_from("<Q", index, int(r[2]) + 32)[0]
    return [struct.unpack_from("<I", index, int(base) + 32 * c + 8)[0] for c in range(nc)]


def _check_files(sa, data, index, refs, dtype, intervals, **kw):
    dec, err, _ = _files_run(sa, data, index, dtype, refs)
    assert err is None, err
    groups, at = [], 0
    for r, n in zip(refs, dec[1].tolist()):
        groups.append((dec[0][at:at + n], _chunk_ns(index, r)))
        assert sum(groups[-1][1]) == n
        at += n
    for lo, hi in intervals:
        aggs, tot, k, err, st, _ = _agg_files(sa, data, index, dtype, refs, lo, hi, **kw)
        assert err is None, (lo, hi, err)
        _check_records(aggs, tot, k, groups, dtype, lo, hi)
        assert st.n_written == len(dec[0]) and st.n_files == len(refs)
    return dec[0]


@pytest.mark.parametrize("dtype", DTYPES)
def test_every_dtype_on_a_batch_of_files(sa, dtype):  # noqa: F811
    xs = [_files_walk(dtype, m, seed=int(np.dtype(dtype).num) + i) for i, m in enumerate([3 * (1 << 14) + 777, 1, 0, 5000, 1 << 14, 257])]
    data, index, refs = _batch(sa, xs, _cfg(1))
    _check_files(sa, data, index, refs, dtype, _intervals(np.concatenate(xs), dtype))


def test_files_refusals_and_spans(sa):  # noqa: F811
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec

    xs = [_walk(np.uint32, s, seed=s) for s in (9000, 20000, 700)]
    cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.no_op(), paging_spec=PagingSpec.equal_pages_up_to(4096))
    data, index, refs = _batch(sa, xs, cfg)
    *_, err, _, spans = _agg_files(sa, data, index, np.uint32, refs, 0, (1 << 32) - 1, profile=True)
    assert err is None
    order = ["ff_map_kernel", "af_files_kernel", "fused_narrow_kernel", "decode_kernel", "ff_cold_list_kernel", "cold_chunks_kernel",
             "af_finish_kernel", "ff_cold_kernel", "ag_files_kernel", "agf_finish_kernel"]
    at = [spans.find(k) for k in order]
    assert all(a >= 0 for a in at) and at == sorted(at), spans
    for kw in ({"rows_cap": 9000 + 100}, {"max_chunks": 2}):
        _, perr, pst = _files_run(sa, data, index, np.uint32, refs, dst_cap=kw.get("rows_cap"), max_chunks=kw.get("max_chunks"))
        aggs, tot, _, err, st, _ = _agg_files(sa, data, index, np.uint32, refs, 0, (1 << 32) - 1, **kw)
        assert perr is not None and err is not None and (err.kind, st.device_status, st.file, st.chunk) == (perr[0], pst.device_status, pst.file, pst.chunk)
        assert (tot == 0).all() and (aggs.view(np.uint64) == UNTOUCHED).all()
    bad = bytearray(data)
    bad[int(refs[1][0]) + int(refs[1][1]) // 2] ^= 0x10
    _, perr, pst = _files_run(sa, bytes(bad), index, np.uint32, refs)
    aggs, tot, _, err, st, _ = _agg_files(sa, bytes(bad), index, np.uint32, refs, 0, (1 << 32) - 1)
    assert (perr is None) == (err is None)
    if perr is not None:
        assert (err.kind, st.file, st.chunk) == (perr[0], pst.file, pst.chunk) and (tot == 0).all()


@pytest.mark.parametrize("name", ["cold_level9", "cold_level12"])
def test_files_with_cold_chunks(sa, name):  # noqa: F811
    """Chunks the fast kernels leave to the catch-all decoder: cold_chunks_kernel stages them and ff_cold_kernel<L, true> reduces them."""
    from tests.test_gpu_async_filter_files import ROUTE_CASES

    dtype, arrays, cfg, _ = ROUTE_CASES[name]
    xs = [np.asarray(a, dtype=dtype) for a in arrays()]
    data, index, refs = _batch(sa, xs, cfg())
    sel = refs[[1, 0, 1]]
    dec = _check_files(sa, data, index, sel, dtype, _intervals(np.concatenate([xs[1], xs[0], xs[1]]), dtype))
    s = np.sort(dec)
    *_, err, _, spans = _agg_files(sa, data, index, dtype, sel, s[len(s) // 3], s[2 * len(s) // 3], profile=True)
    assert err is None and "ff_cold_kernel" in spans and "cold_chunks_kernel" in spans, spans


def test_files_graph_replays_new_refs_counts_and_bounds(sa):  # noqa: F811
    import torch

    from pcodec_b200 import wrapped

    xs = [_files_walk(np.int64, m, seed=m) for m in (70000, 1, 5000, 1 << 16, 300)]
    data, index, refs = _batch(sa, xs, _cfg(1))
    mf, nc = 8, 64
    rows = 4 * sum(len(x) for x in xs)
    a = sa.AsyncFilesAggregate(data[:32], np.int64, len(data), len(index), mf, nc, rows)
    d_data = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    d_index = torch.frombuffer(bytearray(index), dtype=torch.uint8).cuda()
    d_files = torch.zeros((mf, 4), dtype=torch.int64, device="cuda")
    nt = torch.zeros(1, dtype=torch.int64, device="cuda")
    iv = torch.zeros(2, dtype=torch.int64, device="cuda")
    aggs = torch.zeros((mf, 6), dtype=torch.int64, device="cuda")
    tot = torch.zeros(6, dtype=torch.int64, device="cuda")
    d_files[:1] = torch.from_numpy(refs[:1].view(np.int64))
    nt.fill_(1)
    a(d_data, d_index, d_files, nt, iv, aggs, tot)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        a(d_data, d_index, d_files, nt, iv, aggs, tot)
    rng = np.random.default_rng(4)
    for trial in range(4):
        order = rng.integers(0, len(refs), size=int(rng.integers(1, mf + 1)))
        sel = refs[order]
        x = np.concatenate([xs[i] for i in order])
        lo, hi = np.sort(x)[len(x) // 7], np.sort(x)[len(x) * 5 // 6]
        d_files.zero_()
        d_files[: len(sel)] = torch.from_numpy(sel.view(np.int64))
        nt.fill_(len(sel))
        iv.copy_(torch.from_numpy(wrapped.pack_interval(lo, hi, np.int64)))
        g.replay()
        k = a.result()
        groups = [(xs[i], _chunk_ns(index, refs[i])) for i in order]
        _check_records(aggs.cpu().numpy()[: len(sel)], tot.cpu().numpy(), k, groups, np.int64, lo, hi)


@pytest.mark.parametrize("dtype", [np.int32, np.float32])
def test_graph_of_compress_then_aggregate(dtype):
    """AsyncChunksCompressor writes the pages a following AsyncPagesAggregate reads, both captured in one graph."""
    import torch

    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec, wrapped
    from pcodec_b200.wrapped import _torch_dtypes

    cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(1), paging_spec=PagingSpec.equal_pages_up_to(1 << 14))
    n_cap = 1 << 17
    comp = wrapped.AsyncChunksCompressor(dtype, cfg, 4, n_cap, n_cap)
    a = wrapped.AsyncPagesAggregate(dtype, comp.metas_cap, comp.pages_cap, comp.max_chunks, n_cap)
    nums = torch.zeros(n_cap, dtype=_torch_dtypes()[np.dtype(dtype)], device="cuda")
    array_ns = torch.zeros(4, dtype=torch.int64, device="cuda")
    n_arrays = torch.ones(1, dtype=torch.int64, device="cuda")
    metas = torch.zeros(comp.metas_cap, dtype=torch.uint8, device="cuda")
    pages = torch.zeros(comp.pages_cap, dtype=torch.uint8, device="cuda")
    refs = torch.zeros((comp.max_chunks, 5), dtype=torch.int64, device="cuda")
    first = torch.zeros(5, dtype=torch.int64, device="cuda")
    iv = torch.zeros(2, dtype=torch.int64, device="cuda")
    aggs = torch.zeros((comp.max_chunks, 6), dtype=torch.int64, device="cuda")
    tot = torch.zeros(6, dtype=torch.int64, device="cuda")
    n_chunks = first[1:2]  # one array: its chunks are refs[0 : first[1]]
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        comp(nums, array_ns, n_arrays, metas, pages, refs, first)
        a(metas, pages, refs, n_chunks, iv, aggs, tot)
    for seed, n in [(1, 100000), (2, 5000), (3, n_cap)]:
        x = _walk(dtype, n, seed=seed)
        nums[:n].copy_(torch.from_numpy(x))
        array_ns[0] = n
        lo, hi = x.dtype.type(np.quantile(x, 0.25)), x.dtype.type(np.quantile(x, 0.9))
        iv.copy_(torch.from_numpy(wrapped.pack_interval(lo, hi, dtype)))
        g.replay()
        torch.cuda.synchronize()
        comp.result()
        k = a.result()
        page_ns = refs[: int(first[1])].cpu().numpy()[:, 4].tolist()
        assert sum(page_ns) == n
        groups, at = [], 0
        for pn in page_ns:
            groups.append((x[at:at + pn], [pn]))
            at += pn
        _check_records(aggs.cpu().numpy()[: len(groups)], tot.cpu().numpy(), k, groups, dtype, lo, hi)
