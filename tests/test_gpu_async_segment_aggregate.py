"""The asynchronous segment aggregates on the GPU (pco_b200_segment_aggregate_pages_async / _files_async,
wrapped.AsyncPagesSegmentAggregate, standalone.AsyncFilesSegmentAggregate): every record is compared with tests/segment_reference.py over
the numbers the matching decompress call returns for the same refs (counts, min and max bits and integer sums exactly, float sums bit for
bit in the specified order); segments equal to the pages or files against the aggregate call itself; every refusal with its kind, status
and index in precedence order against the decompress call's."""
import math

import numpy as np
import pytest

from tests import aggregate_reference as ref
from tests import segment_reference as sr
from tests.test_gpu_async_aggregate import (DTYPES, UNTOUCHED, _agg_files, _agg_pages, _chunk_ns, _frames, _outcome)
from tests.test_gpu_async_files import _batch, _cfg, _run as _files_run, _walk as _files_walk
from tests.test_gpu_async_filter_files import sa  # noqa: F401  (fixture)
from tests.test_gpu_async_filter_pages import _intervals
from tests.test_gpu_async_pages import _cold_batch, _dev, _refs_dev, _run as _pages_run
from tests.test_gpu_encode import _walk
from tests.test_gpu_wrapped_batch import _container, _mixed_chunks, _shuffled, _six_pages

pytestmark = pytest.mark.gpu

TOO_MANY, ORDER, PAST = 0x401, 0x402, 0x403


def _bounds_dev(bounds, max_segments):
    import torch

    b = np.zeros(max_segments + 1, np.int64)
    b[: len(bounds)] = bounds
    return torch.from_numpy(b).cuda()


def _seg_pages(metas, pages, refs, dtype, bounds, lo, hi, max_segments=None, n_segments=None, max_pages=None, rows_cap=None, n=None,
               profile=False):
    import torch

    from pcodec_b200 import wrapped

    total = int(np.asarray(refs)["page_n"].sum()) if len(refs) else 0
    max_pages = max_pages or max(len(refs), 1)
    ms = max_segments or max(len(bounds) - 1, 1)
    a = wrapped.AsyncPagesSegmentAggregate(dtype, len(metas), len(pages), max_pages, total if rows_cap is None else rows_cap, ms,
                                           frame_cap=_frames(metas, pages, refs, max_pages))
    iv = torch.from_numpy(wrapped.pack_interval(lo, hi, dtype)).cuda()
    nt = torch.tensor([len(refs) if n is None else n], dtype=torch.int64).cuda()
    ns = torch.tensor([len(bounds) - 1 if n_segments is None else n_segments], dtype=torch.int64).cuda()
    m, p, r, b = _dev(metas), _dev(pages), _refs_dev(refs, max_pages), _bounds_dev(bounds, max(ms, len(bounds) - 1))
    return _outcome(lambda aggs, tot: a(m, p, r, nt, b, ns, iv, aggs, tot), a, ms, profile)


def _seg_files(sa, data, index, dtype, refs, bounds, lo, hi, max_segments=None, n_segments=None, rows_cap=None, max_chunks=None, profile=False):
    import struct

    import torch

    from pcodec_b200 import wrapped
    from tests.test_gpu_async_files import _n_chunks

    nc = sum(_n_chunks(index, r) for r in refs)
    if rows_cap is None:
        rows_cap = sum(int(struct.unpack_from("<Q", index, int(r[2]) + 16)[0]) for r in refs)
    mf = max(len(refs), 1)
    ms = max_segments or max(len(bounds) - 1, 1)
    a = sa.AsyncFilesSegmentAggregate(data[int(refs[0][0]):int(refs[0][0]) + 32], dtype, len(data), len(index), mf, max_chunks or max(nc, 1),
                                      rows_cap, ms)
    d_data = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    d_index = torch.frombuffer(bytearray(index), dtype=torch.uint8).cuda()
    fr = np.zeros((mf, 4), np.uint64)
    fr[: len(refs)] = refs
    d_files = torch.from_numpy(fr.view(np.int64)).cuda()
    nt = torch.tensor([len(refs)], dtype=torch.int64, device="cuda")
    ns = torch.tensor([len(bounds) - 1 if n_segments is None else n_segments], dtype=torch.int64).cuda()
    iv = torch.from_numpy(wrapped.pack_interval(lo, hi, dtype)).cuda()
    b = _bounds_dev(bounds, max(ms, len(bounds) - 1))
    return _outcome(lambda aggs, tot: a(d_data, d_index, d_files, nt, b, ns, iv, aggs, tot), a, ms, profile)


def _edge_bounds(pieces, seed):
    """Bounds with empty segments and runs of equal bounds, 1-row segments, bounds on and +-1 around page / chunk starts, segments
    spanning many pages, bounds[0] > 0 and bounds[M] < rows; and one set of every batch edge (each segment one whole batch: 256 rows
    but for a page's / chunk's last)."""
    rows = int(sum(pieces))
    starts = np.concatenate([[0], np.cumsum(pieces)]).astype(np.int64)
    rng = np.random.default_rng(seed)
    b = set(int(v) for v in rng.integers(0, rows + 1, size=40))
    for s in starts[1:-1][:: max(1, len(starts) // 12)]:
        b |= {int(s) - 1, int(s), int(s) + 1, int(s) + 256, int(s) + 257}
    b |= {5, 6, 256, 512, 768}
    b = sorted(v for v in b if 0 <= v <= rows)
    b = b[:3] + [b[3]] * 3 + b[3:]  # a run of equal bounds
    batch_edges = np.concatenate([o + np.arange(0, n, 256) for o, n in zip(starts[:-1], pieces) if n] + [[rows]]).astype(np.int64)
    out = [np.array(b, np.int64), starts, batch_edges, np.array([0, rows], np.int64),
           np.array([min(3, rows), max(rows - 2, min(3, rows))], np.int64)]
    return out


def _check(aggs, tot, k, st, x, pieces, bounds, dtype, lo, hi):
    floats = np.dtype(dtype).kind == "f"
    want, wt = sr.segment_records(x, pieces, bounds, lo, hi)
    for g, (w, _) in enumerate(want):
        assert ref.same(aggs[g], w, floats), (g, bounds[g], bounds[g + 1], lo, hi, [int(v) & ref.MASK64 for v in aggs[g]], w)
    assert (aggs[len(want):].view(np.uint64) == UNTOUCHED).all(), "records past the count written"
    assert ref.same(tot, wt, floats), (lo, hi, [int(v) & ref.MASK64 for v in tot], wt)
    assert k == wt[1] and st.n_matches == k and st.n_segments == len(bounds) - 1


def _check_pages(metas, pages, refs, dtype, intervals, bounds_sets=None):
    got, nw, err, _ = _pages_run(metas, pages, refs, dtype, frame_cap=_frames(metas, pages, refs, max(len(refs), 1)))
    assert err is None, err
    x = got[:nw]
    pieces = np.asarray(refs)["page_n"].tolist()
    for bounds in bounds_sets or _edge_bounds(pieces, seed=len(x)):
        for lo, hi in intervals:
            aggs, tot, k, err, st, _ = _seg_pages(metas, pages, refs, dtype, bounds, lo, hi)
            assert err is None, (lo, hi, err)
            _check(aggs, tot, k, st, x, pieces, bounds, dtype, lo, hi)
    return x


def _decoded_files(sa, data, index, refs, dtype):
    dec, err, _ = _files_run(sa, data, index, dtype, refs)
    assert err is None, err
    pieces = [n for r in refs for n in _chunk_ns(index, r)]
    assert sum(pieces) == len(dec[0])
    return dec[0], pieces


def _check_files(sa, data, index, refs, dtype, intervals):
    x, pieces = _decoded_files(sa, data, index, refs, dtype)
    for bounds in _edge_bounds(pieces, seed=len(x)):
        for lo, hi in intervals:
            aggs, tot, k, err, st, _ = _seg_files(sa, data, index, dtype, refs, bounds, lo, hi)
            assert err is None, (lo, hi, err)
            _check(aggs, tot, k, st, x, pieces, bounds, dtype, lo, hi)
    return x, pieces


@pytest.mark.parametrize("dtype", DTYPES)
def test_every_dtype_on_a_mixed_batch_of_pages(oracle, dtype):
    metas, pages, refs, pieces = _container(_mixed_chunks(oracle, dtype))
    refs, pieces = _shuffled(refs, pieces, seed=int(np.dtype(dtype).num))
    _check_pages(metas, pages, refs, dtype, _intervals(np.concatenate(pieces), dtype)[:3])


@pytest.mark.parametrize("dtype", DTYPES)
def test_every_dtype_on_a_batch_of_files(sa, dtype):  # noqa: F811
    xs = [_files_walk(dtype, m, seed=int(np.dtype(dtype).num) + i) for i, m in enumerate([3 * (1 << 14) + 777, 1, 0, 5000, 1 << 14, 257])]
    data, index, refs = _batch(sa, xs, _cfg(1))
    _check_files(sa, data, index, refs, dtype, _intervals(np.concatenate(xs), dtype)[:3])


@pytest.mark.parametrize("dtype", [np.float32, np.int64, np.uint16])
def test_segments_equal_to_pages_give_the_aggregate_call(oracle, dtype):
    metas, pages, refs, pieces = _container(_mixed_chunks(oracle, dtype))
    x = np.concatenate(pieces)
    page_n = np.asarray(refs)["page_n"].astype(np.int64)
    starts = np.concatenate([[0], np.cumsum(page_n)])
    for lo, hi in _intervals(x, dtype)[:3]:
        a_aggs, a_tot, a_k, a_err, *_ = _agg_pages(metas, pages, refs, dtype, lo, hi)
        s_aggs, s_tot, s_k, s_err, *_ = _seg_pages(metas, pages, refs, dtype, starts, lo, hi)
        assert a_err is None and s_err is None
        assert np.array_equal(a_aggs[: len(refs)], s_aggs[: len(refs)]) and np.array_equal(a_tot, s_tot) and a_k == s_k
        # one segment over a single page is the aggregate's total of that page alone
        one = refs[:1]
        _, o_tot, *_ = _agg_pages(metas, pages, one, dtype, lo, hi)
        w_aggs, *_ = _seg_pages(metas, pages, one, dtype, [0, int(one["page_n"][0])], lo, hi)
        assert np.array_equal(w_aggs[0], o_tot)


def test_segments_equal_to_files_give_the_aggregate_call(sa):  # noqa: F811
    xs = [_files_walk(np.float64, m, seed=m) for m in (70000, 1, 5000, 1 << 16, 300)]
    data, index, refs = _batch(sa, xs, _cfg(1))
    starts = np.concatenate([[0], np.cumsum([len(x) for x in xs])])
    x = np.concatenate(xs)
    for lo, hi in [(-math.inf, math.inf), (float(np.quantile(x, 0.3)), float(np.quantile(x, 0.8)))]:
        a_aggs, a_tot, a_k, a_err, *_ = _agg_files(sa, data, index, np.float64, refs, lo, hi)
        s_aggs, s_tot, s_k, s_err, *_ = _seg_files(sa, data, index, np.float64, refs, starts, lo, hi)
        assert a_err is None and s_err is None
        assert np.array_equal(a_aggs[: len(refs)], s_aggs[: len(refs)]) and np.array_equal(a_tot, s_tot) and a_k == s_k
        _, o_tot, *_ = _agg_files(sa, data, index, np.float64, refs[:1], lo, hi)
        w_aggs, *_ = _seg_files(sa, data, index, np.float64, refs[:1], [0, len(xs[0])], lo, hi)
        assert np.array_equal(w_aggs[0], o_tot)


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
    _check_pages(metas, pages, refs, dtype, [(-1.0, 1.0), (-0.0, -0.0), (-math.inf, math.inf), (1.0, math.inf)])


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
    """The fused kernel, the general pair and cold pages (Lookback, Dict, Conv1) in one batch, with segments over all of them."""
    metas, pages, refs, pieces = _cold_batch(oracle)
    x = _check_pages(metas, pages, refs, np.int32, _intervals(np.sort(np.concatenate(pieces)), np.int32)[:2])
    rows = len(x)
    *_, err, _, spans = _seg_pages(metas, pages, refs, np.int32, np.linspace(0, rows, 301).astype(np.int64), int(np.median(x)), int(np.max(x)),
                                   profile=True)
    assert err is None
    order = ["ap_pages_kernel", "walk_kernel", "sg_front_pages_kernel", "sg_check_kernel", "sg_mark_kernel", "tk_cold_list_kernel",
             "fused_narrow_kernel", "symwalk_kernel", "decode_kernel", "ap_cold_kernel", "ap_finish_kernel", "sg_cold_pages_kernel",
             "sg_group_kernel", "sg_finish_pages_kernel"]
    at = [spans.find(k) for k in order]
    assert all(a >= 0 for a in at) and at == sorted(at), spans


@pytest.mark.parametrize("name", ["cold_level9", "cold_level12"])
def test_files_with_cold_chunks(sa, name):  # noqa: F811
    """Chunks with tables above 2^10 states go to the catch-all decoder; sg_cold_files_kernel reduces them."""
    from tests.test_gpu_async_filter_files import ROUTE_CASES

    dtype, arrays, cfg, _ = ROUTE_CASES[name]
    xs = [np.asarray(a, dtype=dtype) for a in arrays()]
    data, index, refs = _batch(sa, xs, cfg())
    sel = refs[[1, 0, 1]]
    x, pieces = _check_files(sa, data, index, sel, dtype, _intervals(np.concatenate([xs[1], xs[0], xs[1]]), dtype)[:2])
    s = np.sort(x)
    *_, err, _, spans = _seg_files(sa, data, index, dtype, sel, [0, len(x) // 3, len(x)], s[len(s) // 3], s[2 * len(s) // 3], profile=True)
    assert err is None and "sg_cold_files_kernel" in spans and "cold_chunks_kernel" in spans, spans


def test_skip_rule_on_pages(oracle):
    """A bit flip in page k fails the call only when the segments cover page k; a walk failure is a refusal either way.  The fast pages'
    flips are all caught by the walk; the cold pages (Lookback, Conv1, Dict), which the walk routes to the catch-all decoder, give decode
    failures that segments away from them skip."""
    rng = np.random.default_rng(1)
    skipped = 0
    for metas, pages, refs, pieces, dtype in [(*_six_pages(oracle), np.uint64), (*_cold_batch(oracle), np.int32)]:
        x = np.concatenate(pieces)
        sizes = [len(p) for p in pieces]
        starts = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        lo, hi = np.iinfo(dtype).min, np.iinfo(dtype).max
        for trial in range(24):
            k = int(rng.integers(0, len(refs)))
            buf = bytearray(pages)
            buf[int(refs[k]["page_offset"] + rng.integers(0, refs[k]["page_len"]))] ^= 1 << int(rng.integers(0, 8))
            _, _, perr, pst = _pages_run(metas, bytes(buf), refs, dtype)
            on = [int(starts[k]), int(starts[k]) + 1, int(starts[k + 1])]
            _, tot, _, err, st, _ = _seg_pages(metas, bytes(buf), refs, dtype, on, lo, hi)
            if perr is None or pst.page != k:
                continue
            assert err is not None and (err.kind, st.page) == (perr.kind, pst.page) and (tot == 0).all(), (trial, err, perr)
            j = 0 if k else 1  # segments over page j only
            away = [int(starts[j]), (int(starts[j]) + int(starts[j + 1])) // 2, int(starts[j + 1])]
            aggs, tot, cnt, err, st, _ = _seg_pages(metas, bytes(buf), refs, dtype, away, lo, hi)
            if err is None:
                skipped += 1
                assert st.records_decoded == 1
                _check(aggs, tot, cnt, st, x, sizes, away, dtype, lo, hi)
            else:
                assert (err.kind, st.device_status, st.page) == (perr.kind, pst.device_status, pst.page)
    assert skipped >= 1, "no flip gave a decode failure that segments away from its page skip"


def test_skip_rule_on_files(sa):  # noqa: F811
    import struct

    xs = [_walk(np.uint64, 1 << 16, seed=s) for s in range(2)]
    data, index, refs = _batch(sa, xs, _cfg(1, page=4096))
    x, sizes = _decoded_files(sa, data, index, refs, np.uint64)
    starts = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    base, co = int(refs[1, 2]), struct.unpack_from("<Q", index, int(refs[1, 2]) + 32)[0]
    c_in_file = 3
    chunk_off = struct.unpack_from("<Q", index, base + co + 32 * c_in_file)[0]
    chunk_len = struct.unpack_from("<Q", index, base + co + 32 * (c_in_file + 1))[0] - chunk_off
    c = len(_chunk_ns(index, refs[0])) + c_in_file  # that chunk in the concatenation
    rng = np.random.default_rng(5)
    for _ in range(40):  # a flip inside the chunk that the files call reports for this chunk
        bad = bytearray(data)
        bad[int(refs[1, 0]) + chunk_off + int(rng.integers(0, chunk_len))] ^= 1 << int(rng.integers(0, 8))
        bad = bytes(bad)
        _, werr, wst = _files_run(sa, bad, index, np.uint64, refs, dst_cap=len(x))
        if werr is not None:
            break
    assert werr is not None and wst.file == 1 and wst.chunk == c_in_file
    away = [5, int(starts[c]) - 300, int(starts[c]), int(starts[c + 1]), int(starts[c + 2]) - 1]  # all but chunk c
    aggs, tot, cnt, err, st, _ = _seg_files(sa, bad, index, np.uint64, refs, away[:3], 0, (1 << 64) - 1)
    assert err is None and st.records_decoded == c, (err, st.records_decoded)
    _check(aggs, tot, cnt, st, x, sizes, away[:3], np.uint64, 0, (1 << 64) - 1)
    aggs, tot, cnt, err, st, _ = _seg_files(sa, bad, index, np.uint64, refs, away[3:], 0, (1 << 64) - 1)
    assert err is None and st.records_decoded == 1, (err, st.records_decoded)
    _check(aggs, tot, cnt, st, x, sizes, away[3:], np.uint64, 0, (1 << 64) - 1)
    _, tot, _, err, st, _ = _seg_files(sa, bad, index, np.uint64, refs, [5, int(starts[c]) + 10], 0, (1 << 64) - 1)
    assert err is not None and err.kind == werr[0] and (st.device_status, st.file, st.chunk) == (wst.device_status, wst.file, wst.chunk)
    assert (tot == 0).all()


def test_refusals_in_precedence_order(oracle):
    metas, pages, refs, pieces = _six_pages(oracle)
    rows = sum(len(p) for p in pieces)

    def refused(bounds, **kw):
        aggs, tot, _, err, st, _ = _seg_pages(metas, pages, refs, np.uint64, bounds, 0, (1 << 64) - 1, **kw)
        assert err is not None and (tot == 0).all() and (aggs.view(np.uint64) == UNTOUCHED).all() and st.n_matches == 0
        return err, st

    # the pages call's own refusal comes first, even with bad bounds
    _, _, perr, pst = _pages_run(metas, pages, refs, np.uint64, max_pages=len(refs), n=len(refs) + 1)
    err, st = refused([5, 3, rows + 9], max_segments=2, n_segments=9, n=len(refs) + 1)
    assert (err.kind, st.device_status) == (perr.kind, pst.device_status)
    err, st = refused([5, 3, rows + 9], max_segments=2, n_segments=3)
    assert (st.kind, st.device_status, st.n_segments) == (3, TOO_MANY, 3) and "*n_segments is 3" in err.message
    err, st = refused([5, 3, rows + 9, 2], max_segments=3)
    assert (st.device_status, st.segment) == (ORDER, 1) and err.message.startswith("segment 1: ")
    err, st = refused([5, 7, rows + 9, rows + 10], max_segments=3)
    assert (st.device_status, st.segment) == (PAST, 2) and err.message.startswith("segment 2: ") and f"{rows} rows" in err.message
    aggs, tot, k, err, st, _ = _seg_pages(metas, pages, refs, np.uint64, [0, rows], 0, (1 << 64) - 1, n_segments=0)
    assert err is None and (tot == 0).all() and k == 0 and st.records_decoded == 0 and (aggs.view(np.uint64) == UNTOUCHED).all()


def test_a_page_of_2_24_numbers_with_2_20_segments(oracle):
    O = oracle
    x = _walk(np.uint32, 1 << 24, seed=4)
    metas, pages, refs, _ = _container([(x, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=1, max_page_n=1 << 24))])
    assert len(refs) == 1
    rng = np.random.default_rng(9)
    bounds = np.concatenate([[0], np.sort(rng.choice(np.arange(1, 1 << 24), (1 << 20) - 1, replace=False)), [1 << 24]]).astype(np.int64)
    lo, hi = x[1000], x[(1 << 24) - 1000]
    if lo > hi:
        lo, hi = hi, lo
    aggs, tot, k, err, st, _ = _seg_pages(metas, pages, refs, np.uint32, bounds, lo, hi)
    assert err is None, err
    want, wt = sr.segment_records_int(x, bounds, lo, hi)
    assert np.array_equal(aggs.view(np.uint64), np.array(want, dtype=np.uint64)) and [int(v) & ref.MASK64 for v in tot] == wt and k == wt[1]


def test_identical_calls_give_identical_records(oracle):
    metas, pages, refs, pieces = _container(_mixed_chunks(oracle, np.float32))
    x = np.concatenate(pieces)
    bounds = np.linspace(0, len(x), 777).astype(np.int64)
    a = _seg_pages(metas, pages, refs, np.float32, bounds, float(np.nanmin(x)), float(np.nanmax(x)))
    b = _seg_pages(metas, pages, refs, np.float32, bounds, float(np.nanmin(x)), float(np.nanmax(x)))
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_graph_replays_new_refs_counts_bounds_and_interval(oracle):
    import torch

    from pcodec_b200 import wrapped

    metas, pages, refs, pieces = _six_pages(oracle)
    mp, total, ms = len(refs), sum(len(p) for p in pieces), 500
    a = wrapped.AsyncPagesSegmentAggregate(np.uint64, len(metas), len(pages), mp, total, ms)
    d_m, d_p, d_r = _dev(metas), _dev(pages), _refs_dev(refs, mp)
    nt = torch.tensor([mp], dtype=torch.int64, device="cuda")
    b = torch.zeros(ms + 1, dtype=torch.int64, device="cuda")
    ns = torch.zeros(1, dtype=torch.int64, device="cuda")
    iv = torch.zeros(2, dtype=torch.int64, device="cuda")
    aggs = torch.full((ms, 6), UNTOUCHED, dtype=torch.int64, device="cuda")
    tot = torch.zeros(6, dtype=torch.int64, device="cuda")
    a(d_m, d_p, d_r, nt, b, ns, iv, aggs, tot)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        a(d_m, d_p, d_r, nt, b, ns, iv, aggs, tot)
    rng = np.random.default_rng(2)
    for trial in range(4):
        order = rng.permutation(mp)[: int(rng.integers(1, mp + 1))]
        sel = refs[order]
        xs = [pieces[i] for i in order]
        x = np.concatenate(xs)
        m = int(rng.integers(1, ms + 1))
        bounds = np.sort(rng.integers(0, len(x) + 1, size=m + 1)).astype(np.int64)
        lo, hi = np.sort(x)[len(x) // 5], np.sort(x)[len(x) * 3 // 4]
        d_r.copy_(_refs_dev(sel, mp))
        nt.fill_(len(sel))
        b[: m + 1].copy_(torch.from_numpy(bounds))
        ns.fill_(m)
        iv.copy_(torch.from_numpy(wrapped.pack_interval(lo, hi, np.uint64)))
        aggs.fill_(UNTOUCHED)
        g.replay()
        k = a.result()
        st = a.status_record()
        _check(aggs.cpu().numpy(), tot.cpu().numpy(), k, st, x, [len(p) for p in xs], bounds, np.uint64, lo, hi)


def test_time_bucket_graph(oracle):
    """One graph: decode a monotone timestamp column, torch.searchsorted of bucket edges into it, segment-aggregate a value column."""
    import torch

    from pcodec_b200 import wrapped

    O = oracle
    rng = np.random.default_rng(11)
    n = 300000
    ts = np.cumsum(rng.integers(1, 50, size=n)).astype(np.int64)
    val = (rng.normal(size=n) * 100).astype(np.float32)
    cfg = O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=1, max_page_n=1 << 15)
    tm, tp, tr, _ = _container([(ts, cfg)])
    vm, vp, vr, _ = _container([(val, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_NOOP, max_page_n=20000))])
    edges_np = np.arange(int(ts[0]) - 1000, int(ts[-1]) + 5000, 5000, dtype=np.int64)
    ms = len(edges_np) - 1
    dec = wrapped.AsyncPagesDecompressor(np.int64, len(tm), len(tp), len(tr), n, frame_cap=_frames(tm, tp, tr, len(tr)))
    seg = wrapped.AsyncPagesSegmentAggregate(np.float32, len(vm), len(vp), len(vr), n, ms, frame_cap=_frames(vm, vp, vr, len(vr)))
    d_tm, d_tp, d_tr = _dev(tm), _dev(tp), _refs_dev(tr, len(tr))
    d_vm, d_vp, d_vr = _dev(vm), _dev(vp), _refs_dev(vr, len(vr))
    nt = torch.tensor([len(tr)], dtype=torch.int64, device="cuda")
    nv = torch.tensor([len(vr)], dtype=torch.int64, device="cuda")
    col = torch.zeros(n, dtype=torch.int64, device="cuda")
    edges = torch.from_numpy(edges_np).cuda()
    bounds = torch.zeros(ms + 1, dtype=torch.int64, device="cuda")
    ns = torch.tensor([ms], dtype=torch.int64, device="cuda")
    iv = torch.from_numpy(wrapped.pack_interval(-math.inf, math.inf, np.float32)).cuda()
    aggs = torch.zeros((ms, 6), dtype=torch.int64, device="cuda")
    tot = torch.zeros(6, dtype=torch.int64, device="cuda")

    def step():
        dec(d_tm, d_tp, d_tr, nt, col)
        bounds.copy_(torch.searchsorted(col, edges))
        seg(d_vm, d_vp, d_vr, nv, bounds, ns, iv, aggs, tot)

    step()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        step()
    aggs.zero_()
    g.replay()
    torch.cuda.synchronize()
    dec.result()
    k = seg.result()
    b = np.searchsorted(ts, edges_np).astype(np.int64)
    assert np.array_equal(bounds.cpu().numpy(), b)
    _check(aggs.cpu().numpy(), tot.cpu().numpy(), k, seg.status_record(), val, np.asarray(vr)["page_n"].tolist(), b, np.float32, -math.inf,
           math.inf)


def test_files_refusals_in_precedence_order(sa):  # noqa: F811
    """The files call's own refusal (rows_cap) before the segment refusals; then TOO_MANY, ORDER, PAST.  With 5000 bounds sg_check_kernel
    runs on several CTAs, and the lowest bad index wins across them."""
    xs = [_files_walk(np.int32, m, seed=m) for m in (20000, 7000, 300)]
    data, index, refs = _batch(sa, xs, _cfg(1, page=4096))
    rows = sum(len(x) for x in xs)
    ms = 5000

    def refused(bounds, **kw):
        aggs, tot, _, err, st, _ = _seg_files(sa, data, index, np.int32, refs, bounds, 0, 100, max_segments=ms, **kw)
        assert err is not None and (tot == 0).all() and (aggs.view(np.uint64) == UNTOUCHED).all() and st.n_matches == 0
        return err, st

    good = np.linspace(0, rows, ms + 1).astype(np.int64)
    bad = good.copy()
    bad[4500] = bad[4499] - 1  # out of order, in a late CTA
    bad[2001] = bad[2000] - 1  # out of order, lower, in an earlier CTA
    bad[1000] = rows + 1       # past the rows, lower still: order comes first
    _, perr, pst = _files_run(sa, data, index, np.int32, refs, dst_cap=rows - 1)
    err, st = refused(bad, rows_cap=rows - 1)
    assert perr is not None and (err.kind, st.device_status, st.file, st.chunk) == (perr[0], pst.device_status, pst.file, pst.chunk)
    err, st = refused(bad, n_segments=ms + 1)
    assert (st.device_status, st.n_segments) == (TOO_MANY, ms + 1) and "*n_segments is 5001" in err.message
    err, st = refused(bad)
    assert (st.device_status, st.segment) == (ORDER, 1001) and err.message.startswith("segment 1001: "), err
    bad = good.copy()
    bad[1234:] = rows + 1
    bad[4800:] = rows + 2
    err, st = refused(bad)
    assert (st.device_status, st.segment) == (PAST, 1234) and f"{rows} rows" in err.message, err
    aggs, tot, k, err, st, _ = _seg_files(sa, data, index, np.int32, refs, good, 0, 100, max_segments=ms)
    assert err is None
    _check(aggs, tot, k, st, np.concatenate(xs), [n for r in refs for n in _chunk_ns(index, r)], good, np.int32, 0, 100)


def test_long_segments_split_over_ctas(sa):  # noqa: F811
    """Segments above 2^18 rows: their order-free parts are spread over sg_long_kernel's CTAs and the float chain stays on one warp."""
    for dtype in (np.int64, np.float64):
        xs = [_files_walk(dtype, m, seed=m) for m in (1 << 20, 300000, 5)]
        data, index, refs = _batch(sa, xs, _cfg(1))
        x, pieces = _decoded_files(sa, data, index, refs, dtype)
        rows = len(x)
        s = np.sort(x)
        for bounds in ([0, rows], [7, 300000, 300001, rows - 3], [0, 1 << 18, (1 << 18) + 1, rows]):
            for lo, hi in [(s[0], s[-1]), (s[rows // 4], s[rows // 2])]:
                aggs, tot, k, err, st, spans = _seg_files(sa, data, index, dtype, refs, np.array(bounds, np.int64), lo, hi, profile=True)
                assert err is None and "sg_long_kernel" in spans
                _check(aggs, tot, k, st, x, pieces, bounds, dtype, lo, hi)


def test_files_graph_replays_new_refs_counts_bounds_and_interval(sa):  # noqa: F811
    import torch

    from pcodec_b200 import wrapped

    xs = [_files_walk(np.float32, m, seed=m) for m in (70000, 1, 5000, 1 << 16, 300)]
    data, index, refs = _batch(sa, xs, _cfg(1))
    mf, nc, ms = 8, 64, 300
    rows = 4 * sum(len(x) for x in xs)
    a = sa.AsyncFilesSegmentAggregate(data[:32], np.float32, len(data), len(index), mf, nc, rows, ms)
    d_data = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    d_index = torch.frombuffer(bytearray(index), dtype=torch.uint8).cuda()
    d_files = torch.zeros((mf, 4), dtype=torch.int64, device="cuda")
    nt = torch.ones(1, dtype=torch.int64, device="cuda")
    b = torch.zeros(ms + 1, dtype=torch.int64, device="cuda")
    ns = torch.zeros(1, dtype=torch.int64, device="cuda")
    iv = torch.zeros(2, dtype=torch.int64, device="cuda")
    aggs = torch.full((ms, 6), UNTOUCHED, dtype=torch.int64, device="cuda")
    tot = torch.zeros(6, dtype=torch.int64, device="cuda")
    d_files[:1] = torch.from_numpy(refs[:1].view(np.int64))
    a(d_data, d_index, d_files, nt, b, ns, iv, aggs, tot)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        a(d_data, d_index, d_files, nt, b, ns, iv, aggs, tot)
    rng = np.random.default_rng(4)
    for trial in range(4):
        order = rng.integers(0, len(refs), size=int(rng.integers(1, mf + 1)))
        sel = refs[order]
        x = np.concatenate([xs[i] for i in order])
        m = int(rng.integers(1, ms + 1))
        bounds = np.sort(rng.integers(0, len(x) + 1, size=m + 1)).astype(np.int64)
        lo, hi = float(np.sort(x)[len(x) // 7]), float(np.sort(x)[len(x) * 5 // 6])
        d_files.zero_()
        d_files[: len(sel)] = torch.from_numpy(sel.view(np.int64))
        nt.fill_(len(sel))
        b[: m + 1].copy_(torch.from_numpy(bounds))
        ns.fill_(m)
        iv.copy_(torch.from_numpy(wrapped.pack_interval(lo, hi, np.float32)))
        aggs.fill_(UNTOUCHED)
        g.replay()
        k = a.result()
        pieces = [n for i in order for n in _chunk_ns(index, refs[i])]
        _check(aggs.cpu().numpy(), tot.cpu().numpy(), k, a.status_record(), x, pieces, bounds, np.float32, lo, hi)
