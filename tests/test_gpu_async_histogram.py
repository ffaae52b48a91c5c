"""The asynchronous histograms on the GPU (pco_b200_histogram_pages_async / _files_async, wrapped.AsyncPagesHistogram,
standalone.AsyncFilesHistogram): every row is compared with tests/histogram_reference.py over the numbers the matching decompress call
returns for the same refs, bucketed by np.searchsorted on the numbers themselves; every refusal with that call's kind and page / file, and
the edge refusal naming the lowest bad edge."""
import ctypes as C
import math

import numpy as np
import pytest

from tests import histogram_reference as hr
from tests.test_gpu_async_aggregate import _chunk_ns, _frames
from tests.test_gpu_async_files import _batch, _cfg, _n_chunks, _run as _files_run, _walk as _files_walk
from tests.test_gpu_async_filter_files import sa  # noqa: F401  (fixture)
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


def _edge_sets(x, dtype):
    """Edge arrays (strictly ascending, of dtype) for the numbers x: quantiles of its distinct values at a few bucket counts, one bucket,
    edges at the type's extremes, and every number in one bucket."""
    dt = np.dtype(dtype)
    u = np.unique(x[~np.isnan(x)] if dt.kind == "f" else x)
    out = []
    for nb in (1, 7, 255):
        if len(u) >= 2:
            out.append(np.unique(u[np.linspace(0, len(u) - 1, min(nb + 1, len(u))).astype(np.int64)]))
    if dt.kind == "f":
        out += [np.array([-np.inf, np.inf], dt), np.array([-np.inf, -1.0, -0.0, 1.0, np.finfo(dt).max, np.inf], dt)]
    else:
        info = np.iinfo(dt)
        out += [np.array([info.min, info.max], dt), np.unique(np.array([info.min, info.min + 1, 0, info.max - 1, info.max], dt))]
    if len(u):
        out.append(np.array([u[0], u[-1]], dt) if len(u) >= 2 else np.array([u[0], u[0] + dt.type(1)], dt))  # one bucket holds all
    return [e.astype(dt) for e in out]


def _outcome(call, h, max_groups, w, profile=False):
    import torch

    from pcodec_b200 import PcoError, _lib

    hists = torch.full((max_groups, w), UNTOUCHED, dtype=torch.int64, device="cuda")
    tot = torch.full((w,), UNTOUCHED, dtype=torch.int64, device="cuda")
    L = _lib.lib()
    if profile:
        L.pco_b200_profile_enable(1)
    try:
        call(hists, tot)
        st = h.status_record()
        spans = _spans(L) if profile else ""
    finally:
        if profile:
            L.pco_b200_profile_enable(0)
    try:
        n, err = h.result(), None
    except PcoError as e:
        n, err = None, e
    return hists.cpu().numpy(), tot.cpu().numpy(), n, err, st, spans


def _hist_pages(metas, pages, refs, dtype, edges, max_pages=None, rows_cap=None, frame_cap=-1, n=None, profile=False):
    import torch

    from pcodec_b200 import wrapped

    total = int(np.asarray(refs)["page_n"].sum()) if len(refs) else 0
    max_pages = max_pages or max(len(refs), 1)
    rows_cap = total if rows_cap is None else rows_cap
    if frame_cap == -1:
        frame_cap = _frames(metas, pages, refs, max_pages)
    nb = len(edges) - 1
    h = wrapped.AsyncPagesHistogram(dtype, len(metas), len(pages), max_pages, rows_cap, nb, frame_cap)
    ed = torch.from_numpy(wrapped.pack_edges(edges, dtype)).cuda()
    nt = torch.tensor([len(refs) if n is None else n], dtype=torch.int64).cuda()
    m, p, r = _dev(metas), _dev(pages), _refs_dev(refs, max_pages)
    return _outcome(lambda hs, tot: h(m, p, r, nt, ed, hs, tot), h, max_pages, nb + 3, profile)


def _check_rows(hists, tot, n, groups, edges):
    """groups: per group, its numbers."""
    want = np.array([hr.row(x, edges) for x in groups], dtype=np.int64).reshape(len(groups), len(edges) + 2)
    assert np.array_equal(hists[: len(groups)], want), (edges, np.argwhere(hists[: len(groups)] != want)[:5])
    assert (hists[len(groups):].view(np.uint64) == UNTOUCHED).all(), "rows past the count written"
    assert np.array_equal(tot, want.sum(axis=0)) and np.array_equal(tot, hists[: len(groups)].sum(axis=0))
    assert [int(r.sum()) for r in hists[: len(groups)]] == [len(x) for x in groups]
    assert n == sum(len(x) for x in groups) == int(tot.sum())


def _check_pages(metas, pages, refs, dtype, edge_sets, **kw):
    got, nw, err, _ = _pages_run(metas, pages, refs, dtype, frame_cap=_frames(metas, pages, refs, max(len(refs), 1)))
    assert err is None, err
    dec = got[:nw]
    groups, at = [], 0
    for n in np.asarray(refs)["page_n"].tolist():
        groups.append(dec[at:at + n])
        at += n
    for edges in edge_sets:
        hists, tot, n, err, st, _ = _hist_pages(metas, pages, refs, dtype, edges, **kw)
        assert err is None, (edges, err)
        _check_rows(hists, tot, n, groups, edges)
        assert st.n_written == nw and st.edge == (1 << 64) - 1
    return dec


@pytest.mark.parametrize("dtype", DTYPES)
def test_every_dtype_on_a_mixed_batch_of_pages(oracle, dtype):
    metas, pages, refs, pieces = _container(_mixed_chunks(oracle, dtype))
    refs, pieces = _shuffled(refs, pieces, seed=int(np.dtype(dtype).num))
    frames = int(sum((4 + r["meta_len"] + r["page_len"] + 15) // 16 * 16 for r in refs))
    _check_pages(metas, pages, refs, dtype, _edge_sets(np.concatenate(pieces), dtype), frame_cap=frames)


@pytest.mark.parametrize("dtype", [np.float16, np.float32, np.float64])
def test_floats_with_nan_payloads_zeros_and_infinities(oracle, dtype):
    dt = np.dtype(dtype)
    ut = np.dtype(f"u{dt.itemsize}")
    rng = np.random.default_rng(7)
    x = (rng.normal(size=5000) * 10).astype(dt)
    special = np.array([math.inf, -math.inf, 0.0, -0.0, math.nan], dtype=dt)
    x[rng.integers(0, x.size, size=300)] = special[rng.integers(0, special.size, size=300)]
    xb = x.view(ut).copy()
    exp = {2: 0x7C00, 4: 0x7F800000, 8: 0x7FF0000000000000}[dt.itemsize]
    sign = {2: 0x8000, 4: 0x80000000, 8: 0x8000000000000000}[dt.itemsize]
    at = rng.integers(0, x.size, size=60)
    xb[at] = (exp | rng.integers(1, 1 << 9, size=60)).astype(ut) | np.where(np.arange(60) % 2 == 1, sign, 0).astype(ut)  # +-NaN payloads
    x = xb.view(dt)
    O = oracle
    chunks = [(x[:3000], O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_NOOP)), (x[3000:], O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=1))]
    metas, pages, refs, _ = _container(chunks)
    zeros = [np.array([-0.0, 1.0], dt), np.array([-1.0, -0.0], dt), np.array([-1.0, 0.0, 1.0], dt), np.array([-np.inf, 0.0, np.inf], dt)]
    _check_pages(metas, pages, refs, dtype, _edge_sets(x, dtype) + zeros)


def test_every_route_with_spans(oracle):
    metas, pages, refs, pieces = _cold_batch(oracle)
    x = np.concatenate(pieces)
    _check_pages(metas, pages, refs, np.int32, _edge_sets(x, np.int32))
    *_, err, _, spans = _hist_pages(metas, pages, refs, np.int32, np.array([x.min(), np.median(x), x.max()], np.int32), profile=True)
    assert err is None
    order = ["ap_pages_kernel", "hg_front_pages_kernel", "hg_check_kernel", "hg_mark_pages_kernel", "fused_narrow_kernel", "decode_kernel",
             "ap_cold_kernel", "ap_finish_kernel", "hg_cold_pages_kernel", "hg_rows_kernel", "hg_finish_pages_kernel"]
    at = [spans.find(k) for k in order]
    assert all(a >= 0 for a in at) and at == sorted(at), spans


def test_4096_buckets_and_one_bucket(oracle):
    O = oracle
    rng = np.random.default_rng(9)
    x = rng.integers(0, 1 << 40, size=300000, dtype=np.uint64)
    metas, pages, refs, _ = _container([(x, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_NOOP, max_page_n=40000))])
    s = np.unique(x)
    wide = np.unique(s[np.linspace(0, len(s) - 1, 4097).astype(np.int64)])
    assert len(wide) == 4097
    _check_pages(metas, pages, refs, np.uint64, [wide, np.array([0, (1 << 64) - 1], np.uint64), np.array([x.max(), (1 << 64) - 1], np.uint64)])
    y = np.full(70000, 12345, np.int64)
    m2, p2, r2, _ = _container([(y, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=1, max_page_n=30000))])
    _check_pages(m2, p2, r2, np.int64, [np.array([12345, 12346], np.int64), np.arange(12000, 12000 + 4097, dtype=np.int64)])


def test_a_page_of_2_24_and_many_small_pages(oracle):
    O = oracle
    x = _walk(np.uint32, 1 << 24, seed=4)
    metas, pages, refs, _ = _container([(x, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=1, max_page_n=1 << 24))])
    assert len(refs) == 1
    s = np.sort(x)
    _check_pages(metas, pages, refs, np.uint32, [np.unique(s[np.linspace(0, len(s) - 1, 1025).astype(np.int64)]), np.array([s[0], s[-1]], np.uint32)])
    y = _walk(np.float32, 1100 * 37, seed=5)
    m2, p2, r2, _ = _container([(y, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=1, max_page_n=37))])
    assert len(r2) >= 1000
    _check_pages(m2, p2, r2, np.float32, [np.array([-np.inf, float(np.nanmedian(y)), np.inf], np.float32)])


def _same_failure(metas, pages, refs, **kw):
    _, _, perr, pst = _pages_run(metas, pages, refs, np.uint64, **{k: v for k, v in kw.items() if k in ("max_pages", "n", "frame_cap")},
                                 dst_cap=kw.get("rows_cap"))
    hists, tot, _, err, st, _ = _hist_pages(metas, pages, refs, np.uint64, np.array([0, 1 << 40, (1 << 64) - 1], np.uint64), **kw)
    assert perr is not None and err is not None, (perr, err)
    assert (err.kind, st.device_status, st.page) == (perr.kind, pst.device_status, pst.page), (err, perr)
    assert err.message.split(":")[0] == perr.message.split(":")[0], (err, perr)
    assert (tot == 0).all() and (hists.view(np.uint64) == UNTOUCHED).all()
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
    rng = np.random.default_rng(1)
    for trial in range(8):
        k = int(rng.integers(0, len(refs)))
        buf = bytearray(pages)
        buf[int(refs[k]["page_offset"] + rng.integers(0, refs[k]["page_len"]))] ^= 1 << int(rng.integers(0, 8))
        _, _, perr, pst = _pages_run(metas, bytes(buf), refs, np.uint64)
        _, tot, _, err, st, _ = _hist_pages(metas, bytes(buf), refs, np.uint64, np.array([0, 1 << 63], np.uint64))
        assert (perr is None) == (err is None), (trial, err, perr)
        if perr is not None:
            assert (err.kind, st.page) == (perr.kind, pst.page) and (tot == 0).all(), (trial, err, perr)


@pytest.mark.parametrize("dtype,edges,bad", [
    (np.int32, [0, 5, 5, 9], 2), (np.int32, [0, 5, 4, 9, 8], 2), (np.uint64, [1, 0], 1), (np.float32, [0.0, np.nan, 1.0], 1),
    (np.float32, [np.nan, 0.0], 0), (np.float64, [-0.0, 0.0], 1), (np.float64, [0.0, -0.0, 1.0], 1), (np.float16, [-1.0, 2.0, -np.inf], 2),
    (np.int8, [-128, 127, 127], 2)])
def test_bad_edges_name_the_lowest_index(oracle, dtype, edges, bad):
    from pcodec_b200 import PcoError

    metas, pages, refs, _ = _container(_mixed_chunks(oracle, dtype))
    edges = np.array(edges, dtype=dtype)
    hists, tot, n, err, st, _ = _hist_pages(metas, pages, refs, dtype, edges)
    assert isinstance(err, PcoError) and err.kind == "InvalidArgument" and st.device_status == 0x501 and st.edge == bad, (err, st.edge)
    assert err.message.startswith(f"edge {bad}: "), err.message
    assert (tot == 0).all() and (hists.view(np.uint64) == UNTOUCHED).all()
    # a refusal of the pages call comes first
    hists, tot, n, err, st, _ = _hist_pages(metas, pages, refs, dtype, edges, rows_cap=1)
    assert err.kind == "InvalidArgument" and st.device_status != 0x501 and "rows_cap" in err.message, err


def test_identical_calls_give_identical_rows(oracle):
    metas, pages, refs, pieces = _container(_mixed_chunks(oracle, np.float32))
    x = np.concatenate(pieces)
    edges = _edge_sets(x, np.float32)[2]
    a = _hist_pages(metas, pages, refs, np.float32, edges)
    b = _hist_pages(metas, pages, refs, np.float32, edges)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_graph_replays_new_refs_counts_and_edges(oracle):
    import torch

    from pcodec_b200 import wrapped

    metas, pages, refs, pieces = _six_pages(oracle)
    mp, total, nb = len(refs), sum(len(p) for p in pieces), 16
    h = wrapped.AsyncPagesHistogram(np.uint64, len(metas), len(pages), mp, total, nb)
    d_m, d_p, d_r = _dev(metas), _dev(pages), _refs_dev(refs, mp)
    nt = torch.tensor([mp], dtype=torch.int64, device="cuda")
    ed = torch.from_numpy(wrapped.pack_edges(np.arange(nb + 1, dtype=np.uint64), np.uint64)).cuda()
    hists = torch.zeros((mp, nb + 3), dtype=torch.int64, device="cuda")
    tot = torch.zeros(nb + 3, dtype=torch.int64, device="cuda")
    h(d_m, d_p, d_r, nt, ed, hists, tot)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        h(d_m, d_p, d_r, nt, ed, hists, tot)
    rng = np.random.default_rng(2)
    for trial in range(4):
        order = rng.permutation(mp)[: int(rng.integers(1, mp + 1))]
        xs = [pieces[i] for i in order]
        u = np.unique(np.concatenate(xs))
        edges = np.unique(u[np.linspace(0, len(u) - 1, nb + 1).astype(np.int64)])
        edges = np.concatenate([edges, np.arange(1, nb + 2 - len(edges), dtype=np.uint64) + edges[-1]])  # nb + 1 of them
        d_r.copy_(_refs_dev(refs[order], mp))
        nt.fill_(len(order))
        ed.copy_(torch.from_numpy(wrapped.pack_edges(edges, np.uint64)))
        g.replay()
        n = h.result()
        _check_rows(hists.cpu().numpy()[: len(order)], tot.cpu().numpy(), n, xs, edges)


# ---- files


def _hist_files(sa, data, index, dtype, refs, edges, max_files=None, max_chunks=None, rows_cap=None, profile=False):
    import torch

    from pcodec_b200 import wrapped

    nc = sum(_n_chunks(index, r) for r in refs)
    if rows_cap is None:
        rows_cap = sum(sum(_chunk_ns(index, r)) for r in refs)
    mf = max_files or max(len(refs), 1)
    nb = len(edges) - 1
    head = data[int(refs[0][0]):int(refs[0][0]) + 32] if len(refs) else data[:32]
    h = sa.AsyncFilesHistogram(head, dtype, len(data), len(index), mf, max_chunks or max(nc, 1), rows_cap, nb)
    d_data = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    d_index = torch.frombuffer(bytearray(index), dtype=torch.uint8).cuda()
    fr = np.zeros((mf, 4), np.uint64)
    fr[: len(refs)] = refs
    d_files = torch.from_numpy(fr.view(np.int64)).cuda()
    nt = torch.tensor([len(refs)], dtype=torch.int64, device="cuda")
    ed = torch.from_numpy(wrapped.pack_edges(edges, dtype)).cuda()
    return _outcome(lambda hs, tot: h(d_data, d_index, d_files, nt, ed, hs, tot), h, mf, nb + 3, profile)


def _check_files(sa, data, index, refs, dtype, edge_sets, **kw):
    dec, err, _ = _files_run(sa, data, index, dtype, refs)
    assert err is None, err
    groups, at = [], 0
    for n in dec[1].tolist():
        groups.append(dec[0][at:at + n])
        at += n
    for edges in edge_sets:
        hists, tot, n, err, st, _ = _hist_files(sa, data, index, dtype, refs, edges, **kw)
        assert err is None, (edges, err)
        _check_rows(hists, tot, n, groups, edges)
        assert st.n_written == len(dec[0]) and st.n_files == len(refs)
    return dec[0]


@pytest.mark.parametrize("dtype", DTYPES)
def test_every_dtype_on_a_batch_of_files(sa, dtype):  # noqa: F811
    xs = [_files_walk(dtype, m, seed=int(np.dtype(dtype).num) + i) for i, m in enumerate([3 * (1 << 14) + 777, 1, 0, 5000, 1 << 14, 257])]
    for order in (0, 1, 3):  # fused orders 0 and 1, the general pair at order 3
        data, index, refs = _batch(sa, xs, _cfg(order))
        _check_files(sa, data, index, refs, dtype, _edge_sets(np.concatenate(xs), dtype))


@pytest.mark.parametrize("dtype,mode", [(np.int64, "int_mult"), (np.float64, "float_mult"), (np.float32, "float_quant")])
def test_two_var_chunks(sa, dtype, mode):  # noqa: F811
    rng = np.random.default_rng(12)
    if mode == "int_mult":
        xs = [(rng.integers(-1000, 1000, size=m) * 8 + rng.integers(0, 3, size=m)).astype(dtype) for m in (20000, 777)]
    else:
        xs = [(np.round(rng.normal(size=m) * 100) * 0.01).astype(dtype) for m in (20000, 777)]
    data, index, refs = _batch(sa, xs, _cfg(0, mode=mode))
    _check_files(sa, data, index, refs, dtype, _edge_sets(np.concatenate(xs), dtype))


@pytest.mark.parametrize("name", ["cold_level9", "cold_level12"])
def test_files_with_cold_chunks(sa, name):  # noqa: F811
    """Chunks the fast kernels leave to the catch-all decoder: cold_chunks_kernel stages them and hg_cold_files_kernel counts them."""
    from tests.test_gpu_async_filter_files import ROUTE_CASES

    dtype, arrays, cfg, _ = ROUTE_CASES[name]
    xs = [np.asarray(a, dtype=dtype) for a in arrays()]
    data, index, refs = _batch(sa, xs, cfg())
    sel = refs[[1, 0, 1]]
    dec = _check_files(sa, data, index, sel, dtype, _edge_sets(np.concatenate([xs[1], xs[0], xs[1]]), dtype))
    s = np.unique(dec)
    *_, err, _, spans = _hist_files(sa, data, index, dtype, sel, np.array([s[0], s[len(s) // 2], s[-1]], dtype), profile=True)
    assert err is None and "hg_cold_files_kernel" in spans and "cold_chunks_kernel" in spans, spans


def test_files_refusals_and_spans(sa):  # noqa: F811
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec

    xs = [_walk(np.uint32, s, seed=s) for s in (9000, 20000, 700)]
    cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.no_op(), paging_spec=PagingSpec.equal_pages_up_to(4096))
    data, index, refs = _batch(sa, xs, cfg)
    edges = np.array([0, 1 << 20, (1 << 32) - 1], np.uint32)
    *_, err, _, spans = _hist_files(sa, data, index, np.uint32, refs, edges, profile=True)
    assert err is None
    order = ["ff_map_kernel", "af_files_kernel", "hg_front_files_kernel", "hg_check_kernel", "hg_mark_files_kernel", "fused_narrow_kernel",
             "decode_kernel", "ff_cold_list_kernel", "cold_chunks_kernel", "af_finish_kernel", "hg_cold_files_kernel", "hg_rows_kernel",
             "hg_finish_files_kernel"]
    at = [spans.find(k) for k in order]
    assert all(a >= 0 for a in at) and at == sorted(at), spans
    for kw in ({"rows_cap": 9000 + 100}, {"max_chunks": 2}):
        _, perr, pst = _files_run(sa, data, index, np.uint32, refs, dst_cap=kw.get("rows_cap"), max_chunks=kw.get("max_chunks"))
        hists, tot, _, err, st, _ = _hist_files(sa, data, index, np.uint32, refs, edges, **kw)
        assert perr is not None and err is not None and (err.kind, st.device_status, st.file, st.chunk) == (perr[0], pst.device_status, pst.file, pst.chunk)
        assert (tot == 0).all() and (hists.view(np.uint64) == UNTOUCHED).all()
    hists, tot, _, err, st, _ = _hist_files(sa, data, index, np.uint32, refs, np.array([3, 1 << 20, 1 << 20], np.uint32))
    assert err.kind == "InvalidArgument" and st.edge == 2 and err.message.startswith("edge 2: ") and (tot == 0).all() and (hists.view(np.uint64) == UNTOUCHED).all()
    bad = bytearray(data)
    bad[int(refs[1][0]) + int(refs[1][1]) // 2] ^= 0x10
    _, perr, pst = _files_run(sa, bytes(bad), index, np.uint32, refs)
    hists, tot, _, err, st, _ = _hist_files(sa, bytes(bad), index, np.uint32, refs, edges)
    assert (perr is None) == (err is None)
    if perr is not None:
        assert (err.kind, st.file, st.chunk) == (perr[0], pst.file, pst.chunk) and (tot == 0).all()


def _graph_inputs(sa, xs, dtype, order=1):
    import torch

    data, index, refs = _batch(sa, xs, _cfg(order))
    d_data = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    d_index = torch.frombuffer(bytearray(index), dtype=torch.uint8).cuda()
    return data, index, refs, d_data, d_index


def test_files_graph_replays_new_refs_counts_and_edges(sa):  # noqa: F811
    import torch

    from pcodec_b200 import wrapped

    xs = [_files_walk(np.int64, m, seed=m) for m in (70000, 1, 5000, 1 << 16, 300)]
    data, index, refs, d_data, d_index = _graph_inputs(sa, xs, np.int64)
    mf, nc, nb = 8, 64, 100
    rows = 4 * sum(len(x) for x in xs)
    h = sa.AsyncFilesHistogram(data[:32], np.int64, len(data), len(index), mf, nc, rows, nb)
    d_files = torch.zeros((mf, 4), dtype=torch.int64, device="cuda")
    nt = torch.ones(1, dtype=torch.int64, device="cuda")
    ed = torch.from_numpy(wrapped.pack_edges(np.arange(nb + 1), np.int64)).cuda()
    hists = torch.zeros((mf, nb + 3), dtype=torch.int64, device="cuda")
    tot = torch.zeros(nb + 3, dtype=torch.int64, device="cuda")
    d_files[:1] = torch.from_numpy(refs[:1].view(np.int64))
    h(d_data, d_index, d_files, nt, ed, hists, tot)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        h(d_data, d_index, d_files, nt, ed, hists, tot)
    rng = np.random.default_rng(4)
    for trial in range(4):
        order = rng.integers(0, len(refs), size=int(rng.integers(1, mf + 1)))
        sel = refs[order]
        x = np.concatenate([xs[i] for i in order])
        edges = np.sort(rng.choice(np.arange(int(x.min()) - 10, int(x.max()) + 10), nb + 1, replace=False)).astype(np.int64)
        d_files.zero_()
        d_files[: len(sel)] = torch.from_numpy(sel.view(np.int64))
        nt.fill_(len(sel))
        ed.copy_(torch.from_numpy(wrapped.pack_edges(edges, np.int64)))
        g.replay()
        n = h.result()
        _check_rows(hists.cpu().numpy()[: len(sel)], tot.cpu().numpy(), n, [xs[i] for i in order], edges)


@pytest.mark.parametrize("dtype", [np.float64, np.int64])
def test_exact_quantiles_in_one_graph(sa, dtype):  # noqa: F811
    """The histogram finds the bucket that holds rank r, a filter of that bucket's closed interval returns its numbers, and the r-th
    number is picked among them on the device: p50 and p99 equal np.partition's, with no trip to the host inside the graph."""
    import torch

    from pcodec_b200 import wrapped

    rng = np.random.default_rng(21)
    xs = [(rng.lognormal(size=m) * 1000).astype(dtype) for m in (200000, 65536, 3333)]
    data, index, refs, d_data, d_index = _graph_inputs(sa, xs, dtype, order=0)
    x = np.concatenate(xs)
    n, mf, nb = len(x), len(xs), 256
    nc = sum(_n_chunks(index, r) for r in refs)
    out_cap = 1 << 16
    h = sa.AsyncFilesHistogram(data[:32], dtype, len(data), len(index), mf, nc, n, nb)
    f = sa.AsyncFilesFilter(data[:32], dtype, len(data), len(index), mf, nc, n, out_cap)
    d_files = torch.from_numpy(refs.view(np.int64)).cuda()
    nt = torch.tensor([mf], dtype=torch.int64, device="cuda")
    s = np.sort(x)
    ed = torch.from_numpy(wrapped.pack_edges(s[np.linspace(0, n - 1, nb + 1).astype(np.int64)], dtype)).cuda()
    hists = torch.zeros((mf, nb + 3), dtype=torch.int64, device="cuda")
    tot = torch.zeros(nb + 3, dtype=torch.int64, device="cuda")
    rank = torch.zeros(1, dtype=torch.int64, device="cuda")
    tdt = torch.float64 if dtype == np.float64 else torch.int64
    vals = torch.zeros(out_cap, dtype=tdt, device="cuda")
    pos = torch.zeros(out_cap, dtype=torch.int64, device="cuda")
    nm = torch.zeros(1, dtype=torch.int64, device="cuda")
    big = torch.tensor(float("inf") if dtype == np.float64 else np.iinfo(np.int64).max, dtype=tdt, device="cuda")
    idx = torch.arange(out_cap, device="cuda")

    def quantile():
        h(d_data, d_index, d_files, nt, ed, hists, tot)
        cum = torch.cumsum(tot, 0)
        c = torch.searchsorted(cum, rank, right=True)  # the column that holds rank r (0-based); indexing by tensors keeps it on the device
        below = torch.where(c > 0, cum.index_select(0, (c - 1).clamp(min=0)), 0)
        iv = torch.cat([ed.index_select(0, (c - 1).clamp(min=0, max=nb)), ed.index_select(0, c.clamp(max=nb))])
        f(d_data, d_index, d_files, nt, iv, vals, pos, nm)
        return torch.sort(torch.where(idx < nm[0], vals, big)).values.index_select(0, rank - below)

    quantile()
    torch.cuda.synchronize()
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        out = quantile()
    for q in (0.5, 0.99):
        r = int(q * (n - 1))
        rank.fill_(r)
        g.replay()
        torch.cuda.synchronize()
        assert h.result() == n and f.result() <= out_cap
        assert out.item() == np.partition(x, r)[r], q
