"""GPU tests of the asynchronous top-k calls (pco_b200_topk_pages_async / _files_async, wrapped.AsyncPagesTopK,
standalone.AsyncFilesTopK): exact equality with topk_reference over the decompress calls' output for every dtype, both directions, k = 1,
k = 1024 and k above the match count, the fused kernel and the general pair, cold pages and chunks of crafted streams, ties, signed zeros,
NaNs and infinities, empty and NaN intervals, zero pages or files, corrupt pages, sorted columns, graph replays, and a top-k feeding a take
in one graph."""
import numpy as np
import pytest

from tests import topk_reference as tr
from tests.test_gpu_async_aggregate import _frames
from tests.test_gpu_async_files import _batch, _cfg, _run as _files_run, _walk as _files_walk
from tests.test_gpu_async_filter_files import ROUTE_CASES, sa  # noqa: F401  (fixture)
from tests.test_gpu_async_pages import _dev, _refs_dev, _run as _pages_run
from tests.test_gpu_crafted_scans import _assert_routes, scans  # noqa: F401  (fixture)
from tests.test_gpu_crafted_streams import BY_DTYPE, crafted  # noqa: F401  (fixture)
from tests.test_gpu_encode import _walk
from tests.test_gpu_wrapped_batch import _container, _mixed_chunks, _shuffled, _six_pages

pytestmark = pytest.mark.gpu

DTYPES = [np.uint8, np.int8, np.uint16, np.int16, np.float16, np.uint32, np.int32, np.float32, np.uint64, np.int64, np.float64]
SENTINEL = 0x5A


def _full(dtype):
    dt = np.dtype(dtype)
    if dt.kind == "f":
        return -np.inf, np.inf
    return np.iinfo(dt).min, np.iinfo(dt).max


def _intervals(x, dtype):
    """The full range, a middle slice of the numbers present, and one present value alone."""
    dt = np.dtype(dtype)
    u = np.unique(x[~np.isnan(x)] if dt.kind == "f" else x)
    out = [_full(dtype)]
    if len(u):
        out += [(u[len(u) // 4], u[3 * len(u) // 4]), (u[len(u) // 2], u[len(u) // 2])]
    return out


def _buffers(k, dtype):
    import torch

    from pcodec_b200 import wrapped

    vals = torch.full((k * np.dtype(dtype).itemsize,), SENTINEL, dtype=torch.uint8, device="cuda").view(wrapped._torch_dtypes()[np.dtype(dtype)])
    pos = torch.full((k,), 0x5A5A5A5A5A5A5A5A, dtype=torch.int64, device="cuda")
    n_out = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    return vals, pos, n_out


def _outcome(h, call, k, dtype, profile=False):
    """Runs call(out_values, out_positions, n_out) and returns (values, positions, n_out, n_matches or None, error or None, status, spans)."""
    import ctypes as C

    from pcodec_b200 import PcoError, _lib

    vals, pos, n_out = _buffers(k, dtype)
    L = _lib.lib()
    if profile:
        L.pco_b200_profile_enable(1)
    try:
        call(vals, pos, n_out)
        st = h.status_record()
        spans = ""
        if profile:
            buf = C.create_string_buffer(1 << 16)
            L.pco_b200_profile_last(buf, C.c_size_t(len(buf)))
            spans = buf.value.decode()
    finally:
        if profile:
            L.pco_b200_profile_enable(0)
    try:
        nm, err = h.result(), None
    except PcoError as e:
        nm, err = None, e
    return vals.cpu().numpy(), pos.cpu().numpy().view(np.uint64), int(n_out.cpu()[0]), nm, err, st, spans


def _check(got, x, lo, hi, k, largest):
    """The outputs equal topk_reference's bit for bit, and the slots past *n_out are untouched."""
    vals, pos, n, nm, err, _, _ = got
    assert err is None, err
    wv, wp = tr.topk(x, lo, hi, k, largest)
    ut = f"u{x.dtype.itemsize}"
    assert n == len(wv) and nm == len(tr.matches(x, lo, hi)), (n, len(wv), nm, lo, hi, k, largest)
    assert np.array_equal(pos[:n], wp), (lo, hi, k, largest, pos[:n][:8], wp[:8])
    assert np.array_equal(vals[:n].view(ut), wv.view(ut)), (lo, hi, k, largest)
    assert (vals[n:].view(np.uint8) == SENTINEL).all() and (pos[n:] == 0x5A5A5A5A5A5A5A5A).all(), "slots past n_out written"


def _topk_pages(metas, pages, refs, dtype, lo, hi, k, largest, max_pages=None, rows_cap=None, frame_cap=-1, n=None, profile=False):
    import torch

    from pcodec_b200 import wrapped

    total = int(np.asarray(refs)["page_n"].sum()) if len(refs) else 0
    max_pages = max_pages or max(len(refs), 1)
    rows_cap = total if rows_cap is None else rows_cap
    if frame_cap == -1:
        frame_cap = _frames(metas, pages, refs, max_pages)
    h = wrapped.AsyncPagesTopK(dtype, len(metas), len(pages), max_pages, rows_cap, k, largest, frame_cap)
    iv = torch.from_numpy(wrapped.pack_interval(lo, hi, dtype)).cuda()
    nt = torch.tensor([len(refs) if n is None else n], dtype=torch.int64).cuda()
    m, p, r = _dev(metas), _dev(pages), _refs_dev(refs, max_pages)
    return _outcome(h, lambda v, ps, no: h(m, p, r, nt, iv, v, ps, no), k, dtype, profile)


def _topk_files(sa, data, index, dtype, refs, lo, hi, k, largest, max_files=None, max_chunks=None, rows_cap=None, profile=False):  # noqa: F811
    import torch

    from pcodec_b200 import wrapped
    from tests.test_gpu_async_files import _n_chunks
    from tests.test_gpu_async_aggregate import _chunk_ns

    nc = sum(_n_chunks(index, r) for r in refs)
    if rows_cap is None:
        rows_cap = sum(sum(_chunk_ns(index, r)) for r in refs)
    mf = max_files or max(len(refs), 1)
    head = data[int(refs[0][0]):int(refs[0][0]) + 32] if len(refs) else data[:32]
    h = sa.AsyncFilesTopK(head, dtype, len(data), len(index), mf, max_chunks or max(nc, 1), rows_cap, k, largest)
    d_data = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    d_index = torch.frombuffer(bytearray(index), dtype=torch.uint8).cuda()
    fr = np.zeros((mf, 4), np.uint64)
    fr[: len(refs)] = refs
    d_files = torch.from_numpy(fr.view(np.int64)).cuda()
    nt = torch.tensor([len(refs)], dtype=torch.int64, device="cuda")
    iv = torch.from_numpy(wrapped.pack_interval(lo, hi, dtype)).cuda()
    return _outcome(h, lambda v, ps, no: h(d_data, d_index, d_files, nt, iv, v, ps, no), k, dtype, profile)


def _files_numbers(sa, data, index, dtype, refs):
    dec, err, _ = _files_run(sa, data, index, dtype, refs)
    assert err is None, err
    return dec[0]


# ---- pages


@pytest.mark.parametrize("dtype", DTYPES)
def test_every_dtype_on_a_mixed_batch_of_pages(oracle, dtype):
    metas, pages, refs, pieces = _container(_mixed_chunks(oracle, dtype))
    refs, pieces = _shuffled(refs, pieces, seed=int(np.dtype(dtype).num))
    got, nw, err, _ = _pages_run(metas, pages, refs, dtype, frame_cap=_frames(metas, pages, refs, len(refs)))
    assert err is None
    x = got[:nw]
    for lo, hi in _intervals(x, dtype):
        for k in (1, 100, 1024):
            for largest in (False, True):
                _check(_topk_pages(metas, pages, refs, dtype, lo, hi, k, largest), x, lo, hi, k, largest)


def test_zero_pages_empty_and_nan_intervals(oracle):
    metas, pages, refs, pieces = _six_pages(oracle)
    x = np.concatenate(pieces)
    got = _topk_pages(metas, pages, refs[:0], np.uint64, 0, (1 << 64) - 1, 10, False, max_pages=len(refs), n=0)
    _check(got, x[:0], 0, (1 << 64) - 1, 10, False)
    _check(_topk_pages(metas, pages, refs, np.uint64, 5, 4, 10, True), x, 5, 4, 10, True)


def test_refusals_and_corrupt_pages_fail_as_the_pages_call(oracle):
    metas, pages, refs, pieces = _six_pages(oracle)
    total = sum(len(p) for p in pieces)
    for kw in ({"max_pages": len(refs), "n": len(refs) + 1, "rows_cap": total}, {"rows_cap": total - 1}):
        _, _, perr, pst = _pages_run(metas, pages, refs, np.uint64, **{k: v for k, v in kw.items() if k in ("max_pages", "n")},
                                     dst_cap=kw.get("rows_cap"), frame_cap=_frames(metas, pages, refs, len(refs)))
        vals, pos, n, _, err, st, _ = _topk_pages(metas, pages, refs, np.uint64, 0, (1 << 64) - 1, 16, False, **kw)
        assert perr is not None and err is not None and (err.kind, st.device_status, st.page) == (perr.kind, pst.device_status, pst.page)
        assert err.message.split(":")[0] == perr.message.split(":")[0]
        assert n == 0 and (vals.view(np.uint8) == SENTINEL).all() and (pos == 0x5A5A5A5A5A5A5A5A).all()
    bad = bytearray(pages)
    r = refs[2]
    bad[int(r["page_offset"]) + int(r["page_len"]) // 2] ^= 0x24
    _, _, perr, pst = _pages_run(metas, bytes(bad), refs, np.uint64, frame_cap=_frames(metas, bytes(bad), refs, len(refs)))
    vals, pos, n, _, err, st, _ = _topk_pages(metas, bytes(bad), refs, np.uint64, 0, (1 << 64) - 1, 16, True)
    assert (perr is None) == (err is None)
    if perr is not None:
        assert (err.kind, st.page) == (perr.kind, pst.page) and n == 0 and (pos == 0x5A5A5A5A5A5A5A5A).all()


def test_pages_graph_replays_new_refs_counts_and_intervals(oracle):
    import torch

    from pcodec_b200 import wrapped

    metas, pages, refs, pieces = _six_pages(oracle)
    mp, total, k = len(refs), sum(len(p) for p in pieces), 50
    h = wrapped.AsyncPagesTopK(np.uint64, len(metas), len(pages), mp, total, k, True)
    d_m, d_p, d_r = _dev(metas), _dev(pages), _refs_dev(refs, mp)
    nt = torch.tensor([mp], dtype=torch.int64, device="cuda")
    iv = torch.from_numpy(wrapped.pack_interval(0, (1 << 64) - 1, np.uint64)).cuda()
    vals, pos, n_out = _buffers(k, np.uint64)
    h(d_m, d_p, d_r, nt, iv, vals, pos, n_out)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        h(d_m, d_p, d_r, nt, iv, vals, pos, n_out)
    rng = np.random.default_rng(3)
    for trial in range(4):
        order = rng.permutation(mp)[: int(rng.integers(1, mp + 1))]
        x = np.concatenate([pieces[i] for i in order])
        u = np.unique(x)
        lo, hi = (u[0], u[-1]) if trial == 0 else (u[len(u) // 3], u[2 * len(u) // 3])
        d_r.copy_(_refs_dev(refs[order], mp))
        nt.fill_(len(order))
        iv.copy_(torch.from_numpy(wrapped.pack_interval(lo, hi, np.uint64)))
        outs = []
        for _ in range(2):
            g.replay()
            nm = h.result()
            outs.append((vals.cpu().numpy().copy(), pos.cpu().numpy().view(np.uint64).copy(), int(n_out.cpu()[0])))
        wv, wp = tr.topk(x, lo, hi, k, True)
        for v, p, n in outs:
            assert n == len(wv) and nm == len(tr.matches(x, lo, hi))
            assert np.array_equal(p[:n], wp) and np.array_equal(v[:n], wv)


# ---- files


@pytest.mark.parametrize("dtype", DTYPES)
def test_every_dtype_on_a_batch_of_files(sa, dtype):  # noqa: F811
    xs = [_files_walk(dtype, m, seed=int(np.dtype(dtype).num) + i) for i, m in enumerate([3 * (1 << 14) + 777, 1, 0, 5000, 1 << 14, 257])]
    for order in (0, 1, 3):  # fused orders 0 and 1, the general pair at order 3
        data, index, refs = _batch(sa, xs, _cfg(order))
        x = _files_numbers(sa, data, index, dtype, refs)
        for lo, hi in _intervals(x, dtype)[:2]:
            for k in (1, 1024, x.size + 5):
                for largest in (False, True):
                    if k <= 1024:
                        _check(_topk_files(sa, data, index, dtype, refs, lo, hi, k, largest), x, lo, hi, k, largest)


@pytest.mark.parametrize("dtype", [np.float16, np.float32, np.float64])
def test_signed_zeros_nans_and_infinities(sa, dtype):  # noqa: F811
    dt = np.dtype(dtype)
    ut = np.dtype(f"u{dt.itemsize}")
    rng = np.random.default_rng(11)
    x = np.round(rng.normal(size=40000) * 3).astype(dt)
    special = np.array([-0.0, 0.0, np.inf, -np.inf, np.nan, -np.nan], dt)
    x[rng.integers(0, x.size, 3000)] = special[rng.integers(0, special.size, 3000)]
    x.view(ut)[rng.integers(0, x.size, 50)] |= ut.type(np.array(np.nan, dt).view(ut)) | ut.type(1)  # NaN payloads of both signs
    data, index, refs = _batch(sa, [x[:25000], x[25000:]], _cfg(0))
    y = _files_numbers(sa, data, index, dtype, refs)
    assert np.array_equal(y.view(ut), x.view(ut))
    for lo, hi in [(-np.inf, np.inf), (-0.0, 0.0), (0.0, -0.0), (0.0, 0.0), (np.inf, np.inf), (-1.0, 1.0), (np.nan, 1.0), (1.0, -1.0)]:
        for k in (1, 1024):
            for largest in (False, True):
                _check(_topk_files(sa, data, index, dtype, refs, lo, hi, k, largest), y, lo, hi, k, largest)


def test_ties_return_the_first_positions(sa):  # noqa: F811
    x = np.full(150000, 7, np.int32)
    for order in (0, 1):
        data, index, refs = _batch(sa, [x[:100000], x[100000:]], _cfg(order))
        for k in (1, 1000, 1024):
            for largest in (False, True):
                got = _topk_files(sa, data, index, np.int32, refs, -10, 10, k, largest)
                _check(got, x, -10, 10, k, largest)
                assert np.array_equal(got[1][:k], np.arange(k, dtype=np.uint64))


def test_ascending_and_descending_columns(sa):  # noqa: F811
    x = np.arange(1 << 19, dtype=np.uint64) * 3 + 11
    for col in (x, x[::-1].copy()):
        for order in (0, 1):
            data, index, refs = _batch(sa, [col[:300000], col[300000:]], _cfg(order, page=1 << 16))
            for k in (1, 100, 1024):
                for largest in (False, True):
                    _check(_topk_files(sa, data, index, np.uint64, refs, 0, (1 << 64) - 1, k, largest), col, 0, (1 << 64) - 1, k, largest)


@pytest.mark.parametrize("name", ["cold_level9", "cold_level12", "general_int_mult", "general_float_mult"])
def test_files_with_cold_chunks_and_two_var_modes(sa, name):  # noqa: F811
    dtype, arrays, cfg, _ = ROUTE_CASES[name]
    xs = [np.asarray(a, dtype=dtype) for a in arrays()]
    data, index, refs = _batch(sa, xs, cfg())
    sel = refs[[1, 0, 1]]
    x = _files_numbers(sa, data, index, dtype, sel)
    for k in (1, 1024):
        for largest in (False, True):
            got = _topk_files(sa, data, index, dtype, sel, *_full(dtype), k, largest, profile=name.startswith("cold"))
            _check(got, x, *_full(dtype), k, largest)
            if name.startswith("cold"):
                assert "topk_cold_files_kernel" in got[6] and "cold_chunks_kernel" in got[6], got[6]


def test_zero_files_and_corrupt_files(sa):  # noqa: F811
    xs = [_walk(np.uint32, s, seed=s) for s in (9000, 20000, 700)]
    data, index, refs = _batch(sa, xs, _cfg(0, page=4096))
    x = _files_numbers(sa, data, index, np.uint32, refs)
    got = _topk_files(sa, data, index, np.uint32, refs[:0], 0, (1 << 32) - 1, 5, False, max_files=3, max_chunks=64, rows_cap=x.size)
    _check(got, x[:0], 0, (1 << 32) - 1, 5, False)
    for kw in ({"rows_cap": 9000 + 100}, {"max_chunks": 2}):
        _, perr, pst = _files_run(sa, data, index, np.uint32, refs, dst_cap=kw.get("rows_cap"), max_chunks=kw.get("max_chunks"))
        vals, pos, n, _, err, st, _ = _topk_files(sa, data, index, np.uint32, refs, 0, (1 << 32) - 1, 5, False, **kw)
        assert perr is not None and err is not None and (err.kind, st.device_status, st.file, st.chunk) == (perr[0], pst.device_status, pst.file, pst.chunk)
        assert n == 0 and (pos == 0x5A5A5A5A5A5A5A5A).all()
    bad = bytearray(data)
    bad[int(refs[1][0]) + int(refs[1][1]) // 2] ^= 0x10
    _, perr, pst = _files_run(sa, bytes(bad), index, np.uint32, refs)
    vals, pos, n, _, err, st, _ = _topk_files(sa, bytes(bad), index, np.uint32, refs, 0, (1 << 32) - 1, 5, True)
    assert (perr is None) == (err is None)
    if perr is not None:
        assert (err.kind, st.file, st.chunk) == (perr[0], pst.file, pst.chunk) and n == 0


def test_files_graph_topk_then_take_from_another_column(sa):  # noqa: F811
    """Top-k on column A, its positions sorted, then a take from column B at those positions, in one graph replayed with new files, a
    new count and a new interval."""
    import torch

    from pcodec_b200 import wrapped

    rng = np.random.default_rng(5)
    sizes = [70000, 1, 5000, 1 << 16, 300]
    a = [rng.integers(0, 1 << 30, size=m).astype(np.int64) for m in sizes]
    b = [np.arange(m, dtype=np.uint32) * 7 + i for i, m in enumerate(sizes)]
    da, ia, ra = _batch(sa, a, _cfg(1))
    db, ib, rb = _batch(sa, b, _cfg(0))
    mf, k = len(sizes), 100
    from tests.test_gpu_async_files import _n_chunks

    nca, ncb = sum(_n_chunks(ia, r) for r in ra), sum(_n_chunks(ib, r) for r in rb)
    rows = sum(sizes)
    top = sa.AsyncFilesTopK(da[:32], np.int64, len(da), len(ia), mf, nca, rows, k, True)
    take = sa.AsyncFilesTake(db[:32], np.uint32, len(db), len(ib), mf, ncb, rows, k)
    t = lambda buf: torch.frombuffer(bytearray(buf), dtype=torch.uint8).cuda()  # noqa: E731
    d_da, d_ia, d_db, d_ib = t(da), t(ia), t(db), t(ib)
    fa = torch.from_numpy(ra.view(np.int64).copy()).cuda()
    fb = torch.from_numpy(rb.view(np.int64).copy()).cuda()
    nt = torch.tensor([mf], dtype=torch.int64, device="cuda")
    iv = torch.from_numpy(wrapped.pack_interval(0, 1 << 40, np.int64)).cuda()
    vals, pos, n_out = _buffers(k, np.int64)
    tv = torch.zeros(k, dtype=torch.uint32, device="cuda")
    idx = torch.arange(k, device="cuda")

    def step():
        top(d_da, d_ia, fa, nt, iv, vals, pos, n_out)
        sp = torch.sort(torch.where(idx < n_out[0], pos, torch.iinfo(torch.int64).max)).values
        take(d_db, d_ib, fb, nt, sp, n_out, tv)
        return sp

    step()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        sp = step()
    for n_files, lo, hi in [(5, 0, 1 << 40), (3, 1 << 20, 1 << 29), (2, 5, 5)]:
        nt.fill_(n_files)
        iv.copy_(torch.from_numpy(wrapped.pack_interval(lo, hi, np.int64)))
        g.replay()
        top.result()
        take.result()
        xa, xb = np.concatenate(a[:n_files]), np.concatenate(b[:n_files])
        wv, wp = tr.topk(xa, lo, hi, k, True)
        n = int(n_out.cpu()[0])
        assert n == len(wv) and np.array_equal(pos.cpu().numpy().view(np.uint64)[:n], wp)
        assert np.array_equal(tv.cpu().numpy()[:n], xb[np.sort(wp).astype(np.int64)])


# ---- crafted streams: Dict, Lookback, Conv1, wide tables; pages and files, every dtype


@pytest.mark.parametrize("kind", ["pages", "files"])
@pytest.mark.parametrize("dtype_str", BY_DTYPE)
def test_crafted_streams(scans, dtype_str, kind):  # noqa: F811
    import torch

    from pcodec_b200 import standalone, wrapped

    s = scans[dtype_str]
    want, groups, args = s.side(kind)
    cls = wrapped.AsyncPagesTopK if kind == "pages" else standalone.AsyncFilesTopK
    first = True
    for k in (1, 1024):
        for largest in (False, True):
            h = cls(dtype=s.dt, **s.plan_args(kind), rows_cap=want.size, k=k, largest=largest)
            lo, hi = _full(s.dt)
            iv = torch.from_numpy(wrapped.pack_interval(lo, hi, s.dt)).cuda()
            got = _outcome(h, lambda v, p, n: h(*args, iv, v, p, n), k, s.dt, profile=first)
            if first:
                spans = {kv.split("=")[0] for kv in got[6].split(";") if kv}
                cold = "ap_cold_kernel" if kind == "pages" else "cold_chunks_kernel"
                assert cold in spans and f"topk_cold_{kind}_kernel" in spans, sorted(spans)
                first = False
            _check(got, want, lo, hi, k, largest)
