"""Host side of the asynchronous histograms (pco_b200_histogram_pages_async_plan / _files_async_plan / _result,
wrapped.AsyncPagesHistogram, standalone.AsyncFilesHistogram, wrapped.pack_edges) without a GPU: the plans' argument checks, their
workspace sizes against the formulas include/pco_b200.h documents, how a status written by the device becomes a kind and a message, the
calls' host-side refusals, the wrappers' argument checks, pack_edges, and the numpy statement of the rows on hand-worked cases."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from tests import histogram_reference as hr
from tests.test_async_files_host import HEAD
from tests.test_async_files_host import _expected_workspace as _files_workspace
from tests.test_async_pages_host import _expected_workspace as _pages_workspace
from tests.test_async_take_host import _FakeTensor, _bare

U64, U32 = 2, 1
NONE = (1 << 64) - 1
ELEM = {1: 4, 2: 8, 3: 4, 4: 8, 5: 4, 6: 8, 7: 2, 8: 2, 9: 2, 10: 1, 11: 1}
EDGES_ORDER = 0x501
DTYPES = [np.uint8, np.int8, np.uint16, np.int16, np.float16, np.uint32, np.int32, np.float32, np.uint64, np.int64, np.float64]
al = lambda x: (x + 255) // 256 * 256  # noqa: E731
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def L():
    from pcodec_b200 import wrapped

    return wrapped._lib_async_histogram()


@pytest.fixture(scope="module")
def LF():
    from pcodec_b200 import standalone

    return standalone._lib_async_histogram_files()


def _plan(L, dtype=U64, metas_cap=1 << 12, pages_cap=1 << 20, max_pages=64, rows_cap=1 << 18, frame_cap=1 << 21, n_buckets=256, plan=True):
    from pcodec_b200 import wrapped

    p = wrapped._CAsyncHistogramPlan()
    rc = L.pco_b200_histogram_pages_async_plan(C.c_ubyte(dtype), C.c_size_t(metas_cap), C.c_size_t(pages_cap), C.c_size_t(max_pages),
                                               C.c_size_t(rows_cap), C.c_size_t(frame_cap), C.c_size_t(n_buckets), C.byref(p) if plan else None)
    return rc, p, L.pco_b200_last_error_message().decode()


def _files_plan(LF, head, dtype=U32, max_files=8, max_chunks=16, rows_cap=1 << 16, n_buckets=256, src_cap=1 << 20, index_cap=1 << 16,
                plan=True):
    from pcodec_b200 import standalone

    p = standalone._CAsyncFilesHistogramPlan()
    buf = C.create_string_buffer(head, len(head))
    rc = LF.pco_b200_histogram_files_async_plan(buf, C.c_size_t(len(head)), C.c_ubyte(dtype), C.c_size_t(src_cap), C.c_size_t(index_cap),
                                                C.c_size_t(max_files), C.c_size_t(max_chunks), C.c_size_t(rows_cap), C.c_size_t(n_buckets),
                                                C.byref(p) if plan else None)
    return rc, p, LF.pco_b200_last_error_message().decode()


def _header_regions(call):
    """The regions the header's workspace paragraph of `call`'s plan lists, as (coefficient, term, name)."""
    text = open(os.path.join(ROOT, "include", "pco_b200.h")).read()
    doc = re.search(r"/\*((?:(?!\*/).)*?)\*/\s*PcoB200Error " + call + r"\(", text, flags=re.S).group(1)
    doc = " ".join(line.strip(" *") for line in doc.splitlines())
    tail = doc.split("E the bytes of a number of dtype:")[1]
    terms = r"W max_pages|W max_files|W|max_pages|max_chunks|rows_cap|\(max_chunks \+ 1\)|\(n_buckets \+ 2\)"
    return re.findall(r"(\d+|E)(?: (" + terms + r"))? \(([^)]*)\)", tail)


def _formula(call, elem, rows_cap, m, groups, nb):
    w = nb + 3
    terms = {"": 1, "W": w, "W max_pages": w * groups, "W max_files": w * groups, "rows_cap": rows_cap, "max_pages": m, "max_chunks": m,
             "(max_chunks + 1)": m + 1, "(n_buckets + 2)": nb + 2}
    return sum(al((elem if coef == "E" else int(coef)) * terms[term]) for coef, term, _ in _header_regions(call))


def test_header_lists_the_regions():
    assert [r[2] for r in _header_regions("pco_b200_histogram_pages_async_plan")] == [
        "the pages status", "the plan's state", "each page's group", "the edge table", "the cold pages' values", "the pages' rows",
        "the column sums"]
    assert [r[2] for r in _header_regions("pco_b200_histogram_files_async_plan")] == [
        "the files status", "the plan's state", "each chunk's group", "the edge table", "the cold chunks' values", "slot map", "cold list",
        "the files' rows", "the column sums"]


def _expected_pages(dtype, max_pages, rows_cap, frame_cap, nb):
    w = nb + 3
    own = sum(al(r) for r in [40, 16, 4 * max_pages, 8 * (nb + 2), ELEM[dtype] * rows_cap, 8 * w * max_pages, 8 * w])
    assert own == _formula("pco_b200_histogram_pages_async_plan", ELEM[dtype], rows_cap, max_pages, max_pages, nb)
    return _pages_workspace(max_pages, rows_cap, frame_cap) + own


def _expected_files(dtype, max_files, max_chunks, rows_cap, nb):
    w = nb + 3
    own = sum(al(r) for r in [40, 16, 4 * max_chunks, 8 * (nb + 2), ELEM[dtype] * rows_cap, 4 * max_chunks, 4 * (max_chunks + 1),
                              8 * w * max_files, 8 * w])
    assert own == _formula("pco_b200_histogram_files_async_plan", ELEM[dtype], rows_cap, max_chunks, max_files, nb)
    return _files_workspace(max_files, max_chunks, rows_cap) + own


def test_argument_checks_come_before_the_device(L):
    rc, _, msg = _plan(L, dtype=99)
    assert rc == 5 and "type" in msg, msg
    for mp in (0, 1 << 31):
        rc, _, msg = _plan(L, max_pages=mp)
        assert rc == 3 and "max_pages" in msg, msg
    for name in ("rows_cap", "frame_cap"):
        rc, _, msg = _plan(L, **{name: (1 << 56) + 1})
        assert rc == 3 and name in msg, msg
    for nb in (0, 4097, 1 << 40):
        rc, _, msg = _plan(L, n_buckets=nb)
        assert rc == 3 and "n_buckets" in msg, msg
    rc, _, _ = _plan(L, plan=False)
    assert rc == 3


def test_n_buckets_range_is_accepted_up_to_the_device(L, LF):
    """1 and 4096 pass the checks: without a device the plan then stops at the device (PCO_B200_CUDA), not at the argument."""
    import torch

    for nb in (1, 2, 255, 4096):
        rc, p, msg = _plan(L, n_buckets=nb)
        assert rc in (0, 6) and "n_buckets" not in msg, msg
        if not torch.cuda.is_available():
            assert rc == 6, msg
        assert p.n_buckets == nb
        rc, p, msg = _files_plan(LF, HEAD, n_buckets=nb)
        assert rc in (0, 6) and "n_buckets" not in msg, msg
        assert p.n_buckets == nb


@pytest.mark.parametrize("dtype", sorted(ELEM))
@pytest.mark.parametrize("mp,rc_,fc,nb", [(1, 0, 0, 1), (3, 255, 17, 5), (257, 12345, 999, 256), (4096, 1 << 24, 1 << 30, 4096)])
def test_pages_workspace_matches_the_formula(L, dtype, mp, rc_, fc, nb):
    _, p, _ = _plan(L, dtype=dtype, max_pages=mp, rows_cap=rc_, frame_cap=fc, n_buckets=nb)
    assert (p.dtype, p.max_pages, p.rows_cap, p.frame_cap, p.n_buckets) == (dtype, mp, rc_, fc, nb)
    assert p.workspace_bytes == _expected_pages(dtype, mp, rc_, fc, nb)


@pytest.mark.parametrize("dtype", sorted(ELEM))
@pytest.mark.parametrize("mf,mc,rows,nb", [(1, 1, 0, 1), (8, 16, 1 << 16, 300), (4096, 5000, 12345, 16), (3, 1 << 20, 1 << 28, 4096)])
def test_files_workspace_matches_the_formula(LF, dtype, mf, mc, rows, nb):
    _, p, _ = _files_plan(LF, HEAD, dtype=dtype, max_files=mf, max_chunks=mc, rows_cap=rows, n_buckets=nb)
    assert (p.dtype, p.max_files, p.max_chunks, p.rows_cap, p.n_buckets) == (dtype, mf, mc, rows, nb)
    assert p.workspace_bytes == _expected_files(dtype, mf, mc, rows, nb)


def test_workspace_does_not_depend_on_the_buffers(L, LF):
    ws = lambda **kw: _plan(L, **kw)[1].workspace_bytes  # noqa: E731
    assert ws(metas_cap=1 << 30, pages_cap=1 << 30) == ws()
    _, p, _ = _files_plan(LF, HEAD)
    _, q, _ = _files_plan(LF, HEAD, src_cap=1 << 40, index_cap=1 << 40)
    assert q.src_cap == 1 << 40 and q.workspace_bytes == p.workspace_bytes


def test_files_plan_checks(LF):
    for kw, words in [({"max_files": 0}, "max_files"), ({"max_chunks": 0}, "max_chunks"), ({"rows_cap": (1 << 56) + 1}, "rows_cap"),
                      ({"n_buckets": 0}, "n_buckets"), ({"n_buckets": 4097}, "n_buckets")]:
        rc, _, msg = _files_plan(LF, HEAD, **kw)
        assert rc == 3 and words in msg, msg
    rc, _, msg = _files_plan(LF, HEAD, dtype=99)
    assert rc == 5


def _result(L, **fields):
    from pcodec_b200 import wrapped

    s = wrapped._CAsyncHistogramStatus(**fields)
    n = C.c_size_t(12345)
    rc = L.pco_b200_histogram_pages_async_result(C.byref(s), C.byref(n))
    return rc, L.pco_b200_last_error_message().decode(), n.value


def _files_result(LF, **fields):
    from pcodec_b200 import standalone

    s = standalone._CAsyncFilesHistogramStatus(**fields)
    n = C.c_size_t(12345)
    rc = LF.pco_b200_histogram_files_async_result(C.byref(s), C.byref(n))
    return rc, LF.pco_b200_last_error_message().decode(), n.value


def test_result_of_success_is_the_rows_counted(L, LF):
    assert _result(L, kind=0, n_written=1000, page=NONE, edge=NONE)[::2] == (0, 1000)
    assert _files_result(LF, kind=0, n_written=77, file=NONE, chunk=NONE, edge=NONE)[::2] == (0, 77)
    assert L.pco_b200_histogram_pages_async_result(None, None) == 3
    assert LF.pco_b200_histogram_files_async_result(None, None) == 3


@pytest.mark.parametrize("res", ["_result", "_files_result"])
def test_result_names_the_edge(L, LF, res):
    f = (lambda **kw: _result(L, **kw)) if res == "_result" else (lambda **kw: _files_result(LF, **kw))
    for edge in (0, 1, 17, 4096):
        rc, msg, n = f(kind=3, device_status=EDGES_ORDER, edge=edge, n_written=1000)
        assert rc == 3 and msg.startswith(f"edge {edge}: ") and "strictly increasing" in msg and n == 12345, msg


def test_result_of_upstream_statuses_is_the_decompress_calls(L, LF):
    rc, msg, _ = _result(L, kind=2, device_status=2, page=17)
    assert rc == 2 and msg.startswith("page 17: ") and "insufficient data" in msg, msg
    rc, msg, _ = _result(L, kind=3, device_status=0x11e, page=4)
    assert rc == 3 and msg.startswith("page 4: ") and "rows_cap" in msg, msg
    rc, msg, _ = _result(L, kind=3, device_status=0x11a, page=NONE, n_pages=99)
    assert rc == 3 and "*n_pages is 99" in msg, msg
    rc, msg, _ = _result(L, kind=4, device_status=0x11f, page=NONE, frames_needed=5000)
    assert rc == 4 and "5000 bytes" in msg, msg
    rc, msg, _ = _files_result(LF, kind=1, device_status=1, file=3, chunk=2)
    assert rc == 1 and msg == "file 3: corrupt data in chunk 2", msg
    rc, msg, _ = _files_result(LF, kind=7, device_status=7, file=0, chunk=5)
    assert rc == 7 and msg.startswith("file 0: "), msg


def test_the_edge_code_is_documented_with_its_kind():
    text = open(os.path.join(ROOT, "include", "pco_b200.h")).read()
    codes = dict((name, int(v, 16)) for name, v in re.findall(r"(PCO_B200_HIST_\w+)\s*=\s*(0x[0-9a-f]+)", text))
    assert codes == {"PCO_B200_HIST_EDGES_ORDER": EDGES_ORDER}
    assert re.search(r"PCO_B200_HIST_EDGES_ORDER\s*=\s*0x501\s*/\*(?:(?!\*/).)*\(PCO_B200_INVALID_ARGUMENT\) \*/", text)


def test_calls_refuse_missing_buffers_without_a_device(L, LF):
    from pcodec_b200 import standalone, wrapped

    _, p, _ = _plan(L)
    nz = C.c_void_p(256)
    s = wrapped._CAsyncHistogramStatus()
    args = [nz] * 8  # metas, pages, refs, n_pages, edges, hists, total, workspace
    for i in range(8):
        a = list(args)
        a[i] = None
        assert L.pco_b200_histogram_pages_async(C.byref(p), *a, C.byref(s), None) == 3
        assert "null buffer" in L.pco_b200_last_error_message().decode()
    assert L.pco_b200_histogram_pages_async(C.byref(p), *args, None, None) == 3  # null status
    assert L.pco_b200_histogram_pages_async(C.byref(p), *args[:7], C.c_void_p(257), C.byref(s), None) == 3
    assert "aligned" in L.pco_b200_last_error_message().decode()
    bad = wrapped._CAsyncHistogramPlan.from_buffer_copy(bytes(p))
    bad.n_buckets = 4097
    assert L.pco_b200_histogram_pages_async(C.byref(bad), *args, C.byref(s), None) == 3
    assert "not made by" in L.pco_b200_last_error_message().decode()
    assert L.pco_b200_histogram_pages_async(C.byref(wrapped._CAsyncHistogramPlan()), *args, C.byref(s), None) == 3
    assert "not made by" in L.pco_b200_last_error_message().decode()

    _, fp, _ = _files_plan(LF, HEAD)
    fs = standalone._CAsyncFilesHistogramStatus()
    for i in range(8):  # src, index, files, n_files, edges, hists, total, workspace
        a = list(args)
        a[i] = None
        assert LF.pco_b200_histogram_files_async(C.byref(fp), *a, C.byref(fs), None) == 3
        assert "null buffer" in LF.pco_b200_last_error_message().decode()
    assert LF.pco_b200_histogram_files_async(C.byref(fp), *args[:7], C.c_void_p(257), C.byref(fs), None) == 3
    assert "aligned" in LF.pco_b200_last_error_message().decode()
    bad = standalone._CAsyncFilesHistogramPlan.from_buffer_copy(bytes(fp))
    bad.workspace_bytes += 1
    assert LF.pco_b200_histogram_files_async(C.byref(bad), *args, C.byref(fs), None) == 3
    assert "not made by" in LF.pco_b200_last_error_message().decode()


def test_new_symbols_are_exported(L, LF):
    for name in ("pco_b200_histogram_pages_async_plan", "pco_b200_histogram_pages_async", "pco_b200_histogram_pages_async_result"):
        assert hasattr(L, name), name
    for name in ("pco_b200_histogram_files_async_plan", "pco_b200_histogram_files_async", "pco_b200_histogram_files_async_result"):
        assert hasattr(LF, name), name
    from pcodec_b200 import standalone, wrapped

    assert callable(wrapped.AsyncPagesHistogram) and callable(standalone.AsyncFilesHistogram) and callable(wrapped.pack_edges)


def test_status_structs_match_the_header():
    from pcodec_b200 import standalone, wrapped

    assert C.sizeof(wrapped._CAsyncHistogramStatus) == 48 and C.sizeof(standalone._CAsyncFilesHistogramStatus) == 48
    assert C.sizeof(wrapped._CAsyncHistogramPlan) == 64 and C.sizeof(standalone._CAsyncFilesHistogramPlan) == 72


def test_pages_wrapper_checks_its_arguments():
    import torch

    from pcodec_b200 import wrapped

    p = wrapped._CAsyncHistogramPlan(dtype=U64, metas_cap=64, pages_cap=64, max_pages=4, rows_cap=1024, frame_cap=256, n_buckets=10)
    t = _bare(wrapped.AsyncPagesHistogram, p, np.uint64)
    T = lambda dt, *shape: _FakeTensor(dt, shape, t.device)  # noqa: E731
    good = dict(metas=T(torch.uint8, 64), pages=T(torch.uint8, 64), refs=T(torch.int64, 4, 5), n_pages=T(torch.int64, 1),
                edges=T(torch.int64, 11), hists=T(torch.int64, 4, 13), total=T(torch.int64, 13))
    for name, bad, words in [("edges", T(torch.int64, 10), "edges"), ("edges", T(torch.int32, 11), "edges"),
                             ("hists", T(torch.int64, 3, 13), "hists"), ("hists", T(torch.int64, 4, 12), "hists"),
                             ("hists", T(torch.int32, 4, 13), "hists"), ("total", T(torch.int64, 12), "total"),
                             ("total", T(torch.float64, 13), "total"), ("refs", T(torch.int64, 3, 5), "refs"),
                             ("n_pages", T(torch.int64, 2), "n_pages"), ("metas", T(torch.uint8, 63), "metas_cap")]:
        with pytest.raises(ValueError, match=words):
            t(**dict(good, **{name: bad}))
    with pytest.raises(ValueError, match="edges must be a contiguous CUDA tensor"):
        t(**dict(good, edges=object()))


def test_files_wrapper_checks_its_arguments():
    import torch

    from pcodec_b200 import standalone

    p = standalone._CAsyncFilesHistogramPlan(dtype=U32, src_cap=64, index_cap=64, max_files=2, max_chunks=4, rows_cap=1024, n_buckets=1)
    t = _bare(standalone.AsyncFilesHistogram, p, np.uint32)
    T = lambda dt, *shape: _FakeTensor(dt, shape, t.device)  # noqa: E731
    good = dict(src=T(torch.uint8, 64), index=T(torch.uint8, 64), files=T(torch.int64, 2, 4), n_files=T(torch.int64, 1),
                edges=T(torch.int64, 2), hists=T(torch.int64, 2, 4), total=T(torch.int64, 4))
    for name, bad, words in [("edges", T(torch.int64, 3), "edges"), ("hists", T(torch.int64, 1, 4), "hists"),
                             ("total", T(torch.int64, 5), "total"), ("files", T(torch.int64, 2, 5), "files"),
                             ("n_files", T(torch.int64, 2), "n_files"), ("src", T(torch.uint8, 63), "src_cap")]:
        with pytest.raises(ValueError, match=words):
            t(**dict(good, **{name: bad}))


# ---- pack_edges


@pytest.mark.parametrize("dtype", DTYPES)
def test_pack_edges_round_trips(dtype):
    from pcodec_b200 import wrapped

    dt = np.dtype(dtype)
    ut = np.dtype(f"u{dt.itemsize}")
    if dt.kind == "f":
        values = [-np.inf, -1.5, -0.0, 0.0, 1e-3, 2.0, np.finfo(dt).max, np.inf]
    else:
        info = np.iinfo(dt)
        values = [info.min, info.min + 1, 0, 1, info.max - 1, info.max]
    packed = wrapped.pack_edges(values, dt)
    assert packed.dtype == np.int64 and packed.shape == (len(values),)
    bits = packed.view(np.uint64)
    assert all(int(b) < (1 << (8 * dt.itemsize)) for b in bits)  # zero-extended
    back = bits.astype(ut).view(dt)
    want = np.array(values, dtype=dt)
    assert np.array_equal(back.view(ut), want.view(ut))  # bit for bit: -0.0 stays -0.0
    assert np.array_equal(packed, wrapped.pack_edges(np.array(values, dtype=dt), dt))
    for j, v in enumerate(values):  # the conversion is pack_interval's
        assert packed[j] == wrapped.pack_interval(v, v, dt)[0]


def test_pack_edges_refuses_values_outside_the_dtype():
    from pcodec_b200 import wrapped

    with pytest.raises(OverflowError, match="edge 256"):
        wrapped.pack_edges([0, 256], np.uint8)
    with pytest.raises(TypeError, match="edge 1.5"):
        wrapped.pack_edges([0, 1.5], np.int32)
    with pytest.raises(OverflowError, match="bound -1"):
        wrapped.pack_interval(-1, 3, np.uint64)
    with pytest.raises(TypeError):
        wrapped.pack_edges([0, 1], np.complex64)


# ---- the numpy statement of the rows


def test_reference_rows_on_hand_worked_cases():
    x = np.array([-5, 0, 1, 2, 3, 9, 10, 11, 10], dtype=np.int32)
    # columns: below 0 | [0, 2) | [2, 10] | above 10 | NaN
    assert hr.row(x, np.array([0, 2, 10], np.int32)).tolist() == [1, 2, 5, 1, 0]
    f = np.array([np.nan, -0.0, 0.0, -np.inf, np.inf, 1.0, -np.nan], dtype=np.float32)
    # edges -inf, 0.0, +inf: -inf in bucket 0, -0.0 and 0.0 and 1.0 in bucket 1 (closed at +inf), +inf in bucket 1 too
    assert hr.row(f, np.array([-np.inf, 0.0, np.inf], np.float32)).tolist() == [0, 1, 4, 0, 2]
    assert hr.row(f, np.array([-0.0, 1.0], np.float32)).tolist() == [1, 3, 1, 2]
    u = np.array([0, 1 << 63, (1 << 64) - 1, (1 << 64) - 2], dtype=np.uint64)
    assert hr.row(u, np.array([(1 << 64) - 2, (1 << 64) - 1], np.uint64)).tolist() == [2, 2, 0, 0]
    assert hr.rows(x, [4, 0, 5], np.array([0, 2, 10], np.int32)).tolist() == [[1, 2, 1, 0, 0], [0, 0, 0, 0, 0], [0, 0, 4, 1, 0]]
