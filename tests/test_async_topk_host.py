"""Host side of the asynchronous top-k calls (pco_b200_topk_pages_async_plan / _files_async_plan / _result, wrapped.AsyncPagesTopK,
standalone.AsyncFilesTopK) without a GPU: the plans' argument checks, their workspace sizes against the formulas include/pco_b200.h
documents, how a status written by the device becomes a kind and a message, the calls' host-side refusals, the wrappers' argument checks,
and the numpy statement of the outputs on hand-worked cases."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from tests import topk_reference as tr
from tests.test_async_files_host import HEAD
from tests.test_async_files_host import _expected_workspace as _files_workspace
from tests.test_async_pages_host import _expected_workspace as _pages_workspace
from tests.test_async_take_host import _FakeTensor, _bare

U64, U32 = 2, 1
NONE = (1 << 64) - 1
ELEM = {1: 4, 2: 8, 3: 4, 4: 8, 5: 4, 6: 8, 7: 2, 8: 2, 9: 2, 10: 1, 11: 1}
al = lambda x: (x + 255) // 256 * 256  # noqa: E731
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def L():
    from pcodec_b200 import wrapped

    return wrapped._lib_async_topk()


@pytest.fixture(scope="module")
def LF():
    from pcodec_b200 import standalone

    return standalone._lib_async_topk_files()


def _plan(L, dtype=U64, metas_cap=1 << 12, pages_cap=1 << 20, max_pages=64, rows_cap=1 << 18, frame_cap=1 << 21, k=100, largest=0, plan=True):
    from pcodec_b200 import wrapped

    p = wrapped._CAsyncTopkPlan()
    rc = L.pco_b200_topk_pages_async_plan(C.c_ubyte(dtype), C.c_size_t(metas_cap), C.c_size_t(pages_cap), C.c_size_t(max_pages),
                                          C.c_size_t(rows_cap), C.c_size_t(frame_cap), C.c_size_t(k), C.c_int(largest),
                                          C.byref(p) if plan else None)
    return rc, p, L.pco_b200_last_error_message().decode()


def _files_plan(LF, head, dtype=U32, max_files=8, max_chunks=16, rows_cap=1 << 16, k=100, largest=0, src_cap=1 << 20, index_cap=1 << 16,
                plan=True):
    from pcodec_b200 import standalone

    p = standalone._CAsyncFilesTopkPlan()
    buf = C.create_string_buffer(head, len(head))
    rc = LF.pco_b200_topk_files_async_plan(buf, C.c_size_t(len(head)), C.c_ubyte(dtype), C.c_size_t(src_cap), C.c_size_t(index_cap),
                                           C.c_size_t(max_files), C.c_size_t(max_chunks), C.c_size_t(rows_cap), C.c_size_t(k), C.c_int(largest),
                                           C.byref(p) if plan else None)
    return rc, p, LF.pco_b200_last_error_message().decode()


def _header_regions(call):
    """The regions the header's workspace paragraph of `call`'s plan lists, as (coefficient, term, name)."""
    text = open(os.path.join(ROOT, "include", "pco_b200.h")).read()
    doc = re.search(r"/\*((?:(?!\*/).)*?)\*/\s*PcoB200Error " + call + r"\(", text, flags=re.S).group(1)
    doc = " ".join(line.strip(" *") for line in doc.splitlines())
    tail = doc.split("E the bytes of a number of dtype:")[1]
    terms = r"k max_pages|k max_chunks|max_pages|max_chunks|rows_cap|\(max_chunks \+ 1\)"
    return re.findall(r"(\d+|E)(?: (" + terms + r"))? \(([^)]*)\)", tail)


def _formula(call, elem, rows_cap, m, k):
    terms = {"": 1, "rows_cap": rows_cap, "max_pages": m, "max_chunks": m, "(max_chunks + 1)": m + 1, "k max_pages": k * m, "k max_chunks": k * m}
    return sum(al((elem if coef == "E" else int(coef)) * terms[term]) for coef, term, _ in _header_regions(call))


def test_header_lists_the_regions():
    assert [r[2] for r in _header_regions("pco_b200_topk_pages_async_plan")] == [
        "the pages status", "the plan's state", "each page's flag", "the top-k table", "the cold pages' values", "the pages' list lengths",
        "the pages' candidate lists"]
    assert [r[2] for r in _header_regions("pco_b200_topk_files_async_plan")] == [
        "the files status", "the plan's state", "each chunk's flag", "the top-k table", "the cold chunks' values", "slot map", "cold list",
        "the chunks' list lengths", "the chunks' candidate lists"]


def _expected_pages(dtype, max_pages, rows_cap, frame_cap, k):
    own = sum(al(r) for r in [40, 16, 4 * max_pages, 48, ELEM[dtype] * rows_cap, 4 * max_pages, 16 * k * max_pages])
    assert own == _formula("pco_b200_topk_pages_async_plan", ELEM[dtype], rows_cap, max_pages, k)
    return _pages_workspace(max_pages, rows_cap, frame_cap) + own


def _expected_files(dtype, max_files, max_chunks, rows_cap, k):
    own = sum(al(r) for r in [40, 16, 4 * max_chunks, 48, ELEM[dtype] * rows_cap, 4 * max_chunks, 4 * (max_chunks + 1), 4 * max_chunks,
                              16 * k * max_chunks])
    assert own == _formula("pco_b200_topk_files_async_plan", ELEM[dtype], rows_cap, max_chunks, k)
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
    for k in (0, 1025, 1 << 40):
        rc, _, msg = _plan(L, k=k)
        assert rc == 3 and "k must be 1 .. 1024" in msg, msg
    for largest in (-1, 2, 7):
        rc, _, msg = _plan(L, largest=largest)
        assert rc == 3 and "largest" in msg, msg
    rc, _, _ = _plan(L, plan=False)
    assert rc == 3


def test_k_and_direction_are_accepted_up_to_the_device(L, LF):
    """k of 1 .. 1024 in either direction passes the checks: without a device the plan then stops at the device (PCO_B200_CUDA), not at
    the argument, with the plan filled."""
    import torch

    for k in (1, 2, 100, 1024):
        for largest in (0, 1):
            rc, p, msg = _plan(L, k=k, largest=largest)
            assert rc in (0, 6) and "k must" not in msg and "largest" not in msg, msg
            if not torch.cuda.is_available():
                assert rc == 6, msg
            assert (p.k, p.largest) == (k, largest)
            rc, p, msg = _files_plan(LF, HEAD, k=k, largest=largest)
            assert rc in (0, 6) and "k must" not in msg and "largest" not in msg, msg
            assert (p.k, p.largest) == (k, largest)


@pytest.mark.parametrize("dtype", sorted(ELEM))
@pytest.mark.parametrize("mp,rc_,fc,k", [(1, 0, 0, 1), (3, 255, 17, 5), (257, 12345, 999, 100), (4096, 1 << 24, 1 << 30, 1024)])
def test_pages_workspace_matches_the_formula(L, dtype, mp, rc_, fc, k):
    _, p, _ = _plan(L, dtype=dtype, max_pages=mp, rows_cap=rc_, frame_cap=fc, k=k)
    assert (p.dtype, p.max_pages, p.rows_cap, p.frame_cap, p.k) == (dtype, mp, rc_, fc, k)
    assert p.workspace_bytes == _expected_pages(dtype, mp, rc_, fc, k)


@pytest.mark.parametrize("dtype", sorted(ELEM))
@pytest.mark.parametrize("mf,mc,rows,k", [(1, 1, 0, 1), (8, 16, 1 << 16, 300), (4096, 5000, 12345, 16), (3, 1 << 20, 1 << 28, 1024)])
def test_files_workspace_matches_the_formula(LF, dtype, mf, mc, rows, k):
    _, p, _ = _files_plan(LF, HEAD, dtype=dtype, max_files=mf, max_chunks=mc, rows_cap=rows, k=k)
    assert (p.dtype, p.max_files, p.max_chunks, p.rows_cap, p.k) == (dtype, mf, mc, rows, k)
    assert p.workspace_bytes == _expected_files(dtype, mf, mc, rows, k)


def test_files_plan_checks(LF):
    for kw, words in [({"max_files": 0}, "max_files"), ({"max_chunks": 0}, "max_chunks"), ({"rows_cap": (1 << 56) + 1}, "rows_cap"),
                      ({"k": 0}, "k must"), ({"k": 1025}, "k must"), ({"largest": 2}, "largest"), ({"largest": -1}, "largest")]:
        rc, _, msg = _files_plan(LF, HEAD, **kw)
        assert rc == 3 and words in msg, msg
    rc, _, msg = _files_plan(LF, HEAD, dtype=99)
    assert rc == 5


def _result(L, **fields):
    from pcodec_b200 import wrapped

    s = wrapped._CAsyncTopkStatus(**fields)
    n = C.c_size_t(12345)
    rc = L.pco_b200_topk_pages_async_result(C.byref(s), C.byref(n))
    return rc, L.pco_b200_last_error_message().decode(), n.value


def _files_result(LF, **fields):
    from pcodec_b200 import standalone

    s = standalone._CAsyncFilesTopkStatus(**fields)
    n = C.c_size_t(12345)
    rc = LF.pco_b200_topk_files_async_result(C.byref(s), C.byref(n))
    return rc, LF.pco_b200_last_error_message().decode(), n.value


def test_result_of_success_is_the_match_count(L, LF):
    assert _result(L, kind=0, n_written=1000, n_matches=700, page=NONE)[::2] == (0, 700)
    assert _files_result(LF, kind=0, n_written=77, n_matches=0, file=NONE, chunk=NONE)[::2] == (0, 0)
    assert L.pco_b200_topk_pages_async_result(None, None) == 3
    assert LF.pco_b200_topk_files_async_result(None, None) == 3


def test_result_of_upstream_statuses_is_the_decompress_calls(L, LF):
    rc, msg, n = _result(L, kind=2, device_status=2, page=17)
    assert rc == 2 and msg.startswith("page 17: ") and "insufficient data" in msg and n == 12345, msg
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


def test_calls_refuse_missing_buffers_without_a_device(L, LF):
    from pcodec_b200 import standalone, wrapped

    _, p, _ = _plan(L)
    nz = C.c_void_p(256)
    s = wrapped._CAsyncTopkStatus()
    args = [nz] * 9  # metas, pages, refs, n_pages, interval, out_values, out_positions, n_out, workspace
    for i in range(9):
        a = list(args)
        a[i] = None
        assert L.pco_b200_topk_pages_async(C.byref(p), *a, C.byref(s), None) == 3
        assert "null buffer" in L.pco_b200_last_error_message().decode()
    assert L.pco_b200_topk_pages_async(C.byref(p), *args, None, None) == 3  # null status
    assert L.pco_b200_topk_pages_async(C.byref(p), *args[:8], C.c_void_p(257), C.byref(s), None) == 3
    assert "aligned" in L.pco_b200_last_error_message().decode()
    for field, value in (("k", 1025), ("k", 0), ("largest", 2)):
        bad = wrapped._CAsyncTopkPlan.from_buffer_copy(bytes(p))
        setattr(bad, field, value)
        assert L.pco_b200_topk_pages_async(C.byref(bad), *args, C.byref(s), None) == 3
        assert "not made by" in L.pco_b200_last_error_message().decode()
    assert L.pco_b200_topk_pages_async(C.byref(wrapped._CAsyncTopkPlan()), *args, C.byref(s), None) == 3
    assert "not made by" in L.pco_b200_last_error_message().decode()

    _, fp, _ = _files_plan(LF, HEAD)
    fs = standalone._CAsyncFilesTopkStatus()
    for i in range(9):  # src, index, files, n_files, interval, out_values, out_positions, n_out, workspace
        a = list(args)
        a[i] = None
        assert LF.pco_b200_topk_files_async(C.byref(fp), *a, C.byref(fs), None) == 3
        assert "null buffer" in LF.pco_b200_last_error_message().decode()
    assert LF.pco_b200_topk_files_async(C.byref(fp), *args[:8], C.c_void_p(257), C.byref(fs), None) == 3
    assert "aligned" in LF.pco_b200_last_error_message().decode()
    bad = standalone._CAsyncFilesTopkPlan.from_buffer_copy(bytes(fp))
    bad.workspace_bytes += 1
    assert LF.pco_b200_topk_files_async(C.byref(bad), *args, C.byref(fs), None) == 3
    assert "not made by" in LF.pco_b200_last_error_message().decode()


def test_a_plan_fails_loudly_without_a_device():
    """Without a device the Python wrappers raise: no plan, no silent fall-back."""
    import torch

    from pcodec_b200 import PcoError, standalone, wrapped

    if torch.cuda.is_available():
        pytest.skip("a device is present")
    with pytest.raises((PcoError, RuntimeError)):
        wrapped.AsyncPagesTopK(np.uint64, 1 << 12, 1 << 20, 4, 1 << 16, 10)
    with pytest.raises((PcoError, RuntimeError)):
        standalone.AsyncFilesTopK(HEAD, np.uint32, 1 << 20, 1 << 16, 2, 4, 1 << 16, 10, largest=True)


def test_new_symbols_are_exported(L, LF):
    for name in ("pco_b200_topk_pages_async_plan", "pco_b200_topk_pages_async", "pco_b200_topk_pages_async_result"):
        assert hasattr(L, name), name
    for name in ("pco_b200_topk_files_async_plan", "pco_b200_topk_files_async", "pco_b200_topk_files_async_result"):
        assert hasattr(LF, name), name


def test_status_and_plan_structs_match_the_header():
    from pcodec_b200 import standalone, wrapped

    assert C.sizeof(wrapped._CAsyncTopkStatus) == 48 and C.sizeof(standalone._CAsyncFilesTopkStatus) == 48
    assert C.sizeof(wrapped._CAsyncTopkPlan) == 64 and C.sizeof(standalone._CAsyncFilesTopkPlan) == 72


def test_pages_wrapper_checks_its_arguments():
    import torch

    from pcodec_b200 import wrapped

    p = wrapped._CAsyncTopkPlan(dtype=U64, metas_cap=64, pages_cap=64, max_pages=4, rows_cap=1024, frame_cap=256, k=10)
    t = _bare(wrapped.AsyncPagesTopK, p, np.uint64)
    T = lambda dt, *shape: _FakeTensor(dt, shape, t.device)  # noqa: E731
    good = dict(metas=T(torch.uint8, 64), pages=T(torch.uint8, 64), refs=T(torch.int64, 4, 5), n_pages=T(torch.int64, 1),
                interval=T(torch.int64, 2), out_values=T(torch.uint64, 10), out_positions=T(torch.int64, 10), n_out=T(torch.int64, 1))
    for name, bad, words in [("interval", T(torch.int64, 3), "interval"), ("interval", T(torch.int32, 2), "interval"),
                             ("out_values", T(torch.uint64, 9), "out_values"), ("out_values", T(torch.int64, 10), "out_values"),
                             ("out_positions", T(torch.int64, 9), "out_positions"), ("out_positions", T(torch.int32, 10), "out_positions"),
                             ("n_out", T(torch.int64, 2), "n_out"), ("n_out", T(torch.int32, 1), "n_out"), ("refs", T(torch.int64, 3, 5), "refs"),
                             ("n_pages", T(torch.int64, 2), "n_pages"), ("metas", T(torch.uint8, 63), "metas_cap")]:
        with pytest.raises(ValueError, match=words):
            t(**dict(good, **{name: bad}))
    with pytest.raises(ValueError, match="interval must be a contiguous CUDA tensor"):
        t(**dict(good, interval=object()))


def test_files_wrapper_checks_its_arguments():
    import torch

    from pcodec_b200 import standalone

    p = standalone._CAsyncFilesTopkPlan(dtype=U32, src_cap=64, index_cap=64, max_files=2, max_chunks=4, rows_cap=1024, k=3, largest=1)
    t = _bare(standalone.AsyncFilesTopK, p, np.uint32)
    T = lambda dt, *shape: _FakeTensor(dt, shape, t.device)  # noqa: E731
    good = dict(src=T(torch.uint8, 64), index=T(torch.uint8, 64), files=T(torch.int64, 2, 4), n_files=T(torch.int64, 1),
                interval=T(torch.int64, 2), out_values=T(torch.uint32, 3), out_positions=T(torch.int64, 3), n_out=T(torch.int64, 1))
    for name, bad, words in [("interval", T(torch.int64, 1), "interval"), ("out_values", T(torch.float32, 3), "out_values"),
                             ("out_positions", T(torch.int64, 2), "out_positions"), ("n_out", T(torch.int64, 2), "n_out"),
                             ("files", T(torch.int64, 2, 5), "files"), ("n_files", T(torch.int64, 2), "n_files"), ("src", T(torch.uint8, 63), "src_cap")]:
        with pytest.raises(ValueError, match=words):
            t(**dict(good, **{name: bad}))


# ---- the numpy statement


def test_reference_ranks_by_value_then_position():
    x = np.array([5, 3, 5, 1, 3, 9, 1], np.int32)
    v, p = tr.topk(x, -100, 100, 4, False)
    assert v.tolist() == [1, 1, 3, 3] and p.tolist() == [3, 6, 1, 4]
    v, p = tr.topk(x, -100, 100, 3, True)
    assert v.tolist() == [9, 5, 5] and p.tolist() == [5, 0, 2]  # ties: the lower position first in both directions
    v, p = tr.topk(x, 2, 5, 10, True)
    assert v.tolist() == [5, 5, 3, 3] and p.tolist() == [0, 2, 1, 4]
    assert tr.topk(x, 5, 4, 3, False)[0].size == 0


def test_reference_floats_signed_zeros_nans_and_infinities():
    x = np.array([0.0, -0.0, np.nan, -np.inf, np.inf, -np.nan, -1.0, 0.0], np.float32)
    v, p = tr.topk(x, -np.inf, np.inf, 8, False)
    assert p.tolist() == [3, 6, 0, 1, 7, 4]  # -0.0 equals +0.0: position order among the zeros; NaNs never match
    assert np.signbit(v[3]) and not np.signbit(v[2])  # each value keeps its bits
    v, p = tr.topk(x, -np.inf, np.inf, 2, True)
    assert p.tolist() == [4, 0]
    assert tr.topk(x, np.nan, 1.0, 3, False)[0].size == 0
    assert tr.topk(x, 0.0, -0.0, 5, False)[1].tolist() == [0, 1, 7]


def test_reference_keeps_64_bit_integers_exact():
    x = np.array([(1 << 63) - 1, (1 << 63) - 2, -(1 << 63), 0], np.int64)
    assert tr.topk(x, -(1 << 63), (1 << 63) - 1, 2, True)[1].tolist() == [0, 1]
    u = np.array([(1 << 64) - 1, (1 << 64) - 2, 0], np.uint64)
    assert tr.topk(u, 0, (1 << 64) - 1, 1, True)[1].tolist() == [0]
    assert tr.topk(u, 0, (1 << 64) - 1, 1, False)[1].tolist() == [2]
