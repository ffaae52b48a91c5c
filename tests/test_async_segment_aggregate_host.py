"""Host side of the asynchronous segment aggregates (pco_b200_segment_aggregate_pages_async_plan / _files_async_plan / _result,
wrapped.AsyncPagesSegmentAggregate, standalone.AsyncFilesSegmentAggregate) without a GPU: the plans' argument checks, their workspace
sizes against the formulas include/pco_b200.h documents, how a status written by the device becomes a kind and a message, the calls'
host-side refusals, the wrappers' argument checks, and the numpy restatement of the segment float order on hand-worked cases."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from tests import aggregate_reference as ar
from tests import segment_reference as sr
from tests.test_async_files_host import HEAD
from tests.test_async_files_host import _expected_workspace as _files_workspace
from tests.test_async_pages_host import _expected_workspace as _pages_workspace
from tests.test_async_take_host import _FakeTensor, _bare

U64, U32 = 2, 1
NONE = (1 << 64) - 1
ELEM = {1: 4, 2: 8, 3: 4, 4: 8, 5: 4, 6: 8, 7: 2, 8: 2, 9: 2, 10: 1, 11: 1}
TOO_MANY, ORDER, PAST = 0x401, 0x402, 0x403
al = lambda x: (x + 255) // 256 * 256  # noqa: E731
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def L():
    from pcodec_b200 import wrapped

    return wrapped._lib_async_segment_aggregate()


@pytest.fixture(scope="module")
def LF():
    from pcodec_b200 import standalone

    return standalone._lib_async_segment_aggregate_files()


def _plan(L, dtype=U64, metas_cap=1 << 12, pages_cap=1 << 20, max_pages=64, rows_cap=1 << 18, frame_cap=1 << 21, max_segments=1 << 10,
          plan=True):
    from pcodec_b200 import wrapped

    p = wrapped._CAsyncSegmentAggregatePlan()
    rc = L.pco_b200_segment_aggregate_pages_async_plan(C.c_ubyte(dtype), C.c_size_t(metas_cap), C.c_size_t(pages_cap), C.c_size_t(max_pages),
                                                       C.c_size_t(rows_cap), C.c_size_t(frame_cap), C.c_size_t(max_segments),
                                                       C.byref(p) if plan else None)
    return rc, p, L.pco_b200_last_error_message().decode()


def _files_plan(LF, head, dtype=U32, max_files=8, max_chunks=16, rows_cap=1 << 16, max_segments=1 << 10, plan=True):
    from pcodec_b200 import standalone

    p = standalone._CAsyncFilesSegmentAggregatePlan()
    buf = C.create_string_buffer(head, len(head))
    rc = LF.pco_b200_segment_aggregate_files_async_plan(buf, C.c_size_t(len(head)), C.c_ubyte(dtype), C.c_size_t(1 << 20), C.c_size_t(1 << 16),
                                                        C.c_size_t(max_files), C.c_size_t(max_chunks), C.c_size_t(rows_cap),
                                                        C.c_size_t(max_segments), C.byref(p) if plan else None)
    return rc, p, LF.pco_b200_last_error_message().decode()


def _header_regions(call):
    """The regions the header's workspace paragraph of `call`'s plan lists, as (coefficient, term, name)."""
    text = open(os.path.join(ROOT, "include", "pco_b200.h")).read()
    doc = re.search(r"/\*((?:(?!\*/).)*?)\*/\s*PcoB200Error " + call + r"\(", text, flags=re.S).group(1)
    doc = " ".join(line.strip(" *") for line in doc.splitlines())
    tail = doc.split("E the bytes of a number of dtype:")[1]
    terms = r"S|R|max_pages|max_chunks|max_segments|rows_cap|\(max_chunks \+ 1\)|\(max_segments \+ 3\)|\(rows_cap / 262144 \+ 2\)"
    return re.findall(r"(\d+|E)(?: (" + terms + r"))? \(([^)]*)\)", tail)


def _formula(call, s, elem, rows_cap, m, ms):
    terms = {"": 1, "S": s, "R": s + ms, "rows_cap": rows_cap, "max_pages": m, "max_chunks": m, "(max_chunks + 1)": m + 1,
             "max_segments": ms, "(max_segments + 3)": ms + 3, "(rows_cap / 262144 + 2)": rows_cap // 262144 + 2}
    return sum(al((elem if coef == "E" else int(coef)) * terms[term]) for coef, term, _ in _header_regions(call))


def test_header_lists_the_regions():
    assert [r[2] for r in _header_regions("pco_b200_segment_aggregate_pages_async_plan")] == [
        "the pages status", "the plan's state", "each slot's run of segments", "touched flags", "the interval and bounds",
        "the batch-segment records", "the cold pages' values", "the segments' accumulators", "the long segments"]
    assert [r[2] for r in _header_regions("pco_b200_segment_aggregate_files_async_plan")] == [
        "the files status", "the plan's state", "each slot's run of segments", "touched flags", "the interval and bounds",
        "the batch-segment records", "the cold chunks' values", "slot map", "cold list", "the segments' accumulators",
        "the long segments"]


def _expected_pages(dtype, max_pages, rows_cap, frame_cap, ms):
    s = rows_cap // 256 + max_pages
    own = sum(al(r) for r in [40, 56, 8 * s, 4 * max_pages, 8 * (ms + 3), 40 * (s + ms), ELEM[dtype] * rows_cap, 48 * ms,
                              24 * (rows_cap // 262144 + 2)])
    assert own == _formula("pco_b200_segment_aggregate_pages_async_plan", s, ELEM[dtype], rows_cap, max_pages, ms)
    return _pages_workspace(max_pages, rows_cap, frame_cap) + own


def _expected_files(dtype, max_files, max_chunks, rows_cap, ms):
    s = rows_cap // 256 + max_chunks
    own = sum(al(r) for r in [40, 56, 8 * s, 4 * max_chunks, 8 * (ms + 3), 40 * (s + ms), ELEM[dtype] * rows_cap, 4 * max_chunks,
                              4 * (max_chunks + 1), 48 * ms, 24 * (rows_cap // 262144 + 2)])
    assert own == _formula("pco_b200_segment_aggregate_files_async_plan", s, ELEM[dtype], rows_cap, max_chunks, ms)
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
    for ms in (0, 1 << 31, 1 << 63):
        rc, _, msg = _plan(L, max_segments=ms)
        assert rc == 3 and "max_segments" in msg, msg
    rc, _, _ = _plan(L, plan=False)
    assert rc == 3


def test_max_segments_range_is_accepted_up_to_the_device(L, LF):
    """1 and 2^31 - 1 pass the checks: without a device the plan then stops at the device (PCO_B200_CUDA), not at the argument."""
    import torch

    for ms in (1, 2, 1 << 20, (1 << 31) - 1):
        rc, p, msg = _plan(L, max_segments=ms)
        assert rc in (0, 6) and "max_segments" not in msg, msg
        if not torch.cuda.is_available():
            assert rc == 6, msg
        assert p.max_segments == ms
        rc, p, msg = _files_plan(LF, HEAD, max_segments=ms)
        assert rc in (0, 6) and "max_segments" not in msg, msg
        assert p.max_segments == ms


@pytest.mark.parametrize("dtype", sorted(ELEM))
@pytest.mark.parametrize("mp,rc_,fc,ms", [(1, 0, 0, 1), (3, 255, 17, 5), (257, 12345, 999, 1000), (4096, 1 << 24, 1 << 30, 1 << 20)])
def test_pages_workspace_matches_the_formula(L, dtype, mp, rc_, fc, ms):
    _, p, _ = _plan(L, dtype=dtype, max_pages=mp, rows_cap=rc_, frame_cap=fc, max_segments=ms)
    assert (p.dtype, p.max_pages, p.rows_cap, p.frame_cap, p.max_segments) == (dtype, mp, rc_, fc, ms)
    assert p.workspace_bytes == _expected_pages(dtype, mp, rc_, fc, ms)


def test_workspace_does_not_depend_on_the_buffers(L, LF):
    ws = lambda **kw: _plan(L, **kw)[1].workspace_bytes  # noqa: E731
    assert ws(metas_cap=1 << 30, pages_cap=1 << 30) == ws()
    from pcodec_b200 import standalone

    _, p, _ = _files_plan(LF, HEAD)
    q = standalone._CAsyncFilesSegmentAggregatePlan()  # src_cap and index_cap of 2^40 bytes
    LF.pco_b200_segment_aggregate_files_async_plan(C.create_string_buffer(HEAD, len(HEAD)), C.c_size_t(len(HEAD)), C.c_ubyte(U32),
                                                   C.c_size_t(1 << 40), C.c_size_t(1 << 40), C.c_size_t(8), C.c_size_t(16), C.c_size_t(1 << 16),
                                                   C.c_size_t(1 << 10), C.byref(q))
    assert q.src_cap == 1 << 40 and q.workspace_bytes == p.workspace_bytes


def test_files_plan_checks(LF):
    for kw, words in [({"max_files": 0}, "max_files"), ({"max_chunks": 0}, "max_chunks"), ({"rows_cap": (1 << 56) + 1}, "rows_cap"),
                      ({"max_segments": 0}, "max_segments"), ({"max_segments": 1 << 31}, "max_segments")]:
        rc, _, msg = _files_plan(LF, HEAD, **kw)
        assert rc == 3 and words in msg, msg
    rc, _, msg = _files_plan(LF, HEAD, dtype=99)
    assert rc == 5


@pytest.mark.parametrize("dtype", sorted(ELEM))
@pytest.mark.parametrize("mf,mc,rows,ms", [(1, 1, 0, 1), (8, 16, 1 << 16, 300), (4096, 5000, 12345, 7), (3, 1 << 20, 1 << 28, 1 << 20)])
def test_files_workspace_matches_the_formula(LF, dtype, mf, mc, rows, ms):
    _, p, _ = _files_plan(LF, HEAD, dtype=dtype, max_files=mf, max_chunks=mc, rows_cap=rows, max_segments=ms)
    assert (p.dtype, p.max_files, p.max_chunks, p.rows_cap, p.max_segments) == (dtype, mf, mc, rows, ms)
    assert p.workspace_bytes == _expected_files(dtype, mf, mc, rows, ms)


def _result(L, **fields):
    from pcodec_b200 import wrapped

    s = wrapped._CAsyncSegmentAggregateStatus(**fields)
    nm = C.c_size_t(12345)
    rc = L.pco_b200_segment_aggregate_pages_async_result(C.byref(s), C.byref(nm))
    return rc, L.pco_b200_last_error_message().decode(), nm.value


def _files_result(LF, **fields):
    from pcodec_b200 import standalone

    s = standalone._CAsyncFilesSegmentAggregateStatus(**fields)
    nm = C.c_size_t(12345)
    rc = LF.pco_b200_segment_aggregate_files_async_result(C.byref(s), C.byref(nm))
    return rc, LF.pco_b200_last_error_message().decode(), nm.value


def test_result_of_success_is_the_match_count(L, LF):
    assert _result(L, kind=0, n_matches=1000, page=NONE, segment=NONE)[::2] == (0, 1000)
    assert _files_result(LF, kind=0, n_matches=77, file=NONE, chunk=NONE, segment=NONE)[::2] == (0, 77)
    assert L.pco_b200_segment_aggregate_pages_async_result(None, None) == 3
    assert LF.pco_b200_segment_aggregate_files_async_result(None, None) == 3


@pytest.mark.parametrize("res", ["_result", "_files_result"])
def test_result_names_the_segment(L, LF, res):
    f = (lambda **kw: _result(L, **kw)) if res == "_result" else (lambda **kw: _files_result(LF, **kw))
    rc, msg, nm = f(kind=3, device_status=TOO_MANY, n_segments=99, segment=NONE)
    assert rc == 3 and msg == "*n_segments is 99, above the plan's max_segments" and nm == 12345, msg
    rc, msg, _ = f(kind=3, device_status=ORDER, n_segments=99, segment=17)
    assert rc == 3 and msg.startswith("segment 17: ") and "non-decreasing" in msg, msg
    rc, msg, _ = f(kind=3, device_status=PAST, n_segments=99, segment=5, n_written=1000)
    assert rc == 3 and msg.startswith("segment 5: ") and "1000 rows" in msg, msg


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


def test_every_segment_code_is_documented_with_its_kind():
    text = open(os.path.join(ROOT, "include", "pco_b200.h")).read()
    codes = dict((name, int(v, 16)) for name, v in re.findall(r"(PCO_B200_SEGMENTS_\w+)\s*=\s*(0x[0-9a-f]+)", text))
    assert codes == {"PCO_B200_SEGMENTS_TOO_MANY": TOO_MANY, "PCO_B200_SEGMENTS_ORDER": ORDER, "PCO_B200_SEGMENTS_PAST": PAST}
    for name in codes:
        assert re.search(name + r"\s*=\s*0x[0-9a-f]+,?\s*/\*(?:(?!\*/).)*\(PCO_B200_INVALID_ARGUMENT\) \*/", text), name


def test_calls_refuse_missing_buffers_without_a_device(L, LF):
    from pcodec_b200 import standalone, wrapped

    _, p, _ = _plan(L)
    nz = C.c_void_p(256)
    s = wrapped._CAsyncSegmentAggregateStatus()
    args = [nz] * 10  # metas, pages, refs, n_pages, bounds, n_segments, interval, aggs, total, workspace
    for i in range(10):
        a = list(args)
        a[i] = None
        assert L.pco_b200_segment_aggregate_pages_async(C.byref(p), *a, C.byref(s), None) == 3
        assert "null buffer" in L.pco_b200_last_error_message().decode()
    assert L.pco_b200_segment_aggregate_pages_async(C.byref(p), *args, None, None) == 3  # null status
    assert L.pco_b200_segment_aggregate_pages_async(C.byref(p), *args[:9], C.c_void_p(257), C.byref(s), None) == 3
    assert "aligned" in L.pco_b200_last_error_message().decode()
    bad = wrapped._CAsyncSegmentAggregatePlan.from_buffer_copy(bytes(p))
    bad.workspace_bytes += 1
    assert L.pco_b200_segment_aggregate_pages_async(C.byref(bad), *args, C.byref(s), None) == 3
    assert "not made by" in L.pco_b200_last_error_message().decode()
    assert L.pco_b200_segment_aggregate_pages_async(C.byref(wrapped._CAsyncSegmentAggregatePlan()), *args, C.byref(s), None) == 3
    assert "not made by" in L.pco_b200_last_error_message().decode()

    _, fp, _ = _files_plan(LF, HEAD)
    fs = standalone._CAsyncFilesSegmentAggregateStatus()
    for i in range(10):  # src, index, files, n_files, bounds, n_segments, interval, aggs, total, workspace
        a = list(args)
        a[i] = None
        assert LF.pco_b200_segment_aggregate_files_async(C.byref(fp), *a, C.byref(fs), None) == 3
        assert "null buffer" in LF.pco_b200_last_error_message().decode()
    assert LF.pco_b200_segment_aggregate_files_async(C.byref(fp), *args[:9], C.c_void_p(257), C.byref(fs), None) == 3
    assert "aligned" in LF.pco_b200_last_error_message().decode()
    assert LF.pco_b200_segment_aggregate_files_async(C.byref(standalone._CAsyncFilesSegmentAggregatePlan()), *args, C.byref(fs), None) == 3
    assert "not made by" in LF.pco_b200_last_error_message().decode()


def test_new_symbols_are_exported(L, LF):
    for name in ("pco_b200_segment_aggregate_pages_async_plan", "pco_b200_segment_aggregate_pages_async",
                 "pco_b200_segment_aggregate_pages_async_result"):
        assert hasattr(L, name), name
    for name in ("pco_b200_segment_aggregate_files_async_plan", "pco_b200_segment_aggregate_files_async",
                 "pco_b200_segment_aggregate_files_async_result"):
        assert hasattr(LF, name), name


def test_status_structs_match_the_header():
    from pcodec_b200 import standalone, wrapped

    assert C.sizeof(wrapped._CAsyncSegmentAggregateStatus) == 72 and C.sizeof(standalone._CAsyncFilesSegmentAggregateStatus) == 72
    assert C.sizeof(wrapped._CAsyncSegmentAggregatePlan) == 64 and C.sizeof(standalone._CAsyncFilesSegmentAggregatePlan) == 72


def test_pages_wrapper_checks_its_arguments():
    import torch

    from pcodec_b200 import wrapped

    p = wrapped._CAsyncSegmentAggregatePlan(dtype=U64, metas_cap=64, pages_cap=64, max_pages=4, rows_cap=1024, frame_cap=256, max_segments=10)
    t = _bare(wrapped.AsyncPagesSegmentAggregate, p, np.uint64)
    T = lambda dt, *shape: _FakeTensor(dt, shape, t.device)  # noqa: E731
    good = dict(metas=T(torch.uint8, 64), pages=T(torch.uint8, 64), refs=T(torch.int64, 4, 5), n_pages=T(torch.int64, 1),
                bounds=T(torch.int64, 11), n_segments=T(torch.int64, 1), interval=T(torch.int64, 2), aggs=T(torch.int64, 10, 6),
                total=T(torch.int64, 6))
    for name, bad, words in [("bounds", T(torch.int64, 10), "bounds"), ("bounds", T(torch.int32, 11), "bounds"),
                             ("n_segments", T(torch.int64, 2), "n_segments"), ("interval", T(torch.int64, 3), "interval"),
                             ("aggs", T(torch.int64, 9, 6), "aggs"), ("total", T(torch.int64, 5), "total"),
                             ("refs", T(torch.int64, 3, 5), "refs"), ("metas", T(torch.uint8, 63), "metas_cap")]:
        with pytest.raises(ValueError, match=words):
            t(**dict(good, **{name: bad}))
    with pytest.raises(ValueError, match="bounds must be a contiguous CUDA tensor"):
        t(**dict(good, bounds=object()))


def test_files_wrapper_checks_its_arguments():
    import torch

    from pcodec_b200 import standalone

    p = standalone._CAsyncFilesSegmentAggregatePlan(dtype=U32, src_cap=64, index_cap=64, max_files=2, max_chunks=4, rows_cap=1024, max_segments=3)
    t = _bare(standalone.AsyncFilesSegmentAggregate, p, np.uint32)
    T = lambda dt, *shape: _FakeTensor(dt, shape, t.device)  # noqa: E731
    good = dict(src=T(torch.uint8, 64), index=T(torch.uint8, 64), files=T(torch.int64, 2, 4), n_files=T(torch.int64, 1),
                bounds=T(torch.int64, 4), n_segments=T(torch.int64, 1), interval=T(torch.int64, 2), aggs=T(torch.int64, 3, 6),
                total=T(torch.int64, 6))
    for name, bad, words in [("bounds", T(torch.int64, 3), "bounds"), ("n_segments", T(torch.int32, 1), "n_segments"),
                             ("files", T(torch.int64, 2, 5), "files"), ("n_files", T(torch.int64, 2), "n_files"),
                             ("aggs", T(torch.int64, 3, 5), "aggs")]:
        with pytest.raises(ValueError, match=words):
            t(**dict(good, **{name: bad}))


# ---- the numpy restatement of the segment float order


def _bits(f):
    return int(np.array([f]).view(np.uint64)[0])


def test_segments_equal_to_pages_give_the_aggregate_records():
    rng = np.random.default_rng(3)
    pieces = [700, 256, 1, 0, 1500, 33]
    x = rng.normal(size=sum(pieces)).astype(np.float32)
    x[5] = np.float32("nan")
    x[900] = -0.0
    bounds = np.concatenate([[0], np.cumsum(pieces)])
    recs, tot = sr.segment_records(x, pieces, bounds, -1.0, 1.0)
    want, at = [], 0
    for n in pieces:
        want.append(ar.record(x[at:at + n], [n], -1.0, 1.0))
        at += n
    for (r, f), (w, wf) in zip(recs, want):
        assert r == w and (f == wf or (np.isnan(f) and np.isnan(wf))), (r, w)
    assert tot == ar.total(want, np.float32)


def test_one_segment_over_one_page_is_its_total():
    rng = np.random.default_rng(4)
    x = rng.normal(size=5000)
    (rec, fs), = sr.segment_records(x, [5000], [0, 5000], -0.5, 2.0)[0]
    want, _ = ar.record(x, [5000], -0.5, 2.0)
    assert rec == want


def test_batch_partials_count_rows_outside_the_segment_as_non_matches():
    """A page of 600: batches [0, 256), [256, 512), [512, 600).  Segment [250, 520) holds 6 rows of batch 0, all of batch 1 and 8 of
    batch 2; its sum is lane 0: batch 0's partial, lane 1: batch 1's, lane 2: batch 2's, then the tree."""
    x = np.arange(600, dtype=np.float64) * 0.1
    (rec, fs), = sr.segment_records(x, [600], [250, 520], -1e9, 1e9)[0]
    parts = []
    for lo_r, hi_r, base in [(250, 256, 0), (256, 512, 256), (512, 520, 512)]:
        v = np.zeros(256)
        v[lo_r - base:hi_r - base] = x[lo_r:hi_r]
        lanes = v.reshape(32, 8)
        acc = np.zeros(32)
        for e in range(8):
            acc = acc + lanes[:, e]
        parts.append(ar.tree(acc))
    lanes = np.zeros(32)
    lanes[:3] = parts
    assert fs == ar.tree(lanes) and rec[:2] == [270, 270]
    assert rec[4] == _bits(fs)


def test_batch_numbers_run_on_across_pages():
    """Segment [200, 1300) over pages of 300 and 1000: batches 0, 1 of page 0 then 0 .. 3 of page 1 are j = 0 .. 5 of the segment."""
    x = np.linspace(-3, 3, 1300)
    (rec, fs), = sr.segment_records(x, [300, 1000], [200, 1300], -10, 10)[0]
    parts = list(ar.batch_sums(np.where(np.arange(300) >= 200, x[:300], 0.0), np.ones(300, bool)))
    parts += list(ar.batch_sums(x[300:], np.ones(1000, bool)))
    assert len(parts) == 6 and fs == ar.strided_sum(parts)


def test_empty_segments_and_totals():
    x = np.arange(1000, dtype=np.int64) - 500
    recs, tot = sr.segment_records(x, [1000], [10, 10, 10, 600, 600, 999], -100, 100)
    m64 = (1 << 64) - 1
    assert [r for r, _ in recs] == [[0] * 6, [0] * 6, [590, 200, -100 & m64, 99, -100 & m64, m64], [0] * 6, [399, 1, 100, 100, 100, 0]]
    assert tot == [989, 201, -100 & m64, 100, 0, 0]
    assert sr.segment_records(x, [1000], [7], 0, 1) == ([], [0] * 6)


def test_vectorised_integer_reference_matches_the_loop():
    rng = np.random.default_rng(5)
    x = rng.integers(-(1 << 31), 1 << 31, size=4096, dtype=np.int64).astype(np.int32)
    bounds = np.concatenate([[3], np.sort(rng.choice(np.arange(4, 4000), 60, replace=False)), [4000]])
    want, wt = sr.segment_records(x, [4096], bounds, -(1 << 30), 1 << 30)
    got, gt = sr.segment_records_int(x, bounds, -(1 << 30), 1 << 30)
    assert got == [r for r, _ in want] and gt == wt
