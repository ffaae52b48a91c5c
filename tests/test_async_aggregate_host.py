"""Host side of the asynchronous aggregates (pco_b200_aggregate_pages_async_plan / _files_async_plan / _result, wrapped.unpack_aggregates)
without a GPU: the plans' argument checks, their workspace sizes against the formulas include/pco_b200.h documents, how a status written by
the device becomes a kind and a message, the calls' host-side refusals, record unpacking, and the suite's numpy emulation of the float sum
order on hand-worked cases."""
import ctypes as C

import numpy as np
import pytest

from tests import aggregate_reference as ref
from tests.test_async_files_host import HEAD
from tests.test_async_files_host import _expected_workspace as _files_workspace
from tests.test_async_pages_host import _expected_workspace as _pages_workspace

U64, U32, F16, U8 = 2, 1, 9, 10
NONE = (1 << 64) - 1
ELEM = {1: 4, 2: 8, 3: 4, 4: 8, 5: 4, 6: 8, 7: 2, 8: 2, 9: 2, 10: 1, 11: 1}
al = lambda x: (x + 255) // 256 * 256  # noqa: E731


@pytest.fixture(scope="module")
def L():
    from pcodec_b200 import wrapped

    return wrapped._lib_async_aggregate()


@pytest.fixture(scope="module")
def LF():
    from pcodec_b200 import standalone

    return standalone._lib_async_aggregate_files()


def _plan(L, dtype=U64, metas_cap=1 << 12, pages_cap=1 << 20, max_pages=64, rows_cap=1 << 18, frame_cap=1 << 21, plan=True):
    from pcodec_b200 import wrapped

    p = wrapped._CAsyncAggregatePlan()
    rc = L.pco_b200_aggregate_pages_async_plan(C.c_ubyte(dtype), C.c_size_t(metas_cap), C.c_size_t(pages_cap), C.c_size_t(max_pages),
                                               C.c_size_t(rows_cap), C.c_size_t(frame_cap), C.byref(p) if plan else None)
    return rc, p, L.pco_b200_last_error_message().decode()


def _expected_pages(dtype, max_pages, rows_cap, frame_cap):
    """The pages call's formula with dst_cap = rows_cap, then: the pages status, slot counts, slot records, the value staging, the
    pages' accumulators."""
    s = rows_cap // 256 + max_pages
    return _pages_workspace(max_pages, rows_cap, frame_cap) + sum(al(r) for r in [40, 4 * s, 32 * s, ELEM[dtype] * rows_cap, 48 * max_pages])


def _files_plan(LF, head, dtype=U32, max_files=8, max_chunks=16, rows_cap=1 << 16, plan=True):
    from pcodec_b200 import standalone

    p = standalone._CAsyncFilesAggregatePlan()
    buf = C.create_string_buffer(head, len(head))
    rc = LF.pco_b200_aggregate_files_async_plan(buf, C.c_size_t(len(head)), C.c_ubyte(dtype), C.c_size_t(1 << 20),
                                                C.c_size_t(1 << 16), C.c_size_t(max_files), C.c_size_t(max_chunks), C.c_size_t(rows_cap),
                                                C.byref(p) if plan else None)
    return rc, p, LF.pco_b200_last_error_message().decode()


def _expected_files(dtype, max_files, max_chunks, rows_cap):
    s = rows_cap // 256 + max_chunks
    return _files_workspace(max_files, max_chunks, rows_cap) + sum(al(r) for r in [48, 4 * s, 32 * s, ELEM[dtype] * rows_cap, 4 * max_chunks,
                                                                                  4 * (max_chunks + 1), 48 * max_files])


def test_argument_checks_come_before_the_device(L):
    rc, _, msg = _plan(L, dtype=99)
    assert rc == 5 and "type" in msg, msg
    for mp in (0, 1 << 31):
        rc, _, msg = _plan(L, max_pages=mp)
        assert rc == 3 and "max_pages" in msg, msg
    for name in ("rows_cap", "frame_cap"):
        rc, _, msg = _plan(L, **{name: (1 << 56) + 1})
        assert rc == 3 and name in msg, msg
    rc, _, _ = _plan(L, plan=False)
    assert rc == 3


@pytest.mark.parametrize("dtype", sorted(ELEM))
@pytest.mark.parametrize("mp,rc_,fc", [(1, 0, 0), (3, 255, 17), (257, 12345, 999), (4096, 1 << 24, 1 << 30)])
def test_pages_workspace_matches_the_formula(L, dtype, mp, rc_, fc):
    _, p, _ = _plan(L, dtype=dtype, max_pages=mp, rows_cap=rc_, frame_cap=fc)
    assert (p.dtype, p.max_pages, p.rows_cap, p.frame_cap) == (dtype, mp, rc_, fc)
    assert p.workspace_bytes == _expected_pages(dtype, mp, rc_, fc)


def test_pages_workspace_does_not_depend_on_the_buffers(L):
    ws = lambda **kw: _plan(L, **kw)[1].workspace_bytes  # noqa: E731
    assert ws(metas_cap=1 << 30, pages_cap=1 << 30) == ws()


def test_files_plan_checks(LF):
    for kw, words in [({"max_files": 0}, "max_files"), ({"max_chunks": 0}, "max_chunks"), ({"rows_cap": (1 << 56) + 1}, "rows_cap")]:
        rc, _, msg = _files_plan(LF, HEAD, **kw)
        assert rc == 3 and words in msg, msg
    rc, _, msg = _files_plan(LF, HEAD, dtype=99)
    assert rc == 5


@pytest.mark.parametrize("dtype", sorted(ELEM))
@pytest.mark.parametrize("mf,mc,rows", [(1, 1, 0), (8, 16, 1 << 16), (4096, 5000, 12345), (3, 1 << 20, 1 << 28)])
def test_files_workspace_matches_the_formula(LF, dtype, mf, mc, rows):
    _, p, _ = _files_plan(LF, HEAD, dtype=dtype, max_files=mf, max_chunks=mc, rows_cap=rows)  # HEAD has no uniform type: every dtype
    assert (p.dtype, p.max_files, p.max_chunks, p.rows_cap) == (dtype, mf, mc, rows)
    assert p.workspace_bytes == _expected_files(dtype, mf, mc, rows)


def test_files_workspace_does_not_depend_on_the_buffers(LF):
    from pcodec_b200 import standalone

    def ws(src_cap, index_cap):
        p = standalone._CAsyncFilesAggregatePlan()
        buf = C.create_string_buffer(HEAD, len(HEAD))
        LF.pco_b200_aggregate_files_async_plan(buf, C.c_size_t(len(HEAD)), C.c_ubyte(U32), C.c_size_t(src_cap), C.c_size_t(index_cap),
                                               C.c_size_t(8), C.c_size_t(16), C.c_size_t(1 << 16), C.byref(p))
        return p.workspace_bytes

    assert ws(1 << 20, 1 << 16) == ws(1 << 34, 1 << 30)


def _result(L, **fields):
    from pcodec_b200 import wrapped

    s = wrapped._CAsyncAggregateStatus(**fields)
    nm = C.c_size_t(12345)
    rc = L.pco_b200_aggregate_pages_async_result(C.byref(s), C.byref(nm))
    return rc, L.pco_b200_last_error_message().decode(), nm.value


def test_result_maps_statuses_to_kinds_and_messages(L, LF):
    from pcodec_b200 import standalone

    assert _result(L, kind=0, n_matches=1000, page=NONE)[::2] == (0, 1000)
    rc, msg, nm = _result(L, kind=2, device_status=2, page=17)
    assert rc == 2 and msg.startswith("page 17: ") and "insufficient data" in msg and nm == 12345, msg
    rc, msg, _ = _result(L, kind=3, device_status=0x11e, page=4)
    assert rc == 3 and msg.startswith("page 4: ") and "rows_cap" in msg, msg
    rc, msg, _ = _result(L, kind=3, device_status=0x11a, page=NONE, n_pages=99)
    assert rc == 3 and "*n_pages is 99" in msg, msg
    assert L.pco_b200_aggregate_pages_async_result(None, None) == 3
    s = standalone._CAsyncFilesAggregateStatus(kind=1, device_status=1, file=3, chunk=2)
    assert LF.pco_b200_aggregate_files_async_result(C.byref(s), None) == 1
    assert LF.pco_b200_last_error_message().decode() == "file 3: corrupt data in chunk 2"
    s = standalone._CAsyncFilesAggregateStatus(kind=0, n_matches=77)
    nm = C.c_size_t()
    assert LF.pco_b200_aggregate_files_async_result(C.byref(s), C.byref(nm)) == 0 and nm.value == 77


def test_calls_refuse_missing_buffers_without_a_device(L, LF):
    from pcodec_b200 import standalone, wrapped

    _, p, _ = _plan(L)
    nz = C.c_void_p(256)
    s = wrapped._CAsyncAggregateStatus()
    args = [nz] * 8
    for i in range(8):
        a = list(args)
        a[i] = None
        assert L.pco_b200_aggregate_pages_async(C.byref(p), *a, C.byref(s), None) == 3
        assert "null buffer" in L.pco_b200_last_error_message().decode()
    assert L.pco_b200_aggregate_pages_async(C.byref(p), *args[:7], C.c_void_p(257), C.byref(s), None) == 3
    bad = wrapped._CAsyncAggregatePlan.from_buffer_copy(bytes(p))
    bad.workspace_bytes += 1
    assert L.pco_b200_aggregate_pages_async(C.byref(bad), *args, C.byref(s), None) == 3
    assert "not made by" in L.pco_b200_last_error_message().decode()
    fp = standalone._CAsyncFilesAggregatePlan()
    fs = standalone._CAsyncFilesAggregateStatus()
    assert LF.pco_b200_aggregate_files_async(C.byref(fp), *args, C.byref(fs), None) == 3
    assert LF.pco_b200_aggregate_files_async(C.byref(fp), None, *args[1:], C.byref(fs), None) == 3


def test_new_symbols_are_exported(L, LF):
    for name in ("pco_b200_aggregate_pages_async_plan", "pco_b200_aggregate_pages_async", "pco_b200_aggregate_pages_async_result"):
        assert hasattr(L, name), name
    for name in ("pco_b200_aggregate_files_async_plan", "pco_b200_aggregate_files_async", "pco_b200_aggregate_files_async_result"):
        assert hasattr(LF, name), name


def test_unpack_aggregates():
    from pcodec_b200 import wrapped

    m = (1 << 64) - 1
    recs = np.array([[10, 2, 5, m, m, m],  # i64: min 5, max -1, sum -1
                     [0, 0, 0, 0, 0, 0],
                     [7, 3, 1, 2, 3, 1]], dtype=np.uint64).view(np.int64)
    got = wrapped.unpack_aggregates(recs, np.int64)
    assert got[0] == (10, 2, np.int64(5), np.int64(-1), -1)
    assert got[1] == (0, 0, np.int64(0), np.int64(0), 0)
    assert got[2][4] == (1 << 64) + 3
    got = wrapped.unpack_aggregates(recs, np.uint64)
    assert got[0][3] == np.uint64(m) and got[0][4] == (1 << 128) - 1
    one = int(np.array([1.5]).view(np.uint64)[0])
    f = wrapped.unpack_aggregates(np.array([4, 1, 0x3E00, 0xBC00, one, 0], dtype=np.uint64).view(np.int64), np.float16)
    assert f == [(4, 1, np.float16(1.5), np.float16(-1.0), 1.5)] and isinstance(f[0][4], float)
    assert wrapped.unpack_aggregates(np.array([1, 1, 0xFF, 0x80, 0xFF + 0x80, 0], dtype=np.uint64).view(np.int64), np.int8)[0][2:] == \
        (np.int8(-1), np.int8(-128), 0xFF + 0x80)


def test_float_order_emulation_on_hand_worked_cases():
    # lane partials are left to right: 1e16 + 1 + 1 - 1e16 is 0 that way (1e16 + 1 rounds back to 1e16), not 2
    v = np.zeros(256)
    v[:4] = [1e16, 1.0, 1.0, -1e16]
    assert ref.batch_sums(v, np.ones(256, bool))[0] == 0.0
    # the lane tree pairs (0, 1) before (2, 3): lanes 1e16, 1, 1, -1e16 give (1e16 + 1) + (1 - 1e16) = 1e16 - 1e16 = 0
    v = np.zeros(256)
    v[[0, 8, 16, 24]] = [1e16, 1.0, 1.0, -1e16]
    assert ref.batch_sums(v, np.ones(256, bool))[0] == 0.0
    # non-matches add nothing, and a sum of -0.0 alone is +0.0
    v = np.full(256, -0.0)
    s = ref.batch_sums(v, np.ones(256, bool))[0]
    assert s == 0.0 and not np.signbit(s)
    # a group's batch j goes to lane j mod 32: batches 0 and 32 share lane 0, added in order before the tree
    sums = np.zeros(64)
    sums[[0, 32, 1]] = [1e16, -1e16, 1.0]
    assert ref.strided_sum(sums) == 1.0
    sums = np.zeros(64)
    sums[[0, 1, 32]] = [1e16, 1.0, -1e16]  # lane 0: 1e16 - 1e16 = 0, lane 1: 1 -> 1
    assert ref.strided_sum(sums) == 1.0
    sums = np.zeros(32)
    sums[[0, 1, 2]] = [1e16, 1.0, -1e16]  # tree: (1e16 + 1) + (-1e16 + 0) = 0
    assert ref.strided_sum(sums) == 0.0
    # +inf and -inf give NaN
    assert np.isnan(ref.strided_sum([np.inf, -np.inf]))
    # batches restart at each page: 300 numbers of one page are batches of 256 and 44
    x = np.arange(300, dtype=np.float32)
    r, fs = ref.record(x, [300], 0.0, 1000.0)
    assert r[:4] == [300, 300, 0, int(np.float32(299).view(np.uint32))] and fs == float(x.sum())
    # the key order puts -0.0 below +0.0
    z = np.array([0.0, -0.0], dtype=np.float64)
    r, _ = ref.record(z, [2], -1.0, 1.0)
    assert r[2] == 1 << 63 and r[3] == 0
