"""Host side of the asynchronous ranges call (pco_b200_decompress_ranges_async_plan / _result) without a GPU: the plan's argument checks,
its workspace size against the formula include/pco_b200.h documents, and how a status written by the device becomes a kind and a message."""
import ctypes as C

import pytest

HEAD = b"pco!\x03\x00\x00\x04\x01\x00"
HEAD_U64 = b"pco!\x03\x02\x00\x04\x01\x00"
U64, U32, F16 = 2, 1, 9
NONE = (1 << 64) - 1


@pytest.fixture(scope="module")
def L():
    from pcodec_b200 import standalone

    return standalone._lib_async_ranges()


def _plan(L, head=HEAD, dtype=U64, src_cap=1 << 20, index_cap=1 << 16, max_chunks=16, max_ranges=64, dst_cap=1 << 18, window_cap=1 << 18):
    from pcodec_b200 import standalone

    p = standalone._CAsyncRangesPlan()
    buf = C.create_string_buffer(head, len(head)) if head is not None else None
    rc = L.pco_b200_decompress_ranges_async_plan(buf, C.c_size_t(len(head) if head is not None else 0), C.c_ubyte(dtype), C.c_size_t(src_cap),
                                                 C.c_size_t(index_cap), C.c_size_t(max_chunks), C.c_size_t(max_ranges), C.c_size_t(dst_cap),
                                                 C.c_size_t(window_cap), C.byref(p))
    return rc, p, L.pco_b200_last_error_message().decode()


def _expected_workspace(max_chunks, max_ranges, window_cap, elem):
    """The formula of include/pco_b200.h, each region rounded up to 256 bytes."""
    al = lambda x: (x + 255) // 256 * 256  # noqa: E731
    ctas = lambda n: (n + 255) // 256  # noqa: E731
    per_var = (1 << 14) * 6 + (1 << 15) * 13 + 288 * 8 + 256 * 4 + 64
    cold = 3 * per_var + 2 * (2 * (1 << 16) * 8) + 8192
    rows = 2 * (window_cap // 256)
    mc, mr = max_chunks, max_ranges
    regions = [32 + 33 * 7 * 8, 48, 32 * mc, 32 * mc, 24 * ctas(mc), 32 * ctas(mr), 8 * mr, 8 * mr, 32 * mc, 24 * mc, 24 * mc, 4 * mc, mc,
               rows * 256, rows * 4, window_cap * elem, cold]
    return sum(al(r) for r in regions)


def test_argument_checks_come_before_the_device(L):
    rc, _, msg = _plan(L, dtype=99)
    assert rc == 5 and "type" in msg, msg
    rc, _, msg = _plan(L, head=b"pcX!\x03\x00\x00\x04\x01\x00")
    assert rc == 1 and "magic" in msg, msg
    rc, _, _ = _plan(L, head=b"pc")
    assert rc == 2
    rc, _, msg = _plan(L, head=HEAD_U64, dtype=U32)
    assert rc == 3 and "uniform type 2" in msg, msg
    for mc in (0, 1 << 32):
        rc, _, msg = _plan(L, max_chunks=mc)
        assert rc == 3 and "max_chunks" in msg, msg
    for mr in (0, 1 << 32):
        rc, _, msg = _plan(L, max_ranges=mr)
        assert rc == 3 and "max_ranges" in msg, msg
    rc, _, msg = _plan(L, dst_cap=(1 << 56) + 1)
    assert rc == 3 and "dst_cap" in msg, msg
    rc, _, msg = _plan(L, window_cap=(1 << 56) + 1)
    assert rc == 3 and "window_cap" in msg, msg
    rc, _, _ = _plan(L, head=None)
    assert rc == 2


def test_valid_plan_fills_the_plan(L):
    rc, p, msg = _plan(L, head=HEAD_U64, src_cap=1000, index_cap=2000, max_chunks=7, max_ranges=9, dst_cap=3000, window_cap=4000)
    assert rc == (0 if L.pco_b200_device_available() else 6), msg
    assert (p.dtype, p.uniform_type, p.format_major) == (U64, U64, 4)
    assert (p.src_cap, p.index_cap, p.max_chunks, p.max_ranges, p.dst_cap, p.window_cap) == (1000, 2000, 7, 9, 3000, 4000)
    assert p.workspace_bytes == _expected_workspace(7, 9, 4000, 8)


@pytest.mark.parametrize("dtype,elem", [(U64, 8), (U32, 4), (F16, 2)])
@pytest.mark.parametrize("mc,mr,wc", [(1, 1, 0), (3, 1, 255), (3, 5, 256), (1024, 4096, 1 << 20), (1 << 20, 7, 12345), (9, 1 << 20, 1 << 24)])
def test_workspace_matches_the_formula(L, dtype, elem, mc, mr, wc):
    _, p, _ = _plan(L, dtype=dtype, max_chunks=mc, max_ranges=mr, window_cap=wc)
    assert p.workspace_bytes == _expected_workspace(mc, mr, wc, elem)


def _result(L, **fields):
    from pcodec_b200 import standalone

    s = standalone._CAsyncRangesStatus(**fields)
    nw = C.c_size_t(12345)
    rc = L.pco_b200_decompress_ranges_async_result(C.byref(s), C.byref(nw))
    return rc, L.pco_b200_last_error_message().decode(), nw.value


def test_result_maps_statuses_to_kinds_and_messages(L):
    assert _result(L, kind=0, n_written=1000, range=NONE, chunk=NONE)[::2] == (0, 1000)
    # chunk failures: the sync call's "range R: <kind words> in chunk C"
    for kind, st, words in [(1, 1, "corrupt data"), (2, 2, "insufficient data"), (3, 3, "invalid argument"), (7, 7, "valid pco outside")]:
        rc, msg, nw = _result(L, kind=kind, device_status=st, range=17, chunk=3)
        assert rc == kind and msg.startswith("range 17: ") and words in msg and msg.endswith("chunk 3"), msg
        assert nw == 12345  # left alone on an error
    cases = [(0x101, 1, "corrupt standalone header"), (0x102, 2, "insufficient data"), (0x103, 3, "differs from the plan"),
             (0x104, 3, "does not belong"), (0x105, 3, "max_chunks"), (0x107, 3, "side index: chunk 5 does not start"),
             (0x108, 3, "side index"), (0x109, 3, "max_ranges"), (0x10a, 3, "range 4: "), (0x10b, 3, "range 4: "),
             (0x10c, 3, "the ranges' 777 numbers"), (0x10d, 4, "window of 1536 numbers")]
    for st, kind, words in cases:
        rc, msg, _ = _result(L, kind=kind, device_status=st, range=4, chunk=5, n_written=777, window_needed=1536)
        assert rc == kind and words in msg, (st, msg)
    rc, _, _ = _result(L, kind=99, device_status=1, range=0, chunk=0)
    assert rc == 1
    assert L.pco_b200_decompress_ranges_async_result(None, None) == 3


def test_call_refuses_missing_buffers_without_a_device(L):
    from pcodec_b200 import standalone

    _, p, _ = _plan(L)
    s = standalone._CAsyncRangesStatus()
    nz = C.c_void_p(256)
    call = lambda plan, src=nz, ranges=nz, n=nz, ws=nz: L.pco_b200_decompress_ranges_async(plan, src, nz, ranges, n, nz, ws, C.byref(s), None)  # noqa: E731
    assert call(None) == 3
    assert call(C.byref(p), src=None) == 3
    assert call(C.byref(p), ranges=None) == 3
    assert call(C.byref(p), n=None) == 3
    assert call(C.byref(p), ws=None) == 3
    bad = standalone._CAsyncRangesPlan.from_buffer_copy(bytes(p))
    bad.workspace_bytes += 1
    assert call(C.byref(bad)) == 3
    assert call(C.byref(p), ws=C.c_void_p(257)) == 3
