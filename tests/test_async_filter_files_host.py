"""Host side of the asynchronous filter of indexed standalone files (pco_b200_filter_files_async_plan / _result) without a GPU: the plan's
argument checks, its workspace size against the formula include/pco_b200.h documents, how a status written by the device becomes a kind
and a "file <i>: " message, and the call's host-side argument checks."""
import ctypes as C

import pytest

from tests.test_async_files_host import HEAD, HEAD_U64, NONE, U32, U64
from tests.test_async_files_host import _expected_workspace as _files_workspace

ELEM = {1: 4, 2: 8, 3: 4, 4: 8, 5: 4, 6: 8, 7: 2, 8: 2, 9: 2, 10: 1, 11: 1}
F16, U8 = 9, 10


@pytest.fixture(scope="module")
def L():
    from pcodec_b200 import standalone

    return standalone._lib_async_filter_files()


def _plan(L, head=HEAD, dtype=U64, src_cap=1 << 20, index_cap=1 << 16, max_files=64, max_chunks=16, rows_cap=1 << 18, out_cap=1 << 10):
    from pcodec_b200 import standalone

    p = standalone._CAsyncFilesFilterPlan()
    buf = C.create_string_buffer(head, len(head)) if head is not None else None
    rc = L.pco_b200_filter_files_async_plan(buf, C.c_size_t(len(head) if head is not None else 0), C.c_ubyte(dtype), C.c_size_t(src_cap),
                                            C.c_size_t(index_cap), C.c_size_t(max_files), C.c_size_t(max_chunks), C.c_size_t(rows_cap),
                                            C.c_size_t(out_cap), C.byref(p))
    return rc, p, L.pco_b200_last_error_message().decode()


def _expected_workspace(dtype, max_files, max_chunks, rows_cap):
    """The formula of include/pco_b200.h: the files plan's with dst_cap = rows_cap, then these regions, each rounded up to 256 bytes."""
    al = lambda x: (x + 255) // 256 * 256  # noqa: E731
    s = rows_cap // 256 + max_chunks
    regions = [48, 16, 4 * s, 8 * s, 8 * ((s + 255) // 256), ELEM[dtype] * rows_cap, rows_cap, 4 * max_chunks, 4 * (max_chunks + 1)]
    return _files_workspace(max_files, max_chunks, rows_cap) + sum(al(r) for r in regions)


def test_argument_checks_come_before_the_device(L):
    rc, _, msg = _plan(L, dtype=99)
    assert rc == 5 and "type" in msg, msg
    rc, _, msg = _plan(L, head=b"pcX!\x03\x00\x00\x04\x01\x00")
    assert rc == 1 and "magic" in msg, msg
    rc, _, _ = _plan(L, head=b"pc")
    assert rc == 2
    rc, _, msg = _plan(L, head=HEAD_U64, dtype=U32)
    assert rc == 3 and "uniform type 2" in msg, msg
    for mf in (0, 1 << 31):
        rc, _, msg = _plan(L, max_files=mf)
        assert rc == 3 and "max_files" in msg, msg
    for mc in (0, 1 << 32):
        rc, _, msg = _plan(L, max_chunks=mc)
        assert rc == 3 and "max_chunks" in msg, msg
    for name in ("rows_cap", "out_cap"):
        rc, _, msg = _plan(L, **{name: (1 << 56) + 1})
        assert rc == 3 and name in msg, msg
    rc, _, _ = _plan(L, head=None)
    assert rc == 2


def test_valid_plan_fills_the_plan_or_needs_a_device(L):
    rc, p, msg = _plan(L, head=HEAD_U64, src_cap=1000, index_cap=2000, max_files=5, max_chunks=7, rows_cap=3000, out_cap=77)
    assert rc == (0 if L.pco_b200_device_available() else 6), msg
    if rc == 6:
        assert "CUDA" in msg or "device" in msg, msg
    assert (p.dtype, p.uniform_type, p.format_major) == (U64, U64, 4)
    assert (p.src_cap, p.index_cap, p.max_files, p.max_chunks, p.rows_cap, p.out_cap) == (1000, 2000, 5, 7, 3000, 77)
    assert p.workspace_bytes == _expected_workspace(U64, 5, 7, 3000)
    _, p, _ = _plan(L, dtype=U8, max_files=(1 << 31) - 1, max_chunks=(1 << 32) - 1, rows_cap=1 << 56, out_cap=1 << 56)
    assert p.workspace_bytes == _expected_workspace(U8, (1 << 31) - 1, (1 << 32) - 1, 1 << 56)


@pytest.mark.parametrize("dtype", sorted(ELEM))
@pytest.mark.parametrize("mf,mc,rc_", [(1, 1, 0), (3, 1, 255), (255, 3, 256), (256, 1024, 1 << 20), (257, 1 << 20, 12345), (4096, 9, 1 << 24)])
def test_workspace_matches_the_formula(L, dtype, mf, mc, rc_):
    _, p, _ = _plan(L, dtype=dtype, max_files=mf, max_chunks=mc, rows_cap=rc_)
    assert p.workspace_bytes == _expected_workspace(dtype, mf, mc, rc_)


def test_workspace_does_not_depend_on_out_cap_or_the_buffers(L):
    ws = lambda **kw: _plan(L, **kw)[1].workspace_bytes  # noqa: E731
    base = ws()
    assert ws(out_cap=0) == ws(out_cap=1 << 40) == base
    assert ws(src_cap=1 << 40, index_cap=1 << 30) == base
    assert ws(max_chunks=17) - base == _expected_workspace(U64, 64, 17, 1 << 18) - _expected_workspace(U64, 64, 16, 1 << 18) > 0


def _result(L, **fields):
    from pcodec_b200 import standalone

    s = standalone._CAsyncFilesFilterStatus(**fields)
    nm = C.c_size_t(12345)
    rc = L.pco_b200_filter_files_async_result(C.byref(s), C.byref(nm))
    return rc, L.pco_b200_last_error_message().decode(), nm.value


def test_result_maps_statuses_to_kinds_and_messages(L):
    assert _result(L, kind=0, n_matches=1000, matches_needed=1000, file=NONE, chunk=NONE)[::2] == (0, 1000)
    for kind, st, words in [(1, 1, "corrupt data"), (2, 2, "insufficient data"), (3, 3, "invalid argument"), (7, 7, "valid pco outside")]:
        rc, msg, nm = _result(L, kind=kind, device_status=st, file=3, chunk=2)
        assert rc == kind and msg.startswith("file 3: ") and words in msg and msg.endswith("chunk 2"), msg
        assert nm == 12345  # left alone on an error
    cases = [(0x101, 1, "corrupt standalone header"), (0x102, 2, "insufficient data"), (0x103, 3, "differs from the plan"),
             (0x104, 3, "does not belong"), (0x105, 3, "max_chunks"), (0x10f, 3, "file lies outside src"),
             (0x110, 3, "index offset is not a multiple of 16"), (0x111, 3, "side index lies outside index"), (0x112, 7, "no side index"),
             (0x113, 3, "misaligned entries"), (0x114, 3, "points outside"), (0x115, 4, "more numbers than rows_cap")]
    for st, kind, words in cases:
        rc, msg, _ = _result(L, kind=kind, device_status=st, file=4, chunk=NONE, n_files=9)
        assert rc == kind and msg.startswith("file 4: ") and words in msg, (st, msg)
    rc, msg, _ = _result(L, kind=3, device_status=0x10e, file=NONE, chunk=NONE, n_files=99)
    assert rc == 3 and "*n_files is 99" in msg and "max_files" in msg and not msg.startswith("file"), msg
    rc, msg, nm = _result(L, kind=4, device_status=0x201, file=NONE, chunk=NONE, n_matches=10, matches_needed=987654)
    assert rc == 4 and "987654 matches" in msg and "out_cap" in msg and nm == 12345, msg
    rc, _, _ = _result(L, kind=99, device_status=1, file=0, chunk=0)
    assert rc == 1
    assert L.pco_b200_filter_files_async_result(None, None) == 3


def test_call_refuses_missing_buffers_without_a_device(L):
    from pcodec_b200 import standalone

    _, p, _ = _plan(L)
    s = standalone._CAsyncFilesFilterStatus()
    nz = C.c_void_p(256)

    def call(plan, src=nz, index=nz, files=nz, n=nz, iv=nz, vals=nz, pos=nz, nm=nz, file_ns=nz, ws=nz, status=C.byref(s)):
        return L.pco_b200_filter_files_async(plan, src, index, files, n, iv, vals, pos, nm, file_ns, ws, status, None)

    assert call(None) == 3
    for kw in ("src", "index", "files", "n", "iv", "vals", "pos", "nm", "ws", "status"):
        assert call(C.byref(p), **{kw: None}) == 3, kw
        assert "null buffer" in L.pco_b200_last_error_message().decode()
    bad = standalone._CAsyncFilesFilterPlan.from_buffer_copy(bytes(p))
    bad.workspace_bytes += 1
    assert call(C.byref(bad)) == 3
    assert "not made by" in L.pco_b200_last_error_message().decode()
    for field, value in (("out_cap", (1 << 56) + 1), ("max_chunks", 0), ("rows_cap", (1 << 56) + 1)):
        bad = standalone._CAsyncFilesFilterPlan.from_buffer_copy(bytes(p))
        setattr(bad, field, value)
        assert call(C.byref(bad)) == 3, field
    assert call(C.byref(standalone._CAsyncFilesFilterPlan())) == 3  # a plan that was never filled
    assert call(C.byref(p), ws=C.c_void_p(257)) == 3
    assert "256-byte aligned" in L.pco_b200_last_error_message().decode()


def test_plan_needs_a_device(L):
    if L.pco_b200_device_available():
        pytest.skip("a CUDA device is present")
    rc, _, msg = _plan(L)
    assert rc == 6 and "no CPU fallback" in msg, msg


def test_new_symbols_are_exported(L):
    for name in ("pco_b200_filter_files_async_plan", "pco_b200_filter_files_async", "pco_b200_filter_files_async_result"):
        assert hasattr(L, name), name
