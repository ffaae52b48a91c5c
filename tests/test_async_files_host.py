"""Host side of the asynchronous batch-of-files call (pco_b200_decompress_files_async_plan / _result) without a GPU: the plan's argument
checks, its workspace size against the formula include/pco_b200.h documents, how a status written by the device becomes a kind and a
"file <i>: " message, and the call's host-side argument checks."""
import ctypes as C

import pytest

HEAD = b"pco!\x03\x00\x00\x04\x01\x00"
HEAD_U64 = b"pco!\x03\x02\x00\x04\x01\x00"
U64, U32, F16 = 2, 1, 9
NONE = (1 << 64) - 1


@pytest.fixture(scope="module")
def L():
    from pcodec_b200 import standalone

    return standalone._lib_async_files()


def _plan(L, head=HEAD, dtype=U64, src_cap=1 << 20, index_cap=1 << 16, max_files=64, max_chunks=16, dst_cap=1 << 18):
    from pcodec_b200 import standalone

    p = standalone._CAsyncFilesPlan()
    buf = C.create_string_buffer(head, len(head)) if head is not None else None
    rc = L.pco_b200_decompress_files_async_plan(buf, C.c_size_t(len(head) if head is not None else 0), C.c_ubyte(dtype), C.c_size_t(src_cap),
                                                C.c_size_t(index_cap), C.c_size_t(max_files), C.c_size_t(max_chunks), C.c_size_t(dst_cap),
                                                C.byref(p))
    return rc, p, L.pco_b200_last_error_message().decode()


def _expected_workspace(max_files, max_chunks, dst_cap):
    """The formula of include/pco_b200.h, each region rounded up to 256 bytes."""
    al = lambda x: (x + 255) // 256 * 256  # noqa: E731
    ctas = lambda n: (n + 255) // 256  # noqa: E731
    per_var = (1 << 14) * 6 + (1 << 15) * 13 + 288 * 8 + 256 * 4 + 64
    cold = 3 * per_var + 2 * (2 * (1 << 16) * 8) + 8192
    rows = 2 * (dst_cap // 256 + max_chunks + 1)
    mf, mc = max_files, max_chunks
    regions = [32 + 33 * 7 * 8, 64, 4 * mf, 64 * mf, 4 * mf, 48 * mf, 48 * ctas(mf), 32 * mc, 4 * mc, mc, rows * 256, rows * 4, cold]
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
    for mf in (0, 1 << 31):
        rc, _, msg = _plan(L, max_files=mf)
        assert rc == 3 and "max_files" in msg, msg
    for mc in (0, 1 << 32):
        rc, _, msg = _plan(L, max_chunks=mc)
        assert rc == 3 and "max_chunks" in msg, msg
    rc, _, msg = _plan(L, dst_cap=(1 << 56) + 1)
    assert rc == 3 and "dst_cap" in msg, msg
    rc, _, _ = _plan(L, head=None)
    assert rc == 2


def test_valid_plan_fills_the_plan_or_needs_a_device(L):
    rc, p, msg = _plan(L, head=HEAD_U64, src_cap=1000, index_cap=2000, max_files=5, max_chunks=7, dst_cap=3000)
    # without a device the set-up fails with Cuda, after the plan is filled
    assert rc == (0 if L.pco_b200_device_available() else 6), msg
    if rc == 6:
        assert "CUDA" in msg or "device" in msg, msg
    assert (p.dtype, p.uniform_type, p.format_major) == (U64, U64, 4)
    assert (p.src_cap, p.index_cap, p.max_files, p.max_chunks, p.dst_cap) == (1000, 2000, 5, 7, 3000)
    assert p.workspace_bytes == _expected_workspace(5, 7, 3000)
    _, p, _ = _plan(L, max_files=(1 << 31) - 1, max_chunks=(1 << 32) - 1, dst_cap=1 << 56)
    assert p.workspace_bytes == _expected_workspace((1 << 31) - 1, (1 << 32) - 1, 1 << 56)


@pytest.mark.parametrize("mf,mc,dc", [(1, 1, 0), (3, 1, 255), (255, 3, 256), (256, 1024, 1 << 20), (257, 1 << 20, 12345), (4096, 9, 1 << 24)])
def test_workspace_matches_the_formula(L, mf, mc, dc):
    _, p, _ = _plan(L, max_files=mf, max_chunks=mc, dst_cap=dc)
    assert p.workspace_bytes == _expected_workspace(mf, mc, dc)


def test_workspace_grows_with_every_capacity(L):
    ws = lambda **kw: _plan(L, **kw)[1].workspace_bytes  # noqa: E731
    base = ws(max_files=1000, max_chunks=1000, dst_cap=1 << 20)
    assert ws(max_files=2000, max_chunks=1000, dst_cap=1 << 20) - base == _expected_workspace(2000, 1000, 1 << 20) - _expected_workspace(1000, 1000, 1 << 20) > 0
    assert ws(max_files=1000, max_chunks=2000, dst_cap=1 << 20) > base
    assert ws(max_files=1000, max_chunks=1000, dst_cap=1 << 21) > base


def _result(L, **fields):
    from pcodec_b200 import standalone

    s = standalone._CAsyncFilesStatus(**fields)
    nw = C.c_size_t(12345)
    rc = L.pco_b200_decompress_files_async_result(C.byref(s), C.byref(nw))
    return rc, L.pco_b200_last_error_message().decode(), nw.value


def test_result_maps_statuses_to_kinds_and_messages(L):
    assert _result(L, kind=0, n_written=1000, file=NONE, chunk=NONE)[::2] == (0, 1000)
    # chunk failures: "file F: <kind words> in chunk C", C counted from the file's first chunk
    for kind, st, words in [(1, 1, "corrupt data"), (2, 2, "insufficient data"), (3, 3, "invalid argument"), (7, 7, "valid pco outside")]:
        rc, msg, nw = _result(L, kind=kind, device_status=st, file=17, chunk=3)
        assert rc == kind and msg.startswith("file 17: ") and words in msg and msg.endswith("chunk 3"), msg
        assert nw == 12345  # left alone on an error
    cases = [(0x101, 1, "corrupt standalone header"), (0x102, 2, "insufficient data"), (0x103, 3, "differs from the plan"),
             (0x104, 3, "does not belong"), (0x105, 3, "max_chunks"), (0x10f, 3, "file lies outside src"),
             (0x110, 3, "index offset is not a multiple of 16"), (0x111, 3, "side index lies outside index"), (0x112, 7, "no side index"),
             (0x113, 3, "misaligned entries"), (0x114, 3, "points outside"), (0x115, 4, "dst holds")]
    for st, kind, words in cases:
        rc, msg, _ = _result(L, kind=kind, device_status=st, file=4, chunk=NONE, n_files=9)
        assert rc == kind and msg.startswith("file 4: ") and words in msg, (st, msg)
    rc, msg, _ = _result(L, kind=3, device_status=0x10e, file=NONE, chunk=NONE, n_files=99)
    assert rc == 3 and "*n_files is 99" in msg and "max_files" in msg and not msg.startswith("file"), msg
    rc, _, _ = _result(L, kind=99, device_status=1, file=0, chunk=0)
    assert rc == 1
    assert L.pco_b200_decompress_files_async_result(None, None) == 3


def test_status_codes_follow_the_other_async_codes():
    import os
    import re

    text = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "pco_b200.h")).read()
    codes = {name: int(v, 16) for name, v in re.findall(r"(PCO_B200_ASYNC_[A-Z_]+) = (0x[0-9a-f]+)", text)}
    assert len(set(codes.values())) == len(codes)
    new = ["TOO_MANY_FILES", "FILE_OUTSIDE", "INDEX_OFFSET", "INDEX_OUTSIDE", "NO_INDEX", "ENTRIES_MISALIGNED", "RECORDS_OUTSIDE", "FILES_DST"]
    assert [codes["PCO_B200_ASYNC_" + n] for n in new] == list(range(0x10e, 0x116))


def test_call_refuses_missing_buffers_without_a_device(L):
    from pcodec_b200 import standalone

    _, p, _ = _plan(L)
    s = standalone._CAsyncFilesStatus()
    nz = C.c_void_p(256)

    def call(plan, src=nz, index=nz, files=nz, n=nz, dst=nz, ws=nz, status=C.byref(s)):
        return L.pco_b200_decompress_files_async(plan, src, index, files, n, dst, nz, ws, status, None)

    assert call(None) == 3
    assert call(C.byref(p), src=None) == 3
    assert call(C.byref(p), index=None) == 3
    assert call(C.byref(p), files=None) == 3
    assert call(C.byref(p), n=None) == 3
    assert call(C.byref(p), dst=None) == 3
    assert call(C.byref(p), ws=None) == 3
    assert call(C.byref(p), status=None) == 3
    bad = standalone._CAsyncFilesPlan.from_buffer_copy(bytes(p))
    bad.workspace_bytes += 1
    assert call(C.byref(bad)) == 3
    assert "not made by" in L.pco_b200_last_error_message().decode()
    bad = standalone._CAsyncFilesPlan.from_buffer_copy(bytes(p))
    bad.max_files = 0
    assert call(C.byref(bad)) == 3
    assert call(C.byref(standalone._CAsyncFilesPlan())) == 3  # a plan that was never filled
    assert call(C.byref(p), ws=C.c_void_p(257)) == 3
    assert "256-byte aligned" in L.pco_b200_last_error_message().decode()


def test_plan_needs_a_device(L):
    if L.pco_b200_device_available():
        pytest.skip("a CUDA device is present")
    # the plan's set-up is where the device is first needed: Cuda, and the message says there is no CPU fallback
    rc, _, msg = _plan(L)
    assert rc == 6 and "no CPU fallback" in msg, msg


def test_new_symbols_are_exported(L):
    for name in ("pco_b200_decompress_files_async_plan", "pco_b200_decompress_files_async", "pco_b200_decompress_files_async_result"):
        assert hasattr(L, name), name
