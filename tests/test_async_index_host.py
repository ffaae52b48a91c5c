"""Host side of the asynchronous side index builder (pco_b200_build_index_async_plan / _result) without a GPU: the plan's argument
checks, its workspace size, and how a status written by the device becomes a kind, a message and an index length."""
import ctypes as C

import pytest

# an empty standalone file: version 3, uniform type byte, 1-byte size hint, format 4.1, terminator
HEAD = b"pco!\x03\x00\x00\x04\x01\x00"
HEAD_U64 = b"pco!\x03\x02\x00\x04\x01\x00"
U64, U32 = 2, 1


@pytest.fixture(scope="module")
def L():
    from pcodec_b200 import standalone

    return standalone._lib_async_index()


def _plan(L, head=HEAD, dtype=U64, src_cap=1 << 20, index_cap=1 << 16, max_chunks=16):
    from pcodec_b200 import standalone

    p = standalone._CAsyncIndexPlan()
    buf = C.create_string_buffer(head, len(head)) if head is not None else None
    rc = L.pco_b200_build_index_async_plan(buf, C.c_size_t(len(head) if head is not None else 0), C.c_ubyte(dtype), C.c_size_t(src_cap),
                                           C.c_size_t(index_cap), C.c_size_t(max_chunks), C.byref(p))
    return rc, p, L.pco_b200_last_error_message().decode()


def _expected_workspace(src_cap, index_cap, max_chunks):
    """The formula include/pco_b200.h states, each term rounded up to 256 bytes."""
    al = lambda x: (x + 255) // 256 * 256  # noqa: E731
    cands, recs = max_chunks + 8, max_chunks + 1
    find = max(1, -(-src_cap // 4096))
    return (256 + al(8 * find) + al(8 * cands) + al(32 * cands) + al(4 * cands) + al(8 * cands) + al(32 * recs) + al(8 * recs)
            + al(2 * index_cap) + al(index_cap))


def test_argument_checks_come_before_the_device(L):
    rc, _, msg = _plan(L, dtype=99)
    assert rc == 5 and "type" in msg, msg  # InvalidType
    rc, _, msg = _plan(L, head=b"pcX!\x03\x00\x00\x04\x01\x00")
    assert rc == 1 and "magic" in msg, msg  # Corruption, as the header parse words it
    rc, _, _ = _plan(L, head=b"pc")
    assert rc == 2  # InsufficientData
    rc, _, _ = _plan(L, head=b"pco!\x05\x00\x00\x04\x01\x00")  # standalone version 5
    assert rc == 1
    rc, _, msg = _plan(L, head=HEAD_U64, dtype=U32)
    assert rc == 3 and "uniform type 2" in msg, msg  # a uniform type other than dtype
    for mc in (0, (1 << 31) - 8, 1 << 32):  # the candidate walks launch max_chunks + 8 CTAs, at most 2^31 - 1
        rc, _, msg = _plan(L, max_chunks=mc)
        assert rc == 3 and "max_chunks" in msg, msg
    rc, _, msg = _plan(L, src_cap=((1 << 31) - 1) * 4096 + 1)  # the find grid: one CTA per 4096 bytes of src_cap
    assert rc == 3 and "src_cap" in msg, msg
    rc, _, _ = _plan(L, head=None)
    assert rc == 2  # no bytes at all
    assert L.pco_b200_build_index_async_plan(C.create_string_buffer(HEAD, len(HEAD)), C.c_size_t(len(HEAD)), C.c_ubyte(U64), C.c_size_t(1),
                                             C.c_size_t(1), C.c_size_t(1), None) == 3  # no plan to fill


def test_valid_plan_fills_the_plan(L):
    rc, p, msg = _plan(L, head=HEAD_U64, dtype=U64, src_cap=1000, index_cap=2000, max_chunks=7)
    assert rc == (0 if L.pco_b200_device_available() else 6), msg  # Cuda without a device, after the plan is filled
    assert (p.dtype, p.uniform_type, p.format_major) == (U64, U64, 4)
    assert (p.src_cap, p.index_cap, p.max_chunks) == (1000, 2000, 7)
    assert p.workspace_bytes == _expected_workspace(1000, 2000, 7)
    rc, p, _ = _plan(L, head=HEAD, dtype=U32)
    assert p.uniform_type == 0 and p.dtype == U32
    rc, p, msg = _plan(L, src_cap=((1 << 31) - 1) * 4096, max_chunks=(1 << 31) - 9)  # the largest grids: filled, never allocated here
    assert rc == (0 if L.pco_b200_device_available() else 6), msg
    assert p.workspace_bytes == _expected_workspace(((1 << 31) - 1) * 4096, 1 << 16, (1 << 31) - 9)
    rc, p, _ = _plan(L, head=b"pco!\x02\x00\x03", dtype=U32)  # standalone version 2, format major 3: an older flavour
    assert (p.uniform_type, p.format_major) == (0, 3)


@pytest.mark.parametrize("src_cap,index_cap,max_chunks", [(0, 0, 1), (1, 64, 1), (4095, 100, 3), (4096, 1 << 20, 4), (4097, 12345, 1024),
                                                           (1 << 28, 13 << 20, 1024), (12345, 1, (1 << 20) - 1)])
def test_workspace_matches_the_formula(L, src_cap, index_cap, max_chunks):
    _, p, _ = _plan(L, src_cap=src_cap, index_cap=index_cap, max_chunks=max_chunks)
    assert p.workspace_bytes == _expected_workspace(src_cap, index_cap, max_chunks)


def _result(L, **fields):
    from pcodec_b200 import standalone

    s = standalone._CAsyncIndexStatus(**fields)
    n = C.c_size_t(12345)
    rc = L.pco_b200_build_index_async_result(C.byref(s), C.byref(n))
    return rc, L.pco_b200_last_error_message().decode(), n.value


def test_result_maps_statuses_to_kinds_messages_and_length(L):
    rc, _, n = _result(L, kind=0, index_bytes=4096, n_chunks=3, chunk=(1 << 64) - 1)
    assert (rc, n) == (0, 4096)
    # chunk failures: the kind, and the message names the chunk as status_to_error words it
    for kind, st, words in [(1, 1, "corrupt data"), (2, 2, "insufficient data"), (3, 3, "invalid argument"), (7, 7, "valid pco outside")]:
        rc, msg, n = _result(L, kind=kind, device_status=st, chunk=17)
        assert rc == kind and msg.startswith("chunk 17: ") and words in msg, msg
        assert n == 12345  # the length is left alone on an error
    # file-level refusals
    cases = [(0x101, 1, "corrupt standalone header"), (0x102, 2, "insufficient data"), (0x103, 3, "differs from the plan"),
             (0x10f, 3, "src_cap"), (0x105, 3, "max_chunks"), (0x119, 4, "index_cap")]
    for st, kind, words in cases:
        rc, msg, _ = _result(L, kind=kind, device_status=st, chunk=(1 << 64) - 1)
        assert rc == kind and words in msg, msg
    # a kind the library does not know reads as Corruption
    rc, _, _ = _result(L, kind=99, device_status=1, chunk=0)
    assert rc == 1
    assert L.pco_b200_build_index_async_result(None, None) == 3


def test_device_kinds_of_the_codes_it_reuses():
    """The status kinds come from the one table every asynchronous call shares."""
    from pcodec_b200 import _lib

    k = _lib.lib().pco_b200_debug_async_kind
    assert [k(s) for s in (0x101, 0x102, 0x103, 0x10f, 0x105, 0x119, 1, 2, 7)] == [1, 2, 3, 3, 3, 4, 1, 2, 7]


def test_call_refuses_bad_buffers_without_a_device(L):
    from pcodec_b200 import standalone

    _, p, _ = _plan(L)
    s = standalone._CAsyncIndexStatus()
    nz = C.c_void_p(256)  # never dereferenced: the call refuses first
    assert L.pco_b200_build_index_async(None, nz, nz, nz, nz, C.byref(s), None) == 3
    assert L.pco_b200_build_index_async(C.byref(p), None, nz, nz, nz, C.byref(s), None) == 3
    assert L.pco_b200_build_index_async(C.byref(p), nz, None, nz, nz, C.byref(s), None) == 3
    assert L.pco_b200_build_index_async(C.byref(p), nz, nz, None, nz, C.byref(s), None) == 3
    assert L.pco_b200_build_index_async(C.byref(p), nz, nz, nz, None, C.byref(s), None) == 3
    bad = standalone._CAsyncIndexPlan.from_buffer_copy(bytes(p))
    bad.workspace_bytes += 1  # not what the plan computed
    assert L.pco_b200_build_index_async(C.byref(bad), nz, nz, nz, nz, C.byref(s), None) == 3
    assert L.pco_b200_build_index_async(C.byref(p), nz, nz, nz, C.c_void_p(257), C.byref(s), None) == 3  # unaligned workspace
    assert L.pco_b200_build_index_async(C.byref(p), nz, nz, C.c_void_p(264), nz, C.byref(s), None) == 3  # index not 16-byte aligned
