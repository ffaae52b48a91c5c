"""Host side of the asynchronous decompress (pco_b200_decompress_async_plan / _result) without a GPU: the plan's argument checks, its
workspace size, and how a status written by the device becomes a kind, a message and a Progress."""
import ctypes as C

import pytest

# an empty standalone file: version 3, uniform type byte, 1-byte size hint, format 4.1, terminator
HEAD = b"pco!\x03\x00\x00\x04\x01\x00"
HEAD_U64 = b"pco!\x03\x02\x00\x04\x01\x00"
U64, U32 = 2, 1


@pytest.fixture(scope="module")
def L():
    from pcodec_b200 import standalone

    return standalone._lib_async()


def _plan(L, head=HEAD, dtype=U64, src_cap=1 << 20, index_cap=1 << 16, dst_cap=1 << 18, max_chunks=16):
    from pcodec_b200 import standalone

    p = standalone._CAsyncPlan()
    buf = C.create_string_buffer(head, len(head)) if head is not None else None
    rc = L.pco_b200_decompress_async_plan(buf, C.c_size_t(len(head) if head is not None else 0), C.c_ubyte(dtype), C.c_size_t(src_cap),
                                          C.c_size_t(index_cap), C.c_size_t(dst_cap), C.c_size_t(max_chunks), C.byref(p))
    return rc, p, L.pco_b200_last_error_message().decode()


def _expected_workspace(dst_cap, max_chunks):
    """The layout include/pco_b200.h and DESIGN §7e describe, each region 256-byte aligned."""
    al = lambda x: (x + 255) // 256 * 256  # noqa: E731
    rows = 2 * (dst_cap // 256 + max_chunks + 1)  # the general pair's rows: scratch_rows_total(dst_cap, max_chunks)
    per_var = (1 << 14) * 6 + (1 << 15) * 13 + 288 * 8 + 256 * 4 + 64
    cold = 3 * per_var + 2 * (2 * (1 << 16) * 8) + 8192  # cold_scratch_bytes(16)
    check = 32 + 33 * 7 * 8  # the check results and the binomial table decode_kernel reads
    return al(check) + al(32 * max_chunks) + al(4 * max_chunks) + al(max_chunks) + al(rows * 256) + al(rows * 4) + al(cold)


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
    for mc in (0, 1 << 32):
        rc, _, msg = _plan(L, max_chunks=mc)
        assert rc == 3 and "max_chunks" in msg, msg
    rc, _, _ = _plan(L, head=None)
    assert rc == 2  # no bytes at all


def test_valid_plan_fills_the_plan(L):
    rc, p, msg = _plan(L, head=HEAD_U64, dtype=U64, src_cap=1000, index_cap=2000, dst_cap=3000, max_chunks=7)
    assert rc == (0 if L.pco_b200_device_available() else 6), msg  # Cuda without a device, after the plan is filled
    assert (p.dtype, p.uniform_type, p.format_major) == (U64, U64, 4)
    assert (p.src_cap, p.index_cap, p.dst_cap, p.max_chunks) == (1000, 2000, 3000, 7)
    assert p.workspace_bytes == _expected_workspace(3000, 7)
    rc, p, _ = _plan(L, head=HEAD, dtype=U32)
    assert p.uniform_type == 0 and p.dtype == U32


@pytest.mark.parametrize("dst_cap,max_chunks", [(0, 1), (1, 1), (255, 3), (256, 3), (1 << 20, 4), (1 << 28, 1024), (1 << 28, 4096), (12345, 1 << 20)])
def test_workspace_matches_the_layout(L, dst_cap, max_chunks):
    _, p, _ = _plan(L, dst_cap=dst_cap, max_chunks=max_chunks)
    assert p.workspace_bytes == _expected_workspace(dst_cap, max_chunks)


def test_workspace_grows_with_dst_cap_and_max_chunks(L):
    sizes = [_plan(L, dst_cap=d, max_chunks=m)[1].workspace_bytes for d, m in [(1 << 16, 8), (1 << 20, 8), (1 << 20, 64), (1 << 24, 64)]]
    assert sizes == sorted(sizes) and len(set(sizes)) == 4
    # about two bytes of symbol scratch per number of dst_cap
    a, b = sizes[1], sizes[3]
    assert 2 * ((1 << 24) - (1 << 20)) <= b - a <= 2.1 * ((1 << 24) - (1 << 20)) + (1 << 16)


def _result(L, **fields):
    from pcodec_b200 import standalone

    s = standalone._CAsyncStatus(**fields)
    prog = standalone._lib._CProgress(n_processed=12345, finished=7)
    rc = L.pco_b200_decompress_async_result(C.byref(s), C.byref(prog))
    return rc, L.pco_b200_last_error_message().decode(), (prog.n_processed, prog.finished)


def test_result_maps_statuses_to_kinds_messages_and_progress(L):
    rc, _, prog = _result(L, kind=0, n_processed=1000, finished=1, n_chunks=3)
    assert (rc, prog) == (0, (1000, 1))
    rc, _, prog = _result(L, kind=0, n_processed=77, finished=0)
    assert (rc, prog) == (0, (77, 0))
    # chunk failures: the kind, and the message names the chunk as status_to_error words it
    for kind, st, words in [(1, 1, "corrupt data"), (2, 2, "insufficient data"), (3, 3, "invalid argument"), (7, 7, "valid pco outside")]:
        rc, msg, prog = _result(L, kind=kind, device_status=st, chunk=17)
        assert rc == kind and msg.startswith("chunk 17: ") and words in msg, msg
        assert prog == (12345, 7)  # Progress is left alone on an error
    # file-level refusals
    cases = [(0x101, 1, "corrupt standalone header"), (0x102, 2, "insufficient data"), (0x103, 3, "differs from the plan"),
             (0x104, 3, "does not belong"), (0x105, 3, "max_chunks")]
    for st, kind, words in cases:
        rc, msg, _ = _result(L, kind=kind, device_status=st, chunk=(1 << 64) - 1, n_chunks=0)
        assert rc == kind and words in msg, msg
    # a kind the library does not know reads as Corruption
    rc, _, _ = _result(L, kind=99, device_status=1, chunk=0)
    assert rc == 1
    assert L.pco_b200_decompress_async_result(None, None) == 3


def test_call_refuses_missing_buffers_without_a_device(L):
    from pcodec_b200 import standalone

    _, p, _ = _plan(L)
    s = standalone._CAsyncStatus()
    nz = C.c_void_p(256)  # never dereferenced: the call refuses first
    assert L.pco_b200_decompress_async(None, nz, nz, nz, nz, C.byref(s), None) == 3
    assert L.pco_b200_decompress_async(C.byref(p), None, nz, nz, nz, C.byref(s), None) == 3
    assert L.pco_b200_decompress_async(C.byref(p), nz, nz, nz, None, C.byref(s), None) == 3
    bad = standalone._CAsyncPlan.from_buffer_copy(bytes(p))
    bad.workspace_bytes += 1  # not what the plan computed
    assert L.pco_b200_decompress_async(C.byref(bad), nz, nz, nz, nz, C.byref(s), None) == 3
    assert L.pco_b200_decompress_async(C.byref(p), nz, nz, nz, C.c_void_p(257), C.byref(s), None) == 3  # unaligned workspace
