"""pco_b200_decompress_pages / pco_b200_compress_wrapped refuse bad arguments before any device work, so these run without a GPU."""
import ctypes as C

import numpy as np
import pytest

OK, INVALID_ARGUMENT, INVALID_TYPE, CUDA = 0, 3, 5, 6


@pytest.fixture(scope="module")
def L():
    from pcodec_b200 import wrapped

    return wrapped._lib_batch()


def _refs(*rows):
    from pcodec_b200 import wrapped

    return np.array(list(rows), dtype=wrapped.PAGE_REF)


def _decompress(L, refs, metas_len=100, pages_len=1000, dtype=2, dst_len=None, null_refs=False):
    metas = np.zeros(max(metas_len, 1), dtype=np.uint8)
    pages = np.zeros(max(pages_len, 1), dtype=np.uint8)
    n_pages = len(refs)
    total = int(refs["page_n"].sum()) if n_pages else 0
    dst = np.zeros(max(total if dst_len is None else dst_len, 1), dtype=np.uint64)
    nw = C.c_size_t(12345)
    rc = L.pco_b200_decompress_pages(metas.ctypes.data_as(C.c_void_p), C.c_size_t(metas_len), pages.ctypes.data_as(C.c_void_p), C.c_size_t(pages_len),
                                     C.c_ubyte(dtype), None if null_refs else refs.ctypes.data_as(C.c_void_p), C.c_size_t(n_pages),
                                     dst.ctypes.data_as(C.c_void_p), C.c_size_t(total if dst_len is None else dst_len), C.byref(nw), C.c_uint32(0), None)
    return rc, nw.value


def _message(L):
    from pcodec_b200 import _lib

    return _lib.lib().pco_b200_last_error_message().decode()


def test_no_pages_is_ok(L):
    rc, nw = _decompress(L, _refs())
    assert rc == OK and nw == 0
    rc, nw = _decompress(L, _refs(), null_refs=True)
    assert rc == OK and nw == 0


def test_null_refs(L):
    rc, _ = _decompress(L, _refs((0, 10, 0, 100, 256)), null_refs=True)
    assert rc == INVALID_ARGUMENT


@pytest.mark.parametrize("row", [
    (95, 10, 0, 100, 256),               # meta runs past the end of metas
    (100, 1, 0, 100, 256),               # meta starts at the end
    (2**64 - 5, 10, 0, 100, 256),        # offset + length wraps around
    (0, 101, 0, 100, 256),               # meta longer than metas
    (0, 10, 900, 101, 256),              # page runs past the end of pages
    (0, 10, 2**64 - 1, 2, 256),          # wraps around
    (0, 10, 0, 1001, 256),               # page longer than pages
])
def test_ranges_outside_their_buffer(L, row):
    rc, _ = _decompress(L, _refs((0, 10, 0, 100, 256), row))
    assert rc == INVALID_ARGUMENT
    assert _message(L).startswith("page 1: ")


@pytest.mark.parametrize("page_n", [0, (1 << 24) + 1, 2**63])
def test_page_n_out_of_range(L, page_n):
    refs = _refs((0, 10, 0, 100, page_n))
    rc, _ = _decompress(L, refs, dst_len=1 << 10)
    assert rc == INVALID_ARGUMENT


def test_destination_too_small(L):
    refs = _refs((0, 10, 0, 100, 300), (0, 10, 100, 100, 300))
    rc, _ = _decompress(L, refs, dst_len=599)
    assert rc == INVALID_ARGUMENT
    assert "dst holds 599" in _message(L)


@pytest.mark.parametrize("dtype", [0, 12, 255])
def test_unknown_dtype(L, dtype):
    rc, _ = _decompress(L, _refs((0, 10, 0, 100, 256)), dtype=dtype)
    assert rc == INVALID_TYPE


def test_arguments_checked_before_the_device(L):
    """Valid arguments reach the device; without one the call reports the missing device and nothing else."""
    from pcodec_b200 import _lib

    if _lib.lib().pco_b200_device_available():
        pytest.skip("a CUDA device is present")
    rc, _ = _decompress(L, _refs((0, 10, 0, 100, 256), (0, 10, 100, 900, 1 << 24)))
    assert rc == CUDA


def test_compress_wrapped_unknown_dtype(L):
    nums = np.arange(10, dtype=np.uint64)
    ml, pl, nc = C.c_size_t(), C.c_size_t(), C.c_size_t()
    rc = L.pco_b200_compress_wrapped(nums.ctypes.data_as(C.c_void_p), C.c_size_t(10), C.c_ubyte(0), None, None, C.c_size_t(0), C.byref(ml),
                                     None, C.c_size_t(0), C.byref(pl), None, C.c_size_t(0), C.byref(nc), C.c_uint32(0), None)
    assert rc == INVALID_TYPE


def test_python_wrapper_reports_argument_errors():
    from pcodec_b200 import PcoError, wrapped

    with pytest.raises(PcoError) as e:
        wrapped.decompress_pages(b"\0" * 8, b"\0" * 8, _refs((4, 8, 0, 8, 10)), np.uint32)
    assert e.value.kind == "InvalidArgument" and "page 0" in e.value.message
    with pytest.raises(PcoError) as e:
        wrapped.decompress_pages(b"\0" * 8, b"\0" * 8, _refs((0, 8, 0, 8, 0)), np.uint32)
    assert e.value.kind == "InvalidArgument"
    assert wrapped.decompress_pages(b"", b"", _refs(), np.float32).size == 0
