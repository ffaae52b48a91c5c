"""pco_b200_compress_files / pco_b200_decompress_files refuse bad arguments before any device work, so these run without a GPU."""
import ctypes as C

import numpy as np
import pytest

OK, INVALID_ARGUMENT, IO, INVALID_TYPE, CUDA, UNSUPPORTED = 0, 3, 4, 5, 6, 7


@pytest.fixture(scope="module")
def L():
    from pcodec_b200 import standalone

    return standalone._lib_files()


def _files(*rows):
    from pcodec_b200 import standalone

    return np.array(list(rows), dtype=standalone.FILE_REF)


def _decompress(L, files, src_len=1000, index_len=0, dtype=2, dst_len=1 << 16, null_files=False):
    src = np.zeros(max(src_len, 1), dtype=np.uint8)
    index = np.zeros(max(index_len, 1), dtype=np.uint8)
    dst = np.zeros(max(dst_len, 1), dtype=np.uint64)
    ns = np.zeros(max(len(files), 1), dtype=np.uint64)
    nw = C.c_size_t(12345)
    rc = L.pco_b200_decompress_files(src.ctypes.data_as(C.c_void_p), C.c_size_t(src_len), index.ctypes.data_as(C.c_void_p) if index_len else None,
                                     C.c_size_t(index_len), C.c_ubyte(dtype), None if null_files else files.ctypes.data_as(C.c_void_p),
                                     C.c_size_t(len(files)), dst.ctypes.data_as(C.c_void_p), C.c_size_t(dst_len), ns.ctypes.data_as(C.c_void_p), C.byref(nw),
                                     C.c_uint32(0), None)
    return rc, nw.value


def _compress(L, file_ns, dtype=2, config=None, flags=0, null_files=False):
    from pcodec_b200 import standalone

    ns = np.ascontiguousarray(file_ns, dtype=np.uint64)
    nums = np.zeros(max(int(ns.sum()), 1), dtype=np.uint64)
    dst = np.zeros(1 << 16, dtype=np.uint8)
    files = np.zeros(max(len(ns), 1), dtype=standalone.FILE_REF)
    cfg = C.byref(config._to_c()) if config is not None else None
    return L.pco_b200_compress_files(nums.ctypes.data_as(C.c_void_p), ns.ctypes.data_as(C.c_void_p), C.c_size_t(len(ns)), C.c_ubyte(dtype), cfg, C.c_int(0),
                                     dst.ctypes.data_as(C.c_void_p), C.c_size_t(dst.size), None, C.c_size_t(0),
                                     None if null_files else files.ctypes.data_as(C.c_void_p), C.c_uint32(flags), None)


def _message():
    from pcodec_b200 import _lib

    return _lib.lib().pco_b200_last_error_message().decode()


def test_no_files_is_ok(L):
    assert _decompress(L, _files()) == (OK, 0)
    assert _decompress(L, _files(), null_files=True) == (OK, 0)
    assert _compress(L, []) == OK


def test_null_files(L):
    rc, _ = _decompress(L, _files((0, 10, 0, 0)), null_files=True)
    assert rc == INVALID_ARGUMENT
    assert _compress(L, [5], null_files=True) == INVALID_ARGUMENT


@pytest.mark.parametrize("row", [
    (995, 10, 0, 0),             # the file runs past the end of src
    (1000, 1, 0, 0),             # starts at the end
    (2**64 - 5, 10, 0, 0),       # offset + length wraps around
    (0, 1001, 0, 0),             # longer than src
    (0, 10, 16, 100),            # the index runs past the end of index
    (0, 10, 2**64 - 16, 32),     # wraps around
    (0, 10, 8, 64),              # index offset not a multiple of 16
    (0, 10, 1, 1),               # the same, however short
])
def test_ranges_outside_their_buffer(L, row):
    rc, _ = _decompress(L, _files((0, 10, 0, 0), row), index_len=100)
    assert rc == INVALID_ARGUMENT
    assert _message().startswith("file 1: ")


@pytest.mark.parametrize("dtype", [0, 12, 255])
def test_unknown_dtype(L, dtype):
    rc, _ = _decompress(L, _files((0, 10, 0, 0)), dtype=dtype)
    assert rc == INVALID_TYPE
    assert _compress(L, [5], dtype=dtype) == INVALID_TYPE


def test_chunks_only_is_refused(L):
    assert _compress(L, [5, 6], flags=8) == INVALID_ARGUMENT
    assert "CHUNKS_ONLY" in _message()


@pytest.mark.parametrize("level,kind", [(13, INVALID_ARGUMENT)])
def test_config_refusal_names_the_first_file(L, level, kind):
    from pcodec_b200 import ChunkConfig

    assert _compress(L, [5, 6], config=ChunkConfig(compression_level=level)) == kind
    assert _message().startswith("file 0: ")


def test_explicit_config_refusal_names_its_file(L):
    """With explicit specs a file's refusal is known on the host, whatever the files in front of it."""
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec

    cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.no_op(), paging_spec=PagingSpec.exact_page_sizes([3, 4]))
    assert _compress(L, [7, 7, 8, 7], config=cfg) == INVALID_ARGUMENT
    assert _message().startswith("file 2: ")
    for delta in (DeltaSpec.try_lookback(), DeltaSpec.try_conv1(2)):
        assert _compress(L, [7], config=ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=delta)) == UNSUPPORTED
        assert _message().startswith("file 0: ")
    assert _compress(L, [7], config=ChunkConfig(mode_spec=ModeSpec.try_dict(), delta_spec=DeltaSpec.no_op())) == UNSUPPORTED


def test_auto_file_whose_chunks_disagree_is_refused(L):
    """compress_ex refuses Auto over chunks of one array whose sizes imply different unoptimized_bins_log; so does the batch, for that file."""
    from pcodec_b200 import ChunkConfig, PagingSpec

    cfg = ChunkConfig(paging_spec=PagingSpec.exact_page_sizes([100, 5000]))
    assert _compress(L, [5100], config=cfg) == UNSUPPORTED
    assert _message().startswith("file 0: ")


def test_arguments_checked_before_the_device(L):
    """Valid arguments reach the device; without one the calls report the missing device and nothing else."""
    from pcodec_b200 import _lib

    if _lib.lib().pco_b200_device_available():
        pytest.skip("a CUDA device is present")
    rc, _ = _decompress(L, _files((0, 10, 0, 0), (10, 990, 0, 64)), index_len=100)
    assert rc == CUDA
    assert _compress(L, [5, 0, 6]) == CUDA


def test_python_wrappers_report_argument_errors():
    from pcodec_b200 import PcoError, standalone

    with pytest.raises(PcoError) as e:
        standalone.decompress_files(b"\0" * 8, _files((4, 8, 0, 0)), np.uint32)
    assert e.value.kind == "InvalidArgument" and "file 0" in e.value.message
    with pytest.raises(ValueError):
        standalone.compress_files(np.zeros(5, np.uint32), [3, 3])
    vals, ns = standalone.decompress_files(b"", _files(), np.float32)
    assert vals.size == 0 and ns.size == 0
