"""CPU-only checks of the drop-in boundary: the C-ABI library loads, exports every symbol the headers
declare, and refuses compute without a CUDA device (no CPU fallback)."""
import ctypes as C
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    syms = set()
    for h in ("cpcodec.h", "pco_b200.h"):
        text = open(os.path.join(ROOT, "include", h)).read()
        text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
        syms |= set(re.findall(r"\b(pco_[a-z0-9_]+)\s*\(", text))
    return syms


def test_library_exports_every_declared_symbol():
    from pcodec_b200 import _lib

    L = _lib.lib()
    syms = _declared_symbols()
    assert {"pco_standalone_guarantee_file_size", "pco_standalone_simple_compress_into", "pco_standalone_simple_decompress_into"} <= syms
    missing = [s for s in sorted(syms) if not hasattr(L, s)]
    assert not missing, missing


def test_guarantee_file_size_matches_reference_formula():  # pco/src/standalone/guarantee.rs:11-38
    from pcodec_b200 import _lib

    f = _lib.lib().pco_standalone_guarantee_file_size
    assert f(0, 3) == 18
    assert f(1 << 18, 2) == 17 + (4 + 150 + (1 << 21)) + 1
    assert f(10, 99) == 0
    # 2^19 + 1 numbers -> three equal pages of 174763 (chunk_config.rs:134-183); u32 baseline meta = 146 bytes
    n = (1 << 19) + 1
    assert f(n, 1) == 17 + 3 * (4 + 146 + 4 * 174763) + 1
    # 2^18 + 1 -> pages of 131073 and 131072
    assert f((1 << 18) + 1, 2) == 17 + (4 + 150 + 8 * 131073) + (4 + 150 + 8 * 131072) + 1


def test_product_never_imports_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "pcodec_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".hpp", ".h", ".cpp")):
                text = open(os.path.join(dirpath, f)).read()
                assert "pyoracle" not in text and "oracle/" not in text.replace("nothing in this\n// directory includes or links oracle/", "") or f == "codec_common.cuh" or f == "host_common.hpp", f


def test_no_gpu_means_loud_failure():
    import pytest

    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from pcodec_b200 import PcoError, standalone

    with pytest.raises(PcoError) as e:
        standalone.simple_decompress(b"pco!\x03\x00\x00\x04\x01\x00", np.uint32)
    assert e.value.kind == "Cuda"


def test_ans_path_counters_without_a_compress_are_zero():
    """pco_b200_profile_ans_paths on a thread that has compressed nothing (so also without a device): 0 rounds, every slot zeroed."""
    import threading

    from pcodec_b200 import _lib

    L = _lib.lib()
    out = {}

    def probe():
        counts = (C.c_uint * 8)(*([7] * 8))
        out["rc"] = L.pco_b200_profile_ans_paths(counts)
        out["counts"] = list(counts)

    t = threading.Thread(target=probe)  # the library's scratch and counters are per thread: a new thread has none
    t.start()
    t.join()
    assert out == {"rc": 0, "counts": [0] * 8}


def test_decompress_chunks_argument_checks_need_no_device():
    """pco_b200_decompress_chunks validates its table before touching the device: nothing to do is fine, a missing table is not."""
    import ctypes as C

    from pcodec_b200 import _lib

    L = _lib.lib()
    n_written = C.c_size_t(123)
    buf = (C.c_uint8 * 16)()
    assert L.pco_b200_decompress_chunks(buf, C.c_size_t(16), C.c_ubyte(2), None, None, C.c_size_t(0), None, C.c_size_t(0), C.byref(n_written), C.c_uint32(0), None) == 0
    assert n_written.value == 0
    rc = L.pco_b200_decompress_chunks(buf, C.c_size_t(16), C.c_ubyte(2), None, None, C.c_size_t(3), None, C.c_size_t(0), C.byref(n_written), C.c_uint32(0), None)
    assert rc == 3  # InvalidArgument
    assert L.pco_b200_decompress_chunks(buf, C.c_size_t(16), C.c_ubyte(99), None, None, C.c_size_t(0), None, C.c_size_t(0), C.byref(n_written), C.c_uint32(0), None) == 5  # InvalidType
