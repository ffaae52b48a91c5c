"""Index-free decompress (what pco_standalone_simple_decompress_into receives: no side index, no chunk offsets) finds runs of
same-sized chunks by their first 4 bytes, walks every candidate in parallel and follows the chain of verified (start, end) pairs
(host_api.cu walk_index_free and speculative_walk_rounds, the walker pco_b200_decompress_files shares; files_kernels.cuh
find_file_starts_kernel).  The numbers must be the oracle's whatever the candidates look like: coincidences inside chunk bodies, chunks
of changing sizes, short last chunks, short destinations, corrupt and truncated files (reference semantics:
pco/src/standalone/simple.rs:100-143, decompressor.rs:150-215)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from oracle import pyoracle as oracle  # noqa: E402
from pcodec_b200 import PcoError, _lib, standalone  # noqa: E402


def _abi3_decompress(data, dtype, n):
    """the reference's own entry point, unmodified (pco_c/include/cpcodec_generated.h:54-64)"""
    L = _lib.lib()
    src = np.frombuffer(data, dtype=np.uint8)
    dst = np.zeros(n, dtype=dtype)
    nd = C.c_size_t()
    rc = L.pco_standalone_simple_decompress_into(src.ctypes.data_as(C.c_void_p), C.c_size_t(src.size), C.c_ubyte(_lib.dtype_byte(dtype)), dst.ctypes.data_as(C.c_void_p),
                                                 C.c_size_t(n), C.byref(nd))
    assert rc == 0, rc
    assert nd.value == n
    return dst


def _planted_file(n0=4096, k=6):
    """Incompressible u64 chunks (one 64-bit-offset bin with lower 0: the numbers sit in the page byte for byte) with numbers whose low
    bytes spell a chunk start of this very file - type byte 2, count - 1 - planted all over them."""
    rng = np.random.default_rng(1)
    x = rng.integers(0, 1 << 63, size=n0 * k, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=n0 * k, dtype=np.uint64)
    pat = np.uint64(((n0 - 1) << 8) | 2)
    for i in range(100, n0 * k, 997):
        x[i] = (x[i] & np.uint64(0xFFFFFFFF00000000)) | pat
    x[::n0] = 0
    data = oracle.simple_compress(x, oracle.make_config(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_NOOP, max_page_n=n0))
    needle = bytes([2]) + int(n0 - 1).to_bytes(3, "little")
    hits = []
    i = data.find(needle)
    while i >= 0:
        hits.append(i)
        i = data.find(needle, i + 1)
    starts = [c["chunk_start"] for c in oracle.inspect(data, np.uint64)["chunks"]]
    assert len(starts) == k and set(starts) <= set(hits) and len(hits) >= len(starts) + 10, "the fixture lost its false chunk starts"
    return x, data


def test_coincidences_inside_chunk_bodies_are_never_taken_for_chunks():
    x, data = _planted_file()
    assert np.array_equal(standalone.simple_decompress(data, np.uint64), x)
    assert np.array_equal(_abi3_decompress(data, np.uint64, x.size), x)


def test_planted_file_with_device_resident_buffers():
    x, data = _planted_file()
    L = _lib.lib()
    dev = torch.device("cuda")
    d_src = torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).to(dev)
    d_out = torch.zeros(x.size, dtype=torch.int64, device=dev)
    prog = _lib._CProgress()
    _lib.check(L.pco_b200_decompress_ex(C.c_void_p(d_src.data_ptr()), C.c_size_t(d_src.numel()), C.c_ubyte(2), C.c_void_p(d_out.data_ptr()), C.c_size_t(x.size), C.byref(prog),
                                        None, C.c_size_t(0), C.c_uint32(3), None))
    assert prog.n_processed == x.size and prog.finished
    assert np.array_equal(d_out.cpu().numpy().view(np.uint64), x)


@pytest.mark.parametrize("dtype,n,page_n,order", [(np.uint64, 10 * 4096 + 123, 4096, 1), (np.uint32, 37 * 1000 + 1, 1000, 0), (np.int64, 3 * (1 << 16) + 5, 1 << 16, 2),
                                                   (np.float32, 20 * 512 + 7, 512, 0), (np.uint16, 9 * 3000 + 2999, 3000, 1)])
def test_runs_of_equal_chunks_and_a_short_last_chunk(dtype, n, page_n, order):
    rng = np.random.default_rng(3)
    if np.dtype(dtype).kind == "f":
        x = np.cumsum(rng.normal(size=n)).astype(dtype)
    else:
        x = (np.cumsum(rng.geometric(0.05, size=n)) % (1 << min(62, 8 * np.dtype(dtype).itemsize - 1))).astype(dtype)
    cfg = oracle.make_config(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_CONSECUTIVE if order else oracle.DELTA_NOOP, delta_order=order, max_page_n=page_n)
    data = oracle.simple_compress(x, cfg)
    got = standalone.simple_decompress(data, dtype)
    assert np.array_equal(got.view(np.uint8), x.view(np.uint8))
    assert np.array_equal(_abi3_decompress(data, dtype, n).view(np.uint8), x.view(np.uint8))


def test_chunk_sizes_that_change_from_chunk_to_chunk():
    rng = np.random.default_rng(4)
    sizes = [700, 700, 300, 700, 1, 300, 300, 2000, 700, 700, 700, 5]
    x = np.cumsum(rng.geometric(0.01, size=sum(sizes))).astype(np.uint64)
    data = oracle.simple_compress(x, oracle.make_config(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_CONSECUTIVE, delta_order=1, exact_pages=sizes))
    assert len(oracle.inspect(data, np.uint64)["chunks"]) == len(sizes)
    assert np.array_equal(standalone.simple_decompress(data, np.uint64), x)


def test_two_latent_var_chunks_and_float_mult():
    rng = np.random.default_rng(5)
    x = (np.round(rng.normal(size=12 * 2048 + 100) * 1000) * 0.01).astype(np.float64)
    data = oracle.simple_compress(x, oracle.make_config(mode=oracle.MODE_FLOAT_MULT, float_mult_base=0.01, delta=oracle.DELTA_NOOP, max_page_n=2048))
    assert np.array_equal(standalone.simple_decompress(data, np.float64).view(np.uint64), x.view(np.uint64))


@pytest.mark.parametrize("short", [1, 4096, 4096 + 17, 5 * 4096])
def test_destination_shorter_than_the_file(short):
    """Progress semantics of simple_decompress_into (standalone/simple.rs:115-140): the numbers that fit, finished = False"""
    rng = np.random.default_rng(6)
    n = 8 * 4096 + 50
    x = np.cumsum(rng.geometric(0.01, size=n)).astype(np.uint64)
    data = oracle.simple_compress(x, oracle.make_config(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_CONSECUTIVE, delta_order=1, max_page_n=4096))
    dst = np.zeros(n - short + 8, dtype=np.uint64)
    prog = standalone.simple_decompress_into(data, dst[: n - short])
    assert prog.n_processed == n - short and not prog.finished
    assert np.array_equal(dst[: n - short], x[: n - short]) and not dst[n - short :].any()
    # and a destination longer than the file
    big = np.zeros(n + 100, dtype=np.uint64)
    prog = standalone.simple_decompress_into(data, big)
    assert prog.n_processed == n and prog.finished and np.array_equal(big[:n], x)


def test_corrupt_and_truncated_files_fail_like_the_serial_walk():
    rng = np.random.default_rng(7)
    n = 9 * 2048
    x = np.cumsum(rng.geometric(0.01, size=n)).astype(np.uint64)
    data = oracle.simple_compress(x, oracle.make_config(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_CONSECUTIVE, delta_order=1, max_page_n=2048))
    starts = [c["chunk_start"] for c in oracle.inspect(data, np.uint64)["chunks"]]
    # the type byte of chunk 4 destroyed: the chain stops in front of it and the serial walker names the problem
    bad = bytearray(data)
    bad[starts[4]] = 0x37
    with pytest.raises(PcoError) as e:
        standalone.simple_decompress(bytes(bad), np.uint64)
    assert e.value.kind in ("Corruption", "InvalidType", "InvalidArgument")
    # the count of chunk 4 changed: another pattern, its walk fails or lands nowhere
    bad = bytearray(data)
    bad[starts[4] + 1] ^= 0x10
    with pytest.raises(PcoError):
        standalone.simple_decompress(bytes(bad), np.uint64)
    # cut inside chunk 6
    cut = data[: (starts[6] + starts[7]) // 2]
    with pytest.raises(PcoError) as e:
        standalone.simple_decompress(cut, np.uint64)
    assert e.value.kind == "InsufficientData"
    # cut exactly behind chunk 5: no terminator
    with pytest.raises(PcoError) as e:
        standalone.simple_decompress(data[: starts[6]], np.uint64)
    assert e.value.kind == "InsufficientData"


@pytest.mark.parametrize("speculative", [None, "0"])
def test_chunks_before_a_failing_chunk_reach_a_device_destination(monkeypatch, speculative):
    """The call fails at a corrupt chunk, and a device destination holds the numbers of the chunks in front of it, as the reference's
    decoder emits them - with the speculative rounds and with the serial walk alone."""
    if speculative is None:
        monkeypatch.delenv("PCOB200_SPECULATIVE_WALK", raising=False)
    else:
        monkeypatch.setenv("PCOB200_SPECULATIVE_WALK", speculative)
    rng = np.random.default_rng(7)
    page_n = 2048
    n = 9 * page_n
    x = np.cumsum(rng.geometric(0.01, size=n)).astype(np.uint64)
    data = oracle.simple_compress(x, oracle.make_config(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_CONSECUTIVE, delta_order=1, max_page_n=page_n))
    starts = [c["chunk_start"] for c in oracle.inspect(data, np.uint64)["chunks"]]
    bad = bytearray(data)
    bad[starts[4]] = 0x37
    L = _lib.lib()
    dev = torch.device("cuda")
    d_src = torch.from_numpy(np.frombuffer(bytes(bad), dtype=np.uint8).copy()).to(dev)
    d_out = torch.zeros(n, dtype=torch.int64, device=dev)
    prog = _lib._CProgress()
    rc = L.pco_b200_decompress_ex(C.c_void_p(d_src.data_ptr()), C.c_size_t(d_src.numel()), C.c_ubyte(2), C.c_void_p(d_out.data_ptr()), C.c_size_t(n), C.byref(prog),
                                  None, C.c_size_t(0), C.c_uint32(3), None)
    with pytest.raises(PcoError) as e:
        _lib.check(rc)
    assert e.value.kind in ("Corruption", "InvalidType", "InvalidArgument")
    assert np.array_equal(d_out.cpu().numpy().view(np.uint64)[: 4 * page_n], x[: 4 * page_n])


def test_many_chunks_in_one_call():
    """more chunks than one wave of walkers, through the reference's three-function ABI"""
    rng = np.random.default_rng(8)
    n = 3000 * 256 + 3
    x = np.cumsum(rng.geometric(0.02, size=n)).astype(np.uint32)
    data = oracle.simple_compress(x, oracle.make_config(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_CONSECUTIVE, delta_order=1, max_page_n=256))
    assert np.array_equal(_abi3_decompress(data, np.uint32, n), x)


def test_the_serial_walk_alone_gives_the_same_numbers(monkeypatch):
    """PCOB200_SPECULATIVE_WALK=0: chunk after chunk, as before - the path that still owns the tail of every file and every error"""
    monkeypatch.setenv("PCOB200_SPECULATIVE_WALK", "0")
    x, data = _planted_file()
    assert np.array_equal(standalone.simple_decompress(data, np.uint64), x)
    rng = np.random.default_rng(11)
    y = np.cumsum(rng.geometric(0.01, size=5 * 2048 + 3)).astype(np.uint64)
    ydata = oracle.simple_compress(y, oracle.make_config(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_CONSECUTIVE, delta_order=1, max_page_n=2048))
    assert np.array_equal(_abi3_decompress(ydata, np.uint64, y.size), y)
