"""GPU parity tests aimed at the narrow class of fused_narrow_kernel (pcodec_b200/csrc/decode_fused.cuh): the lean decode
for classic-mode chunks with consecutive delta order 0 / 1, bin lowers within 2^16 of the first bin and offsets of
<= 15 bits.  Streams come from the oracle; the GPU decode must equal the original numbers and the oracle's decode
bit for bit, and pco_b200_profile_chunk_classes must show that the narrow kernel (class 3 / 4) really served them -
or, for the boundary cases built to miss a condition, that it did not.
"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DTYPES = [np.uint32, np.int32, np.float32, np.uint64, np.int64, np.float64]


@pytest.fixture(scope="module")
def sa():
    from pcodec_b200 import standalone

    return standalone


def _classes():
    from pcodec_b200 import _lib

    counts = (C.c_uint * 8)()
    n = _lib.lib().pco_b200_profile_chunk_classes(counts)
    return n, list(counts)


def _narrow_data(dtype, n, seed, order):
    """Numbers whose order-`order` latents are a small multi-bin distribution around a (possibly negative) centre."""
    rng = np.random.default_rng(seed)
    if seed == 2:  # a cluster of 2^15 values (15-bit offsets, the widest the narrow kernel takes) and a tight one 60000 above
        pick = rng.integers(0, 2, size=n).astype(np.int64)
        steps = np.where(pick == 0, rng.integers(0, 1 << 15, size=n), 60000 + rng.integers(0, 1 << 10, size=n)).astype(np.int64) - 30000
    else:
        steps = rng.geometric(0.002 if seed < 2 else 0.0004, size=n).astype(np.int64) - (250 if seed % 2 else 0)  # odd seeds: both signs
    vals = np.cumsum(steps) if order == 1 else steps + 100000
    dt = np.dtype(dtype)
    if dt.kind == "f":
        # consecutive floats: ordered latents differ by the integer steps
        u = np.dtype(f"u{dt.itemsize}")
        mid = 1 << (8 * dt.itemsize - 1)
        lat = (vals.astype(np.uint64) + np.uint64(mid) + np.uint64(5000000)).astype(u)  # wraps like the latent arithmetic
        bits = np.where(lat & u.type(mid), lat ^ u.type(mid), ~lat)
        return bits.astype(u).view(dtype)
    return vals.astype(np.uint64).astype(np.dtype(f"u{dt.itemsize}")).view(dtype)


def _cfg(oracle, order, max_page_n=1 << 18):
    if order == 0:
        return oracle.make_config(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_NOOP, max_page_n=max_page_n)
    return oracle.make_config(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_CONSECUTIVE, delta_order=order, max_page_n=max_page_n)


def _bits(a):
    return a.view(np.dtype(f"u{a.dtype.itemsize}"))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("order", [0, 1])
@pytest.mark.parametrize("n", [1, 2, 255, 256, 257, 513, 5000, 3 * 4096 + 1])
def test_narrow_chunks_vs_oracle(sa, oracle, dtype, order, n):
    for seed in (0, 1, 2, 3):
        nums = _narrow_data(dtype, n, seed, order)
        data = oracle.simple_compress(nums, _cfg(oracle, order, max_page_n=4096))
        got = sa.simple_decompress(data, dtype)
        assert np.array_equal(_bits(got), _bits(nums)), (dtype, order, n, seed)
        assert np.array_equal(_bits(got), _bits(oracle.simple_decompress(data, dtype)))


@pytest.mark.parametrize("dtype", [np.uint64, np.int32, np.float64])
@pytest.mark.parametrize("order", [0, 1])
def test_narrow_kernel_is_the_one_that_runs(sa, oracle, dtype, order, monkeypatch):
    # the class counters describe the LAST decode launch: the speculative walk decodes runs of same-sized chunks launch by launch (five
    # chunks of 7033 numbers, then two of 7032), the serial walk hands all seven chunks over at once
    monkeypatch.setenv("PCOB200_SPECULATIVE_WALK", "0")
    nums = _narrow_data(dtype, 6 * 8192 + 77, 1, order)
    data = oracle.simple_compress(nums, _cfg(oracle, order, max_page_n=8192))
    got = sa.simple_decompress(data, dtype)
    assert np.array_equal(_bits(got), _bits(nums))
    n_chunks, counts = _classes()
    assert n_chunks == 7
    assert counts[4 if order == 1 else 3] == 7, counts


def test_full_size_chunks_take_the_narrow_path(sa, oracle):
    from pcodec_b200 import datagen

    nums = np.concatenate([datagen.c2_u64_cumsum_geometric(seed=s) for s in (11, 12, 13)])
    data = oracle.simple_compress(nums, _cfg(oracle, 1))
    got = sa.simple_decompress(data, np.uint64)
    assert np.array_equal(got, nums)
    n_chunks, counts = _classes()
    assert n_chunks == 3 and counts[4] == 3, counts


def test_conditions_that_must_miss_the_narrow_path(sa, oracle):
    rng = np.random.default_rng(5)
    # offsets of 16+ bits: two far-apart clusters of 2^17 distinct values each -> wide bins
    wide = rng.integers(0, 1 << 20, size=20000).astype(np.uint64)
    # lowers spread over more than 2^16: many tight clusters 2^20 apart
    spread = (rng.integers(0, 64, size=20000).astype(np.uint64) << np.uint64(20)) + rng.integers(0, 4, size=20000).astype(np.uint64)
    for nums in (wide, spread):
        data = oracle.simple_compress(nums, _cfg(oracle, 0))
        got = sa.simple_decompress(data, np.uint64)
        assert np.array_equal(got, nums)
        n_chunks, counts = _classes()
        assert n_chunks == 1 and counts[1] == 1, counts
    # delta orders 2..7 are served by the fused kernel too (class 5)
    for order in (2, 3, 7):
        steps = rng.geometric(0.002, size=9000).astype(np.int64)  # the order-th differences: a small multi-bin distribution
        vals = steps
        for _ in range(order):
            vals = np.cumsum(vals)
        nums = vals.astype(np.uint64)  # wraps like the latent arithmetic
        data = oracle.simple_compress(nums, _cfg(oracle, order))
        assert np.array_equal(sa.simple_decompress(data, np.uint64), nums)
        n_chunks, counts = _classes()
        assert n_chunks == 1 and counts[5] == 1, (order, counts)
    # 16-bit (and 8-bit) types are served by the fused kernel as well
    nums16 = (np.cumsum(rng.integers(0, 5, size=9000)) % 60000).astype(np.uint16)
    data = oracle.simple_compress(nums16, _cfg(oracle, 1))
    assert np.array_equal(sa.simple_decompress(data, np.uint16), nums16)
    assert _classes()[1][4] == 1


def test_mixed_classes_in_one_file(sa, oracle):
    """Chunks of different classes in one file: each is decoded by exactly one kernel."""
    rng = np.random.default_rng(9)
    parts = [_narrow_data(np.uint64, 4096, 0, 0), rng.integers(0, 1 << 62, size=4096).astype(np.uint64),
             np.full(4096, 7, dtype=np.uint64), _narrow_data(np.uint64, 4096, 1, 0) + np.uint64(1 << 40)]
    nums = np.concatenate(parts)
    data = oracle.simple_compress(nums, _cfg(oracle, 0, max_page_n=4096))
    got = sa.simple_decompress(data, np.uint64)
    assert np.array_equal(got, nums)
    n_chunks, counts = _classes()
    assert n_chunks == 4 and counts[3] == 2 and counts[1] == 2, counts


def test_partial_destination_and_odd_offsets_on_the_narrow_path(sa, oracle):  # pco/src/standalone/simple.rs:100-143
    nums = _narrow_data(np.uint64, 3 * 1000 + 3, 1, 1)  # chunks of 1001: later chunks start at odd element offsets
    data = oracle.simple_compress(nums, _cfg(oracle, 1, max_page_n=1001))
    got = sa.simple_decompress(data, np.uint64)
    assert np.array_equal(got, nums)
    assert _classes()[1][4] == 3
    for m in (0, 1, 255, 256, 257, 1000, 1001, 1002, 1500, 2999):
        dst = np.zeros(m, dtype=np.uint64)
        prog = sa.simple_decompress_into(data, dst)
        want = np.zeros(m, dtype=np.uint64)
        oprog = oracle.simple_decompress_into(data, want)
        assert prog.n_processed == oprog[0] and bool(prog.finished) == bool(oprog[1]), (m, prog, oprog)
        assert np.array_equal(dst[: prog.n_processed], want[: prog.n_processed]), m
