"""Chunks of more than 2^18 numbers, up to the format's limit of 2^24 (pco/src/constants.rs MAX_ENTRIES), on the GPU.

The default PagingSpec cuts chunks of 2^18, but a caller may ask for up to 2^24 numbers per chunk, and above 2^18 the device code
takes branches that 2^18-number chunks never reach:
* ans_encode_kernel cuts a page into segments of at most 16 batches and resolves them in rounds of 64 segments, so pages of more than
  2^18 numbers take several rounds: the carry from one round to the next, partial last rounds, rounds whose only segment is the one
  that knows its input, and the in-order pass called from a later round;
* plan_solve_kernel computes bin indices by a 64-bit division once a var stores more than 2^20 latents;
* the decode kernels walk and decode more than 1024 batches per chunk, and the front end streams up to 2^24 numbers per CTA.

Every file is compared with the oracle's bytes, and every GPU decode with the input and with the oracle's decode, bit for bit.  The
tANS round counters (pco_b200_profile_ans_paths) show which way each round of a page was resolved.
"""
import ctypes as C

import numpy as np
import pytest

from pcodec_b200 import datagen
from tests.golden_generators import bits_view

pytestmark = pytest.mark.gpu

K18, K20, K24 = 1 << 18, 1 << 20, 1 << 24
# slots of pco_b200_profile_ans_paths: rounds by resolution; the same + 4 counts the rounds after a page's first
SPECULATION, FIXUP, TRANSFER, IN_ORDER, LATER = 0, 1, 2, 3, 4
# fast decode kernels take tables of up to 2^10 states and 256 bins; anything larger decodes through cold_decode_kernel (one thread)
FAST_SIZE_LOG, FAST_BINS = 10, 256


@pytest.fixture(scope="module")
def sa():
    from pcodec_b200 import _lib, standalone

    yield standalone
    # the grow-only scratch of 2^24-number chunks runs to several GB: give it back before the next module
    _lib.lib().pco_b200_thread_release()


def _cfgs(oracle, n_page=None, exact=None, level=8, mode="classic", order=0, base=0.01, ibase=7, k=30, auto=False):
    """(ChunkConfig, oracle config) for the same settings.  `order` is a consecutive delta order (0 = NoOp)."""
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec

    ps = PagingSpec.exact_page_sizes(exact) if exact else PagingSpec.equal_pages_up_to(n_page)
    if auto:
        return (ChunkConfig(paging_spec=ps),
                oracle.make_config(mode=oracle.MODE_AUTO, delta=oracle.DELTA_AUTO, max_page_n=0 if exact else n_page, exact_pages=exact))
    ms = {"classic": ModeSpec.classic(), "float_mult": ModeSpec.try_float_mult(base), "int_mult": ModeSpec.try_int_mult(ibase),
          "float_quant": ModeSpec.try_float_quant(k)}[mode]
    om = {"classic": oracle.MODE_CLASSIC, "float_mult": oracle.MODE_FLOAT_MULT, "int_mult": oracle.MODE_INT_MULT, "float_quant": oracle.MODE_FLOAT_QUANT}[mode]
    ours = ChunkConfig(compression_level=level, mode_spec=ms, delta_spec=DeltaSpec.try_consecutive(order), paging_spec=ps)
    theirs = oracle.make_config(level=level, mode=om, delta=oracle.DELTA_CONSECUTIVE, delta_order=order, float_mult_base=base, int_mult_base=ibase,
                                float_quant_k=k, max_page_n=0 if exact else n_page, exact_pages=exact)
    return ours, theirs


def _first_diff(a, b):
    m = min(len(a), len(b))
    d = np.flatnonzero(np.frombuffer(a[:m], np.uint8) != np.frombuffer(b[:m], np.uint8))
    return int(d[0]) if d.size else m


def _fast_decodable(oracle, data, dtype):
    """True when every var of every chunk fits the fast decode kernels (no cold_decode_kernel)."""
    for ch in oracle.inspect(data, dtype)["chunks"]:
        for v in ch["vars"]:
            if v.get("ans_size_log", 0) > FAST_SIZE_LOG or len(v.get("bins", [])) > FAST_BINS:
                return False
    return True


def _check(sa, oracle, nums, ours, theirs, gpu_decode=True):
    """GPU bytes == oracle bytes; GPU decode == input == oracle decode.  Returns the file."""
    want = oracle.simple_compress(nums, theirs)
    got = sa.simple_compress(nums, ours)
    assert got == want, f"n={nums.size}: {len(got)} bytes vs the oracle's {len(want)}, first difference at byte {_first_diff(got, want)}"
    back = oracle.simple_decompress(got, nums.dtype)
    np.testing.assert_array_equal(bits_view(back), bits_view(nums))
    if gpu_decode:
        dec = sa.simple_decompress(got, nums.dtype)
        assert dec.size == nums.size
        np.testing.assert_array_equal(bits_view(dec), bits_view(back))
    return got


def _ans_paths():
    from pcodec_b200 import _lib

    counts = (C.c_uint * 8)()
    rounds = _lib.lib().pco_b200_profile_ans_paths(counts)
    return rounds, list(counts)


def _c2(n, seed=0):
    return datagen.c2_u64_cumsum_geometric(n, seed=seed)


def _wide_uniform(n, seed, bits=40):
    """Uniform numbers over a wide range: at order 0 one bin whose offsets are far wider than 15 bits (so decode_kernel, not the fused
    kernel, decodes it), and a key range the planner sorts (radix_sort_segments_kernel)."""
    return np.random.default_rng(seed).integers(0, 1 << bits, size=n, dtype=np.uint64)


# ---- where the rounds start and end: stored counts on both sides of 2^18 (one full round of 64 segments of 16 batches) and 2^20

STORED = [
    K18 - 1,             # one round (control)
    K18,                 # one full round (control)
    K18 + 1,             # 65 segments: round 0 ends in the 1-number short batch, round 1 is segment 0 alone (s == 0, no speculation)
    K18 + 2 * 4096 + 3,  # round 1 holds three segments: one speculating segment and a partial round
    (1 << 19) + 77,      # several rounds
    K20,                 # four full rounds; plan_solve_kernel's estimate branch with num above 2^24
    K20 + 1,             # small_n == false in plan_solve_kernel: the 64-bit division
]


@pytest.mark.parametrize("order", [0, 1])
@pytest.mark.parametrize("stored", STORED)
def test_round_thresholds_c2(sa, oracle, stored, order):
    n = stored + order
    nums = _c2(n, seed=stored % 97 + order)
    _check(sa, oracle, nums, *_cfgs(oracle, n_page=n, order=order))


# ---- dtypes and delta orders at the 2^19 / 2^20 tier


@pytest.mark.parametrize("order", [0, 1, 2, 7])
@pytest.mark.parametrize("dtype", [np.uint32, np.int64, np.float32, np.float64, np.uint16])
def test_dtypes_and_orders(sa, oracle, dtype, order):
    # alternate the sizes; order 2 and 7 also store just above 2^20 latents
    n = {0: (1 << 19) + 77, 1: K20, 2: K20 + 2 + 1, 7: K20 + 7 + 1}[order]
    nums = datagen.c5_sweep(dtype, n, seed=order + 3)
    _check(sa, oracle, nums, *_cfgs(oracle, n_page=n, order=order))


def test_u32_lomax_order0_stored_above_2_20(sa, oracle):
    n = K20 + 1
    _check(sa, oracle, datagen.c1_u32_lomax(n, seed=4), *_cfgs(oracle, n_page=n, order=0))


# ---- two latent vars (symwalk_kernel + decode_kernel, the two-kernel front end) and wide offsets


def test_float_mult_c3_order2(sa, oracle):
    n = K20 + 2 + 1  # the primary stores 2^20 + 1 latents, the secondary 2^20 + 3
    _check(sa, oracle, datagen.c3_f64_decimal_sinusoid(n), *_cfgs(oracle, n_page=n, mode="float_mult", order=2, base=0.01))


@pytest.mark.parametrize("n", [(1 << 19) + 77, K20 + 1])
def test_int_mult(sa, oracle, n):
    rng = np.random.default_rng(5)
    nums = (_c2(n, seed=6) * np.uint64(7) + rng.integers(0, 7, size=n, dtype=np.uint64) * (rng.random(n) < 0.05)).astype(np.uint64)
    _check(sa, oracle, nums, *_cfgs(oracle, n_page=n, mode="int_mult", order=1, ibase=7))


def test_float_quant(sa, oracle):
    n = K20
    nums = datagen.c5_sweep(np.float64, n, seed=7)
    q = (nums.view(np.uint64) & ~np.uint64((1 << 30) - 1)).view(np.float64)  # most numbers on the k = 30 grid, a few off it
    q[::1000] = nums[::1000]
    _check(sa, oracle, q, *_cfgs(oracle, n_page=n, mode="float_quant", order=1, k=30))


@pytest.mark.parametrize("n", [K20, K20 + 1])
def test_wide_offsets_and_wide_key_range(sa, oracle, n):
    _check(sa, oracle, _wide_uniform(n, seed=8), *_cfgs(oracle, n_page=n, order=0))
    signed = np.random.default_rng(9).integers(-(1 << 62), 1 << 62, size=n, dtype=np.int64)
    _check(sa, oracle, signed, *_cfgs(oracle, n_page=n, order=1))


# ---- levels 9 and 12 (plan_solve_wide_kernel, the wide instantiations)


def _level_data(n, seed):
    rng = np.random.default_rng(seed)
    steps = rng.lognormal(0.0, 2.0, size=n) * rng.choice([-1.0, 1.0], size=n)
    return np.cumsum(np.round(steps * 300.0)).astype(np.int64).astype(np.uint64)


@pytest.mark.parametrize("level", [9, 12])
@pytest.mark.parametrize("n", [K20, K24])
def test_high_levels(sa, oracle, level, n):
    nums = _level_data(n, seed=level)
    ours, theirs = _cfgs(oracle, n_page=n, level=level, order=1)
    got = _check(sa, oracle, nums, ours, theirs, gpu_decode=False)
    # the GPU decodes what its fast kernels take; the catch-all decoder (a few MB/s) only up to 2^20 numbers
    if n <= K20 or _fast_decodable(oracle, got, nums.dtype):
        np.testing.assert_array_equal(bits_view(sa.simple_decompress(got, nums.dtype)), bits_view(nums))


# ---- Auto / Auto: the mode sample and the delta search at large n


@pytest.mark.parametrize("n", [K20, K24])
def test_auto_auto_c2(sa, oracle, n):
    _check(sa, oracle, _c2(n, seed=10), *_cfgs(oracle, n_page=n, auto=True))


def test_auto_auto_c3_float_mult(sa, oracle):
    n = K20 + 3
    _check(sa, oracle, datagen.c3_f64_decimal_sinusoid(n, seed=1), *_cfgs(oracle, n_page=n, auto=True))


# ---- the format limit


def test_2_24_u64_c2_order1(sa, oracle):
    for n in (K24 - 1, K24):
        _check(sa, oracle, _c2(n, seed=11), *_cfgs(oracle, n_page=n, order=1))


def test_2_24_f64_order0(sa, oracle):
    _check(sa, oracle, datagen.c5_sweep(np.float64, K24, seed=12), *_cfgs(oracle, n_page=K24, order=0))


def test_2_24_near_incompressible(sa, oracle):
    """63 random bits per number: about 2^30 bits of offsets in one chunk, just under the size at which the chunk falls back to
    uncompressed storage (the side index's bit positions are 32-bit)."""
    nums = np.random.default_rng(13).integers(0, 1 << 63, size=K24, dtype=np.uint64)
    data = _check(sa, oracle, nums, *_cfgs(oracle, n_page=K24, order=0))
    assert len(data) > K24 * 63 // 8


# ---- one call that mixes chunk sizes: runs of different unoptimized_bins_log share scratch sized by the largest chunk


@pytest.mark.parametrize("order", [0, 1])
def test_mixed_chunk_sizes_one_call(sa, oracle, order):
    sizes = [K24, 1, K18 + 1, 257, 3]
    nums = _c2(sum(sizes), seed=14)
    data = _check(sa, oracle, nums, *_cfgs(oracle, exact=sizes, order=order))
    assert [c["n"] for c in oracle.inspect(data, np.uint64)["chunks"]] == sizes


# ---- every resolution of a tANS round, in one round (2^18) and in four (2^20)


def _profiled_compress(sa, oracle, nums, ours, theirs):
    from pcodec_b200 import _lib

    L = _lib.lib()
    L.pco_b200_profile_enable(1)
    try:
        got = sa.simple_compress(nums, ours)
        rounds, counts = _ans_paths()
    finally:
        L.pco_b200_profile_enable(0)
    want = oracle.simple_compress(nums, theirs)
    assert got == want, f"{len(got)} bytes vs the oracle's {len(want)}, first difference at byte {_first_diff(got, want)}"
    np.testing.assert_array_equal(bits_view(sa.simple_decompress(got, nums.dtype)), bits_view(nums))
    return rounds, counts


def _in_order_late(n):
    """A page whose last quarter (round 0: the encoder starts at the end) resolves without the in-order pass, and whose front needs it:
    C5 i64 (a slow walk, so heavy symbols in long runs) with the last quarter shuffled.  The shuffle keeps the histogram, so the
    tANS table is the walk's; only the order of the symbols changes, and mixed symbols make trajectories merge."""
    x = datagen.c5_sweep(np.int64, n, seed=15)
    q = n // 4
    x[n - q:] = np.random.default_rng(16).permutation(x[n - q:])
    return x


def _staircase(n, seed, levels=200):
    """Sorted draws from 200 far-apart values: one bin per value, equal weights (5 and 6 of 2^10 states), and symbols in runs of ~n/200.
    Runs of one symbol of a light weight permute the states, so no correction ever meets the guessed trajectory."""
    rng = np.random.default_rng(seed)
    vals = np.sort(rng.integers(0, 1 << 40, size=levels, dtype=np.int64))
    return np.sort(vals[rng.integers(0, levels, size=n)])


# data shapes that reach each resolution (DESIGN.md §4): (slot, generator, delta order)
RESOLUTIONS = {
    "speculation": (SPECULATION, lambda n: _c2(n, seed=17), 1),                             # C2: trajectories merge within the warm-up
    "fixup": (FIXUP, lambda n: datagen.c5_sweep(np.float64, n, seed=18), 0),               # C5 f64 order 0: wrong guesses, corrections meet
    "transfer": (TRANSFER, lambda n: _staircase(n, seed=19), 0),                           # equal light weights in long runs
    "in_order": (IN_ORDER, lambda n: datagen.c5_sweep(np.int64, n, seed=20), 0),           # C5 i64 order 0: weights 205 / 51 in long runs
}


@pytest.mark.parametrize("n_rounds", [1, 4])
@pytest.mark.parametrize("name", list(RESOLUTIONS))
def test_ans_resolution(sa, oracle, name, n_rounds):
    path, gen, order = RESOLUTIONS[name]
    n = n_rounds * K18 + order
    rounds, counts = _profiled_compress(sa, oracle, gen(n), *_cfgs(oracle, n_page=n, order=order))
    assert counts[path] >= 1, (name, counts)
    if path == IN_ORDER:
        # the in-order pass covers the whole page: no round runs after it
        assert counts[IN_ORDER] == 1 and rounds <= n_rounds, counts
    else:
        assert rounds == n_rounds, counts
        assert sum(counts[LATER:]) == n_rounds - 1, counts
        if n_rounds > 1:
            assert counts[LATER + path] >= 1, (name, counts)


def test_ans_in_order_pass_from_a_later_round(sa, oracle):
    n = 4 * K18
    rounds, counts = _profiled_compress(sa, oracle, _in_order_late(n), *_cfgs(oracle, n_page=n, order=0))
    assert counts[LATER + IN_ORDER] == 1, counts
    assert sum(counts[:IN_ORDER]) >= 1, counts


def test_ans_counters_are_per_call(sa, oracle):
    """Several chunks in one call count every (chunk, var, round); a call without profiling leaves nothing to report."""
    n = 3 * (K20 + 1)  # three chunks that store 2^20 latents each: four rounds apiece
    rounds, counts = _profiled_compress(sa, oracle, _c2(n, seed=21), *_cfgs(oracle, n_page=K20 + 1, order=1))
    assert rounds == 3 * 4 and sum(counts[LATER:]) == 3 * 3, counts
    sa.simple_compress(_c2(1000), _cfgs(oracle, n_page=K18, order=1)[0])
    assert _ans_paths() == (0, [0] * 8)


# ---- decode entry points on large chunks


def _multi_chunk_file(oracle):
    sizes = [K20, K20, K20, 5000]
    nums = _c2(sum(sizes), seed=22)
    ours, theirs = _cfgs(oracle, exact=sizes, order=1)
    return nums, sizes, ours, oracle.simple_compress(nums, theirs)


def test_side_index_and_index_free_walk(sa, oracle):
    nums, sizes, ours, data = _multi_chunk_file(oracle)
    got, index = sa.simple_compress_with_index(nums, ours)
    assert got == data
    np.testing.assert_array_equal(sa.simple_decompress(data, np.uint64, index=index), nums)
    built = sa.build_index(data, np.uint64)
    np.testing.assert_array_equal(sa.simple_decompress(data, np.uint64, index=built), nums)
    # no index: the speculative walk finds the chunk starts (one candidate's index is 1.5 MB)
    np.testing.assert_array_equal(sa.simple_decompress(data, np.uint64), nums)
    np.testing.assert_array_equal(sa.simple_decompress(data, np.uint64), oracle.simple_decompress(data, np.uint64))


def test_two_var_side_index_and_walk(sa, oracle):
    n = 2 * K20 + 3
    nums = datagen.c3_f64_decimal_sinusoid(n, seed=2)
    ours, theirs = _cfgs(oracle, n_page=K20 + 2, mode="float_mult", order=2, base=0.01)
    data = oracle.simple_compress(nums, theirs)
    got, index = sa.simple_compress_with_index(nums, ours)
    assert got == data
    for idx in (index, None):
        np.testing.assert_array_equal(bits_view(sa.simple_decompress(data, np.float64, index=idx)), bits_view(nums))


def test_decompress_chunks_at_known_offsets(sa, oracle):
    nums, sizes, _, data = _multi_chunk_file(oracle)
    info = oracle.inspect(data, np.uint64)["chunks"]
    offs, ns = [c["chunk_start"] for c in info], [c["n"] for c in info]
    assert ns == sizes
    np.testing.assert_array_equal(sa.decompress_chunks(data, np.uint64, offs, ns), nums)
    pick = [3, 1, 0]
    starts = np.concatenate([[0], np.cumsum(sizes)])
    want = np.concatenate([nums[starts[i]:starts[i + 1]] for i in pick])
    np.testing.assert_array_equal(sa.decompress_chunks(data, np.uint64, [offs[i] for i in pick], [ns[i] for i in pick]), want)


def test_files_with_one_large_file(sa, oracle):
    ns = [1000, K20, 3, 70000]
    nums = _c2(sum(ns), seed=23)
    ours, theirs = _cfgs(oracle, n_page=K20, order=1)
    data, files, index = sa.compress_files(nums, ns, ours)
    at = np.concatenate([[0], np.cumsum(ns)])
    for i in range(len(ns)):
        piece = bytes(data[int(files[i]["offset"]):int(files[i]["offset"] + files[i]["len"])])
        assert piece == oracle.simple_compress(nums[at[i]:at[i + 1]], theirs), f"file {i}"
    for idx in (index, None):
        refs = files.copy()
        if idx is None:
            refs["index_len"] = 0
        back, file_ns = sa.decompress_files(data, refs, np.uint64, index=idx)
        assert list(file_ns) == ns
        np.testing.assert_array_equal(back, nums)


def test_wrapped_one_page_chunk(oracle):
    from pcodec_b200 import wrapped

    n = K20
    nums = _c2(n, seed=24)
    ours, theirs = _cfgs(oracle, exact=[n], order=1)
    cc = oracle.ChunkCompressor(nums, theirs)
    meta, page = cc.write_meta(), cc.write_page(0)
    refs = np.zeros(1, dtype=wrapped.PAGE_REF)
    refs[0] = (0, len(meta), 0, len(page), n)
    np.testing.assert_array_equal(wrapped.decompress_pages(meta, page, refs, np.uint64), nums)
    metas, pages, _ = wrapped.compress_chunks(nums, ours)
    assert bytes(metas) == meta and bytes(pages) == page


@pytest.mark.parametrize("cap", [0, K20 - 1, K20, K20 + 1, 3 * K20 - 1])
def test_partial_destination(sa, oracle, cap):
    n = 3 * K20
    nums = _c2(n, seed=25)
    data = oracle.simple_compress(nums, _cfgs(oracle, n_page=K20, order=1)[1])
    dst, want = np.zeros(cap, dtype=np.uint64), np.zeros(cap, dtype=np.uint64)
    prog = sa.simple_decompress_into(data, dst)
    n_proc, finished = oracle.simple_decompress_into(data, want)
    assert (prog.n_processed, prog.finished) == (n_proc, finished) == (cap, False)
    np.testing.assert_array_equal(dst, want)
    np.testing.assert_array_equal(dst, nums[:cap])


def test_calls_after_thread_release(sa, oracle):
    """pco_b200_thread_release frees the thread's scratch (this module calls it when it ends); the same thread's next calls must build
    what they need again.  A two-var file decodes through decode_kernel, which reads the per-thread binomial table."""
    from pcodec_b200 import _lib

    _lib.lib().pco_b200_thread_release()
    nums = datagen.c3_f64_decimal_sinusoid(5000)
    data = oracle.simple_compress(nums, _cfgs(oracle, n_page=K18, mode="float_mult", order=2, base=0.01)[1])
    np.testing.assert_array_equal(bits_view(sa.simple_decompress(data, np.float64)), bits_view(nums))
    _lib.lib().pco_b200_thread_release()
    _check(sa, oracle, _c2(5000, seed=26), *_cfgs(oracle, n_page=K18, order=1))
