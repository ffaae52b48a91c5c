"""The catch-all device decoder (cold_decode_kernel, pcodec_b200/csrc/decode_cold.cuh) on full-size files: Lookback chunks longer than
their 2^15 window (the window buffer cycles, lookbacks of exactly window_n), Lookback windows above 2^16 (the second scratch pass of
cold_decode_jobs), Dict chunks of 2^18 and 2^20 numbers with up to 65,536 values, Conv1 at orders 1 to 32 with predictions clamped at
zero, through every entry point that reaches the decoder, and a property test over the oracle's whole config space.

Every case follows one pattern: the oracle writes the file; pcodec_b200.inspect shows that the targeted feature is in it (delta kind,
window, order, dictionary length, bins); the GPU decode equals the input and the oracle's decode bit for bit; and where the route
matters, the profiler's spans show that cold_decode_kernel served the cold chunks.  The window-patch helper and its oracle self-test
need no GPU."""
import ctypes as C

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

from pcodec_b200 import inspect as insp
from tests.golden_generators import bits_view
from tests.test_gpu_properties import _dump_failure
from tests.test_oracle_properties import DTYPES, arrays, configs

gpu = pytest.mark.gpu

W = 1 << 15  # the largest window the encoder writes (window_n_log = clamp(bits(n - 1), 4, 15))
KIND = {"noop": 0, "consecutive": 1, "lookback": 2, "conv1": 3}
MODE_KIND = {"classic": 0, "int_mult": 1, "float_mult": 2, "float_quant": 3, "dict": 4}
ALL_TYPES = [np.uint8, np.int8, np.uint16, np.int16, np.float16, np.uint32, np.int32, np.float32, np.uint64, np.int64, np.float64]


# ---- data ---------------------------------------------------------------------------------------------------------------------
def _u(dtype):
    return np.dtype(f"u{np.dtype(dtype).itemsize}")


def _nbits(dtype):
    return 8 * np.dtype(dtype).itemsize


def _motif(dtype, n, period=97, seed=0, edit_every=211):
    """`n` numbers repeating a random motif of `period` values (full-range bits for integers, normal values for floats), with one
    number in every `edit_every` nudged by 3 units in the last place."""
    dt, u = np.dtype(dtype), _u(dtype)
    rng = np.random.default_rng(seed)
    if dt.kind == "f":
        motif = (rng.normal(size=period) * 1000).astype(dt).view(u)
    else:
        motif = rng.integers(0, 1 << _nbits(dt), size=period, dtype=np.uint64).astype(u)
    x = np.resize(motif, n)
    if edit_every:
        x[::edit_every] += u.type(3)
    return x.view(dt)


def _special_bits(dtype):
    """Bits of floats that must survive untouched: quiet NaNs with payloads (positive and negative), a signalling NaN, +inf, -inf,
    0.0 and -0.0."""
    b = _nbits(dtype)
    mant = {16: 10, 32: 23, 64: 52}[b]
    inf, sign = ((1 << (b - 1 - mant)) - 1) << mant, 1 << (b - 1)
    quiet = inf | (1 << (mant - 1))
    return np.array([quiet | 5, quiet | 3 | sign, inf | 1, inf, inf | sign, 0, sign], dtype=np.uint64).astype(_u(dtype))


def _with_specials(x):
    """Floats with the special values of _special_bits spread through them."""
    y = x.copy().view(_u(x.dtype))
    y[5::997] = np.resize(_special_bits(x.dtype), y[5::997].size)
    return y.view(x.dtype)


def _to_latents(x):
    """pco's order-preserving unsigned latents of the numbers (data_types/{unsigned,signed,float}.rs)."""
    dt, u = x.dtype, _u(x.dtype)
    mid = u.type(1 << (_nbits(dt) - 1))
    v = x.view(u)
    if dt.kind == "u":
        return v.copy()
    if dt.kind == "i":
        return v ^ mid
    return np.where(v & mid, ~v, v ^ mid).astype(u)


def _from_latents(lat, dtype):
    dt, u = np.dtype(dtype), _u(dtype)
    mid = u.type(1 << (_nbits(dt) - 1))
    lat = np.asarray(lat).astype(u)
    if dt.kind == "u":
        return lat.view(dt)
    if dt.kind == "i":
        return (lat ^ mid).view(dt)
    return np.where(lat & mid, lat ^ mid, ~lat).astype(u).view(dt)


def _conv1_nums(dtype, n, shape, seed=0):
    """Conv1 inputs, built in latent space: a smooth wave; sawtooth teeth that climb from latent 0 to the type's largest latent and
    drop back (a linear prediction after the drop is negative and the decoder clamps it at zero); alternating extremes."""
    lmax = float((1 << _nbits(dtype)) - 1)
    i = np.arange(n, dtype=np.float64)
    rng = np.random.default_rng(seed)
    if shape == "smooth":
        lat = lmax / 2 + lmax / 5 * np.sin(i / 30.0) + lmax / 40 * np.cos(i / 7.0)
    elif shape == "sawtooth":
        lat = np.round((i % 37) / 36 * lmax)
    else:  # extremes: 0, max, 0, max with a few middle values
        lat = np.where(i % 2 == 0, 0.0, lmax)
        lat[rng.integers(0, n, size=max(n // 50, 1))] = lmax / 2
    return _from_latents(np.clip(lat, 0, lmax).astype(np.uint64), dtype)


def _negative_predictions(x, delta):
    """How many Conv1 predictions of the chunk are negative before quantization, so that the decoder clamps them at zero (pco's
    conv1.rs): prediction of latent p = bias + sum_j w[j] * latent[p - order + j], for p >= order."""
    w = np.array(delta["weights"], dtype=np.int64)
    lat = _to_latents(x).astype(np.int64)
    if lat.size <= w.size:
        return 0
    win = np.lib.stride_tricks.sliding_window_view(lat, w.size)[:-1]
    return int(((win @ w) + delta["bias"] < 0).sum())


def _distinct(dtype, k, rng):
    """`k` numbers of `dtype` with distinct bits; float pools hold NaNs with payloads of both signs, both infinities, 0.0 and -0.0."""
    dt, u = np.dtype(dtype), _u(dtype)
    pool = _special_bits(dt).tolist()[:k] if dt.kind == "f" else []
    seen = set(pool)
    while len(pool) < k:
        if dt.kind == "f":
            cand = (rng.normal(size=2 * k) * 1000).astype(dt).view(u)
        elif k == 1 << _nbits(dt):
            cand = rng.permutation(np.arange(k, dtype=np.uint64)).astype(u)
        else:
            cand = rng.integers(0, 1 << _nbits(dt), size=2 * k, dtype=np.uint64).astype(u)
        for v in cand.tolist():
            if v not in seen:
                seen.add(v)
                pool.append(v)
    return np.array(pool[:k], dtype=np.uint64).astype(u).view(dt)


# ---- files --------------------------------------------------------------------------------------------------------------------
def _chunks(oracle, data, dtype):
    """Every chunk's meta as pcodec_b200.inspect reads it, with its count and where the meta starts (chunk boundaries from the
    oracle)."""
    info = oracle.inspect(data, dtype)
    out = []
    for c in info["chunks"]:
        meta, _ = insp.read_chunk_meta(data, c["meta_start"], _nbits(dtype), info["format"][0])
        meta["n"], meta["meta_start"] = c["n"], c["meta_start"]
        out.append(meta)
    return out


def _window_log(n):
    return min(15, max(4, (n - 1).bit_length()))


def _assert_lookback(meta, window_n_log):
    d = meta["delta"]
    assert d["kind"] == KIND["lookback"], d
    assert d["window_n_log"] == window_n_log and d["state_n_log"] == 0 and not d["secondary_uses_delta"], d


def _lookbacks(meta):
    return {lower for _, lower, _ in meta["vars"]["delta"]["bins"]}


def _window_field_bit(buf, meta_byte, number_bits):
    """Bit position of a Lookback chunk meta's 5-bit `window_n_log - 1` field (pco's metadata/{mode,delta_encoding}.rs): behind the
    4-bit mode and its parameters (IntMult and FloatMult base: number_bits; FloatQuant k: 8 bits; Dict: 25-bit length, byte padding
    and the values) and the 4-bit delta variant."""
    mode = buf[meta_byte] & 15
    bit = 8 * meta_byte + 4
    if mode in (1, 2):
        bit += number_bits
    elif mode == 3:
        bit += 8
    elif mode == 4:
        dict_len = (int.from_bytes(buf[meta_byte:meta_byte + 8], "little") >> 4) & ((1 << 25) - 1)
        bit = -(-(bit + 25) // 8) * 8 + dict_len * number_bits
    return bit + 4


def patch_window(data, meta_byte, number_bits, window_n_log):
    """`data` with the Lookback chunk meta at `meta_byte` re-written to a window of 2^window_n_log numbers.  The encoder never writes a
    window above 2^15, but any window up to 2^24 that holds the chunk's lookbacks is valid pco and decodes to the same numbers (with
    state_n_log = 0 and secondary_uses_delta = false: a larger window only adds zeros before the page)."""
    before, _ = insp.read_chunk_meta(data, meta_byte, number_bits)
    assert before["delta"]["kind"] == KIND["lookback"] and before["delta"]["state_n_log"] == 0 and not before["delta"]["secondary_uses_delta"]
    assert 1 <= window_n_log <= 24 and max(_lookbacks(before)) <= 1 << window_n_log
    bit = _window_field_bit(data, meta_byte, number_bits)
    b = bytearray(data)
    word = int.from_bytes(b[bit // 8:bit // 8 + 2], "little")
    word = (word & ~(31 << (bit % 8))) | ((window_n_log - 1) << (bit % 8))
    b[bit // 8:bit // 8 + 2] = word.to_bytes(2, "little")
    out = bytes(b)
    after, _ = insp.read_chunk_meta(out, meta_byte, number_bits)
    assert after["delta"]["window_n_log"] == window_n_log
    after["delta"]["window_n_log"] = before["delta"]["window_n_log"]
    assert after == before, "the patch touched more than the window"
    return out


# ---- decoding -----------------------------------------------------------------------------------------------------------------
def _sa():
    from pcodec_b200 import standalone

    return standalone


def _profiled(fn):
    """fn()'s result and the "kernel=ms;" spans of the library call it made."""
    from pcodec_b200 import _lib

    L = _lib.lib()
    L.pco_b200_profile_enable(1)
    try:
        out = fn()
        buf = C.create_string_buffer(1 << 16)
        L.pco_b200_profile_last(buf, C.c_size_t(len(buf)))
    finally:
        L.pco_b200_profile_enable(0)
    return out, buf.value.decode()


def _same(got, want):
    np.testing.assert_array_equal(bits_view(np.asarray(got)), bits_view(np.asarray(want)))


def _decode(oracle, data, nums, cold_passes=1):
    """standalone.simple_decompress on the GPU: the input and the oracle's decode, served by cold_decode_kernel in `cold_passes`
    launches (2 when the first pass met a window above 2^16)."""
    got, prof = _profiled(lambda: _sa().simple_decompress(data, nums.dtype))
    _same(got, nums)
    _same(got, oracle.simple_decompress(data, nums.dtype))
    assert prof.count("cold_decode_kernel=") == cold_passes, prof
    return got


# ==== 1. Lookback at scale =====================================================================================================
LOOKBACK_SIZES = [1 << 14, W - 1, W, W + 1, W + 255, W + 256, W + 257, 1 << 16, (1 << 16) + 1, 3 * W + 77, 1 << 18, 1 << 20]


def _lookback_file(oracle, nums, mode="classic", level=8, **kw):
    ocfg = oracle.make_config(level=level, mode={"classic": oracle.MODE_CLASSIC, "int_mult": oracle.MODE_INT_MULT, "float_mult": oracle.MODE_FLOAT_MULT,
                                                 "float_quant": oracle.MODE_FLOAT_QUANT, "dict": oracle.MODE_DICT}[mode],
                              delta=oracle.DELTA_LOOKBACK, max_page_n=nums.size, **kw)
    data = oracle.simple_compress(nums, ocfg)
    metas = _chunks(oracle, data, nums.dtype)
    assert len(metas) == 1 and metas[0]["n"] == nums.size
    assert metas[0]["mode"]["kind"] == MODE_KIND[mode], metas[0]["mode"]
    _assert_lookback(metas[0], _window_log(nums.size))
    return data, metas[0]


@gpu
@pytest.mark.parametrize("n", LOOKBACK_SIZES)
def test_lookback_chunk_sizes(oracle, n):
    """At n = 2^15 the last batch ends exactly at the end of the window buffer; from 2^15 + 1 on the buffer cycles."""
    nums = _motif(np.uint32, n, seed=n)
    data, _ = _lookback_file(oracle, nums)
    _decode(oracle, data, nums)


def _shape(name, n):
    if name == "constant":
        return np.full(n, 0x9E3779B9, dtype=np.uint32)
    if name == "period_changes":  # period 97 up to the first cycle, then a period that reaches back across it
        return np.concatenate([_motif(np.uint32, W, period=97, seed=1), _motif(np.uint32, n - W, period=W - 100, seed=2, edit_every=0)])
    period = {"period_w": W, "period_w_minus_1": W - 1, "period_w_minus_255": W - 255, "period_w_minus_256": W - 256}[name]
    return _motif(np.uint32, n, period=period, seed=period, edit_every=0)


@gpu
@pytest.mark.parametrize("shape", ["period_w", "period_w_minus_1", "period_w_minus_255", "period_w_minus_256", "period_changes", "constant"])
def test_lookback_data_shapes(oracle, shape):
    n = 3 * W + 77
    nums = _shape(shape, n)
    data, meta = _lookback_file(oracle, nums)
    if shape == "period_w":
        assert W in _lookbacks(meta), "a lookback of exactly window_n"
    elif shape.startswith("period_w_minus"):
        assert W - int(shape.rsplit("_", 1)[1]) in _lookbacks(meta)
    _decode(oracle, data, nums)


@gpu
@pytest.mark.parametrize("dtype", ALL_TYPES)
def test_lookback_every_type(oracle, dtype):
    nums = _motif(dtype, W + 257, seed=3)
    data, _ = _lookback_file(oracle, nums)
    _decode(oracle, data, nums)


def _two_var_nums(mode, dtype, n, seed=4):
    rng = np.random.default_rng(seed)
    dt = np.dtype(dtype)
    if mode == "int_mult":
        lo = -(1 << 40) if dt.kind == "i" else 0
        motif = rng.integers(lo, 1 << (28 if dt.itemsize == 4 else 40), size=97)
        return (np.resize(motif, n) * 8 + rng.integers(0, 3, size=n)).astype(dtype)
    if mode == "float_mult":
        base = 0.25 if dt.itemsize == 2 else 0.01
        x = (np.resize(np.round(rng.normal(size=97) * (40 if dt.itemsize == 2 else 1000)), n) * base).astype(dtype)
        x[::211] = (x[::211].astype(np.float64) + base / 3).astype(dtype)
        return _with_specials(x)
    if mode == "float_quant":
        k = 7 if dt.itemsize == 4 else 13
        u = _u(dt)
        x = np.resize((rng.normal(size=97) * 1000).astype(dt).view(u) & ~u.type((1 << k) - 1), n)
        x[::211] |= u.type(5)
        return _with_specials(x.view(dt))
    pool = _distinct(dt, 300, rng)  # dict
    idx = np.resize(rng.integers(0, 300, size=97), n)
    idx[::211] = rng.integers(0, 300, size=idx[::211].size)
    return pool[idx]


@gpu
@pytest.mark.parametrize("mode,dtype", [("int_mult", np.uint32), ("int_mult", np.int64), ("float_mult", np.float32), ("float_mult", np.float64),
                                        ("float_mult", np.float16), ("float_quant", np.float32), ("float_quant", np.float64), ("dict", np.uint32),
                                        ("dict", np.float64)])
def test_lookback_with_two_var_and_dict_modes(oracle, mode, dtype):
    """The secondary var (IntMult, FloatMult, FloatQuant) and the Dict index var beside a cycling window."""
    nums = _two_var_nums(mode, dtype, W + 3001)
    kw = {"int_mult": dict(int_mult_base=8), "float_mult": dict(float_mult_base=0.25 if np.dtype(dtype).itemsize == 2 else 0.01),
          "float_quant": dict(float_quant_k=7 if np.dtype(dtype).itemsize == 4 else 13), "dict": {}}[mode]
    data, _ = _lookback_file(oracle, nums, mode=mode, **kw)
    _decode(oracle, data, nums)


@gpu
@pytest.mark.parametrize("level", [2, 8, 12])
def test_lookback_levels(oracle, level):
    """The decoder's large tables (up to 2^12 states at level 12) beside the window cycle.  Level 2 is the lowest at which the
    encoder writes Lookback on this data: at levels 0 and 1 it keeps one bin and no delta."""
    rng = np.random.default_rng(level)
    n = 3 * W + 77
    nums = _motif(np.uint32, n, period=1000, seed=5, edit_every=0)
    noisy = rng.random(n) < 0.5
    nums[noisy] += rng.integers(0, 1 << 12, size=int(noisy.sum())).astype(np.uint32)
    data, meta = _lookback_file(oracle, nums, level=level)
    if level == 12:
        assert meta["vars"]["primary"]["ans_size_log"] > 10, meta["vars"]["primary"]["ans_size_log"]
    _decode(oracle, data, nums)


@gpu
def test_default_config_picks_lookback(oracle):
    """The reference's default config (Auto mode and delta, 2^18-number chunks) on repetitive data: the most common file only the
    catch-all decoder reads."""
    nums = _motif(np.uint32, 1 << 18, seed=6)
    data = oracle.simple_compress(nums, None)
    metas = _chunks(oracle, data, np.uint32)
    assert len(metas) == 1
    _assert_lookback(metas[0], 15)
    _decode(oracle, data, nums)


@gpu
def test_default_config_mixes_fast_and_cold_chunks(oracle):
    """Four chunks of 2^18 under the default config: Lookback, consecutive, Lookback, no delta.  A file with a cold chunk is decoded
    again from its first chunk by the catch-all decoder."""
    from tests.test_gpu_encode import _walk

    n = 1 << 18
    rng = np.random.default_rng(7)
    nums = np.concatenate([_motif(np.uint32, n, seed=8), _walk(np.uint32, n, seed=9), _motif(np.uint32, n, period=W - 3, seed=10),
                           rng.integers(0, 1 << 32, size=n, dtype=np.uint64).astype(np.uint32)])
    data = oracle.simple_compress(nums, None)
    metas = _chunks(oracle, data, np.uint32)
    assert [m["n"] for m in metas] == [n] * 4
    assert [m["delta"]["kind"] for m in metas] == [KIND["lookback"], KIND["consecutive"], KIND["lookback"], KIND["noop"]], [m["delta"] for m in metas]
    _decode(oracle, data, nums)


# ==== 2. Windows above 2^15: the second scratch pass ============================================================================
def _patch_cases(oracle):
    """(mode, dtype, numbers, oracle config keywords) with a Lookback chunk of more than 2^15 numbers."""
    n = W + 300
    return [("classic", np.uint32, _motif(np.uint32, n, seed=11), {}),
            ("int_mult", np.uint32, _two_var_nums("int_mult", np.uint32, n), dict(int_mult_base=8)),
            ("float_mult", np.float64, _two_var_nums("float_mult", np.float64, n), dict(float_mult_base=0.01)),
            ("float_quant", np.float32, _two_var_nums("float_quant", np.float32, n), dict(float_quant_k=7)),
            ("dict", np.uint32, _two_var_nums("dict", np.uint32, n), {})]


def test_window_patch_keeps_the_numbers(oracle):
    """The patch helper's self-test: in every mode the patched file is valid pco and the oracle decodes it to the input."""
    for mode, dtype, nums, kw in _patch_cases(oracle):
        data, meta = _lookback_file(oracle, nums, mode=mode, **kw)
        for log in (16, 17, 20, 24):
            patched = patch_window(data, meta["meta_start"], _nbits(dtype), log)
            assert _chunks(oracle, patched, dtype)[0]["delta"]["window_n_log"] == log
            _same(oracle.simple_decompress(patched, dtype), nums)


@gpu
@pytest.mark.parametrize("mode,log", [("classic", 16), ("classic", 17), ("classic", 20), ("classic", 24), ("int_mult", 17), ("dict", 20),
                                      ("float_mult", 24)])
def test_patched_window_standalone(oracle, mode, log):
    """Window 16 fits the first pass's scratch (and cycles in a chunk of 3 * 2^15 + 77); 17 and above need the second pass."""
    n = 3 * W + 77
    dtype = np.float64 if mode == "float_mult" else np.uint32
    nums = _motif(dtype, n, seed=12) if mode == "classic" else _two_var_nums(mode, dtype, n)
    kw = {"classic": {}, "int_mult": dict(int_mult_base=8), "dict": {}, "float_mult": dict(float_mult_base=0.01)}[mode]
    data, meta = _lookback_file(oracle, nums, mode=mode, **kw)
    patched = patch_window(data, meta["meta_start"], _nbits(dtype), log)
    _decode(oracle, patched, nums, cold_passes=1 if log <= 16 else 2)


@gpu
def test_patched_window_in_the_second_chunk(oracle):
    """Chunk 0 keeps window 15, chunk 1 has window 17: the first pass decodes chunk 0, is refused at chunk 1, and the whole file is
    decoded again with the large scratch."""
    n = 2 * (W + 300)
    nums = _motif(np.uint32, n, seed=13)
    data = oracle.simple_compress(nums, oracle.make_config(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_LOOKBACK, max_page_n=W + 300))
    metas = _chunks(oracle, data, np.uint32)
    assert [m["n"] for m in metas] == [W + 300, W + 300]
    for m in metas:
        _assert_lookback(m, 15)
    patched = patch_window(data, metas[1]["meta_start"], 32, 17)
    assert [m["delta"]["window_n_log"] for m in _chunks(oracle, patched, np.uint32)] == [15, 17]
    _decode(oracle, patched, nums, cold_passes=2)


# ==== 3. Dict at scale =========================================================================================================
# (dtype, n, dictionary values, index distribution, level, delta)
DICT_CASES = [(np.uint32, 1 << 18, k, "uniform", 8, "noop") for k in (1, 2, 255, 256, 257, 4096, 65536)] + [
    (np.uint32, 1 << 18, 257, "zipf", 8, "noop"),
    (np.uint32, 1 << 18, 65536, "zipf", 8, "noop"),
    (np.uint32, 1 << 18, 4096, "uniform", 0, "noop"),
    (np.uint32, 1 << 18, 4096, "uniform", 12, "noop"),
    (np.uint32, 1 << 18, 4096, "uniform", 8, "consecutive"),
    (np.uint32, 1 << 18, 4096, "uniform", 8, "lookback"),
    (np.uint8, 1 << 18, 255, "zipf", 8, "noop"),
    (np.uint8, 1 << 18, 100, "uniform", 8, "noop"),
    (np.int16, 1 << 18, 4096, "zipf", 12, "noop"),
    (np.int64, 1 << 18, 65536, "uniform", 8, "noop"),
    (np.float32, 1 << 18, 257, "uniform", 8, "lookback"),
    (np.float64, 1 << 18, 4096, "zipf", 8, "consecutive"),
    (np.uint32, 1 << 20, 65536, "uniform", 12, "noop"),
    (np.float64, 1 << 20, 257, "zipf", 8, "noop"),
]


def _dict_nums(dtype, n, k, dist, delta, seed):
    rng = np.random.default_rng(seed)
    pool = _distinct(dtype, k, rng)
    if dist == "uniform":
        idx = rng.integers(0, k, size=n)
    else:
        idx = np.minimum(rng.zipf(1.3, size=n) - 1, k - 1)
    if delta == "lookback":  # repeats the Lookback can find
        idx = np.resize(idx[:4099], n)
        idx[::211] = rng.integers(0, k, size=idx[::211].size)
    return pool[idx]


@gpu
@pytest.mark.parametrize("dtype,n,k,dist,level,delta", DICT_CASES, ids=[f"{np.dtype(c[0]).name}-n{c[1]}-k{c[2]}-{c[3]}-L{c[4]}-{c[5]}" for c in DICT_CASES])
def test_dict_at_scale(oracle, dtype, n, k, dist, level, delta):
    nums = _dict_nums(dtype, n, k, dist, delta, seed=k + level)
    odelta = {"noop": oracle.DELTA_NOOP, "consecutive": oracle.DELTA_CONSECUTIVE, "lookback": oracle.DELTA_LOOKBACK}[delta]
    data = oracle.simple_compress(nums, oracle.make_config(level=level, mode=oracle.MODE_DICT, delta=odelta, delta_order=1 if delta == "consecutive" else 0,
                                                           enable_8_bit=True))
    metas = _chunks(oracle, data, dtype)
    assert sum(m["n"] for m in metas) == n
    for m, part in zip(metas, np.split(nums, np.cumsum([m["n"] for m in metas])[:-1])):
        assert m["mode"]["kind"] == MODE_KIND["dict"], m["mode"]
        assert sorted(m["mode"]["dict"]) == sorted(np.unique(_to_latents(part)).tolist())
        assert m["delta"]["kind"] == KIND[delta], m["delta"]
        if delta == "consecutive":
            assert m["delta"]["order"] == 1
    primary = metas[0]["vars"]["primary"]
    if n == 1 << 20 and level == 12:  # a 2^12-state table on the index var
        assert len(primary["bins"]) > 256 or primary["ans_size_log"] > 10, (len(primary["bins"]), primary["ans_size_log"])
    _decode(oracle, data, nums)


# ==== 4. Conv1 at every order ==================================================================================================
CONV1_TYPES = [np.uint8, np.int8, np.uint16, np.int16, np.uint32, np.int32, np.float16, np.float32]
CONV1_ORDERS = [1, 2, 7, 8, 16, 31, 32]
CONV1_MIN_CASES = 8  # files per (type, order) the oracle must really write as Conv1


def _conv1_sizes(order):
    return sorted({1, order - 1, order, order + 1, 256, 256 + order - 1, 256 + order, 256 + order + 1} - {0})


def _conv1_cases(order):
    """(shape, n): every size on the smooth wave (and a chunk of 2^17), the clamping shapes at every size up to 256 + order + 1 and
    at 4096."""
    cases = [("smooth", n) for n in _conv1_sizes(order) + [1 << 17]]
    for shape in ("sawtooth", "extremes"):
        cases += [(shape, n) for n in _conv1_sizes(order) + [4096]]
    return cases


@gpu
@pytest.mark.parametrize("order", CONV1_ORDERS)
@pytest.mark.parametrize("dtype", CONV1_TYPES)
def test_conv1_every_order(oracle, dtype, order):
    """Chunks no longer than their state (n <= order: no body), chunks around a batch of 256 and one of 2^17.  Where the oracle
    declines Conv1 (always at n <= 2, and on the smooth wave at high orders for 32-bit types) the file is still decoded, but does not
    count; enough cases must really be Conv1, and from order 7 on some must have predictions clamped at zero."""
    conv1, clamped = 0, 0
    for shape, n in _conv1_cases(order):
        nums = _conv1_nums(dtype, n, shape, seed=order)
        data = oracle.simple_compress(nums, oracle.make_config(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_CONV1, delta_order=order, max_page_n=n))
        (meta,) = _chunks(oracle, data, dtype)
        got = _sa().simple_decompress(data, dtype)
        _same(got, nums)
        _same(got, oracle.simple_decompress(data, dtype))
        if meta["delta"]["kind"] != KIND["conv1"]:
            continue
        assert len(meta["delta"]["weights"]) == order, meta["delta"]
        conv1 += 1
        clamped += _negative_predictions(nums, meta["delta"]) > 0
    assert conv1 >= CONV1_MIN_CASES, f"only {conv1} of {len(_conv1_cases(order))} files were Conv1"
    if order >= 7:  # at orders 1 and 2 the encoder's fits on these shapes never predict below zero
        assert clamped >= 1, "no Conv1 chunk had a prediction clamped at zero"



# ==== 5. Every entry point that reaches the catch-all decoder ===================================================================
@pytest.fixture(scope="module")
def cold_files(oracle):
    """u32 files only the catch-all decoder reads: name -> (file, numbers, chunk metas)."""
    out = {}

    def add(name, nums, data):
        out[name] = (data, nums, _chunks(oracle, data, np.uint32))

    lb = _motif(np.uint32, 1 << 18, seed=20)
    add("lookback_2p18", lb, oracle.simple_compress(lb, oracle.make_config(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_LOOKBACK)))
    lb3 = _motif(np.uint32, 3 * W + 77, seed=21)
    add("lookback_3_chunks", lb3, oracle.simple_compress(lb3, oracle.make_config(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_LOOKBACK, max_page_n=W + 300)))
    one = oracle.simple_compress(lb3, oracle.make_config(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_LOOKBACK, max_page_n=lb3.size))
    add("window_17", lb3, patch_window(one, _chunks(oracle, one, np.uint32)[0]["meta_start"], 32, 17))
    d = _dict_nums(np.uint32, 1 << 20, 4096, "uniform", "noop", seed=22)
    add("dict_2p20", d, oracle.simple_compress(d, oracle.make_config(mode=oracle.MODE_DICT, delta=oracle.DELTA_NOOP)))
    cv = _conv1_nums(np.uint32, 1 << 17, "smooth")
    add("conv1_2p17", cv, oracle.simple_compress(cv, oracle.make_config(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_CONV1, delta_order=2, max_page_n=1 << 17)))
    for m in out["lookback_2p18"][2] + out["lookback_3_chunks"][2]:
        _assert_lookback(m, 15)
    assert len(out["lookback_3_chunks"][2]) == 3 and all(m["n"] > W for m in out["lookback_3_chunks"][2])
    assert [m["delta"]["window_n_log"] for m in out["window_17"][2]] == [17]
    assert all(m["mode"]["kind"] == MODE_KIND["dict"] and len(m["mode"]["dict"]) == 4096 for m in out["dict_2p20"][2])
    assert [m["delta"]["kind"] for m in out["conv1_2p17"][2]] == [KIND["conv1"]]
    return out


SENTINEL = np.uint32(0xA5A5A5A5)


@gpu
@pytest.mark.parametrize("name", ["lookback_2p18", "window_17", "dict_2p20", "conv1_2p17"])
def test_reference_c_abi(cold_files, name):
    """pco_standalone_simple_decompress_into, the reference's decode function: the whole file into dst_cap = n; one number less is
    PcoDecompressionError; nothing lands past dst_cap."""
    from pcodec_b200 import _lib

    data, nums, _ = cold_files[name]
    L = _lib.lib()
    src = np.frombuffer(data, dtype=np.uint8)
    for cap, rc_want in ((nums.size, 0), (nums.size - 1, 3)):
        dst = np.full(cap + 64, SENTINEL, dtype=np.uint32)
        n = C.c_size_t()
        rc = L.pco_standalone_simple_decompress_into(src.ctypes.data_as(C.c_void_p), C.c_size_t(len(data)), C.c_ubyte(1), dst.ctypes.data_as(C.c_void_p),
                                                     C.c_size_t(cap), C.byref(n))
        assert rc == rc_want, (cap, rc)
        if rc == 0:
            assert n.value == nums.size
            _same(dst[:cap], nums)
        assert (dst[cap:] == SENTINEL).all()


def _caps(metas):
    n = sum(m["n"] for m in metas)
    b = metas[0]["n"]
    return sorted({0, 1, 255, 256, W - 1, W, W + 1, b - 1, b, b + 1, n - 1, n, n + 1})


@gpu
@pytest.mark.parametrize("name", ["lookback_3_chunks", "window_17", "conv1_2p17"])
def test_partial_destinations(oracle, cold_files, name):
    """pco_b200_simple_decompress_into with caps around a batch, the window, a chunk boundary and the end: the reference's Progress
    (standalone/simple.rs:100-143), the numbers up to the cap, and nothing past it."""
    from pcodec_b200 import _lib

    data, nums, metas = cold_files[name]
    L = _lib.lib()
    for cap in _caps(metas):
        dst = np.full(cap + 64, SENTINEL, dtype=np.uint32)
        prog = _lib._CProgress()
        rc = L.pco_b200_simple_decompress_into(data, C.c_size_t(len(data)), C.c_ubyte(1), dst.ctypes.data_as(C.c_void_p), C.c_size_t(cap), C.byref(prog))
        assert rc == 0, (cap, _lib.lib().pco_b200_last_error_message())
        want = oracle.simple_decompress_into(data, np.zeros(cap, dtype=np.uint32))
        assert (prog.n_processed, bool(prog.finished)) == want == (min(cap, nums.size), cap >= nums.size), cap
        _same(dst[:prog.n_processed], nums[:prog.n_processed])
        assert (dst[prog.n_processed:] == SENTINEL).all(), cap


@gpu
@pytest.mark.parametrize("name", ["lookback_3_chunks", "window_17", "dict_2p20", "conv1_2p17"])
def test_device_resident_source_and_destination(cold_files, name):
    """pco_b200_decompress_ex with the file and dst in device memory, with sentinel guard zones on both sides of dst; the whole file
    and a cap one past the first chunk."""
    import torch

    from pcodec_b200 import _lib

    data, nums, metas = cold_files[name]
    L = _lib.lib()
    guard = 4096
    src = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    for cap in (nums.size, metas[0]["n"] + 1):
        buf = torch.full(((2 * guard + cap) * 4,), 0xA5, dtype=torch.uint8, device="cuda")
        prog = _lib._CProgress()
        rc = L.pco_b200_decompress_ex(C.c_void_p(src.data_ptr()), C.c_size_t(len(data)), C.c_ubyte(1), C.c_void_p(buf.data_ptr() + 4 * guard), C.c_size_t(cap),
                                      C.byref(prog), None, C.c_size_t(0), C.c_uint32(_lib.SRC_ON_DEVICE | _lib.DST_ON_DEVICE),
                                      C.c_void_p(torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        assert rc == 0, _lib.lib().pco_b200_last_error_message()
        got = buf.cpu().numpy().view(np.uint32)
        k = min(cap, nums.size)
        assert (prog.n_processed, bool(prog.finished)) == (k, cap >= nums.size)
        _same(got[guard:guard + k], nums[:k])
        assert (got[:guard] == SENTINEL).all() and (got[guard + k:] == SENTINEL).all()


@gpu
def test_decompress_files_with_full_size_cold_files(oracle, cold_files):
    """pco_b200_decompress_files: Lookback 2^18, Dict 2^20, Conv1 2^17 and a window-17 file between fast files, with and without
    side indexes on the fast ones."""
    from tests.test_gpu_encode import _walk

    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec

    sa = _sa()
    fast_a = _walk(np.uint32, 70000, seed=23)
    fast_b = _walk(np.uint32, 3001, seed=24)
    fa = oracle.simple_compress(fast_a, oracle.make_config(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_CONSECUTIVE, delta_order=1))
    fb, fb_index = sa.simple_compress_with_index(fast_b, ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(1)))
    fa_index = sa.build_index(fa, np.uint32)
    items = [(fa, fast_a, fa_index)] + [(cold_files[k][0], cold_files[k][1], None) for k in ("lookback_2p18",)] + [(fb, fast_b, fb_index)] + \
            [(cold_files[k][0], cold_files[k][1], None) for k in ("dict_2p20", "conv1_2p17")] + [(fa, fast_a, fa_index)] + \
            [(cold_files["window_17"][0], cold_files["window_17"][1], None), (fb, fast_b, fb_index)]
    for with_index in (True, False):
        data, index, refs = bytearray(), bytearray(), []
        for blob, _, ix in items:
            io, il = 0, 0
            if with_index and ix is not None:
                index += b"\0" * (-len(index) % 16)
                io, il = len(index), len(ix)
                index += ix
            refs.append((len(data), len(blob), io, il))
            data += blob + b"\x07"
        files = np.array(refs, dtype=sa.FILE_REF)
        (vals, ns), prof = _profiled(lambda: sa.decompress_files(bytes(data), files, np.uint32, bytes(index) if with_index else None))
        np.testing.assert_array_equal(ns, [it[1].size for it in items])
        _same(vals, np.concatenate([it[1] for it in items]))
        assert "cold_decode_kernel=" in prof and "fused_narrow_kernel=" in prof, prof


@gpu
def test_decompress_pages_with_lookback_pages(oracle):
    """pco_b200_decompress_pages: wrapped Lookback chunks written by the oracle's ChunkCompressor, with pages of exactly 2^15 and of
    more than 2^15 numbers (each page restarts its window), the same pages under a meta patched to window 17, between fast pages."""
    from tests.test_gpu_encode import _walk

    from pcodec_b200 import wrapped

    O = oracle
    a = _motif(np.uint32, 3 * W + 77, seed=25)
    b = _motif(np.uint32, 2 * W + 600, seed=26)
    fast = _walk(np.uint32, 5000, seed=27)
    chunks = []
    for nums, cfg in [(fast, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=1)),
                      (a, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_LOOKBACK, exact_pages=[W, W + 1, W + 76])),
                      (b, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_LOOKBACK, max_page_n=W + 300))]:
        occ = O.ChunkCompressor(nums, cfg)
        meta = occ.write_meta()
        pages, start = [], 0
        for i, pn in enumerate(occ.n_per_page()):
            pages.append((occ.write_page(i), nums[start:start + pn]))
            start += pn
        chunks.append((meta, pages))
    for meta, _ in chunks[1:]:
        m, _ = insp.read_chunk_meta(meta, 0, 32)
        _assert_lookback(m, 15)
    assert [len(p) for _, p in chunks] == [1, 3, 2] and [p[1].size for p in chunks[1][1]] == [W, W + 1, W + 76]
    patched = (patch_window(chunks[1][0], 0, 32, 17), chunks[1][1])
    order = [chunks[0], chunks[1], chunks[0], patched, chunks[2], chunks[0]]
    metas, pages, refs, pieces, originals = bytearray(), bytearray(), [], [], []
    for (meta, pg), orig in zip(order, [c[0] for c in (chunks[0], chunks[1], chunks[0], chunks[1], chunks[2], chunks[0])]):
        m_off = len(metas)
        metas += meta
        for page, nums in pg:
            refs.append((m_off, len(meta), len(pages), len(page), nums.size))
            pages += page
            pieces.append(nums)
            originals.append((orig, page, nums))
    refs = np.array(refs, dtype=wrapped.PAGE_REF)
    got, prof = _profiled(lambda: wrapped.decompress_pages(bytes(metas), bytes(pages), refs, np.uint32))
    _same(got, np.concatenate(pieces))
    assert "fused_narrow_kernel=" in prof and prof.count("cold_decode_kernel=") == 2, prof
    at = 0
    for meta, page, nums in originals:
        theirs, _, _ = oracle.wrapped_decompress_page(meta, page, np.uint32, nums.size)
        _same(got[at:at + nums.size], theirs)
        at += nums.size


@gpu
@pytest.mark.parametrize("name", ["lookback_2p18", "lookback_3_chunks", "dict_2p20", "conv1_2p17"])
def test_index_paths_refuse_cold_files(cold_files, name):
    """build_index and decompress_ranges (which builds the index) decline files with chunks the fast kernels do not take: Unsupported,
    never numbers."""
    from pcodec_b200 import PcoError

    sa = _sa()
    data, _, _ = cold_files[name]
    with pytest.raises(PcoError) as e:
        sa.build_index(data, np.uint32)
    assert e.value.kind == "Unsupported", e.value
    with pytest.raises(PcoError) as e:
        sa.decompress_ranges(data, np.uint32, None, [(0, 10), (W, 5)])
    assert e.value.kind == "Unsupported", e.value


# ==== 6. The oracle's whole config space ========================================================================================
@st.composite
def _long_arrays(draw):
    """Motifs in chunks around the window size: 2^15 +- 1, 2^15 + 256, 2^16 + 1."""
    dtype = draw(st.sampled_from(DTYPES))
    n = draw(st.sampled_from([W - 1, W + 1, W + 256, (1 << 16) + 1]))
    period = draw(st.sampled_from([97, W - 1, W]))
    return _motif(dtype, n, period=period, seed=draw(st.integers(0, 2**31 - 1)), edit_every=draw(st.sampled_from([0, 211])))


@gpu
@settings(max_examples=300, deadline=None, suppress_health_check=[HealthCheck.too_slow, HealthCheck.data_too_large])
@given(data=st.data())
def test_gpu_decodes_every_oracle_config(oracle, data):
    """Auto, Dict, Lookback, Conv1, levels 0 to 12 and paging: whatever the oracle writes, the GPU decodes, whole and into partial
    destinations."""
    from pcodec_b200 import PcoError

    sa = _sa()
    long = data.draw(st.integers(0, 4)) == 0
    nums = data.draw(_long_arrays() if long else arrays())
    kw = data.draw(configs(nums.dtype))
    if long:
        kw["max_page_n"] = data.draw(st.sampled_from([0, W, W + 1]))
    cfg = oracle.make_config(**{k: getattr(oracle, v) if isinstance(v, str) else v for k, v in kw.items()})
    blob = oracle.simple_compress(nums, cfg)
    try:
        back = sa.simple_decompress(blob, nums.dtype)
    except PcoError as e:
        _dump_failure(nums, dict(kw, error=str(e), where="decompress"), None, blob)
        raise
    if back.size != nums.size or not np.array_equal(bits_view(back), bits_view(nums)):
        _dump_failure(nums, dict(kw, where="decode differs"), back.tobytes(), blob)
        raise AssertionError(f"GPU decode of the oracle's file differs: {kw}, dtype {nums.dtype}, n {nums.size} vs {back.size}")
    for m in sorted({0, min(3, nums.size), min(256, nums.size), nums.size // 2}):
        dst = np.zeros(m + 8, dtype=nums.dtype)
        prog = sa.simple_decompress_into(blob, dst[:m])
        assert (prog.n_processed, prog.finished) == (min(m, nums.size), m >= nums.size), (kw, m)
        _same(dst[:prog.n_processed], nums[:prog.n_processed])
        assert not bits_view(dst[m:]).any()
