"""The GPU planner at the edges of the equal-count histogram, on every planner path, against the oracle.

Each layout of tests/planner_layouts.py (runs that fill a bin, end on a boundary, straddle it by one, span several bins, have
their midpoint on a boundary, follow each other, ...) is turned into numbers whose stored latents are that layout, and compressed
through each way the GPU builds a histogram:

* the one-pass front end (split_count_kernel) - classic mode, key range below 2^15, levels up to 8;
* the redo on the sort path (split_count_kernel flags the chunk; sort_keys_kernel + radix_sort_segments_kernel +
  plan_probe_kernel_sorted) - a key range of exactly 2^15, wider gaps, and a file mixing a narrow chunk with a wide one;
* the two-kernel counting path (plan_probe_kernel_counting) - IntMult, whose two latent vars are both layouts;
* the wide solver (plan_solve_wide_kernel) - levels 9-12 at unoptimized bins logs 9-12, counting and sorted keys;
* the pages of one wrapped chunk (union_probe_kernel, or the union sort when the pages together span 2^15 or more);
* per-chunk bins logs (compress_files, and the CHUNK_BINS kernels of AsyncFilesCompressor), files on both sides of powers of two;
* the asynchronous compress (AsyncCompressor).

Every file must equal the oracle's byte for byte and decode on the GPU to the input.  The profiler's kernel spans show which path
ran.  A mismatch prints both files' bins and keeps the case (numbers, config, both files) like test_gpu_properties.
"""
import ctypes as C

import numpy as np
import pytest

from tests import planner_layouts as pl
from tests.golden_generators import bits_view
from tests.test_gpu_properties import _dump_failure

pytestmark = pytest.mark.gpu

COUNT_LIMIT = (1 << 15) - 1  # widest key range (max - min) the counting planner takes
DT = {"u8": np.uint8, "u16": np.uint16, "u32": np.uint32, "u64": np.uint64, "i64": np.int64, "f32": np.float32}


# ---- numbers whose stored latents are a layout

def from_latents(lat, dtype):
    """Classic order 0: the numbers whose ordered latents are `lat` (uint64)."""
    dt = np.dtype(dtype)
    bits = dt.itemsize * 8
    u = lat.astype(np.uint64) & np.uint64((1 << bits) - 1)
    if dt.kind == "u":
        return u.astype(dt)
    ut = np.dtype(f"u{dt.itemsize}")
    mid = np.uint64(1 << (bits - 1))
    if dt.kind == "i":
        return (u ^ mid).astype(ut).view(dt)
    # floats: the order-preserving bit map (positive: sign bit set in the latent; negative: all bits flipped)
    x = u.astype(ut)
    m = ut.type(1 << (bits - 1))
    return np.where(x & m, x ^ m, ~x).astype(ut).view(dt)


def from_deltas(stored, order, dtype, seed=0):
    """Unsigned numbers whose consecutive deltas of `order` (centred: + MID, delta/mod.rs toggle_center) are `stored`."""
    dt = np.dtype(dtype)
    bits = dt.itemsize * 8
    mask = (1 << bits) - 1
    d = (stored.astype(np.uint64) - np.uint64(1 << (bits - 1))) & np.uint64(mask)
    rng = np.random.default_rng(seed)
    for _ in range(order):
        head = np.array([int(rng.integers(0, 1 << 30))], dtype=np.uint64)
        d = np.cumsum(np.concatenate([head, d]), dtype=np.uint64) & np.uint64(mask)
    return d.astype(dt)


def _layout_cases(n, log, fill=1):
    out = []
    for fam, layouts in pl.families(n, log, seed=n, fill=fill).items():
        for i, counts in enumerate(layouts):
            out.append((f"{fam}.{i}", counts))
    return out


def _counting_gap(counts, want=1031):
    """The largest gap up to `want` that keeps the layout's key range countable, or None."""
    if len(counts) < 2:
        return want
    g = min(want, COUNT_LIMIT // (len(counts) - 1))
    return g if g >= 1 else None


# ---- configs, profiling, checks

def _cfgs(oracle, level=8, mode="classic", order=0, ibase=0, exact=None):
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec

    ms = ModeSpec.try_int_mult(ibase) if mode == "int_mult" else ModeSpec.classic()
    om = oracle.MODE_INT_MULT if mode == "int_mult" else oracle.MODE_CLASSIC
    ps = PagingSpec.exact_page_sizes(exact) if exact else PagingSpec.equal_pages_up_to(1 << 18)
    ours = ChunkConfig(compression_level=level, mode_spec=ms, delta_spec=DeltaSpec.try_consecutive(order) if order else DeltaSpec.no_op(), paging_spec=ps,
                       enable_8_bit=True)
    theirs = oracle.make_config(level=level, mode=om, delta=oracle.DELTA_CONSECUTIVE if order else oracle.DELTA_NOOP, delta_order=order,
                                int_mult_base=ibase, exact_pages=exact)
    return ours, theirs


class _Spans:
    """Kernel spans of the calls made inside the block (pco_b200_profile_enable / pco_b200_profile_last)."""

    def __enter__(self):
        from pcodec_b200 import _lib

        self.L = _lib.lib()
        self.L.pco_b200_profile_enable(1)
        return self

    def read(self):
        buf = C.create_string_buffer(1 << 16)
        self.L.pco_b200_profile_last(buf, C.c_size_t(len(buf)))
        return {kv.split("=")[0] for kv in buf.value.decode().split(";") if kv}

    def __exit__(self, *exc):
        self.L.pco_b200_profile_enable(0)


def _bins(oracle, data, dtype):
    """[weight, lower, offset bits] of every bin of every chunk and var, as the oracle reads the file."""
    try:
        return [v.get("bins", []) for ch in oracle.inspect(data, dtype)["chunks"] for v in ch["vars"]]
    except Exception as e:  # a file the oracle cannot even read is its own finding
        return f"unreadable: {e}"


def _mismatch(oracle, nums, kw, got, want):
    _dump_failure(nums, kw, got, want)
    print("GPU bins:   ", _bins(oracle, got, nums.dtype))
    print("oracle bins:", _bins(oracle, want, nums.dtype))
    m = min(len(got), len(want))
    d = np.flatnonzero(np.frombuffer(got[:m], np.uint8) != np.frombuffer(want[:m], np.uint8))
    return f"{kw}: {len(got)} bytes vs the oracle's {len(want)}, first difference at byte {int(d[0]) if d.size else m}"


def _check(oracle, nums, kw, want_spans=(), no_spans=(), **cfg):
    """GPU bytes == oracle bytes and GPU decode == input, with the spans the path must (and must not) show."""
    from pcodec_b200 import standalone

    ours, theirs = _cfgs(oracle, **cfg)
    want = oracle.simple_compress(nums, theirs)
    with _Spans() as sp:
        got = standalone.simple_compress(nums, ours)
        spans = sp.read()
    if got != want:
        raise AssertionError(_mismatch(oracle, nums, kw, got, want))
    for s in want_spans:
        assert s in spans, (kw, s, sorted(spans))
    for s in no_spans:
        assert s not in spans, (kw, s, sorted(spans))
    back = standalone.simple_decompress(got, nums.dtype)
    if not np.array_equal(bits_view(back), bits_view(nums)):
        _dump_failure(nums, dict(kw, where="decode differs"), back.tobytes(), want)
        raise AssertionError(f"{kw}: the GPU decode differs from the input")
    return got


ONE_PASS = ("split_count_kernel",), ("split_delta_kernel",)
SORTED = ("split_delta_kernel", "radix_sort_segments_kernel", "plan_probe_kernel_sorted", "plan_solve_kernel")


# ---- one-pass front end: classic, key range below 2^15, levels <= 8

ONE_PASS_SIZES = [(4095, 8), (4096, 8), (4097, 8), (3 * 2048 + 5, 8), (1000, 8), (300, 8), (16, 8), (17, 8), (31, 8), (2049, 4)]


@pytest.mark.parametrize("dtype", ["u32", "u64", "i64", "f32", "u16", "u8"])
@pytest.mark.parametrize("n,level", ONE_PASS_SIZES, ids=[f"n{n}-L{lv}" for n, lv in ONE_PASS_SIZES])
def test_one_pass(oracle, dtype, n, level):
    dt = np.dtype(DT[dtype])
    log = pl.choose_unoptimized_bins_log(level, n)
    base = {"f32": 0xBF800000, "i64": (1 << 63) - 5000}.get(dtype, 3)
    limit = 255 if dtype == "u8" else COUNT_LIMIT
    # u8 holds at most 256 distinct latents: longer filler runs between the shaped ones
    for name, counts in _layout_cases(n, log, fill=-(-n // 160) if dtype == "u8" else 1):
        gap = 1 if dtype == "u8" else _counting_gap(counts)
        if gap is None or pl.key_span(counts, gap) > limit:
            continue
        s = pl.sorted_latents(counts, gap=gap, base=base)
        orders = pl.ORDERS if dtype in ("u32", "u16") else ("shuffled",)
        for order in orders:
            nums = from_latents(pl.arrange(s, order, seed=n), dt)
            _check(oracle, nums, dict(path="one_pass", layout=name, gap=gap, order=order, level=level), *ONE_PASS, level=level)
        if dtype in ("u32", "u16") and len(counts) > 1:  # the widest countable range: the last value at min + 2^15 - 1
            s = pl.sorted_latents(counts, gap=1, base=base, span=COUNT_LIMIT)
            _check(oracle, from_latents(pl.arrange(s, "shuffled", seed=1), dt), dict(path="one_pass", layout=name, span=COUNT_LIMIT), *ONE_PASS, level=level)


@pytest.mark.parametrize("order", [1, 2])
@pytest.mark.parametrize("dtype", ["u32", "u64"])
def test_one_pass_consecutive(oracle, dtype, order):
    """Consecutive orders 1 and 2: numbers whose stored deltas are the layout (confirmed by the oracle's encode for u32)."""
    dt = np.dtype(DT[dtype])
    for n_stored in (4096, 4097, 3 * 2048 + 5):
        log = pl.choose_unoptimized_bins_log(8, n_stored + order)
        for name, counts in _layout_cases(n_stored, log):
            gap = _counting_gap(counts)
            if gap is None:
                continue
            stored = pl.sorted_latents(counts, gap=gap, base=(1 << (dt.itemsize * 8 - 1)) - 20000)
            stored = pl.arrange(stored, "shuffled", seed=n_stored)
            nums = from_deltas(stored, order, dt, seed=n_stored)
            if dtype == "u32":
                lat = nums.copy()
                mom = (C.c_uint32 * order)()
                assert oracle.lib().pco_oracle_kat_consecutive_encode_u32(lat.ctypes.data_as(C.c_void_p), C.c_size_t(lat.size), C.c_size_t(order), mom) == 0
                np.testing.assert_array_equal(lat[order:], stored.astype(np.uint32))
            _check(oracle, nums, dict(path="one_pass", layout=name, order=order), *ONE_PASS, level=8, order=order)


# ---- redo on the sort path: key range exactly 2^15, wide gaps, a narrow and a wide chunk in one call

@pytest.mark.parametrize("dtype", ["u32", "u64", "u16"])
@pytest.mark.parametrize("n", [4096, 4097, 3 * 2048 + 5, 1000])
def test_redo_sorted(oracle, dtype, n):
    dt = np.dtype(DT[dtype])
    log = pl.choose_unoptimized_bins_log(8, n)
    for name, counts in _layout_cases(n, log):
        if len(counts) < 2:
            continue
        for gap, span in ((1, 1 << 15), (1031, None)):
            if span is None and (dtype == "u16" or pl.key_span(counts, gap) < (1 << 15)):
                continue
            s = pl.sorted_latents(counts, gap=gap, base=11, span=span)
            assert pl.key_span(counts, gap, span) >= (1 << 15)
            nums = from_latents(pl.arrange(s, "shuffled", seed=n), dt)
            _check(oracle, nums, dict(path="redo_sorted", layout=name, gap=gap, span=span), ("split_count_kernel",) + SORTED, level=8)


@pytest.mark.parametrize("dtype", ["u32", "u64"])
def test_narrow_and_wide_chunk_in_one_call(oracle, dtype):
    dt = np.dtype(DT[dtype])
    n1, n2 = 4097, 3 * 2048 + 5
    l1, l2 = (pl.choose_unoptimized_bins_log(8, n) for n in (n1, n2))
    narrow = dict(_layout_cases(n1, l1))
    wide = dict(_layout_cases(n2, l2))
    for name in sorted(set(narrow) & set(wide)):
        if len(narrow[name]) < 2 or len(wide[name]) < 2:
            continue
        a = pl.sorted_latents(narrow[name], gap=1, base=5, span=COUNT_LIMIT)
        b = pl.sorted_latents(wide[name], gap=1, base=5, span=1 << 15)
        for first, second in ((a, b), (b, a)):
            nums = from_latents(np.concatenate([pl.arrange(first, "shuffled", 1), pl.arrange(second, "reversed")]), dt)
            _check(oracle, nums, dict(path="mixed_chunks", layout=name), ("split_count_kernel",) + SORTED, level=8, exact=[first.size, second.size])


# ---- two-kernel counting path: IntMult (two latent vars, both layouts)

@pytest.mark.parametrize("dtype", ["u32", "u64"])
@pytest.mark.parametrize("n", [4096, 4097, 3 * 2048 + 5])
def test_int_mult_counting(oracle, dtype, n):
    dt = np.dtype(DT[dtype])
    ibase = 4099
    log = pl.choose_unoptimized_bins_log(8, n)
    adj_layouts = [c for _, c in _layout_cases(n, min(log, 6)) if len(c) <= ibase]
    for i, (name, counts) in enumerate(_layout_cases(n, log)):
        gap = _counting_gap(counts, 7)
        if gap is None:
            continue
        mult = pl.arrange(pl.sorted_latents(counts, gap=gap, base=100), "shuffled", seed=i)
        adj = pl.arrange(pl.sorted_latents(adj_layouts[i % len(adj_layouts)], gap=1, base=0), "shuffled", seed=i + 1)
        assert int(adj.max()) < ibase
        nums = (mult * np.uint64(ibase) + adj).astype(dt)
        _check(oracle, nums, dict(path="int_mult", layout=name), ("split_delta_kernel", "plan_probe_kernel_counting", "plan_solve_kernel"),
               ("split_count_kernel",), level=8, mode="int_mult", ibase=ibase)


# ---- wide solver: levels 9-12 at unoptimized bins logs 9-12, counting and sorted keys

WIDE_CASES = [(lv, n, dtype) for lv in (9, 10, 11, 12) for n in ((1 << (lv + 4)) + 1, 3 * (1 << (lv + 3)) + 5)
              for dtype in (("u32", "u64") if lv in (9, 12) else ("u32",))] + [(9, 1 << 13, "u32"), (12, (1 << 16) - 1, "u32")]


@pytest.mark.parametrize("level,n,dtype", WIDE_CASES, ids=[f"L{lv}-n{n}-{d}" for lv, n, d in WIDE_CASES])
def test_wide(oracle, level, n, dtype):
    dt = np.dtype(DT[dtype])
    log = pl.choose_unoptimized_bins_log(level, n)
    assert log >= 9 or n < (1 << (level + 4))
    for name, counts in _layout_cases(n, log, fill=3):
        gap = _counting_gap(counts)
        if gap is not None and len(counts) > 1:
            s = pl.sorted_latents(counts, gap=gap, base=9)
            _check(oracle, from_latents(pl.arrange(s, "shuffled", seed=n), dt), dict(path="wide_counting", layout=name, level=level),
                   ("plan_probe_kernel_counting", "plan_solve_wide_kernel"), ("plan_probe_kernel_sorted",), level=level)
        if len(counts) > 1:
            s = pl.sorted_latents(counts, gap=1031, base=9, span=None if pl.key_span(counts, 1031) >= (1 << 15) else 1 << 15)
            _check(oracle, from_latents(pl.arrange(s, "shuffled", seed=n + 1), dt), dict(path="wide_sorted", layout=name, level=level),
                   ("radix_sort_segments_kernel", "plan_probe_kernel_sorted", "plan_solve_wide_kernel"), level=level)


# ---- pages of one wrapped chunk: shared bins over the union of the pages

def _wrapped_check(oracle, nums, pages, kw, want_spans, no_spans=()):
    from pcodec_b200 import wrapped

    ours, theirs = _cfgs(oracle, exact=pages)
    occ = oracle.ChunkCompressor(nums, theirs)
    with _Spans() as sp:
        cc = wrapped.FileCompressor().chunk_compressor(nums, ours)
        spans = sp.read()
    meta = cc.write_meta()
    want_meta = occ.write_meta()
    if meta != want_meta:
        raise AssertionError(_mismatch(oracle, nums, dict(kw, part="meta"), meta, want_meta))
    assert cc.n_per_page() == list(pages)
    off = 0
    for i, pn in enumerate(pages):
        page, want_page = cc.write_page(i), occ.write_page(i)
        if page != want_page:
            raise AssertionError(_mismatch(oracle, nums[off: off + pn], dict(kw, part=f"page {i}"), page, want_page))
        back, _, _ = oracle.wrapped_decompress_page(meta, page, nums.dtype, pn)
        np.testing.assert_array_equal(bits_view(back), bits_view(nums[off: off + pn]))
        off += pn
    for s in want_spans:
        assert s in spans, (kw, s, sorted(spans))
    for s in no_spans:
        assert s not in spans, (kw, s, sorted(spans))


@pytest.mark.parametrize("n", [4096, 4097, 3 * 2048 + 5])
def test_shared_pages(oracle, n):
    log = pl.choose_unoptimized_bins_log(8, n)
    pages = [n // 3, n // 3, n - 2 * (n // 3)]
    union_wide = 0
    for name, counts in _layout_cases(n, log):
        gap = _counting_gap(counts)
        if gap is None:
            continue
        s = pl.sorted_latents(counts, gap=gap, base=3)
        for order in pl.ORDERS:
            nums = pl.arrange(s, order, seed=n).astype(np.uint32)
            _wrapped_check(oracle, nums, pages, dict(path="union_narrow", layout=name, order=order), ("split_count_kernel", "union_probe_kernel"),
                           ("union_sort_keys_kernel", "split_delta_kernel"))
        # every page narrow, the union not: values spread over 2^15 + 2^13, which sorted order cuts into three narrower spans
        if len(counts) < 2:
            continue
        s = pl.sorted_latents(counts, gap=-(-((1 << 15) + (1 << 13)) // (len(counts) - 1)), base=3)
        cuts = np.cumsum([0] + pages)
        if all(int(s[b - 1]) - int(s[a]) <= COUNT_LIMIT for a, b in zip(cuts[:-1], cuts[1:])):
            union_wide += 1
            _wrapped_check(oracle, s.astype(np.uint32), pages, dict(path="union_wide", layout=name), ("union_probe_kernel", "union_range_kernel",
                           "union_sort_keys_kernel", "union_radix_sort_kernel", "union_plan_probe_kernel_sorted"))
    assert union_wide >= 5  # the generator must keep reaching the case


# ---- per-chunk bins logs: a batch of files on both sides of powers of two, each with a layout made for its own n

FILE_NS = [16, 17, 31, 32, 33, 255, 256, 257, 1023, 1024, 1025, 4095, 4096, 4097]


def _files(level, seed):
    rng = np.random.default_rng(seed)
    parts = []
    for n in FILE_NS:
        log = pl.choose_unoptimized_bins_log(level, n)
        cases = _layout_cases(n, log)
        name, counts = cases[int(rng.integers(len(cases)))]
        gap = _counting_gap(counts) or 1
        parts.append(pl.arrange(pl.sorted_latents(counts, gap=gap, base=1), "shuffled", seed=seed + n))
    return parts


@pytest.mark.parametrize("dtype", ["u32", "u64"])
@pytest.mark.parametrize("seed", range(4))
def test_files_per_chunk_bins_log(oracle, dtype, seed):
    import torch

    from pcodec_b200 import standalone

    dt = np.dtype(DT[dtype])
    parts = [p.astype(dt) for p in _files(8, seed)]
    ns = [p.size for p in parts]
    nums = np.concatenate(parts)
    ours, theirs = _cfgs(oracle)
    data, files, _ = standalone.compress_files(nums, ns, ours)
    wants = [oracle.simple_compress(p, theirs) for p in parts]
    for i, (p, w) in enumerate(zip(parts, wants)):
        got = data[int(files[i]["offset"]): int(files[i]["offset"] + files[i]["len"])]
        if got != w:
            raise AssertionError(_mismatch(oracle, p, dict(path="compress_files", file=i, n=p.size, seed=seed), got, w))
        np.testing.assert_array_equal(standalone.simple_decompress(got, dt), p)
    # the CHUNK_BINS kernels: the same batch through AsyncFilesCompressor, sizes in device memory
    comp = standalone.AsyncFilesCompressor(dt, ours, max_files=len(ns), nums_cap=nums.size, max_file_n=max(ns))
    dev = torch.from_numpy(nums).cuda()
    file_ns = torch.tensor(ns, dtype=torch.int64, device="cuda")
    n_files = torch.tensor([len(ns)], dtype=torch.int64, device="cuda")
    dst = torch.empty(comp.dst_cap, dtype=torch.uint8, device="cuda")
    refs = torch.zeros((comp.max_files, 4), dtype=torch.int64, device="cuda")
    comp(dev, file_ns, n_files, dst, None, refs)
    dl, _ = comp.result()
    out = dst[:dl].cpu().numpy().tobytes()
    r = refs.cpu().numpy()
    for i, (p, w) in enumerate(zip(parts, wants)):
        got = out[int(r[i, 0]): int(r[i, 0] + r[i, 1])]
        if got != w:
            raise AssertionError(_mismatch(oracle, p, dict(path="compress_files_async", file=i, n=p.size, seed=seed), got, w))


# ---- the asynchronous compress on a subset

@pytest.mark.parametrize("dtype", ["u32", "u64"])
@pytest.mark.parametrize("n,level", [(4097, 8), (3 * 2048 + 5, 8), (2049, 4), (300, 8)])
def test_async_compress(oracle, dtype, n, level):
    import torch

    from pcodec_b200 import standalone

    dt = np.dtype(DT[dtype])
    log = pl.choose_unoptimized_bins_log(level, n)
    ours, theirs = _cfgs(oracle, level=level)
    comp = standalone.AsyncCompressor(n, dt, ours, index=False)
    dst = torch.empty(comp.dst_cap, dtype=torch.uint8, device="cuda")
    for name, counts in _layout_cases(n, log):
        for gap, span in ((_counting_gap(counts), None), (1, 1 << 15)):
            if gap is None or (span is not None and len(counts) < 2):
                continue
            nums = from_latents(pl.arrange(pl.sorted_latents(counts, gap=gap, base=2, span=span), "shuffled", seed=n), dt)
            want = oracle.simple_compress(nums, theirs)
            assert standalone.simple_compress(nums, ours) == want, (name, gap, span)
            comp(torch.from_numpy(nums).cuda(), dst)
            nw, _ = comp.result()
            got = dst[:nw].cpu().numpy().tobytes()
            if got != want:
                raise AssertionError(_mismatch(oracle, nums, dict(path="async", layout=name, gap=gap, span=span), got, want))
