"""The GPU planner's premise, checked on the CPU: replaying apply_incomplete / complete_bin / apply_constant_run from the order
statistics at the equal-count boundaries (DESIGN.md section 5, tests/planner_layouts.replay) gives the bins of the reference's
partial quicksort (the oracle's histograms.rs restatement), on layouts built to put runs exactly on, across and around the
boundaries, in shuffled, sorted and reversed order.  The replay counts the branches it takes, and each family of layouts must
reach the branch it was built for; the oracle counts its heapsort fallbacks, and no layout compared here may take one."""
import ctypes as C

import numpy as np
import pytest

from tests import planner_layouts as pl


def _hist(oracle, latents, log):
    a = np.ascontiguousarray(latents, dtype=np.uint64)
    out = (C.c_uint64 * (3 * (1 << log)))()
    n = C.c_size_t()
    assert oracle.lib().pco_oracle_kat_histogram_u64(a.ctypes.data_as(C.c_void_p), C.c_size_t(a.size), log, out, C.byref(n)) == 0
    return [tuple(out[3 * i: 3 * i + 3]) for i in range(n.value)]


def _hist_sorted(oracle, s, log):
    """apply_sorted over the whole sorted array in one slice (the tail of the reference's heapsort fallback)."""
    a = np.ascontiguousarray(s, dtype=np.uint32)
    lens = (C.c_size_t * 1)(a.size)
    out = (C.c_uint64 * (3 * (1 << log)))()
    inc = (C.c_uint64 * 3)()
    n_, has = C.c_size_t(), C.c_int()
    assert oracle.lib().pco_oracle_kat_histogram_sorted_u32(a.ctypes.data_as(C.c_void_p), lens, C.c_size_t(1), C.c_size_t(a.size), log, out,
                                                           C.byref(n_), inc, C.byref(has)) == 0
    assert not has.value
    return [tuple(out[3 * i: 3 * i + 3]) for i in range(n_.value)]


def _fallbacks(oracle):
    f = oracle.lib().pco_oracle_heapsort_fallbacks
    f.restype = C.c_uint64
    return int(f())


def _cases():
    """(n, bins_log): n around 2^(bins_log + 4) for every bins_log the levels reach, and small n whose bins hold one or two latents
    (bins_log = log2 n), or none at all (more bins than latents), as choose_unoptimized_bins_log gives them."""
    out = []
    for log in range(13):
        base = 1 << (log + 4)
        for n in (base - 1, base, base + 1, 3 * (1 << (log + 3)) + 5):
            out.append((n, log))
    for level, ns in ((8, (1, 2, 3, 5, 8, 15, 16, 17, 31)), (9, (32, 47, 63)), (10, (64, 100, 127)), (8, (300, 1000))):
        for n in ns:
            out.append((n, pl.choose_unoptimized_bins_log(level, n)))
    return sorted(set(out))


CASES = _cases()


def test_cases_cover_the_bin_logs():
    assert {log for _, log in CASES} == set(range(13))
    assert (16, 4) in CASES and (32, 5) in CASES and (64, 6) in CASES  # bins of one latent
    assert (300, 6) in CASES and (1000, 6) in CASES


@pytest.mark.parametrize("n,log", CASES, ids=[f"n{n}-log{log}" for n, log in CASES])
def test_replay_equals_the_quicksort(oracle, n, log):
    before = _fallbacks(oracle)
    for fam, layouts in pl.families(n, log, seed=n).items():
        for li, counts in enumerate(layouts):
            for gap in (1, 1031):
                s = pl.sorted_latents(counts, gap=gap, base=7)
                want = pl.replay(s, log)
                assert sum(c for c, _, _ in want) == n
                for order in pl.ORDERS:
                    got = _hist(oracle, pl.arrange(s, order, seed=li), log)
                    assert got == want, (fam, li, gap, order, counts[:20])
    assert _fallbacks(oracle) == before, "a layout took the heapsort fallback: its bins are not the replay's to compare"


# the branch each family is built to reach, where the bins are large enough to hold the shape
DESIGNED = {
    "F1": ("exact_fill",),
    "F2": ("run_ends_at_boundary",),
    "F3": ("straddle_by_one",),
    "F4": ("spare_completed", "spare_declined"),
    "F5": ("mid_on_boundary", "mid_next_to_boundary"),
    "F6": ("back_to_back", "skipped_bins"),
    "F7": ("clean", "straddle", "spare_declined"),
    "F8": ("straddle",),
}
SHAPED = [(n, log) for n, log in CASES if log >= 3 and n >= 8 << log]


@pytest.mark.parametrize("n,log", SHAPED, ids=[f"n{n}-log{log}" for n, log in SHAPED])
def test_every_family_reaches_its_branch(n, log):
    for fam, layouts in pl.families(n, log, seed=n).items():
        stats = {}
        for counts in layouts:
            pl.replay(pl.sorted_latents(counts), log, stats)
        for branch in DESIGNED[fam]:
            assert stats[branch] > 0, (fam, branch, stats)


def test_f2_after_skipped_bins_pins_the_apply_sorted_divergence(oracle):
    """histograms.rs:250-258: after too many bad pivots the reference heapsorts a slice and runs apply_sorted over it.  apply_sorted
    treats the latent at every boundary as a constant run even when the boundary is clean, so a run that ends exactly at C(k) behind
    distinct values, after a multi-bin run that left next_avail_bin_idx behind, completes the distinct values as a spare bin of
    their own.  The quicksort (and the GPU's replay) keeps them with the run.  64 latents, 4 bins of 16: a run of 40 zeros, then
    1, 2, 3, 4 and four 5s ending at C(2) = 48, then 16 distinct values."""
    counts = [40, 1, 1, 1, 1, 4] + [1] * 16
    s = pl.sorted_latents(counts, dtype=np.uint32)
    stats = {}
    replayed = pl.replay(s, 2, stats)
    assert stats["run_ends_at_boundary"] == 1 and stats["spare_declined"] == 1
    assert replayed == [(40, 0, 0), (8, 1, 5), (16, 6, 21)]
    assert _hist(oracle, np.random.default_rng(3).permutation(s), 2) == replayed
    assert _hist_sorted(oracle, s, 2) == [(40, 0, 0), (4, 1, 4), (4, 5, 5), (16, 6, 21)]
