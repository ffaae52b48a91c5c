"""Layouts of stored latents at the edges of the equal-count histogram, and a plain restatement of the GPU planner's replay.

pco's unoptimized histogram (pco/src/histograms.rs:87-281) cuts the sorted latents at the boundaries B = c_count(k) =
ceil((k + 1) * n / 2^bins_log) (:132-140).  A run of equal latents never splits, so a run that meets a boundary decides where a
bin ends: `apply_constant_run` (:142-161) puts it in the bin of its midpoint, and first completes the bin before that ("the spare
bin") when the run's midpoint lies beyond the next free bin index.  The GPU planner does not sort like the reference: its probe
kernels read the order statistics at every boundary (s[B-1], s[B] and, where they are equal, the run's extent [l, r)) and the
solvers replay apply_incomplete / complete_bin / apply_constant_run from them (DESIGN.md section 5).  `replay` below is that replay
over a sorted array, in Python; `families` builds sorted run lists that put runs exactly where the replay branches:

* F1: a run that fills a bin [C(k-1), C(k)) exactly;
* F2: a run that ends exactly at C(k), behind distinct values of the same bin (also after skipped bin indices);
* F3: runs [C(k)-1, C(k)+1), [C(k)-1, C(k)+m) and [C(k), C(k)+m);
* F4: runs over 2, 3 and nbk-1 bins that start one before, at and one after a boundary (spare bin completed or declined);
* F5: runs whose midpoint start + len/2 is C(k) or C(k) +- 1;
* F6: multi-bin runs back to back (bin indices skipped);
* F7: all distinct, all one value, n-1 copies of one value and one other value below or above;
* F8: seeded random compositions of run lengths near the bin size.

A layout is a list of run lengths in value order; `sorted_latents` gives them values `gap` apart (and optionally stretches the
last value to a given key range), `arrange` puts them in a seeded shuffled, sorted or reversed order.
"""
import numpy as np


def c_count(k, n, log):  # histograms.rs:139
    return ((k + 1) * n + (1 << log) - 1) >> log


def bin_idx(c, n, log):  # histograms.rs:135
    return (c << log) // n


def choose_unoptimized_bins_log(level, n):  # pco/src/wrapped/chunk_compressor.rs:362-371
    log_n = max(int(n).bit_length() - 1, 0)
    fast = log_n - 4 if log_n >= 4 else 0
    return level if level <= fast else fast + (level - fast) // 2


# ---- building run lists

def compose(n, runs, fill=1):
    """Run lengths summing to n: the runs [start, start + length) given (sorted, non-overlapping, clipped to n), and between them
    filler runs of `fill` latents each (distinct values)."""
    out, pos = [], 0
    for start, length in sorted(runs):
        start, end = max(start, pos), min(start + length, n)
        if end <= start:
            continue
        while pos < start:
            step = min(fill, start - pos)
            out.append(step)
            pos += step
        out.append(end - start)
        pos = end
    while pos < n:
        step = min(fill, n - pos)
        out.append(step)
        pos += step
    assert sum(out) == n and all(c > 0 for c in out)
    return out


def _ks(nbk, *picks):
    """Distinct bin indices in range, in order: picks may be negative (from the end)."""
    ks = sorted({(k if k >= 0 else nbk + k) for k in picks if -nbk <= k < nbk})
    return ks


def families(n, log, seed=0, fill=1):
    """{family: [run lengths, ...]} for n latents and 2^log bins."""
    nbk = 1 << log
    C = lambda k: c_count(k, n, log) if k >= 0 else 0  # noqa: E731
    bin_n = max(n // nbk, 1)
    fam = {f"F{i}": [] for i in range(1, 9)}
    # F1: runs that fill bins exactly (every third bin from a few places, so that the runs do not touch)
    fam["F1"].append(compose(n, [(C(k - 1), C(k) - C(k - 1)) for k in _ks(nbk, 0, 2, nbk // 2, -1)], fill))
    fam["F1"].append(compose(n, [(C(k - 1), C(k) - C(k - 1)) for k in range(1, nbk, 3)], fill))
    # F2: a run ending exactly at C(k) behind distinct values of the bin
    if bin_n >= 3:
        runs = []
        for k in _ks(nbk, 1, nbk // 2, -1):
            length = max(2, (C(k) - C(k - 1)) // 2)
            runs.append((C(k) - length, length))
        fam["F2"].append(compose(n, runs, 1))
        # ... after skipped bin indices: a run over 2.5 bins from 0 leaves next_avail_bin_idx behind the bin it ends in
        if nbk >= 4:
            k = bin_idx(C(1) + bin_n // 2, n, log)
            length = max(2, (C(k) - C(1) - bin_n // 2) // 2)
            fam["F2"].append(compose(n, [(0, C(1) + bin_n // 2), (C(k) - length, length)], 1))
    # F3: runs straddling a boundary by one
    if nbk >= 2:
        m = max(2, bin_n // 2)
        ks = _ks(nbk, 0, nbk // 3, (2 * nbk) // 3)
        shapes = [(-1, 2), (-1, 1 + m), (0, m)]
        runs = [(C(k) + d, length) for k, (d, length) in zip(ks, shapes)]
        fam["F3"].append(compose(n, runs, fill))
        for d, length in shapes:  # each shape at every boundary it fits, far apart
            fam["F3"].append(compose(n, [(C(k) + d, length) for k in range(0, nbk - 1, 4)], fill))
    # F4: multi-bin runs, starting one before, at and one after a boundary
    for span in sorted({2, 3, nbk - 1}):
        if span < 2 or span >= nbk + 1:
            continue
        for d in (-1, 0, 1):
            for k in _ks(nbk, 0, nbk // 2 - 1):
                start = C(k) + d
                if start < 0 or start >= n:
                    continue
                fam["F4"].append(compose(n, [(start, span * bin_n)], fill))
    # F5: midpoints on and next to a boundary
    for d in (-1, 0, 1):
        for length in sorted({bin_n, bin_n + 1, 2 * bin_n + 1, 3}):
            runs, last = [], -1
            for k in range(0, nbk - 1, max(1, nbk // 4)):
                start = C(k) + d - length // 2
                if start > last and start >= 0:
                    runs.append((start, length))
                    last = start + length
            if runs:
                fam["F5"].append(compose(n, runs, fill))
    # F6: multi-bin runs back to back
    if nbk >= 4:
        for first in (C(0), C(0) + 1, 1):
            runs, pos = [], first
            for length in (2 * bin_n, 2 * bin_n + 1, 3 * bin_n - 1, bin_n + 1):
                runs.append((pos, length))
                pos += length
            fam["F6"].append(compose(n, runs, fill))
    # F7: degenerate layouts
    fam["F7"] += [[1] * n, [n]]
    if n >= 2:
        fam["F7"] += [[1, n - 1], [n - 1, 1]]
    # F8: seeded random compositions of lengths near the bin size
    rng = np.random.default_rng(seed * 1000003 + n * 31 + log)
    choices = sorted({1, 2, max(bin_n - 1, 1), bin_n, bin_n + 1, max(2 * bin_n - 1, 1), 2 * bin_n + 1, 3 * bin_n, max(bin_n // 2, 1)})
    for _ in range(3):
        out, left = [], n
        while left > 0:
            c = min(int(rng.choice(choices)), left)
            out.append(c)
            left -= c
        fam["F8"].append(out)
    return {k: v for k, v in fam.items() if v}


def sorted_latents(counts, gap=1, base=0, span=None, dtype=np.uint64):
    """The sorted latents of a run list: run i takes base + i * gap; with `span`, the last run's value is base + span instead (the
    key range max - min of the layout, chosen on purpose)."""
    m = len(counts)
    vals = base + np.arange(m, dtype=np.uint64) * np.uint64(gap)
    if span is not None and m > 1:
        assert span > (m - 2) * gap, (span, m, gap)
        vals[-1] = np.uint64(base + span)
    return np.repeat(vals, counts).astype(dtype)


def key_span(counts, gap, span=None):
    return 0 if len(counts) < 2 else (span if span is not None else (len(counts) - 1) * gap)


ORDERS = ("shuffled", "sorted", "reversed")


def arrange(s, order, seed=0):
    if order == "sorted":
        return s.copy()
    if order == "reversed":
        return s[::-1].copy()
    return np.random.default_rng(seed).permutation(s)


# ---- the replay (DESIGN.md section 5; plan_solve_kernel / plan_solve_wide_kernel do the same from the probes)

BRANCHES = ("clean", "exact_fill","run_ends_at_boundary", "straddle", "straddle_by_one", "spare_completed", "spare_declined",
            "mid_on_boundary", "mid_next_to_boundary", "skipped_bins", "back_to_back")


def replay(s, log, stats=None):
    """The unoptimized histogram of the sorted latents `s` as [(count, lower, upper)], replayed boundary by boundary from the order
    statistics the probe kernels read.  `stats` (a dict) counts the branches taken."""
    s = np.asarray(s)
    n = int(s.size)
    st = stats if stats is not None else {}
    for b in BRANCHES:
        st.setdefault(b, 0)
    if n == 0:
        return []
    C = lambda k: c_count(k, n, log)  # noqa: E731
    B_of = lambda c: bin_idx(c, n, log)  # noqa: E731
    hist = []
    inc = None  # [count, lower, upper] of the incomplete bin
    next_avail = 0

    def apply_incomplete(cnt, lo, hi):
        nonlocal inc
        if cnt == 0:
            return
        if inc is None:
            inc = [cnt, lo, hi]
        else:
            inc[0] += cnt
            inc[2] = hi

    def complete_bin(b):
        nonlocal inc, next_avail
        if inc is None:
            return False
        if b > next_avail:
            st["skipped_bins"] += 1
        next_avail = b + 1
        hist.append(tuple(inc))
        inc = None
        return True

    pos, prev_run_end = 0, -1
    while pos < n:
        k = B_of(pos)
        B = C(k)
        vb1 = int(s[B - 1])
        if B >= n or vb1 != int(s[B]):
            first = int(s[pos])
            start_k = C(k - 1) if k > 0 else 0
            st["clean"] += 1
            if first == vb1 and pos == start_k:
                st["exact_fill"] += 1
            elif first != vb1 and B >= 2 and int(s[B - 2]) == vb1:
                st["run_ends_at_boundary"] += 1
            apply_incomplete(B - pos, first, vb1)
            complete_bin(k)
            pos = B
            continue
        l = int(np.searchsorted(s, s[B - 1], "left"))
        r = int(np.searchsorted(s, s[B - 1], "right"))
        st["straddle"] += 1
        if l == B - 1 or r == B + 1:
            st["straddle_by_one"] += 1
        if l == pos and prev_run_end == pos:
            st["back_to_back"] += 1
        if l > pos:
            apply_incomplete(l - pos, int(s[pos]), int(s[l - 1]))
        # apply_constant_run (histograms.rs:142-161)
        mid = l + (r - l) // 2
        b = B_of(mid)
        j = B_of(mid)
        near = [abs(mid - C(q)) for q in (j - 1, j) if q >= 0]
        if 0 in near:
            st["mid_on_boundary"] += 1
        elif 1 in near:
            st["mid_next_to_boundary"] += 1
        if b > next_avail:
            if complete_bin(b - 1):
                st["spare_completed"] += 1
            else:
                st["spare_declined"] += 1
                b -= 1
        apply_incomplete(r - l, vb1, vb1)
        if r >= C(b):
            complete_bin(b)
        pos = prev_run_end = r
    return hist
