"""numpy reference of the segment aggregate calls (pco_b200_segment_aggregate_pages_async / _files_async), built on aggregate_reference: the
PcoB200Aggregate record of each row segment [bounds[g], bounds[g + 1]) of a concatenation of pages / chunks, with the float sums in the
order include/pco_b200.h specifies (a batch's partial of a segment counts the batch's rows outside it as non-matches; the batches that
hold rows of the segment, in row order across pages and chunks, go to lane j mod 32; the total puts segment g on lane g mod 32)."""
import numpy as np

from tests import aggregate_reference as ar


def segment_record(x, pieces, a, b, lo, hi):
    """The record of the rows [a, b) of x (the concatenation, whose pages / chunks have the lengths `pieces`), and its f64 sum (None for
    integers)."""
    x = np.asarray(x)
    rec, _ = ar.record(x[a:b], [b - a], lo, hi)  # count, min, max and integer sums do not depend on the batches
    if x.dtype.kind != "f":
        return rec, None
    parts, o = [], 0
    for n in pieces:
        lo_r, hi_r = max(a, o), min(b, o + n)
        if lo_r < hi_r:
            bf, bl = (lo_r - o) // 256, (hi_r - 1 - o) // 256
            with np.errstate(invalid="ignore"):  # NaN payloads widen to f64 NaNs
                v = x[o + bf * 256:o + min(n, (bl + 1) * 256)].astype(np.float64)
            rows = np.arange(o + bf * 256, o + bf * 256 + len(v))
            m = ar.matches(x[o + bf * 256:o + bf * 256 + len(v)], lo, hi) & (rows >= a) & (rows < b)
            parts.extend(ar.batch_sums(v, m))
        o += n
    fs = ar.strided_sum(parts) if parts else 0.0
    rec[4] = int(np.array([fs]).view(np.uint64)[0])
    return rec, fs


def segment_records(x, pieces, bounds, lo, hi):
    """The records of every segment of `bounds` (M + 1 non-decreasing row indices) and the total, as ([(record, fs)], total record)."""
    x = np.asarray(x)
    recs = [segment_record(x, pieces, int(bounds[g]), int(bounds[g + 1]), lo, hi) for g in range(len(bounds) - 1)]
    tot = ar.total(recs, x.dtype) if recs else [0] * 6
    return recs, tot


def segment_records_int(x, bounds, lo, hi):
    """segment_records for integers of at most 32 bits and non-empty segments, vectorised (for millions of segments): the records as an
    (M, 6) list of Python ints per row, and the total."""
    x = np.asarray(x)
    assert x.dtype.kind in "iu" and x.dtype.itemsize <= 4
    bounds = np.asarray(bounds, dtype=np.int64)
    starts = bounds[:-1]
    assert np.all(np.diff(bounds) > 0)
    seg = x[bounds[0]:bounds[-1]]
    m = ar.matches(seg, lo, hi)
    at = starts - bounds[0]
    cnt = np.add.reduceat(m.astype(np.int64), at)
    k = ar.keys(seg).astype(np.uint64)
    kmin = np.minimum.reduceat(np.where(m, k, np.uint64(~np.uint64(0))), at)
    kmax = np.maximum.reduceat(np.where(m, k, np.uint64(0)), at)
    s = np.add.reduceat(np.where(m, seg.astype(np.int64), 0), at)
    ut = np.dtype(f"u{x.dtype.itemsize}")
    top = np.uint64(1 << (8 * x.dtype.itemsize - 1)) if x.dtype.kind == "i" else np.uint64(0)
    unkey = lambda kk: (kk ^ top).astype(ut).astype(np.uint64)  # noqa: E731
    mn = np.where(cnt > 0, unkey(kmin), 0)
    mx = np.where(cnt > 0, unkey(kmax), 0)
    rows = np.diff(bounds)
    recs = []
    for i in range(len(starts)):
        v = int(s[i]) & ((1 << 128) - 1)
        recs.append([int(rows[i]), int(cnt[i]), int(mn[i]), int(mx[i]), v & ar.MASK64, v >> 64])
    tot = ar.total([(r, None) for r in recs], x.dtype)
    return recs, tot
