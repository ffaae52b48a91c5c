"""The numpy statement of the top-k calls' outputs (include/pco_b200.h): the min(k, matches) best numbers x with lo <= x <= hi, ranked
by (value, position) with the lower position winning a tie in both directions, and their positions.  Numbers compare as the filter calls
compare them: integers in their own order, floats as IEEE values (-0.0 equals +0.0, NaN never matches); the ranking sorts an unsigned
key built from the bit patterns, so 64-bit integers never pass through a float."""
import numpy as np


def ordered_key(x):
    """An unsigned 64-bit key per number whose order is the numbers' (floats: -0.0 and +0.0 get one key; NaNs are not ranked)."""
    x = np.asarray(x)
    bits = x.dtype.itemsize * 8
    top = np.uint64(1) << np.uint64(bits - 1)
    u = x.view(f"u{x.dtype.itemsize}").astype(np.uint64)
    if x.dtype.kind == "i":
        return u ^ top
    if x.dtype.kind == "f":
        u = np.where(u == top, np.uint64(0), u)  # -0.0 as +0.0
        mask = np.uint64((1 << bits) - 1)
        return np.where(u & top, ~u & mask, u | top)
    return u


def matches(x, lo, hi):
    """The positions of the numbers inside the closed interval [lo, hi] (none when lo > hi or a bound is NaN)."""
    x = np.asarray(x)
    lo, hi = x.dtype.type(lo), x.dtype.type(hi)
    with np.errstate(invalid="ignore"):
        return np.nonzero((x >= lo) & (x <= hi))[0].astype(np.uint64)


def topk(x, lo, hi, k, largest):
    """(values, positions) of the call's output: values of x's dtype, positions uint64, both of length min(k, matches)."""
    x = np.asarray(x)
    pos = matches(x, lo, hi)
    key = ordered_key(x[pos])
    if largest:
        key = ~key
    order = np.lexsort((pos, key))[:k]
    return x[pos[order]], pos[order]
