"""The numpy statement of the histogram calls' rows (include/pco_b200.h): for B + 1 edges, W = B + 3 counts per group: below edge 0, the
buckets (the last one closed), above the last edge, NaN.  Numbers are bucketed by np.searchsorted on the numbers themselves, in their own
dtype, so 64-bit integers never pass through a float."""
import numpy as np


def columns(x, edges):
    """The column of every number of x (a numpy array) for the edges (an array of x's dtype, strictly ascending)."""
    x = np.asarray(x)
    edges = np.asarray(edges, dtype=x.dtype)
    b = edges.size - 1
    c = np.searchsorted(edges, x, side="right").astype(np.int64)  # the edges at or below each number
    c[(c == b + 1) & (x == edges[b])] = b  # the last bucket is closed
    if x.dtype.kind == "f":
        c[np.isnan(x)] = b + 2
    return c


def row(x, edges):
    """The W counts of the numbers x."""
    return np.bincount(columns(x, edges), minlength=np.asarray(edges).size + 2).astype(np.int64)


def rows(x, sizes, edges):
    """The rows of groups of `sizes` consecutive numbers of x, as an int64 array of shape (len(sizes), W)."""
    out, at = [], 0
    for n in sizes:
        out.append(row(x[at:at + n], edges))
        at += n
    return np.array(out, dtype=np.int64).reshape(len(sizes), np.asarray(edges).size + 2)
