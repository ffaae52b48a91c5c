"""numpy reference of the aggregate calls (pco_b200_aggregate_pages_async / _files_async): the PcoB200Aggregate records of groups of
decoded numbers, with the float sums in the order include/pco_b200.h specifies (lane partials of 8, pairwise trees of 32 lanes, batch j and
group g on lane j mod 32)."""
import numpy as np

MASK64 = (1 << 64) - 1


def _key_kind(dt):
    return 2 if dt.kind == "f" else 1 if dt.kind == "i" else 0


def keys(x):
    """The unsigned key whose order is the numbers' (floats: IEEE order with -0.0 right below +0.0), as uint64."""
    x = np.asarray(x)
    dt = x.dtype
    ut = np.dtype(f"u{dt.itemsize}")
    b = x.view(ut).astype(np.uint64)
    top = np.uint64(1 << (8 * dt.itemsize - 1))
    full = np.uint64((1 << (8 * dt.itemsize)) - 1)
    kind = _key_kind(dt)
    if kind == 1:
        return b ^ top
    if kind == 2:
        return np.where(b & top, ~b & full, b | top)
    return b


def matches(x, lo, hi):
    """lo <= x <= hi: integers in their order, floats as IEEE values (NaN never matches, a NaN bound selects nothing)."""
    x = np.asarray(x)
    with np.errstate(invalid="ignore"):
        return (x >= x.dtype.type(lo)) & (x <= x.dtype.type(hi))


def tree(v):
    """Pairwise tree over the last axis (a power of two): (0, 1), (2, 3), ..., then pairs of pairs."""
    with np.errstate(invalid="ignore", over="ignore"):  # +inf + -inf is NaN, a finite sum may overflow to +-inf, as on the device
        while v.shape[-1] > 1:
            v = v[..., 0::2] + v[..., 1::2]
    return v[..., 0]


def strided_sum(sums):
    """Item j on lane j mod 32, each lane adding its items in order from +0.0, then the tree."""
    s = np.asarray(sums, dtype=np.float64)
    s = np.concatenate([s, np.zeros((-len(s)) % 32)]).reshape(-1, 32)
    acc = np.zeros(32)
    with np.errstate(invalid="ignore", over="ignore"):
        for row in s:
            acc = acc + row
    return float(tree(acc))


def batch_sums(v, m):
    """Per 256-number batch of one page / chunk (v as f64, m the matches): each lane's 8 numbers left to right, then the tree."""
    x = np.where(m, v, 0.0)  # non-matches add +0.0, which changes no sum that starts from +0.0
    x = np.concatenate([x, np.zeros((-len(x)) % 256)]).reshape(-1, 32, 8)
    acc = np.zeros(x.shape[:2])
    with np.errstate(invalid="ignore", over="ignore"):
        for e in range(8):
            acc = acc + x[:, :, e]
    return tree(acc)


def record(x, pieces, lo, hi):
    """The record of one group: x its numbers, pieces the lengths of its pages / chunks (batches restart at each).  Returns the 6 fields
    as Python ints (sum_lo of a float sum: its f64 bit pattern), and the f64 sum for floats (None for integers)."""
    x = np.asarray(x)
    dt = x.dtype
    m = matches(x, lo, hi)
    cnt = int(m.sum())
    mn = mx = 0
    if cnt:
        k = keys(x[m])
        ut = np.dtype(f"u{dt.itemsize}")
        mn = int(x[m][np.argmin(k)].view(ut))
        mx = int(x[m][np.argmax(k)].view(ut))
    if dt.kind == "f":
        bs, at = [], 0
        for n in pieces:
            with np.errstate(invalid="ignore"):  # NaN payloads widen to f64 NaNs
                v = x[at:at + n].astype(np.float64)
            bs.extend(batch_sums(v, m[at:at + n]))
            at += n
        fs = strided_sum(bs)
        return [len(x), cnt, mn, mx, int(np.array([fs]).view(np.uint64)[0]), 0], fs
    s = sum(int(v) for v in x[m].astype(object)) if cnt < 4096 else _exact_sum(x[m])
    s &= (1 << 128) - 1
    return [len(x), cnt, mn, mx, s & MASK64, s >> 64], None


def _exact_sum(v):
    """Exact sum of integers, as a Python int, without a per-element loop."""
    if v.dtype.kind == "i":
        neg = int((v < 0).sum())
        u = v.astype(np.int64).view(np.uint64)
        return _exact_sum(u) - neg * (1 << 64)
    u = v.astype(np.uint64)
    return int((u >> np.uint64(32)).sum()) * (1 << 32) + int((u & np.uint64(0xFFFFFFFF)).sum())


def total(records, dtype):
    """The total record from the groups' (record, f64 sum) pairs of numbers of dtype."""
    dt = np.dtype(dtype)
    ut = np.dtype(f"u{dt.itemsize}")
    floats = dt.kind == "f"
    rs = [r for r, _ in records]
    out = [sum(r[0] for r in rs), sum(r[1] for r in rs), 0, 0, 0, 0]
    have = [r for r in rs if r[1]]
    if have:
        mins = np.array([r[2] for r in have], dtype=np.uint64).astype(ut).view(dt)
        maxs = np.array([r[3] for r in have], dtype=np.uint64).astype(ut).view(dt)
        out[2] = int(mins[np.argmin(keys(mins))].view(ut))
        out[3] = int(maxs[np.argmax(keys(maxs))].view(ut))
    if floats:
        fs = strided_sum([f if r[1] else 0.0 for r, f in records])
        out[4] = int(np.array([fs]).view(np.uint64)[0])
    else:
        s = sum((r[5] << 64 | r[4]) for r in rs) & ((1 << 128) - 1)
        out[4], out[5] = s & MASK64, s >> 64
    return out


def same(got, want, floats):
    """Records equal, float sums bit-equal (any NaN matching any NaN)."""
    got = [int(v) & MASK64 for v in got]
    if floats and got[:4] == want[:4]:
        a, b = (np.array([v], dtype=np.uint64).view(np.float64)[0] for v in (got[4], want[4]))
        return (np.isnan(a) and np.isnan(b)) or got[4:] == want[4:]
    return got == want
