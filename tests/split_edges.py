"""Numbers at the edges of the per-chunk mode split and of the size-guarantee fallback, and the split restated in numpy.

The split (pco/src/mode/{classic,int_mult,float_mult,float_quant}.rs) takes each number to a primary latent and, for the
two-var modes, a secondary one.  The GPU runs it in split_delta_kernel and gather_primary_sample_kernel, and for FloatMult it
is float arithmetic that has to match the CPU bit for bit.  `split` restates it under the x86 rules the reference runs by:

* FloatMult's multiplier is round(x * inv_base), rounding half away from zero;
* a NaN operand propagates with its sign and payload and the quiet bit set;
* a NaN the multiply produces (0 * inf, when a subnormal base has an infinite reciprocal) is x86's default NaN: sign set,
  quiet, zero payload;
* the multiplier becomes a latent by int_float_to_latent (data_types/float.rs:229-244): integers below 2^MANTISSA_DIGITS
  count by value, above it by ulps.

`families()` builds seeded families of numbers per mode and number type, each with its config; `BOUNDARY` lists chunks that
sit one byte below, on and one byte above the size guarantee (chunk_compressor.rs:502-541), found by `search_boundary`.
"""
import numpy as np

DTYPES = {"u8": np.uint8, "i8": np.int8, "u16": np.uint16, "i16": np.int16, "f16": np.float16, "u32": np.uint32, "i32": np.int32,
          "f32": np.float32, "u64": np.uint64, "i64": np.int64, "f64": np.float64}
FLOAT_LAYOUT = {16: (5, 10), 32: (8, 23), 64: (11, 52)}  # exponent bits, mantissa bits
MANTISSA_DIGITS = {32: 24, 64: 53}
MODE_CODE = {"classic": 0, "int_mult": 1, "float_mult": 2, "float_quant": 3}  # ModeKind in the chunk meta
ORDERS = (0, 1, 2, 7)


def nbits(dtype):
    return 8 * np.dtype(dtype).itemsize


def _u(dtype):
    return np.dtype(f"u{np.dtype(dtype).itemsize}")


def _mask(bits):
    return (1 << bits) - 1


def from_bits(bits, dtype):
    return np.asarray(bits, dtype=np.uint64).astype(_u(dtype)).view(dtype)


def to_latents(x):
    """to_latent_ordered (data_types/{unsigned,signed,float}.rs) as uint64."""
    dt, u = x.dtype, _u(x.dtype)
    mid = u.type(1 << (nbits(dt) - 1))
    v = x.view(u)
    if dt.kind == "u":
        return v.astype(np.uint64)
    if dt.kind == "i":
        return (v ^ mid).astype(np.uint64)
    return np.where(v & mid, ~v, v ^ mid).astype(u).astype(np.uint64)


def from_latents(lat, dtype):
    dt, u = np.dtype(dtype), _u(dtype)
    mid = u.type(1 << (nbits(dt) - 1))
    lat = np.asarray(lat, dtype=np.uint64).astype(u)
    if dt.kind == "u":
        return lat.view(dt)
    if dt.kind == "i":
        return (lat ^ mid).view(dt)
    return np.where(lat & mid, lat ^ mid, ~lat).astype(u).view(dt)


# ---- the split, restated ------------------------------------------------------------------------------------------------------
def _round_half_away(q):
    """Rust's f32/f64::round: half away from zero, keeping the sign of zero and passing infinities and NaNs through."""
    with np.errstate(invalid="ignore"):
        t = np.trunc(q)
        away = np.abs(q - t) >= q.dtype.type(0.5)
        return np.where(away, t + np.copysign(q.dtype.type(1), q), t).astype(q.dtype)


def int_float_to_latent(mult_bits, bits):
    """float.rs:229-244 on bit patterns: |mult| below 2^MANTISSA_DIGITS counts by value, above it by ulps from there."""
    mid = 1 << (bits - 1)
    f = np.dtype(f"f{bits // 8}")
    abs_bits = mult_bits & np.uint64(mid - 1)
    gpi = 1 << MANTISSA_DIGITS[bits]
    gpi_bits = int(np.array([gpi], dtype=f).view(_u(f))[0])
    a = abs_bits.astype(_u(f)).view(f)
    with np.errstate(invalid="ignore"):
        small = a < f.type(gpi)
        small_int = np.where(small, a, 0).astype(np.uint64)
    abs_int = np.where(small, small_int, np.uint64(gpi) + (abs_bits - np.uint64(gpi_bits)))
    neg = (mult_bits & np.uint64(mid)) != 0
    return np.where(neg, np.uint64(mid - 1) - abs_int, np.uint64(mid) + abs_int) & np.uint64(_mask(bits))


def float_mult_mults(x, base):
    """The multiplier round(x * inv_base) of each number as bit patterns, with the x86 NaN rules."""
    bits = nbits(x.dtype)
    u = _u(x.dtype)
    _, m = FLOAT_LAYOUT[bits]
    quiet = np.uint64(1 << (m - 1))
    default_nan = np.uint64(((1 << (bits - 1)) | (_mask(bits - 1) ^ _mask(m)) | (1 << (m - 1))))
    b = x.dtype.type(base)
    with np.errstate(over="ignore", divide="ignore", invalid="ignore", under="ignore"):
        inv = x.dtype.type(1) / b
        q = (x * inv).astype(x.dtype)
    mult = _round_half_away(q).view(u).astype(np.uint64)
    xb = x.view(u).astype(np.uint64)
    mult = np.where(np.isnan(q), default_nan, mult)
    return np.where(np.isnan(x), xb | quiet, mult)


def split(x, mode="classic", base=None, k=None):
    """(primary, secondary) latents of the numbers `x` (uint64 arrays; secondary None for one-var modes)."""
    bits = nbits(x.dtype)
    mask = np.uint64(_mask(bits))
    mid = np.uint64(1 << (bits - 1))
    lat = to_latents(x)
    if mode == "classic":
        return lat, None
    if mode == "int_mult":
        b = np.uint64(int(base) & _mask(bits))  # L::from_u64 keeps the low bits
        return lat // b, lat % b
    if mode == "float_quant":
        kmax = np.uint64((1 << k) - 1)
        lowest = lat & kmax
        neg = (x.view(_u(x.dtype)).astype(np.uint64) & mid) != 0
        return lat >> np.uint64(k), np.where(neg, kmax - lowest, lowest)
    # float_mult (float_mult.rs:38-60)
    u = _u(x.dtype)
    _, m = FLOAT_LAYOUT[bits]
    mult_bits = float_mult_mults(x, base)
    primary = int_float_to_latent(mult_bits, bits)
    mult = mult_bits.astype(u).view(x.dtype)
    with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        prod = (mult * x.dtype.type(base)).astype(x.dtype).view(u).astype(np.uint64)
    prod = np.where(np.isnan(mult), mult_bits | np.uint64(1 << (m - 1)), prod)
    prod_lat = to_latents(prod.astype(u).view(x.dtype))
    return primary, (lat - prod_lat + mid) & mask


def delta_encode(lat, order, bits):
    """Consecutive delta (delta/consecutive.rs:19-33): `order` passes of x[i] -= x[i-1], each keeping its first latent as a
    moment, then the stored deltas centred (+ MID).  Returns (stored, moments)."""
    mask = np.uint64(_mask(bits))
    d = lat.astype(np.uint64)
    moments = []
    for _ in range(order):
        moments.append(int(d[0]))
        d = (d[1:] - d[:-1]) & mask
    return (d + np.uint64(1 << (bits - 1))) & mask if order else d, moments


def dissect(stored, bins):
    """(bin index, offset) of each stored latent under the bins [weight, lower, offset bits] of a chunk meta: the bin with the
    largest lower at or below the latent, which for pco's sorted, disjoint bins is the one the encoder chose."""
    lowers = np.array([b[1] for b in bins], dtype=np.uint64)
    order = np.argsort(lowers, kind="stable")
    sym = order[np.searchsorted(lowers[order], stored, side="right") - 1]
    off = stored - lowers[sym]
    return sym.astype(np.int64), off


# ---- special values ------------------------------------------------------------------------------------------------------------
def float_specials(dtype):
    """Bit patterns of ±0, ±smallest and ±largest subnormal, ±smallest normal, ±max finite, ±inf, and quiet and signalling NaNs of
    both signs with payloads 1, the top payload bit and a full payload."""
    bits = nbits(dtype)
    e, m = FLOAT_LAYOUT[bits]
    sign = 1 << (bits - 1)
    inf = _mask(e) << m
    quiet = 1 << (m - 1)
    pos = [0, 1, _mask(m), 1 << m, inf - 1, inf]
    for q in (quiet, 0):
        pos += [inf | q | 1, inf | q | (1 << (m - 2)), inf | q | _mask(m - 1)]
    return np.array(pos + [p | sign for p in pos], dtype=np.uint64)


def int_extremes(dtype):
    info = np.iinfo(dtype)
    vals = [info.min, info.min + 1, info.max, info.max - 1, 0, 1]
    if info.min < 0:
        vals.append(-1)
    return np.array(vals, dtype=object).astype(dtype)


def _mix(walk, extra, rng, runs=3):
    """`extra` dropped into `walk` in a few runs, so the walk stays a walk around them and no chunk is all specials."""
    out = walk.copy()
    cuts = np.sort(rng.choice(np.arange(1, extra.size), size=min(runs - 1, extra.size - 1), replace=False)) if extra.size > 1 else []
    pieces = np.split(extra, cuts)
    slots = np.sort(rng.choice(np.arange(8, walk.size - extra.size - 8), size=len(pieces), replace=False))
    shift = 0
    for piece, at in zip(pieces, slots):
        at = at + shift
        out[at: at + piece.size] = piece
        shift += piece.size
    return out


# ---- families ------------------------------------------------------------------------------------------------------------------
def family(name, dtype, nums, mode="classic", order=0, level=8, path=None, **params):
    return dict(name=name, dtype=np.dtype(dtype), nums=np.ascontiguousarray(nums), mode=mode, order=order, level=level, path=path,
                base=params.get("base"), k=params.get("k"))


def _float_walk(dtype, n, rng, scale=1.0):
    return (np.cumsum(rng.integers(-3, 4, size=n)) * scale + 1000 * scale).astype(dtype)


def _neighbours(v, dtype):
    """v and the floats one ulp either side (as far as they exist)."""
    v = np.asarray(v, dtype=dtype)
    with np.errstate(over="ignore", invalid="ignore"):
        return np.concatenate([v, np.nextafter(v, dtype(np.inf)), np.nextafter(v, dtype(-np.inf))]).astype(dtype)


def float_mult_bases(dtype):
    big = {np.float32: [float(np.finfo(np.float32).max), 2.0 ** 100], np.float64: [float(np.finfo(np.float64).max), 2.0 ** 1000]}[dtype]
    sub = {np.float32: [2.0 ** -127, 1e-39], np.float64: [2.0 ** -1023, 1e-310]}[dtype]
    return [0.01, 1 / 7, 2.0 ** -20, 0.5, 3.0, -0.25, -3.0] + big + sub


def float_mult_values(dtype, base, rng):
    """The edges of the FloatMult split at `base`: specials, ties at k + 1/2, x * inv overflowing, multipliers on both sides of
    2^MANTISSA_DIGITS, mult * base rounding past max finite, and values one ulp off a multiple."""
    dt = np.dtype(dtype).type
    bits = nbits(dtype)
    b = dt(base)
    fmax = np.finfo(dtype).max
    vals = [from_bits(float_specials(dtype), dtype)]
    with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        ks = np.array([0, 1, 2, 3, 7, 100, 12345], dtype=dtype) + dt(0.5)
        ties = np.concatenate([ks, -ks]) * b
        vals.append(ties.astype(dtype))
        g = float(1 << MANTISSA_DIGITS[bits])
        mults = np.array([g - 1, g, g + 2, g + 4, 2 * g, 3.0], dtype=dtype)
        vals.append(_neighbours(np.concatenate([mults, -mults]) * b, dtype))
        vals.append(_neighbours(np.array([fmax, -fmax, fmax / 2, fmax / 3, dt(1e30), dt(-1e30)], dtype=dtype), dtype))
        m = np.floor(fmax / np.abs(b)) if np.isfinite(fmax / np.abs(b)) else dt(0)
        vals.append(_neighbours(np.array([m, m - 1, -m], dtype=dtype) * b, dtype))
        vals.append(_neighbours(rng.integers(-50, 50, size=6).astype(dtype) * b, dtype))
    return np.concatenate(vals).astype(dtype)


def _float_mult_walk(dtype, base, n, rng):
    b = np.dtype(dtype).type(base)
    with np.errstate(over="ignore", invalid="ignore"):
        k = np.cumsum(rng.integers(-2, 3, size=n)) + (0 if abs(base) > 1e30 else 200)
        return (k.astype(dtype) * b).astype(dtype)


def _float_quant_values(dtype, k, rng):
    bits = nbits(dtype)
    u = _u(dtype)
    low = np.uint64(_mask(k))
    raw = (rng.normal(size=24) * 1000).astype(dtype)
    raw = np.concatenate([raw, -np.abs(raw)]).astype(dtype).view(u).astype(np.uint64)
    zero_low = raw & ~low
    ones_low = raw | low
    vals = [zero_low, ones_low, float_specials(dtype)]
    e, m = FLOAT_LAYOUT[bits]
    inf = _mask(e) << m
    sign = 1 << (bits - 1)
    pay = [1 << min(k - 1, m - 1), _mask(min(k, m - 1)), (1 << (m - 1)) | _mask(min(k, m - 1))]
    vals.append(np.array([inf | p for p in pay] + [sign | inf | p for p in pay], dtype=np.uint64))
    return from_bits(np.concatenate(vals), dtype)


def families():
    """Every family of the split edges, seeded."""
    out = []
    n = 2500
    # special values, every float type, Classic on the sort path
    for i, ds in enumerate(("f16", "f32", "f64", "u8", "i8", "u16", "i16", "u32", "i32", "u64", "i64")):
        dt = DTYPES[ds]
        rng = np.random.default_rng(100 + i)
        if np.dtype(dt).kind == "f":
            walk, extra = _float_walk(dt, n, rng, 0.37), from_bits(float_specials(dt), dt)
        else:
            walk = (np.cumsum(rng.integers(-3, 4, size=n)) + 100).astype(dt)
            extra = int_extremes(dt)
        for order in ORDERS:
            out.append(family(f"classic-sorted-{ds}-o{order}", dt, _mix(walk, extra, rng), order=order, path="sorted"))
        # the one-pass front end: every stored latent within 2^15 of the others - clusters of specials that sit together
        if np.dtype(dt).kind == "f":
            e, m = FLOAT_LAYOUT[nbits(dt)]
            centres = {"zero": int(to_latents(np.array([0], dtype=dt))[0]), "inf": int(to_latents(from_bits([_mask(e) << m], dt))[0])}
        else:
            centres = {"min": 0, "zero": int(to_latents(np.array([0], dtype=dt))[0]), "max": _mask(nbits(dt))}
        span = min(1 << 13, 1 << (nbits(dt) - 2))
        for where, centre in centres.items():
            lo, hi = max(centre - span, 0), min(centre + span, _mask(nbits(dt)))
            lat = rng.integers(lo, hi, size=n, dtype=np.uint64, endpoint=True)
            lat[:8] = [lo, hi, centre, min(centre + 1, hi), max(centre - 1, lo), max(centre - 2, lo), min(centre + 2, hi), centre]
            out.append(family(f"classic-one_pass-{ds}-{where}", dt, rng.permutation(from_latents(lat, dt)), path="one_pass"))
    # FloatMult, f32 and f64
    for ds in ("f32", "f64"):
        dt = DTYPES[ds]
        for j, base in enumerate(float_mult_bases(dt)):
            rng = np.random.default_rng(1000 + j + (50 if ds == "f64" else 0))
            extra = float_mult_values(dt, base, rng)
            walk = _float_mult_walk(dt, base, n, rng)
            for order in ORDERS:
                out.append(family(f"float_mult-{ds}-b{base!r}-o{order}", dt, _mix(walk, extra, rng), "float_mult", order, base=base))
    # FloatQuant, every float type
    for ds in ("f16", "f32", "f64"):
        dt = DTYPES[ds]
        p = FLOAT_LAYOUT[nbits(dt)][1]
        for j, k in enumerate(sorted({1, 2, p // 2, p - 1, p})):
            rng = np.random.default_rng(2000 + 10 * j + nbits(dt))
            walk = _float_walk(dt, n, rng, 0.25).view(_u(dt)).astype(np.uint64) & ~np.uint64(_mask(k))
            walk = from_bits(walk, dt)
            extra = _float_quant_values(dt, k, rng)
            for order in ORDERS:
                out.append(family(f"float_quant-{ds}-k{k}-o{order}", dt, _mix(walk, extra, rng), "float_quant", order, k=k))
    # IntMult, every integer type.  The config carries the base as given: a base with bits above the type width (2^bits + 3) is
    # truncated by the compressor like L::from_u64, so its split uses 3.  "above" is a base above every latent of its chunk
    # (3 * 2^(bits-2) + 1, the data below it): every primary latent is 0 and every secondary is the number's latent.
    for i, ds in enumerate(("u8", "i8", "u16", "i16", "u32", "i32", "u64", "i64")):
        dt = DTYPES[ds]
        bits = nbits(dt)
        bases = [1, 2, 3, 7, 1 << (bits - 1), _mask(bits), "above"] + ([(1 << bits) + 3] if bits < 64 else [])
        for j, base in enumerate(bases):
            rng = np.random.default_rng(3000 + 16 * i + j)
            cfg_base = 3 * (1 << (bits - 2)) + 1 if base == "above" else int(base)
            b = cfg_base & _mask(bits)
            top = b - 1 if base == "above" else _mask(bits)  # the largest latent in the data
            ks = np.arange(0, 5, dtype=object)
            lat = [k * b + d for k in ks for d in (-1, 0, 1)] + [0, top, 1 << (bits - 1), (1 << (bits - 1)) - 1]
            lat = np.array([v for v in lat if 0 <= v <= top], dtype=np.uint64)
            ext = int_extremes(dt)  # type min and max among them
            extra = np.concatenate([from_latents(lat, dt), ext[to_latents(ext) <= np.uint64(top)]])
            span = max(min(b, 1 << 20) // 4, 1)
            kk = np.cumsum(rng.integers(-2, 3, size=n)) + 300
            mult = kk % max(top // max(b, 1), 1) if b > 1 else kk
            wlat = mult.astype(np.uint64) * np.uint64(b) + rng.integers(0, span, size=n).astype(np.uint64) % np.uint64(b)
            walk = from_latents(np.minimum(wlat & np.uint64(_mask(bits)), np.uint64(top)), dt)
            order = ORDERS[(i + j) % len(ORDERS)]
            out.append(family(f"int_mult-{ds}-b{base}-o{order}", dt, _mix(walk, extra, rng), "int_mult", order, base=cfg_base))
    # levels 0 and 12 for a subset
    subset = ["classic-sorted-f64-o1", "float_mult-f64-b0.01-o0", "float_mult-f32-b1e-39-o1", "float_quant-f32-k11-o0", "int_mult-u32-b7-"]
    for prefix in subset:
        base = next(f for f in out if f["name"].startswith(prefix))
        for level in (0, 12):
            f = dict(base)
            f["name"], f["level"] = f"{base['name']}-L{level}", level
            out.append(f)
    return out


# ---- chunks at the size guarantee ---------------------------------------------------------------------------------------------
# combo -> (dtype, mode, params, order, level, wrapped pages).  The numbers of a combo are `smooth` numbers the config compresses
# well with a fraction `frac` replaced by noise over the whole type; the chunk size, the fraction and the seed move the chunk's
# worst case size across the baseline one byte at a time.
BOUNDARY_COMBOS = {
    "classic-o1-u8": ("u8", "classic", {}, 1, 8, None),
    "classic-o7-u8": ("u8", "classic", {}, 7, 8, None),
    "classic-o1-u16": ("u16", "classic", {}, 1, 8, None),
    "classic-o7-u16": ("u16", "classic", {}, 7, 8, None),
    "classic-o1-u32": ("u32", "classic", {}, 1, 8, None),
    "classic-o7-u32": ("u32", "classic", {}, 7, 8, None),
    "classic-o1-f64": ("f64", "classic", {}, 1, 8, None),
    "classic-o7-f64": ("f64", "classic", {}, 7, 8, None),
    "int_mult-u32": ("u32", "int_mult", {"base": 7}, 0, 8, None),
    "float_mult-f64": ("f64", "float_mult", {"base": 0.01}, 0, 8, None),
    "float_quant-f32": ("f32", "float_quant", {"k": 4}, 0, 8, None),
    "classic-o1-u32-L12": ("u32", "classic", {}, 1, 12, None),
    "wrapped-o2-u32": ("u32", "classic", {}, 2, 8, 3),
}


def boundary_nums(combo, n, frac, seed):
    ds, mode, params = BOUNDARY_COMBOS[combo][:3]
    dt = DTYPES[ds]
    bits = nbits(dt)
    rng = np.random.default_rng(seed)
    noise = rng.random(n) < frac
    if mode == "classic":  # a walk that rarely steps, so even its 7th differences are mostly 0; noise over every latent
        steps = rng.integers(-2, 3, size=n) * (rng.random(n) < 0.1)
        lat = np.cumsum(steps).astype(np.uint64) + np.uint64(1 << (bits - 1))
        lat = np.where(noise, rng.integers(0, _mask(bits), size=n, dtype=np.uint64, endpoint=True), lat)
        return from_latents(lat, dt)
    if mode == "int_mult":  # multiples of the base over the whole type; the noisy ones are off the grid
        b = np.uint64(params["base"])
        x = rng.integers(0, _mask(bits), size=n, dtype=np.uint64, endpoint=True) // b * b
        return np.where(noise, x + rng.integers(0, params["base"], size=n).astype(np.uint64), x).astype(dt)
    if mode == "float_mult":  # multiples of the base of either sign and every magnitude up to 2^513; the noisy ones are ulps off
        sign = rng.integers(0, 2, size=n, dtype=np.uint64) << np.uint64(63)
        mult = np.round(from_bits(rng.integers(0x3FF0000000000000, 0x6000000000000000, size=n, dtype=np.uint64) | sign, dt))
        x = (mult * dt(params["base"])).astype(dt)
        return np.where(noise, np.nextafter(np.nextafter(x, dt(np.inf)), dt(np.inf)), x).astype(dt)
    # float_quant: numbers of either sign with the low k bits clear over the whole finite range; the noisy ones have them set
    u = _u(dt)
    sign = rng.integers(0, 2, size=n, dtype=np.uint64) << np.uint64(31)
    x = (rng.integers(0, 0x7f800000, size=n, dtype=np.uint64) & ~np.uint64(_mask(params["k"]))) | sign
    x = np.where(noise, x | rng.integers(0, 1 << params["k"], size=n, dtype=np.uint64), x)
    return x.astype(u).view(dt)


def boundary_pages(combo, n):
    pages = BOUNDARY_COMBOS[combo][5]
    if not pages:
        return None
    return [n // pages] * (pages - 1) + [n - (pages - 1) * (n // pages)]


# margins found by search_boundary: (combo, margin) -> (n, frac, seed); a combination missing from here was not reached
BOUNDARY = {
    ('classic-o1-u8', -1): (1109, 0.581, 428), ('classic-o1-u8', 0): (74, 0.525, 671), ('classic-o1-u8', 1): (143, 0.668, 300),
    ('classic-o7-u8', -1): (1260, 0.118, 219), ('classic-o7-u8', 0): (325, 0.095, 873), ('classic-o7-u8', 1): (1420, 0.274, 625),
    ('classic-o1-u16', -1): (743, 0.735, 91), ('classic-o1-u16', 0): (607, 0.701, 853), ('classic-o1-u16', 1): (143, 0.818, 300),
    ('classic-o7-u16', -1): (794, 0.254, 184), ('classic-o7-u16', 0): (219, 0.197, 59), ('classic-o7-u16', 1): (143, 0.318, 300),
    ('classic-o1-u32', -1): (1109, 0.831, 428), ('classic-o1-u32', 0): (341, 0.791, 198), ('classic-o1-u32', 1): (1420, 0.924, 625),
    ('classic-o7-u32', -1): (1430, 0.29, 562), ('classic-o7-u32', 0): (466, 0.284, 266), ('classic-o7-u32', 1): (143, 0.368, 300),
    ('classic-o1-f64', -1): (270, 0.829, 114), ('classic-o1-f64', 0): (83, 0.791, 183), ('classic-o1-f64', 1): (1420, 0.974, 625),
    ('classic-o7-f64', -1): (498, 0.362, 269), ('classic-o7-f64', 0): (583, 0.431, 327), ('classic-o7-f64', 1): (1420, 0.474, 625),
    ('int_mult-u32', -1): (1420, 0.224, 625), ('int_mult-u32', 0): (878, 0.137, 467), ('int_mult-u32', 1): (374, 0.048, 610),
    ('float_mult-f64', -1): (452, 0.542, 807), ('float_mult-f64', 0): (374, 0.943, 452), ('float_mult-f64', 1): (404, 0.96, 801),
    ('float_quant-f32', -1): (384, 0.578, 866), ('float_quant-f32', 0): (1049, 0.65, 361), ('float_quant-f32', 1): (760, 0.628, 793),
    ('classic-o1-u32-L12', -1): (11125, 0.805, 903), ('classic-o1-u32-L12', 0): (9434, 0.812, 381), ('classic-o1-u32-L12', 1): (10858, 0.947, 622),
    ('wrapped-o2-u32', -1): (989, 0.644, 806), ('wrapped-o2-u32', 0): (1132, 0.647, 134), ('wrapped-o2-u32', 1): (647, 0.654, 967),
}
# (combo, margin) that search_boundary did not reach within its budget
UNREACHED = []


def boundary_family(combo, n, frac, seed):
    ds, mode, params, order, level, _ = BOUNDARY_COMBOS[combo]
    f = family(f"boundary-{combo}-n{n}-f{frac}-s{seed}", DTYPES[ds], boundary_nums(combo, n, frac, seed), mode, order, level, **params)
    f["pages"] = boundary_pages(combo, n)
    return f


def oracle_configs(oracle, fam, delta_auto=False):
    """The oracle's config for a family."""
    mode = {"classic": oracle.MODE_CLASSIC, "int_mult": oracle.MODE_INT_MULT, "float_mult": oracle.MODE_FLOAT_MULT,
            "float_quant": oracle.MODE_FLOAT_QUANT}[fam["mode"]]
    delta = oracle.DELTA_AUTO if delta_auto else oracle.DELTA_CONSECUTIVE if fam["order"] else oracle.DELTA_NOOP
    return oracle.make_config(level=fam["level"], mode=mode, delta=delta, delta_order=fam["order"], float_mult_base=fam["base"] or 0.0,
                              int_mult_base=int(fam["base"] or 0) if fam["mode"] == "int_mult" else 0, float_quant_k=fam["k"] or 0,
                              exact_pages=fam.get("pages"))


def margin(oracle, fam):
    """worst_case_size - baseline of the family's (single) chunk, as the oracle computes it."""
    cfg = oracle_configs(oracle, fam)
    if fam.get("pages"):
        oracle.ChunkCompressor(fam["nums"], cfg)
    else:
        oracle.simple_compress(fam["nums"], cfg)
    (w, b), = oracle.last_fallback_margins()
    return w - b


def search_boundary(oracle, combo, targets=(-1, 0, 1), budget=3000):
    """(n, frac, seed) for each reachable target margin of `combo`: a scan over the noise fraction finds where the margin changes
    sign, then a seeded random walk over chunk size, fraction and seed near there looks for each target."""
    found = {}
    lo, hi = (8192, 12000) if BOUNDARY_COMBOS[combo][4] == 12 else (64, 1500)
    mid = (lo + hi) // 2
    fracs = np.linspace(0, 1, 21)
    ms = [margin(oracle, boundary_family(combo, mid, round(float(f), 3), 1)) for f in fracs]
    cross = [i for i in range(len(fracs) - 1) if (ms[i] <= 0) != (ms[i + 1] <= 0)]
    f_lo, f_hi = (fracs[max(cross[0] - 2, 0)], fracs[min(cross[-1] + 3, len(fracs) - 1)]) if cross else (0.0, 1.0)
    rng = np.random.default_rng(7)
    for _ in range(budget):
        n = int(rng.integers(lo, hi))
        frac = round(float(rng.uniform(f_lo, f_hi)), 3)
        seed = int(rng.integers(0, 1000))
        m = margin(oracle, boundary_family(combo, n, frac, seed))
        if m in targets and m not in found:
            found[m] = (n, frac, seed)
            if len(found) == len(targets):
                break
    return found
