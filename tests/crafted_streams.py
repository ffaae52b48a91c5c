"""Valid pco streams that pco's own encoder never writes, for testing the decoders.

pco's planner writes bins sorted by lower and disjoint, offsets that fill their bins the way its histogram made them, table sizes
that follow unoptimized_bins_log + 2, and secondary latents inside what the mode's split produces.  The format allows much more:
bins in any order, duplicated or overlapping, lowers whose `lower + offset` passes the top of the latent type (the decoder adds with
wrapping), offsets as wide as the type in tables of many bins, all-weight-1 tables up to 2^14 states, moments anywhere, IntMult
adjustments at or above the base, FloatMult adjustments that land on NaN payloads or infinities.

Each family here describes chunks by their bins and (bin index, offset) pairs; the oracle's explicit writer
(oracle.pyoracle.write_explicit_file) turns them into a file, and `expected` restates the decode in numpy - `lower + offset` mod
2^bits, the consecutive un-delta from the moments with wrapping, then the mode's join - as a third opinion beside the oracle's
decoder and the GPU.  Every chunk names the GPU decoder it is built for:

* "fused3" / "fused4" / "fused5": fused_narrow_kernel at delta order 0 / 1 / 2..7 (chunk classes 3, 4, 5);
* "general1" / "general2": symwalk_kernel + decode_kernel with one / two latent vars (classes 1, 2);
* "cold": cold_decode_kernel, the catch-all (tables above 2^10 states or 256 bins, FloatMult below 32 bits, secondary_uses_delta).
"""
import numpy as np

DTYPES = {"u8": np.uint8, "i8": np.int8, "u16": np.uint16, "i16": np.int16, "f16": np.float16, "u32": np.uint32, "i32": np.int32,
          "f32": np.float32, "u64": np.uint64, "i64": np.int64, "f64": np.float64}
PRECISION = {16: 10, 32: 23, 64: 52}  # float mantissa bits: FloatQuant's largest k
MANTISSA_DIGITS = {16: 11, 32: 24, 64: 53}
ROUTE_CLASS = {"general1": 1, "general2": 2, "fused3": 3, "fused4": 4, "fused5": 5}


def nbits(dtype):
    return 8 * np.dtype(DTYPES.get(dtype, dtype) if isinstance(dtype, str) else dtype).itemsize


def _u(dtype):
    return np.dtype(f"u{np.dtype(dtype).itemsize}")


def _mask(bits):
    return np.uint64((1 << bits) - 1)


# ---- latent-ordered bits <-> numbers (pco/src/data_types/{unsigned,signed,float}.rs) ----------------------------------------------
def from_latents(lat, dtype):
    dt, u = np.dtype(dtype), _u(dtype)
    mid = u.type(1 << (nbits(dt) - 1))
    lat = np.asarray(lat, dtype=np.uint64).astype(u)
    if dt.kind == "u":
        return lat.view(dt)
    if dt.kind == "i":
        return (lat ^ mid).view(dt)
    return np.where(lat & mid, lat ^ mid, ~lat).astype(u).view(dt)


def to_latents(x):
    dt, u = x.dtype, _u(x.dtype)
    mid = u.type(1 << (nbits(dt) - 1))
    v = x.view(u)
    if dt.kind == "u":
        return v.astype(np.uint64)
    if dt.kind == "i":
        return (v ^ mid).astype(np.uint64)
    return np.where(v & mid, ~v, v ^ mid).astype(u).astype(np.uint64)


def float_latent(value, dtype):
    """The latent-ordered bits of one float (FloatMult's base is stored this way)."""
    return int(to_latents(np.array([value], dtype=dtype))[0])


# ---- the decode, restated --------------------------------------------------------------------------------------------------------
def stored_latents(var, bits):
    """lower[bin] + offset, wrapping at 2^bits (page_latent_decompressor.rs: lower.wrapping_add(offset))."""
    lowers = np.array([b[1] for b in var["bins"]] or [0], dtype=np.uint64)
    sym = np.asarray(var["symbols"], dtype=np.int64)
    off = np.asarray(var["offsets"], dtype=np.uint64)
    return (lowers[sym] + off) & _mask(bits)


def undelta(stored, moments, bits):
    """Consecutive decode (delta/consecutive.rs:35-50): centre the stored deltas, then one prefix sum per order from the innermost
    moment out, each adding one number in front."""
    mask = _mask(bits)
    x = (stored + np.uint64(1 << (bits - 1))) & mask
    for m in reversed([np.uint64(v) for v in moments]):
        x = np.concatenate([[m], (m + np.cumsum(x, dtype=np.uint64)) & mask]).astype(np.uint64) & mask
    return x


def _int_float_from_latent(lat, dtype):
    """float.rs:208-226: the float of integer value `lat - MID` (exact below 2^MANTISSA_DIGITS, then counting ulps)."""
    bits = nbits(dtype)
    u = _u(dtype)
    mid = np.uint64(1 << (bits - 1))
    neg = lat < mid
    abs_int = np.where(neg, mid - np.uint64(1) - lat, lat - mid)
    gpi = np.uint64(1 << MANTISSA_DIGITS[bits])
    gpi_bits = np.uint64(int(np.array([1 << MANTISSA_DIGITS[bits]], dtype=dtype).view(u)[0]))
    small_bits = np.minimum(abs_int, gpi).astype(dtype).view(u).astype(np.uint64)
    abs_bits = np.where(abs_int < gpi, small_bits, gpi_bits + (abs_int - gpi))
    abs_bits = np.where(neg, abs_bits ^ mid, abs_bits)
    return abs_bits.astype(u).view(dtype)


def join(chunk, dtype, prim, sec):
    """mode/{classic,int_mult,float_mult,float_quant}.rs join_latents, all with wrapping arithmetic."""
    bits = nbits(dtype)
    mask = _mask(bits)
    mid = np.uint64(1 << (bits - 1))
    mode = chunk.get("mode", "classic")
    if mode == "classic":
        return from_latents(prim, dtype)
    if mode == "int_mult":
        return from_latents((prim * np.uint64(chunk["base"]) + sec) & mask, dtype)
    if mode == "float_mult":
        base = from_latents(np.array([chunk["base"]], dtype=np.uint64), dtype)[0]
        unadjusted = _int_float_from_latent(prim, dtype) * base
        u = to_latents(np.asarray(unadjusted, dtype=dtype))
        return from_latents((u + sec + mid) & mask, dtype)
    k = chunk["k"]
    cutoff = mid >> np.uint64(k)
    kmax = np.uint64((1 << k) - 1)
    lowest = np.where(prim >= cutoff, sec, (kmax - sec) & mask)
    return from_latents(((prim << np.uint64(k)) + lowest) & mask, dtype)


def expected_chunk(chunk, dtype):
    bits = nbits(dtype)
    order = chunk.get("order", 0)
    lat = []
    for v, var in enumerate(chunk["vars"]):
        s = stored_latents(var, bits)
        if order and (v == 0 or chunk.get("secondary_uses_delta")):
            s = undelta(s, var["moments"], bits)[: chunk["n"]]
        lat.append(s)
    return join(chunk, dtype, lat[0], lat[1] if len(lat) > 1 else None)


def expected(fam):
    return np.concatenate([expected_chunk(c, fam["dtype"]) for c in fam["chunks"]])


def write(oracle, fam):
    """(file, [(meta, page) per chunk]) of a family, from the oracle's explicit writer."""
    return oracle.write_explicit_file(fam["dtype"], [{k: v for k, v in c.items() if k != "route"} for c in fam["chunks"]])


# ---- building blocks -----------------------------------------------------------------------------------------------------------
def table_log(bins):
    w = sum(b[0] for b in bins)
    assert w & (w - 1) == 0, w
    return w.bit_length() - 1


def var(bins, n_stored, rng, offsets="random", moments=None, symbols=None):
    """A latent var over `bins` [(weight, lower, offset_bits)] with `n_stored` latents: symbols drawn by weight (or given), offsets
    random, all ones ("max") or zero."""
    w = np.array([b[0] for b in bins], dtype=np.float64)
    if symbols is None:
        symbols = rng.choice(len(bins), size=n_stored, p=w / w.sum()) if len(bins) > 1 else np.zeros(n_stored, np.int64)
    symbols = np.asarray(symbols, dtype=np.int64)
    ob = np.array([b[2] for b in bins], dtype=np.uint64)[symbols]
    full = np.uint64(0xFFFFFFFFFFFFFFFF)
    omask = np.where(ob >= 64, full, (np.uint64(1) << np.minimum(ob, np.uint64(63))) - np.uint64(1))
    if offsets == "max":
        offs = omask
    elif offsets == "zero":
        offs = np.zeros(n_stored, np.uint64)
    else:
        offs = rng.integers(0, 1 << 64, size=n_stored, dtype=np.uint64, endpoint=False) & omask
    out = {"ans_size_log": table_log(bins), "bins": [tuple(int(x) for x in b) for b in bins], "symbols": symbols, "offsets": offs}
    if moments is not None:
        out["moments"] = [int(m) for m in moments]
    return out


def chunk(route, n, vars_, order=0, **mode):
    return dict(route=route, n=n, order=order, vars=vars_, **mode)


def classic(route, dtype, n, bins, rng, order=0, offsets="random", moments=None):
    if order and moments is None:
        moments = rng.integers(0, 1 << nbits(dtype), size=order, dtype=np.uint64, endpoint=False)
    return chunk(route, n, [var(bins, max(n - order, 0), rng, offsets, moments)], order=order)


def fam(name, dtype, chunks):
    return {"name": name, "dtype": np.dtype(DTYPES[dtype] if isinstance(dtype, str) else dtype), "chunks": chunks}


def _fused(order):
    return "fused3" if order == 0 else "fused4" if order == 1 else "fused5"


def _top(dtype):
    return (1 << nbits(dtype)) - 1


# ---- the families --------------------------------------------------------------------------------------------------------------
def f1_fused_edges():
    """fused_narrow_kernel's limits: max offset bits 15 (every offset 0x7fff) against 16; lowers spanning 2^16 - 1 against 2^16;
    2 and 256 bins against 257; ans_size_log 10 against 11; delta orders 0, 1, 2 and 7."""
    out = []
    rng = np.random.default_rng(1)
    for dt in ("u16", "u32", "u64"):
        b = 1 << (nbits(dt) - 2)
        for order in (0, 1, 2, 7):
            bins = [(3, b, 15), (1, b + 40000, 15), (4, b + 9, 15), (8, b + 20000, 15)]
            out.append(fam(f"f1_ob15_all_ones_{dt}_o{order}", dt, [classic(_fused(order), dt, 2048 + 3, bins, rng, order, "max")]))
        for order in (0, 1):
            bins = [(3, b, 16), (1, b + 40000, 15), (4, b + 9, 2), (8, b + 20000, 15)]
            out.append(fam(f"f1_ob16_{dt}_o{order}", dt, [classic("general1", dt, 2048 + 3, bins, rng, order, "max")]))
    for dt in ("u32", "u64"):
        b = (1 << nbits(dt)) - 70000
        for span, route in (((1 << 16) - 1, "fused3"), (1 << 16, "general1")):
            out.append(fam(f"f1_span_{span}_{dt}", dt, [classic(route, dt, 1500, [(2, b, 7), (2, b + span, 7)], rng)]))
    for n_bins, log, route in ((2, 1, "fused3"), (256, 8, "fused3"), (257, 9, "cold")):
        bins = [(1, 7 * i, 3) for i in range(n_bins)]
        bins[0] = (1 + (1 << log) - n_bins, 0, 3)
        out.append(fam(f"f1_bins_{n_bins}", "u32", [classic(route, "u32", 3000, bins, rng)]))
    for log, route in ((10, "fused4"), (11, "cold")):
        bins = [((1 << log) - 5, 50, 4), (3, 300, 5), (2, 100, 1)]
        out.append(fam(f"f1_ans_size_log_{log}", "u32", [classic(route, "u32", 3000, bins, rng, order=1)]))
    return out


def f2_bin_order():
    """Bins not sorted by lower: the first bin not the lowest, descending lowers, duplicated lowers, overlapping ranges."""
    out = []
    rng = np.random.default_rng(2)
    for dt, b in (("u32", 1 << 20), ("u64", 1 << 40), ("u16", 1000)):
        cases = {
            "first_not_lowest": [(2, b + 100, 6), (1, b, 6), (1, b + 500, 6)],
            "descending": [(1, b + 3000, 10), (1, b + 2000, 10), (1, b + 1000, 10), (1, b, 10)],
            "duplicate": [(2, b, 4), (1, b, 4), (1, b + 10, 2)],
            "overlapping": [(1, b, 4), (1, b + 5, 4), (1, b + 3, 8), (1, b + 1, 0)],
        }
        for name, bins in cases.items():
            # u16 lowers always lie within 2^16 of the first bin modulo 2^16: bins below the first are narrow there
            route = "fused3" if (dt == "u16" or name in ("duplicate", "overlapping")) else "general1"
            for order in (0, 1):
                r = route if order == 0 or route.startswith("general") else "fused4"
                out.append(fam(f"f2_{name}_{dt}_o{order}", dt, [classic(r, dt, 1000 + 17, bins, rng, order)]))
        bins = [(2, b, 20 if dt != "u16" else 16), (1, b, 3), (1, b + 7, 20 if dt != "u16" else 16)]
        out.append(fam(f"f2_duplicate_wide_{dt}", dt, [classic("general1", dt, 1000, bins, rng)]))
    return out


def f3_wrapping():
    """lower + offset past 2^bits for every width and its signed and float views, on the fused, general and catch-all routes; moments
    within a few units of the wrap at orders 1, 2 and 7."""
    out = []
    rng = np.random.default_rng(3)
    for dt in DTYPES:
        bits = nbits(dt)
        top = _top(dt)
        ob = min(15, bits)
        fused = [(2, top - 40 if bits > 8 else top - 100, ob), (1, top - 3, ob), (1, top, 2)]
        wide_ob = min(20, bits)
        general = [(2, top - 5, wide_ob), (1, top - (1 << (wide_ob - 1)), wide_ob), (1, 0, 1)]
        cold = [((1 << 11) - 2, top - 5, wide_ob), (1, top - 1000 if bits > 8 else top - 50, ob), (1, top, 1)]
        if bits == 8:
            general = [(1, top - 5, 8)]  # every 8-bit table of 2 or more bins is narrow: one bin is what the general pair takes
        out.append(fam(f"f3_wrap_fused_{dt}", dt, [classic("fused3", dt, 2000, fused, rng, offsets="max")]))
        out.append(fam(f"f3_wrap_general_{dt}", dt, [classic("general1", dt, 2000, general, rng)]))
        out.append(fam(f"f3_wrap_cold_{dt}", dt, [classic("cold", dt, 2000, cold, rng)]))
    for dt in ("u8", "u16", "u32", "u64", "i32", "f64"):
        top = _top(dt)
        for order in (1, 2, 7):
            moments = [(top - i) if i % 2 == 0 else i for i in range(order)]
            bins = [(2, top - 30 if nbits(dt) > 8 else 200, min(15, nbits(dt))), (2, top - 2, 3)]
            out.append(fam(f"f3_moments_{dt}_o{order}", dt, [classic(_fused(order), dt, 3000, bins, rng, order, moments=moments)]))
        bins = [(1, top - 2, nbits(dt)), (1, top, 3)]
        route = "fused5" if nbits(dt) == 8 else "general1"
        out.append(fam(f"f3_moments_general_{dt}_o2", dt, [classic(route, dt, 3000, bins, rng, 2, moments=[top - 1, 2])]))
    return out


def f4_full_width():
    """offset_bits == bits in tables of 2 or more bins, including all-ones offsets."""
    out = []
    rng = np.random.default_rng(4)
    for dt in ("u8", "u16", "u32", "u64", "i64", "f64", "f32"):
        bits = nbits(dt)
        route = "fused3" if bits == 8 else "general1"
        for offsets in ("random", "max"):
            bins = [(1, 3, bits), (1, _top(dt) - 1, bits)]
            out.append(fam(f"f4_two_bins_{offsets}_{dt}", dt, [classic(route, dt, 1300, bins, rng, offsets=offsets)]))
        bins = [(4, 0, bits), (2, 1 << (bits - 1), bits - 1), (1, 5, 1), (1, _top(dt), bits)]
        out.append(fam(f"f4_four_bins_o1_{dt}", dt, [classic("fused4" if bits == 8 else "general1", dt, 1300, bins, rng, order=1)]))
    for dt in ("u32", "u64"):
        bins = [((1 << 12) - 1, 0, nbits(dt)), (1, 9, nbits(dt))]
        out.append(fam(f"f4_cold_{dt}", dt, [classic("cold", dt, 1300, bins, rng, offsets="max")]))
    return out


def f5_table_shapes():
    """One bin with offsets at ans_size_log 0; weights 1 and 2^k - 1; all-weight-1 tables at ans_size_log 1..14; ans_size_log 11-14 with
    a few bins."""
    out = []
    rng = np.random.default_rng(5)
    for dt, ob in (("u8", 8), ("u32", 12), ("u64", 64), ("f32", 32)):
        out.append(fam(f"f5_one_bin_{dt}", dt, [classic("general1", dt, 1000, [(1, 77, ob)], rng)]))
        out.append(fam(f"f5_one_bin_o2_{dt}", dt, [classic("general1", dt, 1000, [(1, 5, ob)], rng, order=2)]))
    out.append(fam("f5_one_bin_no_offsets", "u32", [classic("general1", "u32", 1000, [(1, 123456, 0)], rng)]))
    for k in (1, 4, 10):
        out.append(fam(f"f5_weights_1_and_2^{k}-1", "u32", [classic("fused3", "u32", 2000, [(1, 0, 4), ((1 << k) - 1, 10, 3)], rng)]))
    out.append(fam("f5_weights_1_and_63_wide", "u64", [classic("general1", "u64", 2000, [(1, 10, 20), (63, 0, 40)], rng)]))
    for log in range(1, 15):
        route = "fused3" if log <= 8 else "cold"
        bins = [(1, 3 * i, 2) for i in range(1 << log)]
        out.append(fam(f"f5_all_weight_1_log{log}", "u32", [classic(route, "u32", max(2000, 4 << log), bins, rng)]))
    for log in (11, 12, 13, 14):
        bins = [((1 << log) - 3, 1000, 5), (1, 0, 7), (1, 1 << 30, 9), (1, 400, 0)]
        out.append(fam(f"f5_few_bins_log{log}", "u32", [classic("cold", "u32", 3000, bins, rng, order=1)]))
    return out


def _two_var(route, n, mode, prim, sec, **params):
    return chunk(route, n, [prim, sec], mode=mode, **params)


def f6_two_var_modes():
    """IntMult with base 3 and 2^63 + 1 and adjustments >= base; FloatMult adjustments that land on NaN payloads, +-inf and -0.0 (f32,
    f64, and f16 on the catch-all route); FloatQuant at k = 1 and k = precision bits."""
    out = []
    rng = np.random.default_rng(6)
    n = 2000
    for dt, base in (("u32", 3), ("i32", 3), ("u64", 3), ("u64", (1 << 63) + 1), ("i64", (1 << 63) + 1), ("u16", 3)):
        bits = nbits(dt)
        top = _top(dt)
        prim = var([(2, top - 100, 7), (1, 0, 5), (1, top - 3, 2)], n, rng)
        sec = var([(1, 0, 3), (1, base - 1 if base < 8 else base, 3), (2, top - 7, 3)], n, rng)
        out.append(fam(f"f6_int_mult_{dt}_{base}", dt, [_two_var("general2", n, "int_mult", prim, sec, base=base)]))
        sec_cold = var([((1 << 11) - 1, 0, min(bits, 20)), (1, top, 3)], n, rng)
        out.append(fam(f"f6_int_mult_cold_{dt}_{base}", dt, [_two_var("cold", n, "int_mult", prim, sec_cold, base=base)]))
        prim1 = var([(1, 0, 4), (1, top - 2, 2)], n - 1, rng, moments=[top - 1])
        out.append(fam(f"f6_int_mult_o1_{dt}_{base}", dt, [_two_var("general2", n, "int_mult", prim1, sec, base=base, order=1)]))
    for dt, base in (("f32", 0.5), ("f32", 1.25), ("f64", 0.1), ("f64", 3.0), ("f16", 0.25)):
        out.append(_float_mult_family(dt, base, n, rng))
    for dt in ("f16", "f32", "f64"):
        bits = nbits(dt)
        top = _top(dt)
        for k in (1, PRECISION[bits]):
            pb = bits - k
            mid_p = 1 << (pb - 1)
            prim = var([(1, mid_p - min(50, mid_p // 2), 6), (1, mid_p + 3, 6), (1, 0, min(pb, 10)), (1, (1 << pb) - 20, 4)], n, rng)
            sec = var([(2, 0, k), (1, (1 << k) - 1, min(bits, k + 3)), (1, top - 1, 2)], n, rng)
            out.append(fam(f"f6_float_quant_{dt}_k{k}", dt, [_two_var("general2", n, "float_quant", prim, sec, k=k)]))
        out.append(fam(f"f6_float_quant_secondary_delta_{dt}", dt, [_two_var(
            "cold", n, "float_quant", var([(1, (1 << (bits - 2)), 5), (1, 0, 3)], n - 2, rng, moments=[1 << (bits - 1), 3]),
            var([(1, 0, 2), (1, top - 1, 2)], n - 2, rng, moments=[top, 1]), k=2, order=2, secondary_uses_delta=True)]))
    return out


def _special_latents(dtype):
    """Latent-ordered bits of quiet NaNs with payloads (both signs), a signalling NaN, +inf, -inf, 0.0 and -0.0."""
    bits = nbits(dtype)
    mant = PRECISION[bits]
    inf, sign = ((1 << (bits - 1 - mant)) - 1) << mant, 1 << (bits - 1)
    quiet = inf | (1 << (mant - 1))
    raw = np.array([quiet | 5, quiet | 3 | sign, inf | 1, inf, inf | sign, 0, sign], dtype=np.uint64).astype(_u(dtype))
    return to_latents(raw.view(dtype))


def _float_mult_family(dt, base, n, rng):
    """FloatMult: primaries of modest size (finite products), secondaries chosen so that every third number lands on a special value;
    the rest are small adjustments, both below and above the product."""
    dtype = np.dtype(DTYPES[dt])
    bits = nbits(dtype)
    mid = 1 << (bits - 1)
    mask = _mask(bits)
    base_lat = float_latent(base, dtype)
    prim = var([(2, mid - 300, 9), (1, mid + 1000, 6), (1, mid - 5, 3)], n, rng)
    p = stored_latents(prim, bits)
    u = to_latents(np.asarray(_int_float_from_latent(p, dtype) * from_latents(np.array([base_lat], np.uint64), dtype)[0], dtype=dtype))
    special = _special_latents(dtype)
    target = (u + rng.integers(0, 8, size=n, dtype=np.uint64) - np.uint64(4)) & mask
    pick = np.arange(n) % 3 == 0
    target[pick] = special[rng.integers(0, special.size, size=int(pick.sum()))]
    s = (target - u - np.uint64(mid)) & mask  # the join: latent = u + s + MID
    sec = var([(1, 0, bits)], n, rng, symbols=np.zeros(n, np.int64))
    sec["offsets"] = s
    route = "cold" if bits < 32 else "general2"
    return fam(f"f6_float_mult_{dt}_{base}", dt, [_two_var(route, n, "float_mult", prim, sec, base=base_lat)])


def f7_shapes():
    """Chunks of 1, 255, 256, 257, 2^15 + 1 and 2^18 numbers, and files whose chunks mix the fast routes (fused and general); the
    catch-all shapes come as files of their own (a cold chunk sends its whole file to the catch-all decoder)."""
    out = []
    rng = np.random.default_rng(7)
    narrow = [(2, (1 << 20) - 7, 9), (1, 1 << 20, 12), (1, (1 << 20) + 300, 15)]
    wide = [(1, 1 << 30, 20), (1, 5, 32), (2, (1 << 30) + 4, 3)]
    for n in (1, 255, 256, 257, (1 << 15) + 1, 1 << 18):
        out.append(fam(f"f7_n{n}_fused", "u32", [classic("fused3", "u32", n, narrow, rng)]))
        out.append(fam(f"f7_n{n}_general_o1", "u32", [classic("general1", "u32", n, wide, rng, order=1)]))
    cold_bins = [(1, 3 * i, 2) for i in range(1 << 14)]
    out.append(fam("f7_n262144_cold", "u32", [classic("cold", "u32", 1 << 18, cold_bins, rng)]))
    out.append(fam("f7_n257_cold_o7", "u32", [classic("cold", "u32", 257, [((1 << 11) - 1, 0, 9), (1, 7, 2)], rng, order=7)]))
    top = _top("u32")
    mixed = [classic("fused3", "u32", 257, narrow, rng), classic("general1", "u32", 1, wide, rng, order=1),
             classic("fused5", "u32", (1 << 15) + 1, [(2, top - 40, 15), (2, top - 2, 3)], rng, order=7),
             classic("general1", "u32", 4097, [(1, top - 5, 20), (1, 2, 32)], rng, order=2),
             classic("fused4", "u32", 255, [(1, 0, 1), (1, 60000, 15)], rng, order=1)]
    out.append(fam("f7_mixed_fast_chunks", "u32", mixed))
    return out


FAMILY_GROUPS = {"f1": f1_fused_edges, "f2": f2_bin_order, "f3": f3_wrapping, "f4": f4_full_width, "f5": f5_table_shapes,
                 "f6": f6_two_var_modes, "f7": f7_shapes}


def all_families():
    out = []
    for fn in FAMILY_GROUPS.values():
        out.extend(fn())
    names = [f["name"] for f in out]
    assert len(set(names)) == len(names), "family names must be unique"
    return out


def is_cold(f):
    return any(c["route"] == "cold" for c in f["chunks"])


def class_counts(f):
    """Expected pco_b200_profile_chunk_classes counts of a fast family (index k = class k)."""
    counts = [0] * 8
    for c in f["chunks"]:
        counts[ROUTE_CLASS[c["route"]]] += 1
    return counts
