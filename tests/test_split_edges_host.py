"""The split restatement and the size-guarantee boundary cases of tests/split_edges.py, pinned to the oracle (no GPU).

* The restated latents, dissected with the oracle's own bins into (bin, offset) pairs and written by the oracle's explicit writer,
  give the oracle's simple_compress file byte for byte - subnormal FloatMult bases, NaN payloads and all.
* The oracle decodes every family back bit for bit.
* Every boundary case sits at the margin (worst case size - baseline) it was found at, and falls back exactly when that is > 0.
* The margins the oracle reports equal the size formula (chunk_compressor.rs:502-541) restated from the chunk's bins and counts.
"""
import numpy as np
import pytest

from tests import split_edges as se

FAMILIES = se.families()
BOUNDARY = [se.boundary_family(combo, *v) | {"margin": m} for (combo, m), v in se.BOUNDARY.items()]
STANDALONE_BOUNDARY = [f for f in BOUNDARY if not f.get("pages")]


def _ids(fams):
    return [f["name"] for f in fams]


def _compress(oracle, fam):
    """The oracle's file and (worst, baseline) of its one chunk."""
    data = oracle.simple_compress(fam["nums"], se.oracle_configs(oracle, fam))
    margins = oracle.last_fallback_margins()
    assert len(margins) == 1, (fam["name"], margins)
    return data, margins[0]


def _stored_vars(fam, chunk):
    """Per latent var of the oracle's chunk meta: (var meta, stored latents, moments) from the restated split."""
    bits = se.nbits(fam["dtype"])
    p, s = se.split(fam["nums"], fam["mode"], fam["base"], fam["k"])
    out = []
    for v, lat in enumerate([p] + ([s] if s is not None else [])):
        stored, moments = se.delta_encode(lat, fam["order"] if v == 0 else 0, bits)
        out.append((chunk["vars"][v], stored, moments))
    return out


def _explicit_spec(fam, chunk):
    vars_ = []
    for meta, stored, moments in _stored_vars(fam, chunk):
        sym, off = se.dissect(stored, meta["bins"])
        vars_.append(dict(ans_size_log=meta["ans_size_log"], bins=meta["bins"], symbols=sym, offsets=off, moments=moments))
    spec = dict(n=fam["nums"].size, mode=fam["mode"], order=fam["order"], vars=vars_)
    if fam["mode"] == "int_mult":
        spec["base"] = int(fam["base"]) & se._mask(se.nbits(fam["dtype"]))
    elif fam["mode"] == "float_mult":
        spec["base"] = int(se.to_latents(np.array([fam["base"]], dtype=fam["dtype"]))[0])
    elif fam["mode"] == "float_quant":
        spec["k"] = fam["k"]
    return spec


def _kept(fam, chunk, worst, baseline):
    """The chunk kept the family's mode and delta exactly when it did not fall back, and fell back to Classic / NoOp otherwise."""
    fell_back = worst > baseline and not (fam["mode"] == "classic" and fam["order"] == 0)
    want = (0, 0, 0) if fell_back else (se.MODE_CODE[fam["mode"]], 1 if fam["order"] else 0, fam["order"])
    assert (chunk["mode"], chunk["delta"], chunk["delta_order"]) == want, (fam["name"], worst - baseline, chunk)
    return not fell_back


@pytest.mark.parametrize("fam", FAMILIES + STANDALONE_BOUNDARY, ids=_ids(FAMILIES + STANDALONE_BOUNDARY))
def test_restated_split_gives_the_oracles_bytes(oracle, fam):
    want, (worst, baseline) = _compress(oracle, fam)
    chunk = oracle.inspect(want, fam["dtype"])["chunks"][0]
    if not _kept(fam, chunk, worst, baseline):
        pytest.skip("the chunk falls back to Classic; its latents are the numbers'")
    got, _ = oracle.write_explicit_file(fam["dtype"], [_explicit_spec(fam, chunk)])
    assert got == want, fam["name"]


def test_families_reach_their_edges(oracle):
    """Enough of each mode is kept for the pinning to mean something; every subnormal-base FloatMult family keeps FloatMult."""
    kept = {}
    for fam in FAMILIES:
        data, (w, b) = _compress(oracle, fam)
        ok = _kept(fam, oracle.inspect(data, fam["dtype"])["chunks"][0], w, b)
        kept.setdefault(fam["mode"], []).append(ok)
        if fam["mode"] == "float_mult" and abs(fam["base"]) < 1e-37 and fam["level"] != 0:
            assert ok, fam["name"]
    for mode, oks in kept.items():
        assert sum(oks) >= 0.85 * len(oks), (mode, sum(oks), len(oks))
    # IntMult bases with bits above the type width reach the compressor as given and are kept as their low bits, for every width
    over = [f for f in FAMILIES if f["mode"] == "int_mult" and f["base"] >> se.nbits(f["dtype"])]
    assert {se.nbits(f["dtype"]) for f in over} == {8, 16, 32}
    for width in (8, 16, 32):
        kept_bases = set()
        for f in over:
            if se.nbits(f["dtype"]) == width:
                data, (w, b) = _compress(oracle, f)
                chunk = oracle.inspect(data, f["dtype"])["chunks"][0]
                if _kept(f, chunk, w, b):
                    kept_bases.add(chunk["mode_base_latent"])
        assert kept_bases == {f["base"] & se._mask(width) for f in over if se.nbits(f["dtype"]) == width}, width
    # a base above every latent of its chunk: every primary latent is 0
    for f in FAMILIES:
        if f["name"].startswith("int_mult-") and "-babove-" in f["name"]:
            p, s = se.split(f["nums"], "int_mult", f["base"])
            assert not p.any() and np.array_equal(s, se.to_latents(f["nums"])), f["name"]
    # 0 * inf is a NaN the multiply produces: the restated multiplier of every zero is x86's default NaN
    f = next(f for f in FAMILIES if f["name"] == "float_mult-f64-b1e-310-o0")
    zeros = f["nums"] == 0
    assert zeros.any()
    assert set(se.float_mult_mults(f["nums"][zeros], f["base"]).tolist()) == {0xFFF8000000000000}


@pytest.mark.parametrize("fam", FAMILIES + BOUNDARY, ids=_ids(FAMILIES + BOUNDARY))
def test_oracle_round_trip(oracle, fam):
    cfg = se.oracle_configs(oracle, fam)
    u = se._u(fam["dtype"])
    if fam.get("pages"):
        occ = oracle.ChunkCompressor(fam["nums"], cfg)
        meta, off = occ.write_meta(), 0
        for i, pn in enumerate(occ.n_per_page()):
            back, _, _ = oracle.wrapped_decompress_page(meta, occ.write_page(i), fam["dtype"], pn)
            np.testing.assert_array_equal(back.view(u), fam["nums"][off: off + pn].view(u))
            off += pn
        return
    back = oracle.simple_decompress(oracle.simple_compress(fam["nums"], cfg), fam["dtype"])
    np.testing.assert_array_equal(back.view(u), fam["nums"].view(u))


def test_every_boundary_target_is_found_or_named():
    for combo in se.BOUNDARY_COMBOS:
        for m in (-1, 0, 1):
            assert ((combo, m) in se.BOUNDARY) != ((combo, m) in se.UNREACHED), (combo, m)


@pytest.mark.parametrize("fam", BOUNDARY, ids=_ids(BOUNDARY))
def test_boundary_margin(oracle, fam):
    assert se.margin(oracle, fam) == fam["margin"], fam["name"]
    if fam.get("pages"):
        return
    data, (w, b) = _compress(oracle, fam)
    assert _kept(fam, oracle.inspect(data, fam["dtype"])["chunks"][0], w, b) == (fam["margin"] <= 0)


def _restated_margins(fam, chunk):
    """worst_case_size and baseline (bytes) of a one-page chunk from its bins and the dissected per-bin counts."""
    lbits = se.nbits(fam["dtype"])
    obb = lbits.bit_length()  # bits of an offset-bits field
    payload = {"classic": 0, "float_quant": 8}.get(fam["mode"], lbits)
    delta_max = 4 + 5 + 5 + 64 + 32 * 32  # DeltaEncoding::MAX_BIT_SIZE
    meta_bits = 4 + payload + delta_max
    page_meta_bits, wc_bits = 0, 7
    for v, (meta, stored, _) in enumerate(_stored_vars(fam, chunk)):
        bins = meta["bins"]
        size_log = meta["ans_size_log"]
        meta_bits += 4 + 15 + len(bins) * (size_log + lbits + obb)
        page_meta_bits += 4 * size_log + (lbits * fam["order"] if v == 0 else 0)
        sym, _ = se.dissect(stored, bins)
        counts = np.bincount(sym, minlength=len(bins))
        wc_bits += sum(int(c) * (ob + size_log - (int(w).bit_length() - 1)) for c, (w, _, ob) in zip(counts, bins))
    worst = -(-meta_bits // 8) + -(-page_meta_bits // 8) + -(-wc_bits // 8)
    baseline = -(-(4 + delta_max + 4 + 15 + lbits + obb) // 8) + -(-(fam["nums"].size * lbits) // 8)
    return worst, baseline


@pytest.mark.parametrize("fam", FAMILIES + STANDALONE_BOUNDARY, ids=_ids(FAMILIES + STANDALONE_BOUNDARY))
def test_margin_hook_matches_the_size_formula(oracle, fam):
    data, (worst, baseline) = _compress(oracle, fam)
    chunk = oracle.inspect(data, fam["dtype"])["chunks"][0]
    if not _kept(fam, chunk, worst, baseline):
        pytest.skip("the chunk falls back; its bins are the fallback's")
    assert _restated_margins(fam, chunk) == (worst, baseline), fam["name"]
