"""The oracle's explicit stream writer (pco_oracle_write_explicit_file) and the crafted families of tests/crafted_streams.py, on the CPU.

The writer is pinned to the format first: fed the bins the oracle's own compressor chose and the (bin, offset) pairs those bins give
the stored latents, it must write the compressor's file byte for byte, for every number type, Classic and IntMult, and consecutive
orders 0-7.  Then every crafted family must decode on the oracle to the numpy restatement of the decode, and pcodec_b200.inspect
must read the crafted bins back.  Specs the format's reader would refuse are refused by the writer."""
import numpy as np
import pytest

from pcodec_b200 import inspect as insp
from tests import crafted_streams as cs

ALL_TYPES = list(cs.DTYPES)
FAMILIES = cs.all_families()


# ---- the writer, pinned to the oracle's compressor ------------------------------------------------------------------------------
def _ordinary(dtype, n, seed):
    """A bounded random walk (so that the consecutive orders find something to take out) in the type's range."""
    dt = np.dtype(cs.DTYPES[dtype])
    rng = np.random.default_rng(seed)
    if dt.kind == "f":
        return np.cumsum(rng.normal(size=n)).astype(dt) * dt.type(3)
    bits = cs.nbits(dt)
    walk = np.cumsum(rng.integers(-40, 41, size=n)) + rng.integers(0, 1 << min(bits - 2, 30))
    return cs.from_latents(np.asarray(walk, dtype=np.int64).astype(np.uint64) & cs._mask(bits), dt)


def _consecutive_encode(lat, order, bits):
    """delta/consecutive.rs:3-33: `order` rounds of differences, each keeping its first value as a moment; the rest centred."""
    mask = cs._mask(bits)
    moments = []
    v = lat.copy()
    for _ in range(order):
        moments.append(int(v[0]) if v.size else 0)
        v = (v[1:] - v[:-1]) & mask
    return (v + np.uint64(1 << (bits - 1))) & mask, moments


def _spec_from_oracle_file(data, nums):
    """The explicit spec of every chunk of an oracle file: bins and mode from oracle.inspect, stored latents and moments from the split
    and delta restated here, each latent's bin the last whose lower is at or below it (what the encoder does for its sorted bins)."""
    from oracle import pyoracle as O

    info = O.inspect(data, nums.dtype)
    bits = cs.nbits(nums.dtype)
    chunks, at = [], 0
    for ch in info["chunks"]:
        x = nums[at:at + ch["n"]]
        at += ch["n"]
        lat = cs.to_latents(x)
        mode = {0: "classic", 1: "int_mult"}[ch["mode"]]
        if mode == "int_mult":
            base = np.uint64(ch["mode_base_latent"])
            split = [lat // base, lat % base]
        else:
            split = [lat]
        order = ch["delta_order"] if ch["delta"] == 1 else 0
        assert ch["delta"] in (0, 1)
        vars_ = []
        for v, (latents, meta) in enumerate(zip(split, ch["vars"])):
            moments = []
            if v == 0 and order:
                latents, moments = _consecutive_encode(latents, order, bits)
            bins = meta["bins"]
            lowers = np.array([b[1] for b in bins], dtype=np.uint64)
            assert np.all(lowers[1:] > lowers[:-1]), "the compressor's bins are sorted by lower"
            sym = np.searchsorted(lowers, latents, side="right") - 1
            vars_.append({"ans_size_log": meta["ans_size_log"], "bins": [tuple(b) for b in bins], "symbols": sym,
                          "offsets": (latents - lowers[sym]) & cs._mask(bits), "moments": moments})
        c = {"n": ch["n"], "mode": mode, "order": order, "vars": vars_}
        if mode == "int_mult":
            c["base"] = ch["mode_base_latent"]
        chunks.append(c)
    return chunks


@pytest.mark.parametrize("mode", ["classic", "int_mult"])
@pytest.mark.parametrize("dtype", ALL_TYPES)
def test_writer_reproduces_the_oracle_compressor(oracle, dtype, mode):
    dt = np.dtype(cs.DTYPES[dtype])
    if mode == "int_mult" and dt.kind == "f":
        pytest.skip("IntMult is for integers")
    base = 7
    for order in range(8):
        for n, page in ((1000, 0), (1000, 600), (9, 0), (300, 0)):
            nums = _ordinary(dtype, n, seed=order * 31 + n)
            if mode == "int_mult":
                lat = cs.to_latents(nums)
                nums = cs.from_latents(lat - lat % np.uint64(base) + np.uint64(2), dt)
            cfg = oracle.make_config(mode=oracle.MODE_INT_MULT if mode == "int_mult" else oracle.MODE_CLASSIC, int_mult_base=base if mode == "int_mult" else 0,
                                     delta=oracle.DELTA_CONSECUTIVE if order else oracle.DELTA_NOOP, delta_order=order, max_page_n=page)
            want = oracle.simple_compress(nums, cfg)
            spec = _spec_from_oracle_file(want, nums)
            got, parts = oracle.write_explicit_file(dt, spec)
            assert got == want, (dtype, mode, order, n, page)
            metas = oracle.inspect(want, dt)["chunks"]
            assert b"".join(m + p for m, p in parts) == b"".join(want[c["meta_start"]:c["chunk_end"]] for c in metas)


def test_writer_pin_reaches_the_modes_and_orders(oracle):
    """The pin above would be empty if the compressor fell back to its one-bin classic chunk: it does keep IntMult and the orders."""
    nums = _ordinary("u32", 1000, seed=5)
    lat = cs.to_latents(nums)
    nums = cs.from_latents(lat - lat % np.uint64(7) + np.uint64(2), np.uint32)
    for order in range(8):
        cfg = oracle.make_config(mode=oracle.MODE_INT_MULT, int_mult_base=7, delta=oracle.DELTA_CONSECUTIVE if order else oracle.DELTA_NOOP, delta_order=order)
        ch = oracle.inspect(oracle.simple_compress(nums, cfg), np.uint32)["chunks"][0]
        assert ch["mode"] == 1 and ch["delta_order"] == order, ch
        assert len(ch["vars"][0]["bins"]) > 1 or order > 2, ch  # at high orders the walk's deltas are noise: one wide bin


# ---- the families ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fam", FAMILIES, ids=[f["name"] for f in FAMILIES])
def test_oracle_decodes_family_to_the_restatement(oracle, fam):
    data, parts = cs.write(oracle, fam)
    got = oracle.simple_decompress(data, fam["dtype"])
    want = cs.expected(fam)
    np.testing.assert_array_equal(got.view(cs._u(fam["dtype"])), want.view(cs._u(fam["dtype"])))
    at = 0
    for (meta, page), c in zip(parts, fam["chunks"]):  # the wrapped meta and page of each chunk decode to the same numbers
        back, mc, pc = oracle.wrapped_decompress_page(meta, page, fam["dtype"], c["n"])
        assert (mc, pc) == (len(meta), len(page))
        np.testing.assert_array_equal(back.view(cs._u(fam["dtype"])), want[at:at + c["n"]].view(cs._u(fam["dtype"])))
        at += c["n"]


@pytest.mark.parametrize("fam", [f for f in FAMILIES if sum(c["n"] for c in f["chunks"]) <= 1 << 16], ids=lambda f: f["name"])
def test_inspect_reports_the_crafted_bins(oracle, fam):
    data, _ = cs.write(oracle, fam)
    summary = insp.inspect(data)
    assert summary["n_chunks"] == len(fam["chunks"]) and summary["compressed"]["unknown_trailing_bytes"] == 0
    for got, c in zip(summary["chunk"], fam["chunks"]):
        assert got["n"] == c["n"]
        for key, v in zip(("primary", "secondary"), c["vars"]):
            lv = got["latent_var"][key]
            assert lv["ans_size_log"] == v["ans_size_log"]
            assert [tuple(b) for b in lv["bins"]] == [tuple(b) for b in v["bins"]]


def test_families_cover_every_route():
    routes = {c["route"] for f in FAMILIES for c in f["chunks"]}
    assert routes == {"fused3", "fused4", "fused5", "general1", "general2", "cold"}


# ---- invalid specs --------------------------------------------------------------------------------------------------------------
def _one(bins, n=8, bits_ob=None, offsets=None, **kw):
    sym = [i % len(bins) for i in range(n)]
    offs = offsets if offsets is not None else [0] * n
    lg = kw.pop("ans_size_log", None)
    if lg is None:
        w = sum(b[0] for b in bins)
        lg = max(w.bit_length() - 1, 0)
    return [dict(n=n, vars=[dict(ans_size_log=lg, bins=bins, symbols=sym, offsets=offs)], **kw)]


INVALID = {
    "weights_short": _one([(1, 0, 0), (2, 5, 0)], ans_size_log=2),
    "weights_long": _one([(3, 0, 0), (2, 5, 0)], ans_size_log=2),
    "more_bins_than_states": _one([(1, 0, 0), (1, 5, 0), (1, 9, 0)], ans_size_log=1),
    "ans_size_log_15": _one([(1 << 14, 0, 0), (1 << 14, 5, 0)], ans_size_log=15),
    "one_bin_log_1": _one([(2, 0, 3)], ans_size_log=1),
    "offset_bits_33": _one([(1, 0, 33), (1, 5, 0)]),
    "offset_too_wide": _one([(1, 0, 3), (1, 5, 0)], offsets=[8] + [0] * 7),
    "int_mult_base_0": [dict(n=4, mode="int_mult", base=0, vars=[dict(ans_size_log=0, bins=[(1, 0, 3)], symbols=[0] * 4, offsets=[1] * 4)] * 2)],
    "float_mode_on_ints": [dict(n=4, mode="float_quant", k=3, vars=[dict(ans_size_log=0, bins=[(1, 0, 3)], symbols=[0] * 4, offsets=[1] * 4)] * 2)],
    "stored_count": [dict(n=5, order=1, vars=[dict(ans_size_log=0, bins=[(1, 0, 3)], symbols=[0] * 5, offsets=[1] * 5, moments=[3])])],
}
FLOAT_INVALID = {
    "float_quant_k_0": dict(mode="float_quant", k=0),
    "float_quant_k_24": dict(mode="float_quant", k=24),
    "float_mult_base_inf": dict(mode="float_mult", base=cs.float_latent(np.inf, np.float32)),
    "float_mult_base_0": dict(mode="float_mult", base=cs.float_latent(0.0, np.float32)),
    "int_mult_on_floats": dict(mode="int_mult", base=3),
}


@pytest.mark.parametrize("name", sorted(INVALID))
def test_invalid_specs_are_refused(oracle, name):
    with pytest.raises(oracle.OracleError) as e:
        oracle.write_explicit_file(np.uint32, INVALID[name])
    assert e.value.kind == "InvalidArgument", e.value


@pytest.mark.parametrize("name", sorted(FLOAT_INVALID))
def test_invalid_float_modes_are_refused(oracle, name):
    v = dict(ans_size_log=0, bins=[(1, 0, 3)], symbols=[0] * 4, offsets=[1] * 4)
    with pytest.raises(oracle.OracleError) as e:
        oracle.write_explicit_file(np.float32, [dict(n=4, vars=[v, v], **FLOAT_INVALID[name])])
    assert e.value.kind == "InvalidArgument", e.value
    ok = dict(FLOAT_INVALID[name], k=23) if name == "float_quant_k_24" else None
    if ok:  # the edge itself is valid
        oracle.write_explicit_file(np.float32, [dict(n=4, vars=[v, v], **ok)])
