"""Property test of the GPU path against the oracle (hypothesis): for any in-scope number type, data shape, mode, consecutive delta
order, level and paging, the GPU writes the oracle's bytes and decodes them back bit for bit; anything the path refuses is refused as
Unsupported, never mis-encoded.  Same generators as tests/test_oracle_properties.py."""
import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

from tests.golden_generators import bits_view
from tests.test_oracle_properties import arrays

pytestmark = pytest.mark.gpu


@st.composite
def gpu_configs(draw, dtype):
    dtype = np.dtype(dtype)
    modes = ["classic"] + (["float_quant"] + (["float_mult"] if dtype.itemsize >= 4 else []) if dtype.kind == "f" else ["int_mult"])
    kw = dict(mode=draw(st.sampled_from(modes)), order=draw(st.integers(0, 7)), level=draw(st.integers(0, 12)), max_page_n=draw(st.sampled_from([0, 100, 256, 300])))
    kw["base"] = draw(st.sampled_from([0.01, 0.5, 1.0, 3.0])) if kw["mode"] == "float_mult" else draw(st.sampled_from([1, 2, 7, 10, 255]))
    kw["k"] = draw(st.integers(1, {2: 10, 4: 23, 8: 52}.get(dtype.itemsize, 1)))
    return kw


def _dump_failure(nums, kw, got, want):
    """A falsifying example is data: keep it (numbers, config, both files) in $PCOB200_PROP_DUMP, or the temporary directory."""
    import hashlib
    import json
    import os
    import tempfile

    root = os.environ.get("PCOB200_PROP_DUMP") or os.path.join(tempfile.gettempdir(), "pcodec_prop_failures")
    try:
        os.makedirs(root, exist_ok=True)
        tag = hashlib.sha1(nums.tobytes() + repr(sorted((k, str(v)) for k, v in kw.items())).encode()).hexdigest()[:12]
        np.save(os.path.join(root, f"prop_fail_{tag}_{nums.dtype.name}.npy"), nums.view(f"u{nums.dtype.itemsize}"))
        with open(os.path.join(root, f"prop_fail_{tag}.json"), "w") as f:
            json.dump({"kw": kw, "dtype": nums.dtype.name, "n": int(nums.size), "got_hex": (got or b"").hex(), "want_hex": want.hex()}, f)
    except OSError:
        pass


@settings(max_examples=400, deadline=None, suppress_health_check=[HealthCheck.too_slow, HealthCheck.data_too_large])
@given(data=st.data())
def test_gpu_bytes_equal_the_oracles(oracle, data):
    import pcodec_b200 as p

    nums = data.draw(arrays())
    kw = data.draw(gpu_configs(nums.dtype))
    mode_spec = {"classic": p.ModeSpec.classic(), "int_mult": p.ModeSpec.try_int_mult(kw["base"]), "float_mult": p.ModeSpec.try_float_mult(kw["base"]),
                 "float_quant": p.ModeSpec.try_float_quant(kw["k"])}[kw["mode"]]
    omode = {"classic": oracle.MODE_CLASSIC, "int_mult": oracle.MODE_INT_MULT, "float_mult": oracle.MODE_FLOAT_MULT, "float_quant": oracle.MODE_FLOAT_QUANT}[kw["mode"]]
    cfg = p.ChunkConfig(compression_level=kw["level"], mode_spec=mode_spec, delta_spec=p.DeltaSpec.try_consecutive(kw["order"]) if kw["order"] else p.DeltaSpec.no_op(),
                        paging_spec=p.PagingSpec.equal_pages_up_to(kw["max_page_n"] or (1 << 18)), enable_8_bit=True)
    ocfg = oracle.make_config(level=kw["level"], mode=omode, delta=oracle.DELTA_CONSECUTIVE if kw["order"] else oracle.DELTA_NOOP, delta_order=kw["order"],
                              float_mult_base=float(kw["base"]), int_mult_base=int(kw["base"]) if kw["mode"] == "int_mult" else 0, float_quant_k=kw["k"],
                              max_page_n=kw["max_page_n"], enable_8_bit=True)
    want = oracle.simple_compress(nums, ocfg)
    try:
        got = p.standalone.simple_compress(nums, cfg)
    except p.PcoError as e:
        if e.kind != "Unsupported":
            _dump_failure(nums, dict(kw, error=str(e), where="compress"), None, want)
        assert e.kind == "Unsupported", (kw, e)  # e.g. more than 256 bins at the highest levels
        got = None
    if got is not None and got != want:
        _dump_failure(nums, kw, got, want)
        assert got == want, kw
    try:
        back = p.standalone.simple_decompress(want, nums.dtype)
    except p.PcoError as e:
        if e.kind != "Unsupported":
            _dump_failure(nums, dict(kw, error=str(e), where="decompress"), None, want)
        assert e.kind == "Unsupported", (kw, e)
        return
    if not np.array_equal(bits_view(back), bits_view(nums)):
        _dump_failure(nums, dict(kw, where="decode differs"), back.tobytes(), want)
        a, b = bits_view(back), bits_view(nums)
        bad = np.nonzero(a != b)[0] if a.shape == b.shape else np.array([], dtype=int)
        raise AssertionError(f"GPU decode of the oracle's file differs: {kw}, dtype {nums.dtype}, n {nums.size} vs {back.size}, first differing indices {bad[:5].tolist()}, "
                             f"got {[hex(int(x)) for x in a[bad[:5]]]} want {[hex(int(x)) for x in b[bad[:5]]]}, nums bits {[hex(int(x)) for x in b[:40]]}")
