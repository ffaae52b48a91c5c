"""Planner parameters of the BASELINE configs (SURVEY.md 8d: "always record ans_size_log, n_bins, mean ans/offset bits per latent,
compressed size"), read with pcodec_b200.inspect from chunk 0 (seed 0, 2^18 numbers) of every config.

The bytes come from the CPU oracle, so this runs without a GPU; tests/test_gpu_baseline_fullsize.py checks that the GPU path writes
these same bytes for C1, C2, C3 and every C5 row.
Usage: python tests/make_chunk_stats.py [out.md]      (tests/ may use the oracle; the product never does)
"""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np

from oracle import pyoracle as o
from pcodec_b200 import datagen
from pcodec_b200 import inspect as insp

N = 1 << 18
rows = []


def add(name, nums, **kw):
    data = o.simple_compress(nums, o.make_config(**kw))
    s = insp.inspect(data)
    c = s["chunk"][0]
    cells = []
    for key in ("primary", "secondary"):
        v = c["latent_var"].get(key)
        cells += ["-"] * 4 if v is None else [str(v["n_bins"]), str(v["ans_size_log"]), f"{v['approx_avg_ans_bits']:.2f}", f"{v['approx_avg_offset_bits']:.2f}"]
    rows.append([name, c["mode"], c["delta_encoding"].replace(", secondary_uses_delta=false", "")] + cells +
                [str(c["meta_size"]), str(c["page_size"]), f"{nums.nbytes / (c['meta_size'] + c['page_size']):.2f}"])
    print(rows[-1], flush=True)


rng = np.random.default_rng(0)
add("C1 u32 lomax", datagen.c1_u32_lomax(seed=0), mode=o.MODE_CLASSIC, delta=o.DELTA_NOOP)
add("C2(i) u64 cumsum geometric(0.001)", datagen.c2_u64_cumsum_geometric(seed=0), mode=o.MODE_CLASSIC, delta=o.DELTA_CONSECUTIVE, delta_order=1)
add("C2(ii) u64 uniform random", rng.integers(0, 1 << 64, size=N, dtype=np.uint64), mode=o.MODE_CLASSIC, delta=o.DELTA_CONSECUTIVE, delta_order=1)
add("C2(iii) u64 arithmetic sequence", (np.arange(N, dtype=np.uint64) * np.uint64(77) + np.uint64(12345)), mode=o.MODE_CLASSIC, delta=o.DELTA_CONSECUTIVE, delta_order=1)
add("C3 f64 decimal sinusoid", datagen.c3_f64_decimal_sinusoid(seed=0), mode=o.MODE_FLOAT_MULT, float_mult_base=0.01, delta=o.DELTA_CONSECUTIVE, delta_order=2)
for dtype in (np.uint8, np.uint16, np.int32, np.int64, np.float32, np.float64):
    nums = datagen.c5_sweep(dtype, seed=0)
    for order in range(8):
        add(f"C5 {np.dtype(dtype).name} order {order}", nums, mode=o.MODE_CLASSIC, delta=o.DELTA_CONSECUTIVE if order else o.DELTA_NOOP, delta_order=order, enable_8_bit=True)

out = sys.argv[1] if len(sys.argv) > 1 else "chunk_stats.md"
with open(out, "w") as f:
    f.write("Planner parameters of the BASELINE configs: chunk 0 (seed 0, 2^18 numbers, level 8) of each config, read by `pcodec_b200.inspect` from\n"
            "the oracle's bytes (`tests/make_chunk_stats.py`; the GPU path writes the same bytes - `tests/test_gpu_baseline_fullsize.py`).\n"
            "avg bits are per stored latent, from the bin weights as `pco inspect` computes them (pco_cli/src/inspect/mod.rs:96-121): tANS part\n"
            "= sum w (size_log - log2 w) / 2^size_log, offset part = sum w offset_bits / 2^size_log.  ratio = number bytes / (chunk meta + page).\n\n")
    f.write("| config | mode | delta | primary n_bins | ans_size_log | avg tANS bits | avg offset bits | secondary n_bins | ans_size_log | avg tANS bits | avg offset bits | meta bytes | page bytes | ratio |\n")
    f.write("|---|---|---|---|---|---|---|---|---|---|---|---|---|---|\n")
    for r in rows:
        f.write("| " + " | ".join(r) + " |\n")
print("wrote", out)
