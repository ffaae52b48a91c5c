"""PCOB200_AUTO_MODE_SEARCH=1: ModeSpec::Auto inside the library resolved by the host-side search over the call's first chunk
(pcodec_b200/csrc/compress_host.cuh, mode_search.hpp).  The search itself is covered on CPU (tests/test_mode_search_host.py); this file
checks the wiring: with an explicit delta, Auto-mode bytes equal the oracle's Auto-mode bytes.

The library keeps this search opt-in and reads the switch once per process, hence the child process.
"""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

CHILD = r"""
import sys
sys.path.insert(0, sys.argv[1])
import numpy as np
from oracle import pyoracle as o
from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec, standalone as sa
rng = np.random.default_rng(3)
n = 20000
cases = {
    "decimals_f64": (rng.integers(-5000, 5000, size=n).astype(np.float64) / 100.0, 2),
    "decimals_f32": ((rng.integers(-5000, 5000, size=n).astype(np.float64) / 100.0).astype(np.float32), 1),
    "int_mult_u32": ((rng.integers(0, 1 << 20, size=n) * 77).astype(np.uint32), 0),
    "int_mult_i64": ((rng.integers(-(1 << 30), 1 << 30, size=n) * 1000).astype(np.int64), 1),
    "quant_f64": (((rng.standard_normal(n).view(np.uint64) >> np.uint64(30)) << np.uint64(30)).view(np.float64), 0),
    "plain_u64": (rng.integers(0, 1 << 40, size=n).astype(np.uint64), 0),
    "plain_f32": (rng.standard_normal(n).astype(np.float32), 0),
}
for name, (nums, order) in cases.items():
    for max_page_n in (1 << 18, 7000):  # one chunk, three chunks (homogeneous data: every chunk makes the same choice)
        delta = DeltaSpec.try_consecutive(order) if order else DeltaSpec.no_op()
        got = sa.simple_compress(nums, ChunkConfig(mode_spec=ModeSpec.auto(), delta_spec=delta, paging_spec=PagingSpec.equal_pages_up_to(max_page_n)))
        want = o.simple_compress(nums, o.make_config(mode=o.MODE_AUTO, delta=o.DELTA_CONSECUTIVE if order else o.DELTA_NOOP, delta_order=order, max_page_n=max_page_n))
        assert got == want, (name, max_page_n, len(got), len(want))
        back = sa.simple_decompress(got, nums.dtype)
        assert np.array_equal(back.view(np.uint8), nums.view(np.uint8)), name
print("AUTO_MODE_SEARCH_OK")
"""


def test_auto_mode_bytes_equal_the_oracles():
    root = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
    env = dict(os.environ, PCOB200_AUTO_MODE_SEARCH="1")
    res = subprocess.run([sys.executable, "-c", CHILD, root], capture_output=True, text=True, timeout=600, env=env)
    assert res.returncode == 0 and "AUTO_MODE_SEARCH_OK" in res.stdout, res.stdout[-2000:] + res.stderr[-4000:]
