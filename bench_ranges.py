#!/usr/bin/env python
"""bench_ranges.py — ranges of an indexed standalone file (pco_b200_decompress_ranges) against decoding the whole file.

Two files of bench.py's size, 1024 chunks of 2^18 u64 (C2 data, chunk c = datagen.c2_u64_cumsum_geometric(seed = c)), classic mode,
each written by pco_b200_compress_ex with its side index, every buffer in HBM:
  - order1: consecutive delta order 1 (bench.py's file): a range decodes its chunks from batch 0 up to its last number;
  - order0: DeltaSpec NoOp: a range decodes only the batches it touches.
Legs per file, with seeded random positions:
  - range_1m: one range of 2^20 numbers;
  - points_1, points_64, points_4096: point lookups (count = 1);
  - ranges_4096: 4096 ranges of 256 to 65,536 numbers;
  - whole_then_slice: pco_b200_decompress_ex of the whole file, then the 4096 point lookups gathered from it on the device (the
    alternative without this call; slicing costs the same for every leg).
One warm-up call each, then `--steps` calls timed with CUDA events (profiler off), then one profiled call for the per-kernel split.
`parity`: every leg's output equals the same positions of the input.  Prints one JSON line; writes nothing.

    python bench_ranges.py [--steps 10] [--chunks 1024]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_levels import CHUNK_N, gpu_description, parse_profile  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--chunks", type=int, default=1024)
    args = ap.parse_args()

    import torch

    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, _lib, datagen, standalone

    L = _lib.lib()
    if not L.pco_b200_device_available():
        raise RuntimeError("libcpcodec.so found no usable CUDA device: " + L.pco_b200_last_error_message().decode())
    L.pco_b200_decompress_ex.argtypes = [C.c_void_p, C.c_size_t, C.c_ubyte, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p]
    dev = torch.device("cuda", 0)
    n_chunks = args.chunks
    n = n_chunks * CHUNK_N
    h_np = np.empty(n, dtype=np.uint64)
    for c in range(n_chunks):
        h_np[c * CHUNK_N:(c + 1) * CHUNK_N] = datagen.c2_u64_cumsum_geometric(CHUNK_N, seed=c)
    nums = torch.from_numpy(h_np.view(np.int64)).to(dev)
    stream = torch.cuda.current_stream()
    sp = C.c_void_p(stream.cuda_stream)
    SRC, DST, IDX = 1, 2, 4
    cap = L.pco_standalone_guarantee_file_size(n, 2)
    icap = L.pco_b200_index_size_bound(n, n_chunks)
    d_whole = torch.empty(n, dtype=torch.int64, device=dev)

    rng = np.random.default_rng(0)
    legs = {"range_1m": [(int(rng.integers(0, n - (1 << 20))), 1 << 20)]}
    for m in (1, 64, 4096):
        legs[f"points_{m}"] = [(int(s), 1) for s in rng.integers(0, n, m)]
    starts = rng.integers(0, n - 65536, 4096)
    legs["ranges_4096"] = [(int(s), int(c)) for s, c in zip(starts, rng.integers(256, 65537, 4096))]
    points = legs["points_4096"]
    d_points = torch.as_tensor(np.array([s for s, _ in points], dtype=np.int64), device=dev)
    max_total = max(sum(c for _, c in v) for v in legs.values())
    d_out = torch.empty(max_total, dtype=torch.int64, device=dev)
    nw = C.c_size_t()

    def timed(fn, steps):
        fn()  # warm-up (modules, scratch)
        torch.cuda.synchronize()
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(max(steps, 1))]
        for a, b in evs:
            a.record(stream)
            fn()
            b.record(stream)
        torch.cuda.synchronize()
        ms = [a.elapsed_time(b) for a, b in evs]
        L.pco_b200_profile_enable(1)
        fn()
        prof = parse_profile(L)
        L.pco_b200_profile_enable(0)
        return {"ms": float(np.mean(ms)), "ms_min": float(np.min(ms)), "ms_max": float(np.max(ms)), "kernel_ms": prof}

    res, parity = {}, {}
    for name, order in (("order1", 1), ("order0", 0)):
        ds = DeltaSpec.try_consecutive(1) if order else DeltaSpec.no_op()
        cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=ds)._to_c()
        d_file = torch.empty(cap, dtype=torch.uint8, device=dev)
        d_index = torch.empty(icap, dtype=torch.uint8, device=dev)
        written, ilen = C.c_size_t(), C.c_size_t()
        _lib.check(L.pco_b200_compress_ex(C.c_void_p(nums.data_ptr()), C.c_size_t(n), C.c_ubyte(2), C.byref(cfg), C.c_int(0), C.c_void_p(d_file.data_ptr()),
                                          C.c_size_t(cap), C.byref(written), C.c_void_p(d_index.data_ptr()), C.c_size_t(icap), C.byref(ilen),
                                          C.c_uint32(SRC | DST | IDX), sp))
        torch.cuda.synchronize()
        out = {"compressed_bytes": written.value}

        for leg, pairs in legs.items():
            r = standalone._ranges_array(pairs)
            total = int(r["count"].sum())

            def call(r=r, total=total):
                _lib.check(L.pco_b200_decompress_ranges(C.c_void_p(d_file.data_ptr()), C.c_size_t(written.value), C.c_ubyte(2), C.c_void_p(d_index.data_ptr()),
                                                        C.c_size_t(ilen.value), r.ctypes.data_as(C.c_void_p), C.c_size_t(r.size), C.c_void_p(d_out.data_ptr()),
                                                        C.c_size_t(total), C.byref(nw), C.c_uint32(SRC | DST | IDX), sp))

            t = timed(call, args.steps)
            t["numbers"] = total
            out[leg] = t
            want = torch.cat([nums[s:s + c] for s, c in pairs])
            parity[f"{name}.{leg}"] = bool(nw.value == total and torch.equal(d_out[:total], want))

        prog = _lib._CProgress()

        def whole_then_slice():
            _lib.check(L.pco_b200_decompress_ex(C.c_void_p(d_file.data_ptr()), C.c_size_t(written.value), C.c_ubyte(2), C.c_void_p(d_whole.data_ptr()),
                                                C.c_size_t(n), C.byref(prog), C.c_void_p(d_index.data_ptr()), C.c_size_t(ilen.value), C.c_uint32(SRC | DST | IDX), sp))
            d_out[:len(points)] = d_whole[d_points]

        out["whole_then_slice"] = timed(whole_then_slice, args.steps)
        parity[f"{name}.whole_then_slice"] = bool(torch.equal(d_whole, nums) and torch.equal(d_out[:len(points)], nums[d_points]))
        res[name] = out
        del d_file, d_index

    # how much of a chunk a point lookup decodes: order 0 starts at the number's batch, order 1 at the chunk's first batch
    k0 = sum(res["order0"]["points_4096"]["kernel_ms"].values())
    k1 = sum(res["order1"]["points_4096"]["kernel_ms"].values())
    res["points_4096_kernel_ms_order0_over_order1"] = k0 / k1 if k1 else None
    res["parity"] = {"all": all(parity.values()), **parity}
    print(json.dumps({"workload": f"C2: {n_chunks} chunks x 2^18 u64, classic mode, order 1 and order 0 (NoOp), side index from compress_ex, device buffers",
                      "unit": "ms per call", "steps": args.steps, "gpu": gpu_description(), **res}))


if __name__ == "__main__":
    main()
