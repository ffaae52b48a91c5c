#!/usr/bin/env python
"""bench_async.py — the asynchronous decompress (pco_b200_decompress_async) against pco_b200_decompress_ex on the same file and index.

Big file: bench.py's array and file - 1024 chunks of 2^18 u64 (C2 data, chunk c = datagen.c2_u64_cumsum_geometric(seed = c)), classic
mode, consecutive delta order 1, written by pco_b200_compress_ex with its side index, every buffer in HBM.  Legs, each timed with CUDA
events around `--steps` calls after one warm-up:
  - ex: pco_b200_decompress_ex (blocks until done; the events bracket its kernels and the host gaps between them);
  - async: pco_b200_decompress_async (enqueues only), and the host time one such call takes to return (`enqueue_us`);
  - graph: one async call captured in a torch.cuda.CUDAGraph, replayed.
A separate profiled call of ex and of async gives the per-kernel split.
Small file: 2^16 u64 numbers (one chunk, order 1) with its index in HBM: host wall time per call of a loop of `--small-steps`
decompress_ex calls, of as many back-to-back async calls with one synchronisation at the end, and of as many graph replays.
`parity`: every leg's output equals the input.  The card's name, power limit and max SM clock are read in the same run.
Prints one JSON line; writes nothing.

    python bench_async.py [--steps 10] [--small-steps 200] [--chunks 1024]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_levels import CHUNK_N, gpu_description, parse_profile  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--small-steps", type=int, default=200)
    ap.add_argument("--chunks", type=int, default=1024)
    args = ap.parse_args()

    import torch

    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, _lib, datagen, standalone

    L = _lib.lib()
    if not L.pco_b200_device_available():
        raise RuntimeError("libcpcodec.so found no usable CUDA device: " + L.pco_b200_last_error_message().decode())
    L.pco_b200_decompress_ex.argtypes = [C.c_void_p, C.c_size_t, C.c_ubyte, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p]
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream()
    sp = C.c_void_p(stream.cuda_stream)
    SRC, DST, IDX = 1, 2, 4
    cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(1))._to_c()

    def compress(nums, n_chunks):
        n = nums.numel()
        cap = L.pco_standalone_guarantee_file_size(n, 2)
        icap = L.pco_b200_index_size_bound(n, n_chunks)
        d_file = torch.empty(cap, dtype=torch.uint8, device=dev)
        d_index = torch.empty(icap, dtype=torch.uint8, device=dev)
        written, ilen = C.c_size_t(), C.c_size_t()
        _lib.check(L.pco_b200_compress_ex(C.c_void_p(nums.data_ptr()), C.c_size_t(n), C.c_ubyte(2), C.byref(cfg), C.c_int(0), C.c_void_p(d_file.data_ptr()),
                                          C.c_size_t(cap), C.byref(written), C.c_void_p(d_index.data_ptr()), C.c_size_t(icap), C.byref(ilen),
                                          C.c_uint32(SRC | DST | IDX), sp))
        torch.cuda.synchronize()
        return d_file[: written.value], d_index[: ilen.value]

    def setup(nums, n_chunks):
        """The file, its index, a destination for each leg and the calls."""
        n = nums.numel()
        d_file, d_index = compress(nums, n_chunks)
        outs = {k: torch.empty(n, dtype=torch.int64, device=dev) for k in ("ex", "async", "graph")}
        prog = _lib._CProgress()

        def ex():
            _lib.check(L.pco_b200_decompress_ex(C.c_void_p(d_file.data_ptr()), C.c_size_t(d_file.numel()), C.c_ubyte(2), C.c_void_p(outs["ex"].data_ptr()),
                                                C.c_size_t(n), C.byref(prog), C.c_void_p(d_index.data_ptr()), C.c_size_t(d_index.numel()),
                                                C.c_uint32(SRC | DST | IDX), C.c_void_p(torch.cuda.current_stream().cuda_stream)))

        head = d_file[:32].cpu().numpy()
        dec = standalone.AsyncDecompressor(head, np.uint64, d_file.numel(), d_index.numel(), n, n_chunks)
        dst_async, dst_graph = outs["async"].view(torch.uint64), outs["graph"].view(torch.uint64)

        def run_async():
            dec(d_file, d_index, dst_async)

        ex()
        run_async()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            dec(d_file, d_index, dst_graph)
        torch.cuda.synchronize()
        return ex, run_async, g, dec, outs, d_file

    def timed(fn, steps):
        fn()
        torch.cuda.synchronize()
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(max(steps, 1))]
        for a, b in evs:
            a.record(stream)
            fn()
            b.record(stream)
        torch.cuda.synchronize()
        ms = [a.elapsed_time(b) for a, b in evs]
        return {"ms": float(np.mean(ms)), "ms_min": float(np.min(ms)), "ms_max": float(np.max(ms))}

    def profiled(fn):
        L.pco_b200_profile_enable(1)
        fn()
        torch.cuda.synchronize()
        prof = parse_profile(L)
        L.pco_b200_profile_enable(0)
        return prof

    res, parity = {}, {}
    # ---- big file
    n_chunks = args.chunks
    n = n_chunks * CHUNK_N
    h_np = np.empty(n, dtype=np.uint64)
    for c in range(n_chunks):
        h_np[c * CHUNK_N:(c + 1) * CHUNK_N] = datagen.c2_u64_cumsum_geometric(CHUNK_N, seed=c)
    nums = torch.from_numpy(h_np.view(np.int64)).to(dev)
    ex, run_async, g, dec, outs, d_file = setup(nums, n_chunks)
    big = {"compressed_bytes": int(d_file.numel()), "workspace_bytes": dec.workspace_bytes}
    big["ex"] = timed(ex, args.steps)
    big["async"] = timed(run_async, args.steps)
    big["graph"] = timed(g.replay, args.steps)
    torch.cuda.synchronize()
    enq = []
    for _ in range(max(args.steps, 1)):
        t0 = time.perf_counter()
        run_async()
        enq.append((time.perf_counter() - t0) * 1e6)
        torch.cuda.synchronize()
    big["enqueue_us"] = {"mean": float(np.mean(enq)), "min": float(np.min(enq))}
    big["kernel_ms"] = {"ex": profiled(ex), "async": profiled(run_async)}
    big["async_over_ex_kernels"] = sum(big["kernel_ms"]["async"].values()) / max(sum(big["kernel_ms"]["ex"].values()), 1e-9)
    prog = dec.result()
    parity["big.ex"] = bool(torch.equal(outs["ex"], nums))
    parity["big.async"] = bool(torch.equal(outs["async"], nums) and (prog.n_processed, prog.finished) == (n, True))
    g.replay()
    prog = dec.result()
    parity["big.graph"] = bool(torch.equal(outs["graph"], nums) and (prog.n_processed, prog.finished) == (n, True))
    res["big"] = big
    del ex, run_async, g, dec, outs, d_file, nums

    # ---- small file: the fixed cost per call
    m = 1 << 16
    small_np = datagen.c2_u64_cumsum_geometric(m, seed=7)
    snums = torch.from_numpy(small_np.view(np.int64)).to(dev)
    ex, run_async, g, dec, outs, _ = setup(snums, 1)
    K = max(args.small_steps, 1)
    small = {}
    for name, fn in (("ex_loop", ex), ("async_back_to_back", run_async), ("graph_replays", g.replay)):
        fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(K):
            fn()
        torch.cuda.synchronize()
        small[name + "_us_per_call"] = (time.perf_counter() - t0) / K * 1e6
    small["kernel_ms"] = {"ex": profiled(ex), "async": profiled(run_async)}
    prog = dec.result()
    parity["small.ex"] = bool(torch.equal(outs["ex"], snums))
    parity["small.async"] = bool(torch.equal(outs["async"], snums) and (prog.n_processed, prog.finished) == (m, True))
    g.replay()
    prog = dec.result()
    parity["small.graph"] = bool(torch.equal(outs["graph"], snums) and (prog.n_processed, prog.finished) == (m, True))
    res["small"] = small
    res["parity"] = {"all": all(parity.values()), **parity}
    print(json.dumps({"workload": f"big: C2 {n_chunks} chunks x 2^18 u64, classic, order 1; small: 2^16 u64 in one chunk; side index from compress_ex, "
                      "device buffers", "unit": "ms per call unless named", "steps": args.steps, "small_steps": K, "gpu": gpu_description(), **res}))


if __name__ == "__main__":
    main()
