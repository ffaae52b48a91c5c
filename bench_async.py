#!/usr/bin/env python
"""bench_async.py — the asynchronous decompress (pco_b200_decompress_async) against pco_b200_decompress_ex on the same file and index,
and the asynchronous compress (pco_b200_compress_async) against pco_b200_compress_ex on the same arrays.

Big file: bench.py's array and file - 1024 chunks of 2^18 u64 (C2 data, chunk c = datagen.c2_u64_cumsum_geometric(seed = c)), classic
mode, consecutive delta order 1, written by pco_b200_compress_ex with its side index, every buffer in HBM.  Legs, each timed with CUDA
events around `--steps` calls after one warm-up:
  - ex: pco_b200_decompress_ex (blocks until done; the events bracket its kernels and the host gaps between them);
  - async: pco_b200_decompress_async (enqueues only), and the host time one such call takes to return (`enqueue_us`);
  - graph: one async call captured in a torch.cuda.CUDAGraph, replayed.
A separate profiled call of ex and of async gives the per-kernel split.
Small file: 2^16 u64 numbers (one chunk, order 1) with its index in HBM: host wall time per call of a loop of `--small-steps`
decompress_ex calls, of as many back-to-back async calls with one synchronisation at the end, and of as many graph replays.
Compress legs (compress_big, compress_small): the same three legs on the same two arrays, for compress_ex and AsyncCompressor (same
config, dst_cap = the size guarantee, side index on).  round_trip: a compress then an AsyncDecompressor call on the file it wrote, eager and
captured in one graph, wall time per call on the small array.
`parity`: every decompress leg's output equals the input; every async compress leg's file and index equal compress_ex's, which decode
to the input.  The card's name, power limit and max SM clock are read in the same run.
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
    del ex, run_async, g, dec, outs
    res["compress_big"], res["compress_small"], res["round_trip"] = compress_legs(args, L, cfg, h_np, snums, parity, timed, profiled)
    res["parity"] = {"all": all(parity.values()), **parity}
    print(json.dumps({"workload": f"big: C2 {n_chunks} chunks x 2^18 u64, classic, order 1; small: 2^16 u64 in one chunk; side index from compress_ex, "
                      "device buffers", "unit": "ms per call unless named", "steps": args.steps, "small_steps": K, "gpu": gpu_description(), **res}))


def compress_legs(args, L, cfg, h_np, snums, parity, timed, profiled):
    """pco_b200_compress_ex against pco_b200_compress_async (AsyncCompressor) and a graph replay of it, on the big array and on the
    2^16-number one, and a compress + AsyncDecompressor round trip captured in one graph.  Parity: the async bytes equal compress_ex's
    and decode to the input."""
    import torch

    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, _lib, standalone

    dev = torch.device("cuda", 0)
    SRC, DST, IDX = 1, 2, 4
    pcfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(1))

    def legs(nums, n_chunks, name):
        n = nums.numel()
        comp = standalone.AsyncCompressor(n, np.uint64, pcfg)
        cap, icap = comp.dst_cap, comp.index_bytes
        bufs = {k: (torch.zeros(cap, dtype=torch.uint8, device=dev), torch.zeros(icap, dtype=torch.uint8, device=dev)) for k in ("ex", "async", "graph")}
        unums = nums.view(torch.uint64)
        written, ilen = C.c_size_t(), C.c_size_t()

        def ex():
            d, i = bufs["ex"]
            _lib.check(L.pco_b200_compress_ex(C.c_void_p(nums.data_ptr()), C.c_size_t(n), C.c_ubyte(2), C.byref(cfg), C.c_int(0), C.c_void_p(d.data_ptr()),
                                              C.c_size_t(cap), C.byref(written), C.c_void_p(i.data_ptr()), C.c_size_t(icap), C.byref(ilen),
                                              C.c_uint32(SRC | DST | IDX), C.c_void_p(torch.cuda.current_stream().cuda_stream)))

        def run_async():
            comp(unums, *bufs["async"])

        ex()
        run_async()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            comp(unums, *bufs["graph"])
        torch.cuda.synchronize()
        out = {"workspace_bytes": comp.workspace_bytes}
        if name == "big":
            out["ex"] = timed(ex, args.steps)
            out["async"] = timed(run_async, args.steps)
            out["graph"] = timed(g.replay, args.steps)
            enq = []
            for _ in range(max(args.steps, 1)):
                t0 = time.perf_counter()
                run_async()
                enq.append((time.perf_counter() - t0) * 1e6)
                torch.cuda.synchronize()
            out["enqueue_us"] = {"mean": float(np.mean(enq)), "min": float(np.min(enq))}
            out["kernel_ms"] = {"ex": profiled(ex), "async": profiled(run_async)}
            out["async_over_ex_kernels"] = sum(out["kernel_ms"]["async"].values()) / max(sum(out["kernel_ms"]["ex"].values()), 1e-9)
        else:
            K = max(args.small_steps, 1)
            for leg, fn in (("ex_loop", ex), ("async_back_to_back", run_async), ("graph_replays", g.replay)):
                fn()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(K):
                    fn()
                torch.cuda.synchronize()
                out[leg + "_us_per_call"] = (time.perf_counter() - t0) / K * 1e6
            out["kernel_ms"] = {"ex": profiled(ex), "async": profiled(run_async)}
        ex()
        torch.cuda.synchronize()
        ref = bufs["ex"][0][: written.value].cpu().numpy().tobytes()
        ref_index = bufs["ex"][1][: ilen.value].cpu().numpy().tobytes()
        for leg in ("async", "graph"):
            if leg == "graph":
                g.replay()
            else:
                run_async()
            fb, ib = comp.result()
            d, i = bufs[leg]
            same = d[:fb].cpu().numpy().tobytes() == ref and i[:ib].cpu().numpy().tobytes() == ref_index
            back = standalone.simple_decompress(ref, np.uint64) if leg == "async" else None
            parity[f"compress_{name}.{leg}"] = bool(same and (back is None or np.array_equal(back, unums.cpu().numpy())))
        out["compressed_bytes"] = len(ref)
        return out, comp, bufs

    big_nums = torch.from_numpy(h_np.view(np.int64)).to(dev)
    big, _, _ = legs(big_nums, args.chunks, "big")
    del big_nums
    small, comp, bufs = legs(snums, 1, "small")
    # round trip: compress, then AsyncDecompressor on the file it wrote, captured in one graph
    m = snums.numel()
    d, i = bufs["async"]
    ref_head = d[:32].cpu().numpy()
    dec = standalone.AsyncDecompressor(ref_head, np.uint64, comp.dst_cap, comp.index_bytes, m, 1)
    back = torch.zeros(m, dtype=torch.int64, device=dev)
    unums = snums.view(torch.uint64)

    def trip():
        comp(unums, d, i)
        dec(d, i, back.view(torch.uint64))

    trip()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        trip()
    K = max(args.small_steps, 1)
    rt = {}
    for leg, fn in (("eager_us_per_call", trip), ("graph_us_per_call", g.replay)):
        fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(K):
            fn()
        torch.cuda.synchronize()
        rt[leg] = (time.perf_counter() - t0) / K * 1e6
    back.zero_()
    g.replay()
    prog = dec.result()
    parity["round_trip.graph"] = bool(torch.equal(back, snums) and (prog.n_processed, prog.finished) == (m, True))
    return big, small, rt


if __name__ == "__main__":
    main()
