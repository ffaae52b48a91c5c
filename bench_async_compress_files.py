#!/usr/bin/env python
"""bench_async_compress_files.py — the asynchronous batch compress (pco_b200_compress_files_async) against the blocking
pco_b200_compress_files on the same files.

The array of bench.py (chunks of 2^18 u64, C2 data, chunk c = datagen.c2_u64_cumsum_geometric(seed = c)), classic mode, consecutive delta
order 1, level 8, every buffer in HBM, cut into files three ways:
  - "uniform": 4096 files of 2^16 numbers (bench_files.py's);
  - "lognormal": seeded lognormal sizes (median 2^16, sigma 1.5) clipped to [1, 2^20] (bench_files.py's);
  - "mixed": seeded lognormal sizes of median 2^10 and sigma 2.5 clipped to [1, 2^20]: the files span every unoptimized_bins_log of level 8,
    so the blocking call makes one pipeline pass per value and the asynchronous one a single pass.
Legs per cut: the blocking call; the asynchronous call (CUDA events, call to call); the same call replayed from a captured CUDA graph; the
host time to enqueue one call; the per-kernel split of one call from the library's profiler (every gated launch included); and a graph that
compresses a device-chosen subset of the files and decodes it with AsyncFilesDecompressor.  `parity` compares dst, the side indexes and
the refs of every leg with the blocking call's, and the decoded subset with its input.  Prints one JSON line; writes nothing.

    python bench_async_compress_files.py [--steps 10] [--chunks 1024]
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


def file_sizes(kind, n, seed=1):
    if kind == "uniform":
        return np.full(min(n >> 16, 4096), 1 << 16, dtype=np.uint64)
    median, sigma = (1 << 16, 1.5) if kind == "lognormal" else (1 << 10, 2.5)
    rng = np.random.default_rng(seed)
    out, left = [], n
    while left > 0:
        s = int(np.clip(rng.lognormal(np.log(median), sigma), 1, 1 << 20))
        out.append(min(s, left))
        left -= out[-1]
    return np.array(out, dtype=np.uint64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--chunks", type=int, default=1024)
    args = ap.parse_args()

    import torch

    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, _lib, datagen, standalone

    L = standalone._lib_files()
    if not L.pco_b200_device_available():
        raise RuntimeError("libcpcodec.so found no usable CUDA device: " + L.pco_b200_last_error_message().decode())
    standalone._lib_async_compress_files()
    dev = torch.device("cuda", 0)
    n = args.chunks * CHUNK_N
    h_np = np.empty(n, dtype=np.uint64)
    for c in range(args.chunks):
        h_np[c * CHUNK_N:(c + 1) * CHUNK_N] = datagen.c2_u64_cumsum_geometric(CHUNK_N, seed=c)
    nums = torch.from_numpy(h_np.view(np.int64)).to(dev)
    cfg_py = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(1))
    cfg = cfg_py._to_c()
    SRC, DST, IDX = 1, 2, 4

    def events(fn, steps):
        fn()
        torch.cuda.synchronize()
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
        for a, b in evs:
            a.record()
            fn()
            b.record()
        torch.cuda.synchronize()
        ms = [a.elapsed_time(b) for a, b in evs]
        return {"ms": float(np.mean(ms)), "ms_min": float(np.min(ms)), "ms_max": float(np.max(ms))}

    results = {}
    for kind in ("uniform", "lognormal", "mixed"):
        ns = file_sizes(kind, n)
        nf = len(ns)
        total = int(ns.sum())
        U = total * 8
        max_file_n = int(ns.max())
        comp = standalone.AsyncFilesCompressor(np.int64, cfg_py, nf, total, max_file_n)
        stream = torch.cuda.current_stream()
        sp = C.c_void_p(stream.cuda_stream)
        # the blocking call, with the capacities of the asynchronous one
        s_data = torch.empty(comp.dst_cap, dtype=torch.uint8, device=dev)
        s_index = torch.empty(comp.index_cap, dtype=torch.uint8, device=dev)
        s_files = np.zeros(nf, dtype=standalone.FILE_REF)

        def sync():
            _lib.check(L.pco_b200_compress_files(C.c_void_p(nums.data_ptr()), ns.ctypes.data_as(C.c_void_p), C.c_size_t(nf), C.c_ubyte(4), C.byref(cfg),
                                                 C.c_int(0), C.c_void_p(s_data.data_ptr()), C.c_size_t(comp.dst_cap), C.c_void_p(s_index.data_ptr()),
                                                 C.c_size_t(comp.index_cap), s_files.ctypes.data_as(C.c_void_p), C.c_uint32(SRC | DST | IDX), sp))

        r = {"files": nf, "file_n_min": int(ns.min()), "file_n_median": int(np.median(ns)), "file_n_max": max_file_n,
             "max_chunks": int(comp._plan.max_chunks), "workspace_mb": comp.workspace_bytes / 1e6}
        r["sync"] = events(sync, args.steps)
        used = int(s_files[-1]["offset"] + s_files[-1]["len"])
        iused = int(s_files[-1]["index_offset"] + s_files[-1]["index_len"])
        want_refs = torch.from_numpy(np.stack([s_files["offset"], s_files["len"], s_files["index_offset"], s_files["index_len"]], axis=1).astype(np.int64)).to(dev)
        d_ns = torch.from_numpy(ns.astype(np.int64)).to(dev)
        d_nf = torch.tensor([nf], dtype=torch.int64, device=dev)
        dst = torch.empty(comp.dst_cap, dtype=torch.uint8, device=dev)
        index = torch.empty(comp.index_cap, dtype=torch.uint8, device=dev)
        files = torch.empty((nf, 4), dtype=torch.int64, device=dev)

        def call():
            comp(nums, d_ns, d_nf, dst, index, files)

        def same():
            dl, il = comp.result()
            return bool(dl == used and il == iused and torch.equal(dst[:used], s_data[:used]) and torch.equal(index[:iused], s_index[:iused])
                        and torch.equal(files, want_refs))

        r["async"] = events(call, args.steps)
        p_async = same()
        # host enqueue time of one call
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.steps):
            call()
        t1 = time.perf_counter()
        torch.cuda.synchronize()
        r["enqueue_ms"] = (t1 - t0) * 1e3 / args.steps
        # per-kernel split
        L.pco_b200_profile_enable(1)
        call()
        torch.cuda.synchronize()
        r["kernel_ms"] = parse_profile(L)
        L.pco_b200_profile_enable(0)
        # graph replay, into cleared outputs
        dst.fill_(0)
        index.fill_(0)
        files.fill_(-1)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                call()
        torch.cuda.current_stream().wait_stream(s)
        r["graph"] = events(g.replay, args.steps)
        p_graph = same()
        # a device-chosen subset (every third file), compressed and decoded in one graph
        pick = torch.arange(0, nf, 3, device=dev)
        sub_ns = torch.zeros(nf, dtype=torch.int64, device=dev)
        sub_nf = torch.zeros(1, dtype=torch.int64, device=dev)
        starts = torch.cumsum(d_ns, 0) - d_ns
        sub_total = int(d_ns[pick].sum())
        sub_nums = torch.empty(total, dtype=torch.int64, device=dev)
        head = s_data[:32]
        dec = standalone.AsyncFilesDecompressor(head, np.int64, comp.dst_cap, comp.index_cap, nf, int(comp._plan.max_chunks), total)
        out = torch.empty(total, dtype=torch.int64, device=dev)
        out_ns = torch.empty(nf, dtype=torch.int64, device=dev)
        idx_of = torch.repeat_interleave(pick, d_ns[pick])
        offs = torch.arange(sub_total, device=dev) - torch.repeat_interleave(torch.cumsum(d_ns[pick], 0) - d_ns[pick], d_ns[pick])
        gather = starts[idx_of] + offs

        def subset():
            sub_nf.fill_(pick.numel())
            sub_ns[:pick.numel()].copy_(d_ns[pick])
            sub_nums[:sub_total].copy_(nums[gather])
            comp(sub_nums, sub_ns, sub_nf, dst, index, files)
            dec(dst, index, files, sub_nf, out, out_ns)

        subset()
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            g2 = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g2, stream=s):
                subset()
        torch.cuda.current_stream().wait_stream(s)
        r["subset_graph"] = events(g2.replay, args.steps)
        r["subset_graph"]["files"] = int(pick.numel())
        p_subset = bool(dec.result() == sub_total and torch.equal(out[:sub_total], nums[gather]))
        for leg in ("sync", "async", "graph"):
            r[leg]["gb_s"] = U / 1e9 / (r[leg]["ms"] / 1e3)
        r["ratio"] = U / used
        r["speedup_graph_vs_sync"] = r["sync"]["ms"] / r["graph"]["ms"]
        r["parity"] = {"async_equals_sync": p_async, "graph_equals_sync": p_graph, "subset_decoded_equals_input": p_subset}
        results[kind] = r
        del comp, dec
        torch.cuda.empty_cache()
    print(json.dumps({"workload": f"C2: {args.chunks} x 2^18 u64 cut into files, classic mode, consecutive delta order 1, level 8, device buffers",
                      "unit": "ms per batch; GB/s of uncompressed bytes", "steps": args.steps, "gpu": gpu_description(), **results}))


if __name__ == "__main__":
    main()
