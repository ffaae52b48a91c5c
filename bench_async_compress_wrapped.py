#!/usr/bin/env python
"""bench_async_compress_wrapped.py — the asynchronous batch compress into wrapped chunks (pco_b200_compress_wrapped_async) against a loop of
the blocking pco_b200_compress_wrapped, one call per array, on the same arrays.

The array of bench.py (chunks of 2^18 u64, C2 data, chunk c = datagen.c2_u64_cumsum_geometric(seed = c)), classic mode, consecutive delta
order 1, level 8, every buffer in HBM, cut into arrays four ways:
  - "one": one array of all the numbers;
  - "uniform": 64 arrays of 2^22 numbers;
  - "lognormal": seeded lognormal sizes (median 2^16, sigma 1.5) clipped to [1, 2^20] (bench_files.py's);
  - "mixed": seeded lognormal sizes of median 2^10 and sigma 2.5 clipped to [1, 2^20] (bench_async_compress_files.py's): the chunks span
    every unoptimized_bins_log of level 8, all in one pass.
Legs per cut: the blocking loop (CUDA events around the first --loop-arrays calls, scaled to all arrays, as bench_pages.py scales its
per-page loop); the asynchronous call (CUDA events, call to call); the same call replayed from a captured CUDA graph; the host time to
enqueue one call (mean and minimum); the per-kernel split of one call from the library's profiler (every gated launch included); and a
graph that compresses a device-chosen subset of the arrays (every third) and decodes it with AsyncPagesDecompressor straight from the
device refs.  `parity` compares the metas, pages, refs and first_chunk of the call and of the graph replay with the whole blocking loop's,
and the decoded subset with its input.  Prints one JSON line with the card's name and power limit; writes nothing.

    python bench_async_compress_wrapped.py [--steps 10] [--chunks 1024] [--loop-arrays 64]
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

from bench_async_compress_files import file_sizes  # noqa: E402
from bench_levels import CHUNK_N, gpu_description, parse_profile  # noqa: E402


def array_sizes(kind, n):
    if kind == "one":
        return np.array([n], dtype=np.uint64)
    if kind == "uniform":
        return np.full(64, n // 64, dtype=np.uint64)
    return file_sizes(kind, n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--chunks", type=int, default=1024)
    ap.add_argument("--loop-arrays", type=int, default=64)
    args = ap.parse_args()

    import torch

    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, _lib, datagen, wrapped

    L = wrapped._lib_batch()
    if not L.pco_b200_device_available():
        raise RuntimeError("libcpcodec.so found no usable CUDA device: " + L.pco_b200_last_error_message().decode())
    wrapped._lib_async_compress_wrapped()
    wrapped._lib_async_pages()
    dev = torch.device("cuda", 0)
    n = args.chunks * CHUNK_N
    h_np = np.empty(n, dtype=np.uint64)
    for c in range(args.chunks):
        h_np[c * CHUNK_N:(c + 1) * CHUNK_N] = datagen.c2_u64_cumsum_geometric(CHUNK_N, seed=c)
    nums = torch.from_numpy(h_np.view(np.int64)).to(dev)
    del h_np
    cfg_py = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(1))
    cfg = cfg_py._to_c()
    SRC, DST = 1, 2

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
    for kind in ("one", "uniform", "lognormal", "mixed"):
        ns = array_sizes(kind, n)
        na = len(ns)
        total = int(ns.sum())
        U = total * 8
        starts = np.concatenate([[0], np.cumsum(ns)]).astype(np.int64)
        comp = wrapped.AsyncChunksCompressor(np.int64, cfg_py, na, total, int(ns.max()))
        stream = torch.cuda.current_stream()
        sp = C.c_void_p(stream.cuda_stream)
        r = {"arrays": na, "array_n_min": int(ns.min()), "array_n_median": int(np.median(ns)), "array_n_max": int(ns.max()),
             "max_chunks": comp.max_chunks, "workspace_mb": comp.workspace_bytes / 1e6}
        # the blocking loop: one compress_wrapped per array, each behind the arrays before it in the same buffers
        s_metas = torch.empty(comp.metas_cap, dtype=torch.uint8, device=dev)
        s_pages = torch.empty(comp.pages_cap, dtype=torch.uint8, device=dev)
        s_refs = np.zeros(comp.max_chunks, dtype=wrapped.PAGE_REF)
        s_first = np.zeros(na + 1, dtype=np.int64)
        ml, pl, nc = C.c_size_t(), C.c_size_t(), C.c_size_t()

        def loop(k):
            mo = po = ro = 0
            for i in range(k):
                refs_at = s_refs[ro:]
                _lib.check(L.pco_b200_compress_wrapped(C.c_void_p(nums.data_ptr() + int(starts[i]) * 8), C.c_size_t(int(ns[i])), C.c_ubyte(4), C.byref(cfg),
                                                       C.c_void_p(s_metas.data_ptr() + mo), C.c_size_t(comp.metas_cap - mo), C.byref(ml),
                                                       C.c_void_p(s_pages.data_ptr() + po), C.c_size_t(comp.pages_cap - po), C.byref(pl),
                                                       refs_at.ctypes.data_as(C.c_void_p), C.c_size_t(len(refs_at)), C.byref(nc), C.c_uint32(SRC | DST), sp))
                refs_at["meta_offset"][:nc.value] += mo
                refs_at["page_offset"][:nc.value] += po
                mo, po, ro = mo + ml.value, po + pl.value, ro + nc.value
                s_first[i + 1] = ro
            return mo, po, ro

        k = min(args.loop_arrays, na)
        loop(min(2, na))  # warm up
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        loop(k)
        b.record()
        torch.cuda.synchronize()
        loop_ms = a.elapsed_time(b) * na / k
        r["sync_loop"] = {"arrays_timed": k, "ms": loop_ms}
        used_m, used_p, used_c = loop(na)  # the whole loop, untimed: the parity reference
        torch.cuda.synchronize()
        want_refs = torch.from_numpy(np.stack([s_refs[f][:used_c] for f in ("meta_offset", "meta_len", "page_offset", "page_len", "page_n")],
                                              axis=1).astype(np.int64)).to(dev)
        want_first = torch.from_numpy(s_first).to(dev)
        d_ns = torch.from_numpy(ns.astype(np.int64)).to(dev)
        d_na = torch.tensor([na], dtype=torch.int64, device=dev)
        metas = torch.empty(comp.metas_cap, dtype=torch.uint8, device=dev)
        pages = torch.empty(comp.pages_cap, dtype=torch.uint8, device=dev)
        refs = torch.empty((comp.max_chunks, 5), dtype=torch.int64, device=dev)
        first = torch.empty(na + 1, dtype=torch.int64, device=dev)

        def call():
            comp(nums, d_ns, d_na, metas, pages, refs, first)

        def same():
            got = comp.result()
            return bool(got == (used_m, used_p, used_c) and torch.equal(metas[:used_m], s_metas[:used_m]) and torch.equal(pages[:used_p], s_pages[:used_p])
                        and torch.equal(refs[:used_c], want_refs) and torch.equal(first, want_first))

        r["async"] = events(call, args.steps)
        p_async = same()
        # host enqueue time of one call
        torch.cuda.synchronize()
        host = []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            call()
            host.append((time.perf_counter() - t0) * 1e3)
        torch.cuda.synchronize()
        r["enqueue_ms"] = {"mean": float(np.mean(host)), "min": float(np.min(host))}
        # per-kernel split
        L.pco_b200_profile_enable(1)
        call()
        torch.cuda.synchronize()
        r["kernel_ms"] = parse_profile(L)
        L.pco_b200_profile_enable(0)
        # graph replay, into cleared outputs
        metas.fill_(0)
        pages.fill_(0)
        refs.fill_(-1)
        first.fill_(-1)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                call()
        torch.cuda.current_stream().wait_stream(s)
        r["graph"] = events(g.replay, args.steps)
        p_graph = same()
        # a device-chosen subset (every third array), compressed and decoded from the device refs in one graph
        pick = torch.arange(0, na, 3, device=dev)
        sub_ns = torch.zeros(na, dtype=torch.int64, device=dev)
        sub_na = torch.zeros(1, dtype=torch.int64, device=dev)
        d_starts = torch.cumsum(d_ns, 0) - d_ns
        sub_total = int(d_ns[pick].sum())
        sub_nums = torch.empty(total, dtype=torch.int64, device=dev)
        dec = wrapped.AsyncPagesDecompressor(np.int64, comp.metas_cap, comp.pages_cap, comp.max_chunks, total)
        out = torch.empty(total, dtype=torch.int64, device=dev)
        n_pages = torch.zeros(1, dtype=torch.int64, device=dev)
        idx_of = torch.repeat_interleave(pick, d_ns[pick])
        offs = torch.arange(sub_total, device=dev) - torch.repeat_interleave(torch.cumsum(d_ns[pick], 0) - d_ns[pick], d_ns[pick])
        gather = d_starts[idx_of] + offs
        del idx_of, offs

        def subset():
            sub_na.fill_(pick.numel())
            sub_ns[:pick.numel()].copy_(d_ns[pick])
            sub_nums[:sub_total].copy_(nums[gather])
            comp(sub_nums, sub_ns, sub_na, metas, pages, refs, first)
            n_pages.copy_(first.index_select(0, sub_na))
            dec(metas, pages, refs, n_pages, out)

        subset()
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            g2 = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g2, stream=s):
                subset()
        torch.cuda.current_stream().wait_stream(s)
        r["subset_graph"] = events(g2.replay, args.steps)
        r["subset_graph"]["arrays"] = int(pick.numel())
        p_subset = bool(dec.result() == sub_total and torch.equal(out[:sub_total], nums[gather]))
        comp.result()
        r["sync_loop"]["gb_s"] = U / 1e9 / (r["sync_loop"]["ms"] / 1e3)
        for leg in ("async", "graph"):
            r[leg]["gb_s"] = U / 1e9 / (r[leg]["ms"] / 1e3)
        r["ratio"] = U / (used_m + used_p)
        r["speedup_async_vs_loop"] = r["sync_loop"]["ms"] / r["async"]["ms"]
        r["speedup_graph_vs_loop"] = r["sync_loop"]["ms"] / r["graph"]["ms"]
        r["parity"] = {"async_equals_loop": p_async, "graph_equals_loop": p_graph, "subset_decoded_equals_input": p_subset}
        results[kind] = r
        del comp, dec, g, g2, metas, pages, refs, first, s_metas, s_pages, sub_nums, out, gather
        torch.cuda.empty_cache()
    print(json.dumps({"workload": f"C2: {args.chunks} x 2^18 u64 cut into arrays, classic mode, consecutive delta order 1, level 8, device buffers",
                      "unit": "ms per batch; GB/s of uncompressed bytes", "steps": args.steps, "gpu": gpu_description(), **results}))


if __name__ == "__main__":
    main()
