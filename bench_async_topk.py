#!/usr/bin/env python
"""bench_async_topk.py — the k smallest or largest numbers selected in the decoder (pco_b200_topk_pages_async / _files_async,
wrapped.AsyncPagesTopK, standalone.AsyncFilesTopK), against decoding everything and selecting afterwards (AsyncPagesDecompressor /
AsyncFilesDecompressor, then torch.topk, captured in one graph), and against the aggregate call (AsyncPagesAggregate /
AsyncFilesAggregate) over every number, the floor a one-pass scan can aim for, on the same input.

Inputs: bench.py's array (1024 chunks of 2^18 u64, C2 data, chunk c = datagen.c2_u64_cumsum_geometric(seed = c)), every buffer in HBM:
  - file_order1 / file_order0: standalone.compress_files, one indexed file of 1024 chunks, consecutive delta order 1 / no_op;
  - files_4096: 4096 files of 2^16 numbers, delta order 1;
  - pages: wrapped.compress_chunks, 1024 pages, delta order 1.
On file_order1 the array also runs in random order (a fixed permutation), sorted ascending and sorted descending: the sorted columns are
the candidate buffers' worst case in one direction each (every number beats the CTA's threshold).
Legs: k = 1, 100 and 1024, smallest and largest.  Per leg: topk_ms (one call) and topk_graph_ms (one replay of the call captured once),
baseline_graph_ms (decode, then torch.topk), CUDA events, median of --steps; enqueue_us (host time of one call); kernel_ms (per-kernel
split of one profiled call); written_mb (HBM bytes written, from the shapes: the top-k's slot lists and outputs; the baseline's decoded
column); parity (values and positions equal a stable sort of the numbers at or beyond torch.kthvalue's, which ranks ties by position as
the call does; torch.topk's values agree).  Per input: aggregate_graph_ms and decode_graph_ms.
Prints one JSON line with the card's name, power limit and max SM clock read in the same run; writes nothing.

    python bench_async_topk.py [--steps 5] [--chunks 1024]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_levels import CHUNK_N, gpu_description, parse_profile  # noqa: E402

KS = [1, 100, 1024]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--chunks", type=int, default=1024)
    args = ap.parse_args()

    import torch

    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec, _lib, datagen, standalone, wrapped

    L = _lib.lib()
    if not L.pco_b200_device_available():
        raise RuntimeError("libcpcodec.so found no usable CUDA device: " + L.pco_b200_last_error_message().decode())
    dev = torch.device("cuda", 0)
    steps = max(args.steps, 1)
    n = args.chunks * CHUNK_N
    h_np = np.empty(n, dtype=np.uint64)
    for c in range(args.chunks):
        h_np[c * CHUNK_N:(c + 1) * CHUNK_N] = datagen.c2_u64_cumsum_geometric(CHUNK_N, seed=c)
    base = torch.from_numpy(h_np.view(np.int64)).to(dev)  # the C2 values stay below 2^63: int64 compares order them as u64 does
    del h_np

    def events(fn):
        stream = torch.cuda.current_stream()
        fn()
        torch.cuda.synchronize()
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
        for a, b in evs:
            a.record(stream)
            fn()
            b.record(stream)
        torch.cuda.synchronize()
        return float(np.median([a.elapsed_time(b) for a, b in evs]))

    def capture(fn):
        fn()  # warm-up outside the capture
        torch.cuda.synchronize()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side):
            out = fn()
        torch.cuda.synchronize()
        return g, out

    def reference(x, k, largest):
        """(values, positions) of the k best of x ranked by (value, position)."""
        v = torch.kthvalue(x, n - k + 1 if largest else k).values
        cand = torch.nonzero(x >= v if largest else x <= v).flatten()  # ascending positions
        order = torch.sort(x[cand], descending=largest, stable=True).indices[:k]
        return x[cand[order]], cand[order]

    def refs_tensor(refs):
        return torch.from_numpy(np.stack([refs[f].astype(np.int64) for f in wrapped.PAGE_REF.names], axis=1)).to(dev)

    perm = torch.randperm(n, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    datas = {"bench": lambda: base, "random": lambda: base[perm], "ascending": lambda: torch.sort(base).values,
             "descending": lambda: torch.sort(base, descending=True).values}
    inputs = [("file_order1", "files", DeltaSpec.try_consecutive(1), [n], list(datas)), ("file_order0", "files", DeltaSpec.no_op(), [n], ["bench"]),
              ("files_4096", "files", DeltaSpec.try_consecutive(1), [1 << 16] * (n >> 16), ["bench"]),
              ("pages", "pages", DeltaSpec.try_consecutive(1), None, ["bench"])]
    res, parity = {}, {}
    for iname, kind, delta, sizes, dnames in inputs:
        for dname in dnames:
            nums = datas[dname]()
            cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=delta, paging_spec=PagingSpec.equal_pages_up_to(CHUNK_N))
            if kind == "pages":
                metas, pages, refs = wrapped.compress_chunks(nums.view(torch.uint64), cfg)
                torch.cuda.synchronize()
                ng = len(refs)
                args_in = (metas, pages, refs_tensor(refs), torch.tensor([ng], dtype=torch.int64, device=dev))
                mk = lambda k, lg: wrapped.AsyncPagesTopK(np.uint64, metas.numel(), pages.numel(), ng, n, k, lg)  # noqa: E731
                agg = wrapped.AsyncPagesAggregate(np.uint64, metas.numel(), pages.numel(), ng, n)
                dec = wrapped.AsyncPagesDecompressor(np.uint64, metas.numel(), pages.numel(), ng, n)
                legs = {"pages": ng}
            else:
                d_data, files, d_index = standalone.compress_files(nums.view(torch.uint64), np.array(sizes, np.uint64), cfg)
                torch.cuda.synchronize()
                frefs = np.stack([files["offset"], files["len"], files["index_offset"], files["index_len"]], axis=1).astype(np.uint64)
                ng = len(frefs)
                nc = int(sum(-(-int(s) // CHUNK_N) for s in sizes))
                args_in = (d_data, d_index, torch.as_tensor(frefs.view(np.int64), device=dev), torch.tensor([ng], dtype=torch.int64, device=dev))
                mk = lambda k, lg: standalone.AsyncFilesTopK(d_data[:32], np.uint64, d_data.numel(), d_index.numel(), ng, nc, n, k, lg)  # noqa: E731
                agg = standalone.AsyncFilesAggregate(d_data[:32], np.uint64, d_data.numel(), d_index.numel(), ng, nc, n)
                dec = standalone.AsyncFilesDecompressor(d_data[:32], np.uint64, d_data.numel(), d_index.numel(), ng, nc, n)
                legs = {"files": ng, "chunks": nc}
            d_out = torch.empty(n, dtype=torch.int64, device=dev)
            if kind == "pages":
                decode = lambda: dec(*args_in, d_out.view(torch.uint64))  # noqa: E731
            else:
                d_ns = torch.zeros(ng, dtype=torch.int64, device=dev)
                decode = lambda: dec(*args_in, d_out.view(torch.uint64), d_ns)  # noqa: E731
            g_dec, _ = capture(decode)
            legs["decode_graph_ms"] = events(g_dec.replay)
            iv = torch.tensor([0, -1], dtype=torch.int64, device=dev)  # [0, 2^64 - 1]: every number
            aggs, atot = torch.zeros((ng, 6), dtype=torch.int64, device=dev), torch.zeros(6, dtype=torch.int64, device=dev)
            g_agg, _ = capture(lambda: agg(*args_in, iv, aggs, atot))
            legs["aggregate_graph_ms"] = events(g_agg.replay)
            del g_agg
            ok_all = agg.result() == n
            for k in KS:
                for largest in (False, True):
                    top = mk(k, largest)
                    vals = torch.zeros(k, dtype=torch.int64, device=dev)
                    pos = torch.zeros(k, dtype=torch.int64, device=dev)
                    n_out = torch.zeros(1, dtype=torch.int64, device=dev)
                    call = lambda: top(*args_in, iv, vals.view(torch.uint64), pos, n_out)  # noqa: E731
                    wv, wp = reference(nums, k, largest)
                    t = {"workspace_bytes": top.workspace_bytes}
                    t["topk_ms"] = events(call)
                    ok_c = top.result() == n and int(n_out) == k and torch.equal(vals, wv) and torch.equal(pos, wp)
                    pos.fill_(-7)
                    g_top, _ = capture(call)
                    t["topk_graph_ms"] = events(g_top.replay)
                    ok_g = top.result() == n and torch.equal(vals, wv) and torch.equal(pos, wp)
                    enq = []
                    for _ in range(steps):
                        t0 = time.perf_counter()
                        call()
                        enq.append(time.perf_counter() - t0)
                        torch.cuda.synchronize()
                    t["enqueue_us"] = float(np.median(enq) * 1e6)
                    L.pco_b200_profile_enable(1)
                    call()
                    torch.cuda.synchronize()
                    t["kernel_ms"] = {kk: round(v, 4) for kk, v in parse_profile(L).items()}
                    L.pco_b200_profile_enable(0)
                    g_base, base_out = capture(lambda: (decode(), torch.topk(d_out, k, largest=largest, sorted=True))[1])
                    t["baseline_graph_ms"] = events(g_base.replay)
                    ok_b = torch.equal(base_out.values, wv)
                    slots = ng if kind == "pages" else nc
                    t["written_mb"] = {"topk": round((16 * k * slots + 16 * k) / 1e6, 3), "baseline": round((8 * n + 16 * k) / 1e6, 3)}
                    t["parity"] = bool(ok_c and ok_g and ok_b)
                    ok_all = ok_all and t["parity"]
                    legs[f"k{k}_{'largest' if largest else 'smallest'}"] = t
                    del g_top, g_base, top
            key = iname if dname == "bench" else f"{iname}_{dname}"
            parity[key] = bool(ok_all)
            res[key] = legs
            del g_dec, agg, dec, d_out
            torch.cuda.empty_cache()
    print(json.dumps({"workload": f"C2: {args.chunks} chunks x 2^18 u64 as one indexed file (order 1 and 0; on order 1 also random, ascending "
                                  f"and descending), {n >> 16} files of 2^16 and 1024 wrapped pages, u64 top-k with k = 1 / 100 / 1024 in both "
                                  "directions, device buffers",
                      "gpu": gpu_description(), "steps": steps, "results": res, "parity": parity}))


if __name__ == "__main__":
    main()
