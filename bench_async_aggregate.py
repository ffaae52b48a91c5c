#!/usr/bin/env python
"""bench_async_aggregate.py — count, min, max and sum of the numbers inside an interval, reduced in the decoder per page / file
(pco_b200_aggregate_pages_async / _files_async, wrapped.AsyncPagesAggregate, standalone.AsyncFilesAggregate), against decoding everything
and reducing afterwards (AsyncPagesDecompressor / AsyncFilesDecompressor, then a torch mask, where and per-group index_add / scatter_reduce,
captured in one graph).

Inputs: bench.py's array (1024 chunks of 2^18 u64, C2 data, chunk c = datagen.c2_u64_cumsum_geometric(seed = c)), every buffer in HBM:
  - pages_order1 / pages_order0: wrapped.compress_chunks, 1024 pages, consecutive delta order 1 (fused_narrow_kernel) / no_op (the general
    pair);
  - file_order1 / file_order0: standalone.compress_files, one indexed file of 1024 chunks (one group of 2^20 batches);
  - files_4096: bench_files.py's uniform cut, 4096 files of 2^16 numbers, delta order 1.
Selectivities 0, 1 %, 50 % and 100 %: the interval spans that share of the sorted numbers around their median (0: lo > hi).
Per leg: agg_ms (one call) and agg_graph_ms (one replay of the call captured once), baseline_graph_ms (one replay of the baseline graph),
decode_graph_ms (the decompressor alone, captured), CUDA events, median of --steps; enqueue_us (host time of one call); kernel_ms (per-kernel
split of one profiled call); written_mb (HBM bytes written, computed from the counts: the aggregate's slot counts, slot records of batches
with a match, group accumulators and records; the baseline's decoded numbers, mask and its per-group outputs); parity (every group's count,
min, max and sum, and the total, from both paths equal a torch reduction over the input; the C2 values stay below 2^63 and their sums
below 2^63, so int64 torch ops are exact on them).
Prints one JSON line; writes nothing.

    python bench_async_aggregate.py [--steps 10] [--chunks 1024]
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

SELECTIVITIES = [0.0, 0.01, 0.5, 1.0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
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
    nums = torch.from_numpy(h_np.view(np.int64)).to(dev)
    srt = torch.sort(nums)[0]
    BIG = torch.iinfo(torch.int64).max

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
            fn()
        torch.cuda.synchronize()
        return g

    def reduce_groups(x, gid, n_groups, lo_t, hi_t, out):
        """The baseline's reduction (also the reference, over the input): per group count, min, max and sum of the matches."""
        m = (x >= lo_t) & (x <= hi_t)
        out["cnt"] = torch.zeros(n_groups, dtype=torch.int64, device=dev).index_add_(0, gid, m.long())
        out["sum"] = torch.zeros(n_groups, dtype=torch.int64, device=dev).index_add_(0, gid, torch.where(m, x, 0))
        out["min"] = torch.full((n_groups,), BIG, dtype=torch.int64, device=dev).scatter_reduce_(0, gid, torch.where(m, x, BIG), "amin")
        out["max"] = torch.full((n_groups,), -1, dtype=torch.int64, device=dev).scatter_reduce_(0, gid, torch.where(m, x, -1), "amax")
        return out

    def same(recs, tot, want):
        """The aggregate's records (n_groups x 6) and total against the reduction `want`."""
        cnt = want["cnt"]
        has = cnt > 0
        ok = torch.equal(recs[:, 1], cnt) and torch.equal(recs[:, 4], want["sum"]) and bool((recs[:, 5] == 0).all())
        ok = ok and torch.equal(recs[:, 2][has], want["min"][has]) and torch.equal(recs[:, 3][has], want["max"][has])
        ok = ok and bool((recs[:, 2][~has] == 0).all()) and bool((recs[:, 3][~has] == 0).all())
        k = int(cnt.sum())
        ok = ok and int(tot[1]) == k and int(tot[4]) == int(want["sum"].sum()) and int(tot[5]) == 0
        if k:
            ok = ok and int(tot[2]) == int(want["min"][has].min()) and int(tot[3]) == int(want["max"][has].max())
        return bool(ok)

    def refs_tensor(refs):
        return torch.from_numpy(np.stack([refs[f].astype(np.int64) for f in wrapped.PAGE_REF.names], axis=1)).to(dev)

    inputs = {}
    for name, delta in (("pages_order1", DeltaSpec.try_consecutive(1)), ("pages_order0", DeltaSpec.no_op())):
        inputs[name] = ("pages", delta, None)
    for name, delta, sizes in (("file_order1", DeltaSpec.try_consecutive(1), [n]), ("file_order0", DeltaSpec.no_op(), [n]),
                               ("files_4096", DeltaSpec.try_consecutive(1), [1 << 16] * (n >> 16))):
        inputs[name] = ("files", delta, sizes)

    res, parity = {}, {}
    for iname, (kind, delta, sizes) in inputs.items():
        cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=delta, paging_spec=PagingSpec.equal_pages_up_to(CHUNK_N))
        if kind == "pages":
            metas, pages, refs = wrapped.compress_chunks(nums.view(torch.uint64), cfg)
            torch.cuda.synchronize()
            ng = len(refs)
            group_ns = refs["page_n"].astype(np.int64)
            d_refs, d_n = refs_tensor(refs), torch.tensor([ng], dtype=torch.int64, device=dev)
            agg = wrapped.AsyncPagesAggregate(np.uint64, metas.numel(), pages.numel(), ng, n)
            dec = wrapped.AsyncPagesDecompressor(np.uint64, metas.numel(), pages.numel(), ng, n)
            args_in = (metas, pages, d_refs, d_n)
            n_batches = int(sum((int(p) + 255) // 256 for p in group_ns))
            legs = {"pages": ng, "pages_bytes": int(pages.numel())}
        else:
            d_data, files, d_index = standalone.compress_files(nums.view(torch.uint64), np.array(sizes, np.uint64), cfg)
            torch.cuda.synchronize()
            frefs = np.stack([files["offset"], files["len"], files["index_offset"], files["index_len"]], axis=1).astype(np.uint64)
            ng = len(frefs)
            group_ns = np.array(sizes, np.int64)
            n_chunks = int(sum(-(-int(s) // CHUNK_N) for s in sizes))
            d_refs, d_n = torch.as_tensor(frefs.view(np.int64), device=dev), torch.tensor([ng], dtype=torch.int64, device=dev)
            agg = standalone.AsyncFilesAggregate(d_data[:32], np.uint64, d_data.numel(), d_index.numel(), ng, n_chunks, n)
            dec = standalone.AsyncFilesDecompressor(d_data[:32], np.uint64, d_data.numel(), d_index.numel(), ng, n_chunks, n)
            args_in = (d_data, d_index, d_refs, d_n)
            n_batches = n // 256  # every chunk holds a multiple of 256 numbers
            legs = {"files": ng, "chunks": n_chunks, "file_bytes": int(d_data.numel())}
        legs.update({"aggregate_workspace_bytes": agg.workspace_bytes, "decompressor_workspace_bytes": dec.workspace_bytes})
        gid = torch.repeat_interleave(torch.arange(ng, device=dev), torch.from_numpy(group_ns).to(dev))
        iv = torch.zeros(2, dtype=torch.int64, device=dev)
        lo_t, hi_t = torch.zeros((), dtype=torch.int64, device=dev), torch.zeros((), dtype=torch.int64, device=dev)
        aggs = torch.zeros((ng, 6), dtype=torch.int64, device=dev)
        tot = torch.zeros(6, dtype=torch.int64, device=dev)
        d_out = torch.empty(n, dtype=torch.int64, device=dev)
        call = lambda: agg(*args_in, iv, aggs, tot)  # noqa: E731
        if kind == "pages":
            decode = lambda: dec(*args_in, d_out.view(torch.uint64))  # noqa: E731
        else:
            d_ns = torch.zeros(ng, dtype=torch.int64, device=dev)
            decode = lambda: dec(*args_in, d_out.view(torch.uint64), d_ns)  # noqa: E731
        g_agg = capture(call)
        g_dec = capture(decode)
        legs["decode_graph_ms"] = events(g_dec.replay)
        out = {}

        def baseline():
            decode()
            reduce_groups(d_out, gid, ng, lo_t, hi_t, out)

        g_base = capture(baseline)
        ok_all = True
        for s in SELECTIVITIES:
            k_want = int(round(s * n))
            mid = n // 2
            if k_want == 0:
                lo, hi = int(srt[mid]) + 1, int(srt[mid])
            else:
                a = max(0, min(n - k_want, mid - k_want // 2))
                lo, hi = int(srt[a]), int(srt[a + k_want - 1])
            iv.copy_(torch.tensor([lo, hi], dtype=torch.int64))
            lo_t.fill_(lo)
            hi_t.fill_(hi)
            want = reduce_groups(nums, gid, ng, lo_t, hi_t, {})
            k = int(want["cnt"].sum())
            t = {"lo": lo, "hi": hi, "matches": k}
            t["agg_ms"] = events(call)
            ok_a = agg.result() == k and same(aggs, tot, want)
            aggs.fill_(-7)
            t["agg_graph_ms"] = events(g_agg.replay)
            ok_g = agg.result() == k and same(aggs, tot, want)
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
            t["baseline_graph_ms"] = events(g_base.replay)
            rec_b = torch.stack([torch.zeros_like(out["cnt"]), out["cnt"], torch.where(out["cnt"] > 0, out["min"], 0),
                                 torch.where(out["cnt"] > 0, out["max"], 0), out["sum"], torch.zeros_like(out["cnt"])], 1)
            tot_b = torch.tensor([0, k, int(want["min"][want["cnt"] > 0].min()) if k else 0, int(want["max"][want["cnt"] > 0].max()) if k else 0,
                                  int(out["sum"].sum()), 0])
            ok_b = same(rec_b, tot_b, want)
            slots = n // 256 + ng if kind == "pages" else n // 256 + n_chunks
            hit = int(torch.unique(torch.nonzero((nums >= lo) & (nums <= hi)).squeeze(1) // 256).numel()) if k else 0
            t["written_mb"] = {"aggregate": round((4 * slots + 32 * hit + 48 * ng + 48 * ng + 48) / 1e6, 3),
                               "baseline": round((8 * n + n + 4 * 8 * ng) / 1e6, 3)}
            t["batches"] = n_batches
            t["parity"] = bool(ok_a and ok_g and ok_b)
            ok_all = ok_all and t["parity"]
            legs[f"sel_{s:g}"] = t
        parity[iname] = ok_all
        res[iname] = legs
        del g_agg, g_dec, g_base, agg, dec
        torch.cuda.empty_cache()
    print(json.dumps({"workload": f"C2: {args.chunks} chunks x 2^18 u64 as 1024 wrapped pages (order 1 and 0), one indexed file (order 1 and 0) "
                                  f"and {n >> 16} files of 2^16, u64 interval aggregates, device buffers",
                      "gpu": gpu_description(), "steps": steps, "results": res, "parity": parity}))


if __name__ == "__main__":
    main()
