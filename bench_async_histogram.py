#!/usr/bin/env python
"""bench_async_histogram.py — per page / file histograms counted in the decoder (pco_b200_histogram_pages_async / _files_async,
wrapped.AsyncPagesHistogram, standalone.AsyncFilesHistogram), against decoding everything and bucketing afterwards (AsyncPagesDecompressor /
AsyncFilesDecompressor, then torch.bucketize and index_add_ into a (groups, W) tensor, captured in one graph), and against the aggregate
call (AsyncPagesAggregate / AsyncFilesAggregate) over the interval of every number, on the same input.

Inputs: bench.py's array (1024 chunks of 2^18 u64, C2 data, chunk c = datagen.c2_u64_cumsum_geometric(seed = c)), every buffer in HBM:
  - file_order1 / file_order0: standalone.compress_files, one indexed file of 1024 chunks, consecutive delta order 1 / no_op;
  - files_4096: 4096 files of 2^16 numbers, delta order 1;
  - pages: wrapped.compress_chunks, 1024 pages, delta order 1.
Bucket counts 16, 256 and 4096, each with three edge layouts: uniform (equal widths over [min, max], which the aggregate call gives),
quantile (edges at sampled quantiles, so every bucket holds about as many numbers) and skew (every number in one bucket: the
contention worst case the CTA-private counters exist for).
Per leg: hist_ms (one call) and hist_graph_ms (one replay of the call captured once), baseline_graph_ms, CUDA events, median of --steps;
enqueue_us (host time of one call); kernel_ms (per-kernel split of one profiled call: the decode kernels count and flush, hg_cold_* and
hg_rows_kernel are the group stage, hg_finish_* the finish); written_mb (HBM bytes written, from the shapes: the histogram's cleared rows,
hists and total; the baseline's decoded numbers, bucket indices, flat indices and its (groups, W) output); parity (every row and the total
from both paths equal np.searchsorted-style counts made by torch.bucketize over the input, and agree with each other).
Per input: aggregate_graph_ms (the aggregate call captured) and decode_graph_ms (the decompressor alone, captured).  On file_order1, the
exact p99 leg: the histogram (256 quantile buckets), the bucket that holds rank r, a filter of that bucket and a sort of its few numbers,
all in one graph, against torch.kthvalue on the decompressed column.
Prints one JSON line with the card's name, power limit and max SM clock read in the same run; writes nothing.

    python bench_async_histogram.py [--steps 5] [--chunks 1024]
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

BUCKETS = [16, 256, 4096]
LAYOUTS = ["uniform", "quantile", "skew"]


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
    nums = torch.from_numpy(h_np.view(np.int64)).to(dev)  # the C2 values stay below 2^63: int64 compares order them as u64 does
    lo_all, hi_all = int(nums.min()), int(nums.max())
    sample = torch.sort(nums[torch.randint(0, n, (1 << 20,), device=dev, generator=torch.Generator(device=dev).manual_seed(0))])[0]

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

    def edges_of(layout, nb):
        if layout == "uniform":
            e = np.unique(np.linspace(lo_all, hi_all, nb + 1).astype(np.int64))
        elif layout == "quantile":
            e = np.unique(sample[torch.linspace(0, sample.numel() - 1, nb + 1, device=dev).long()].cpu().numpy())
            e[0], e[-1] = min(e[0], lo_all), max(e[-1], hi_all)
        else:  # every number in bucket 0: the others lie above the largest number
            e = np.concatenate([[lo_all], hi_all + 1 + np.arange(nb, dtype=np.int64)])
        assert len(e) == nb + 1 and (np.diff(e) > 0).all(), (layout, nb)
        return torch.from_numpy(e.astype(np.int64)).to(dev)

    def bucket_rows(x, gid, ng, ed, ones):
        """The baseline's bucketing (also the reference, over the input): the (ng, W) rows of x."""
        nb = ed.numel() - 1
        col = torch.bucketize(x, ed, right=True)  # the edges at or below each number
        col = torch.where((col == nb + 1) & (x == ed[nb]), nb, col)
        flat = gid * (nb + 3) + col
        return torch.zeros(ng * (nb + 3), dtype=torch.int64, device=dev).index_add_(0, flat, ones).view(ng, nb + 3)

    def refs_tensor(refs):
        return torch.from_numpy(np.stack([refs[f].astype(np.int64) for f in wrapped.PAGE_REF.names], axis=1)).to(dev)

    inputs = {"file_order1": ("files", DeltaSpec.try_consecutive(1), [n]), "file_order0": ("files", DeltaSpec.no_op(), [n]),
              "files_4096": ("files", DeltaSpec.try_consecutive(1), [1 << 16] * (n >> 16)), "pages": ("pages", DeltaSpec.try_consecutive(1), None)}
    ones = torch.ones(n, dtype=torch.int64, device=dev)
    res, parity = {}, {}
    for iname, (kind, delta, sizes) in inputs.items():
        cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=delta, paging_spec=PagingSpec.equal_pages_up_to(CHUNK_N))
        if kind == "pages":
            metas, pages, refs = wrapped.compress_chunks(nums.view(torch.uint64), cfg)
            torch.cuda.synchronize()
            ng = len(refs)
            group_ns = refs["page_n"].astype(np.int64)
            args_in = (metas, pages, refs_tensor(refs), torch.tensor([ng], dtype=torch.int64, device=dev))
            mk_hist = lambda nb: wrapped.AsyncPagesHistogram(np.uint64, metas.numel(), pages.numel(), ng, n, nb)  # noqa: E731
            agg = wrapped.AsyncPagesAggregate(np.uint64, metas.numel(), pages.numel(), ng, n)
            dec = wrapped.AsyncPagesDecompressor(np.uint64, metas.numel(), pages.numel(), ng, n)
            legs = {"pages": ng}
        else:
            d_data, files, d_index = standalone.compress_files(nums.view(torch.uint64), np.array(sizes, np.uint64), cfg)
            torch.cuda.synchronize()
            frefs = np.stack([files["offset"], files["len"], files["index_offset"], files["index_len"]], axis=1).astype(np.uint64)
            ng = len(frefs)
            group_ns = np.array(sizes, np.int64)
            nc = int(sum(-(-int(s) // CHUNK_N) for s in sizes))
            args_in = (d_data, d_index, torch.as_tensor(frefs.view(np.int64), device=dev), torch.tensor([ng], dtype=torch.int64, device=dev))
            mk_hist = lambda nb: standalone.AsyncFilesHistogram(d_data[:32], np.uint64, d_data.numel(), d_index.numel(), ng, nc, n, nb)  # noqa: E731
            agg = standalone.AsyncFilesAggregate(d_data[:32], np.uint64, d_data.numel(), d_index.numel(), ng, nc, n)
            dec = standalone.AsyncFilesDecompressor(d_data[:32], np.uint64, d_data.numel(), d_index.numel(), ng, nc, n)
            legs = {"files": ng, "chunks": nc}
        gid = torch.repeat_interleave(torch.arange(ng, device=dev), torch.from_numpy(group_ns).to(dev))
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
        legs["aggregate_parity"] = agg.result() == n
        del g_agg
        ok_all = legs["aggregate_parity"]
        for nb in BUCKETS:
            w = nb + 3
            hist = mk_hist(nb)
            hists = torch.zeros((ng, w), dtype=torch.int64, device=dev)
            tot = torch.zeros(w, dtype=torch.int64, device=dev)
            ed = torch.zeros(nb + 1, dtype=torch.int64, device=dev)
            call = lambda: hist(*args_in, ed, hists, tot)  # noqa: E731
            g_hist, _ = capture(call)
            g_base, base_out = capture(lambda: (decode(), bucket_rows(d_out, gid, ng, ed, ones))[1])
            for layout in LAYOUTS:
                ed.copy_(edges_of(layout, nb))
                want = bucket_rows(nums, gid, ng, ed, ones)
                t = {"workspace_bytes": hist.workspace_bytes}
                t["hist_ms"] = events(call)
                ok_c = hist.result() == n and torch.equal(hists, want) and torch.equal(tot, want.sum(0))
                hists.fill_(-7)
                t["hist_graph_ms"] = events(g_hist.replay)
                ok_g = hist.result() == n and torch.equal(hists, want) and torch.equal(tot, want.sum(0))
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
                t["kernel_ms"] = {k: round(v, 4) for k, v in parse_profile(L).items()}
                L.pco_b200_profile_enable(0)
                t["baseline_graph_ms"] = events(g_base.replay)
                ok_b = torch.equal(base_out, want)
                t["written_mb"] = {"histogram": round((2 * 8 * ng * w + 16 * w) / 1e6, 3), "baseline": round((3 * 8 * n + 8 * ng * w) / 1e6, 3)}
                t["fullest_bucket_share"] = round(float(want.sum(0).max()) / n, 4)
                t["parity"] = bool(ok_c and ok_g and ok_b)
                ok_all = ok_all and t["parity"]
                legs[f"b{nb}_{layout}"] = t
            del g_hist, g_base, hist
            torch.cuda.empty_cache()
        if iname == "file_order1":
            legs["p99"] = p99_leg(args_in, d_data, d_index, ng, nc, n, decode, d_out, edges_of("quantile", 256), events, capture, standalone)
            ok_all = ok_all and legs["p99"]["parity"]
        parity[iname] = ok_all
        res[iname] = legs
        del g_dec, agg, dec
        torch.cuda.empty_cache()
    print(json.dumps({"workload": f"C2: {args.chunks} chunks x 2^18 u64 as one indexed file (order 1 and 0), {n >> 16} files of 2^16 and 1024 "
                                  "wrapped pages, u64 histograms of 16 / 256 / 4096 buckets, device buffers",
                      "gpu": gpu_description(), "steps": steps, "results": res, "parity": parity}))


def p99_leg(args_in, d_data, d_index, ng, nc, n, decode, d_out, ed, events, capture, standalone):
    """The exact p99 in one graph (histogram, bucket of rank r, filter of the bucket, sort of its numbers) against torch.kthvalue."""
    import torch

    dev = d_out.device
    nb, out_cap = ed.numel() - 1, 1 << 22
    hist = standalone.AsyncFilesHistogram(d_data[:32], np.uint64, d_data.numel(), d_index.numel(), ng, nc, n, nb)
    filt = standalone.AsyncFilesFilter(d_data[:32], np.uint64, d_data.numel(), d_index.numel(), ng, nc, n, out_cap)
    hists = torch.zeros((ng, nb + 3), dtype=torch.int64, device=dev)
    tot = torch.zeros(nb + 3, dtype=torch.int64, device=dev)
    vals = torch.zeros(out_cap, dtype=torch.int64, device=dev)
    pos = torch.zeros(out_cap, dtype=torch.int64, device=dev)
    nm = torch.zeros(1, dtype=torch.int64, device=dev)
    idx = torch.arange(out_cap, device=dev)
    big = torch.tensor(torch.iinfo(torch.int64).max, device=dev)
    r = int(0.99 * (n - 1))
    rank = torch.tensor([r], device=dev)

    def quantile():
        hist(*args_in, ed, hists, tot)
        cum = torch.cumsum(tot, 0)
        c = torch.searchsorted(cum, rank, right=True)  # indexing by tensors keeps every step on the device
        below = torch.where(c > 0, cum.index_select(0, (c - 1).clamp(min=0)), 0)
        iv = torch.cat([ed.index_select(0, (c - 1).clamp(min=0, max=nb)), ed.index_select(0, c.clamp(max=nb))])
        filt(*args_in, iv, vals.view(torch.uint64), pos, nm)
        return torch.sort(torch.where(idx < nm[0], vals, big)).values.index_select(0, rank - below)

    g, out = capture(quantile)
    t = {"graph_ms": events(g.replay)}
    hist.result()
    got = int(out)

    def base():
        decode()
        return torch.kthvalue(d_out, r + 1).values

    gb, bout = capture(base)
    t["baseline_graph_ms"] = events(gb.replay)
    t["bucket_numbers"] = int(filt.result())
    t["parity"] = got == int(bout)
    return t


if __name__ == "__main__":
    main()
