#!/usr/bin/env python
"""bench_async_segment_aggregate.py — count, min, max and sum of the numbers inside an interval per row segment [bounds[g], bounds[g + 1]),
reduced in the decoder (pco_b200_segment_aggregate_pages_async / _files_async, wrapped.AsyncPagesSegmentAggregate,
standalone.AsyncFilesSegmentAggregate), against decoding everything and reducing afterwards (AsyncPagesDecompressor /
AsyncFilesDecompressor, then torch bucketize segment ids, a mask and index_add / scatter_reduce, captured in one graph).

Inputs: bench.py's array (1024 chunks of 2^18 u64, C2 data, chunk c = datagen.c2_u64_cumsum_geometric(seed = c)), every buffer in HBM:
  - file_order1 / file_order0: standalone.compress_files, one indexed file of 1024 chunks, consecutive delta order 1 / no_op;
  - files_4096: bench_files.py's uniform cut, 4096 files of 2^16 numbers, delta order 1;
  - pages_order1: wrapped.compress_chunks, 1024 pages, delta order 1.
Segment shapes over the n rows: uniform widths of 300 rows (a bound in most batches), 4096, 100000 and 2^22 rows; segments equal to the
pages / files (beside the aggregate call, agg_ms); one segment over every row (likewise); a 1 % window around the middle cut into 1000
segments; 2^20 segments of 256 rows on batch edges.  Intervals: everything, and the middle half of the sorted numbers (about 50 %).
Per leg: seg_ms (one call) and seg_graph_ms (one replay of the call captured once), CUDA events, median of --steps; enqueue_us (host time
of one call); kernel_ms (per-kernel split of one profiled call: plan = sg_*check/mark, decode = the decode stage, group = sg_group_kernel,
finish = sg_finish_*); records_decoded; written_mb (HBM bytes the call writes, an upper bound computed from the counts: each slot's run,
one 40-byte record per (batch, segment) pair, the segments' accumulators and records); parity (every segment's count, min, max and sum and
the total equal a torch reduction over the input; the C2 values and their sums stay below 2^63, so int64 torch ops are exact on them).
The baseline (decoder + torch, captured) runs once per input and shape, with the interval of everything: baseline_graph_ms.
Prints one JSON line with the card name and power limit read in the same run; writes nothing.

    python bench_async_segment_aggregate.py [--steps 10] [--chunks 1024]
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
    rows_idx = torch.arange(n, device=dev)

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

    def reduce_segments(x, bounds, m, lo_t, hi_t, out):
        """The baseline's reduction (also the reference, over the input): segment ids by bucketize (rows outside every segment go to an
        extra group m), then per segment count, min, max and sum of the matches."""
        gid = torch.bucketize(rows_idx, bounds[: m + 1], right=True) - 1
        gid = torch.where((gid >= 0) & (gid < m), gid, m)
        mk = (x >= lo_t) & (x <= hi_t)
        out["cnt"] = torch.zeros(m + 1, dtype=torch.int64, device=dev).index_add_(0, gid, mk.long())[:m]
        out["sum"] = torch.zeros(m + 1, dtype=torch.int64, device=dev).index_add_(0, gid, torch.where(mk, x, 0))[:m]
        out["min"] = torch.full((m + 1,), BIG, dtype=torch.int64, device=dev).scatter_reduce_(0, gid, torch.where(mk, x, BIG), "amin")[:m]
        out["max"] = torch.full((m + 1,), -1, dtype=torch.int64, device=dev).scatter_reduce_(0, gid, torch.where(mk, x, -1), "amax")[:m]
        return out

    def same(recs, tot, want, bounds):
        cnt = want["cnt"]
        has = cnt > 0
        m = cnt.numel()
        ok = torch.equal(recs[:, 0], bounds[1:m + 1] - bounds[:m]) and torch.equal(recs[:, 1], cnt) and torch.equal(recs[:, 4], want["sum"])
        ok = ok and bool((recs[:, 5] == 0).all()) and torch.equal(recs[:, 2][has], want["min"][has]) and torch.equal(recs[:, 3][has], want["max"][has])
        ok = ok and bool((recs[:, 2][~has] == 0).all()) and bool((recs[:, 3][~has] == 0).all())
        k = int(cnt.sum())
        ok = ok and int(tot[0]) == int(bounds[m] - bounds[0]) and int(tot[1]) == k and int(tot[4]) == int(want["sum"].sum()) and int(tot[5]) == 0
        if k:
            ok = ok and int(tot[2]) == int(want["min"][has].min()) and int(tot[3]) == int(want["max"][has].max())
        return bool(ok)

    def refs_tensor(refs):
        return torch.from_numpy(np.stack([refs[f].astype(np.int64) for f in wrapped.PAGE_REF.names], axis=1)).to(dev)

    mid = n // 2
    win = n // 100
    shapes = {
        "w300": np.append(np.arange(0, n, 300), n),
        "w4096": np.append(np.arange(0, n, 4096), n),
        "w100000": np.append(np.arange(0, n, 100000), n),
        "w2^22": np.append(np.arange(0, n, 1 << 22), n),
        "groups": None,  # the pages' / files' starts, beside the aggregate call
        "whole": np.array([0, n]),
        "window1pct_1000": np.linspace(mid - win // 2, mid + win // 2, 1001).astype(np.int64),
        "aligned256_2^20": np.arange(0, min(n, 256 << 20) + 1, 256),
    }
    max_segments = max(len(b) - 1 for b in shapes.values() if b is not None) + 4096
    half = (int(srt[n // 4]), int(srt[3 * n // 4]))
    intervals = {"all": (0, BIG), "half": half}

    res, parity = {}, {}
    for iname, (kind, delta, sizes) in {"file_order1": ("files", DeltaSpec.try_consecutive(1), [n]),
                                        "file_order0": ("files", DeltaSpec.no_op(), [n]),
                                        "files_4096": ("files", DeltaSpec.try_consecutive(1), [1 << 16] * (n >> 16)),
                                        "pages_order1": ("pages", DeltaSpec.try_consecutive(1), None)}.items():
        cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=delta, paging_spec=PagingSpec.equal_pages_up_to(CHUNK_N))
        if kind == "pages":
            metas, pages, refs = wrapped.compress_chunks(nums.view(torch.uint64), cfg)
            torch.cuda.synchronize()
            ng = len(refs)
            group_ns = refs["page_n"].astype(np.int64)
            d_refs, d_n = refs_tensor(refs), torch.tensor([ng], dtype=torch.int64, device=dev)
            seg = wrapped.AsyncPagesSegmentAggregate(np.uint64, metas.numel(), pages.numel(), ng, n, max_segments)
            agg = wrapped.AsyncPagesAggregate(np.uint64, metas.numel(), pages.numel(), ng, n)
            dec = wrapped.AsyncPagesDecompressor(np.uint64, metas.numel(), pages.numel(), ng, n)
            args_in = (metas, pages, d_refs, d_n)
            legs = {"pages": ng}
        else:
            d_data, files, d_index = standalone.compress_files(nums.view(torch.uint64), np.array(sizes, np.uint64), cfg)
            torch.cuda.synchronize()
            frefs = np.stack([files["offset"], files["len"], files["index_offset"], files["index_len"]], axis=1).astype(np.uint64)
            ng = len(frefs)
            group_ns = np.array(sizes, np.int64)
            n_chunks = int(sum(-(-int(s) // CHUNK_N) for s in sizes))
            d_refs, d_n = torch.as_tensor(frefs.view(np.int64), device=dev), torch.tensor([ng], dtype=torch.int64, device=dev)
            seg = standalone.AsyncFilesSegmentAggregate(d_data[:32], np.uint64, d_data.numel(), d_index.numel(), ng, n_chunks, n, max_segments)
            agg = standalone.AsyncFilesAggregate(d_data[:32], np.uint64, d_data.numel(), d_index.numel(), ng, n_chunks, n)
            dec = standalone.AsyncFilesDecompressor(d_data[:32], np.uint64, d_data.numel(), d_index.numel(), ng, n_chunks, n)
            args_in = (d_data, d_index, d_refs, d_n)
            legs = {"files": ng, "chunks": n_chunks}
        legs["segment_workspace_bytes"] = seg.workspace_bytes
        starts = np.concatenate([[0], np.cumsum(group_ns)])
        iv = torch.zeros(2, dtype=torch.int64, device=dev)
        lo_t, hi_t = torch.zeros((), dtype=torch.int64, device=dev), torch.full((), BIG, dtype=torch.int64, device=dev)
        d_bounds = torch.zeros(max_segments + 1, dtype=torch.int64, device=dev)
        d_ns = torch.zeros(1, dtype=torch.int64, device=dev)
        aggs = torch.zeros((max_segments, 6), dtype=torch.int64, device=dev)
        tot = torch.zeros(6, dtype=torch.int64, device=dev)
        a_aggs = torch.zeros((ng, 6), dtype=torch.int64, device=dev)
        a_tot = torch.zeros(6, dtype=torch.int64, device=dev)
        d_out = torch.empty(n, dtype=torch.int64, device=dev)
        call = lambda: seg(*args_in, d_bounds, d_ns, iv, aggs, tot)  # noqa: E731
        if kind == "pages":
            decode = lambda: dec(*args_in, d_out.view(torch.uint64))  # noqa: E731
        else:
            d_fns = torch.zeros(ng, dtype=torch.int64, device=dev)
            decode = lambda: dec(*args_in, d_out.view(torch.uint64), d_fns)  # noqa: E731
        g_seg = capture(call)
        ok_all = True
        for sname, b in shapes.items():
            b = starts if b is None else b
            m = len(b) - 1
            d_bounds.zero_()
            d_bounds[: m + 1].copy_(torch.from_numpy(b.astype(np.int64)))
            d_ns.fill_(m)
            leg = {"segments": m}
            out = {}

            def baseline():
                decode()
                reduce_segments(d_out, d_bounds, m, lo_t, hi_t, out)

            iv.copy_(torch.tensor([0, BIG], dtype=torch.int64))
            g_base = capture(baseline)
            leg["baseline_graph_ms"] = events(g_base.replay)
            del g_base
            for vname, (lo, hi) in intervals.items():
                iv.copy_(torch.tensor([lo, hi], dtype=torch.int64))
                lo_t.fill_(lo)
                hi_t.fill_(hi)
                want = reduce_segments(nums, d_bounds, m, lo_t, hi_t, {})
                k = int(want["cnt"].sum())
                t = {"matches": k, "seg_ms": events(call)}
                ok_c = seg.result() == k and same(aggs[:m], tot, want, d_bounds)
                st = seg.status_record()
                aggs.fill_(-7)
                t["seg_graph_ms"] = events(g_seg.replay)
                ok_g = seg.result() == k and same(aggs[:m], tot, want, d_bounds)
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
                t["records_decoded"] = int(st.records_decoded)
                covered = int(b[-1] - b[0])
                t["written_mb"] = round((8 * (n // 256 + len(group_ns)) + 40 * (covered // 256 + 2 * m) + 96 * m + 48) / 1e6, 3)
                if sname in ("groups", "whole"):
                    agg(*args_in, iv, a_aggs, a_tot)
                    t["agg_ms"] = events(lambda: agg(*args_in, iv, a_aggs, a_tot))
                    agg.result()
                    if sname == "groups":
                        ok_c = ok_c and torch.equal(a_aggs, aggs[:m]) and torch.equal(a_tot, tot)
                t["parity"] = bool(ok_c and ok_g)
                ok_all = ok_all and t["parity"]
                leg[vname] = t
            legs[sname] = leg
            torch.cuda.empty_cache()
        parity[iname] = ok_all
        res[iname] = legs
        del g_seg, seg, agg, dec
        torch.cuda.empty_cache()
    print(json.dumps({"workload": f"C2: {args.chunks} chunks x 2^18 u64 as one indexed file (order 1 and 0), {n >> 16} files of 2^16 and "
                                  f"{args.chunks} wrapped pages; u64 segment aggregates, device buffers",
                      "gpu": gpu_description(), "steps": steps, "results": res, "parity": parity}))


if __name__ == "__main__":
    main()
