#!/usr/bin/env python
"""bench_async_pages_to_file.py — the transcode of wrapped pages into one indexed standalone file (pco_b200_pages_to_file_async,
wrapped.AsyncPagesToFile), and what it buys: the files calls on its output against the pages calls on the pages.

Inputs (every buffer in HBM): bench.py's array (1024 chunks of 2^18 u64, C2 data, chunk c = datagen.c2_u64_cumsum_geometric(seed = c))
as 1024 wrapped pages (wrapped.compress_chunks) at consecutive delta order 1 (pages_1024_order1) and with no delta (pages_1024_order0), and
its first 2^19 numbers as 64 pages of 2^13 (pages_64x8192, order 1).
Per leg:
  - transcode_ms (one call) and transcode_graph_ms (one replay of the call captured once), CUDA events, median of --steps; kernel_ms (the
    per-kernel split of one profiled call); read_mb / written_mb (HBM bytes: the front end reads the metas and pages and writes the frames,
    the file writer reads the frames' chunk bytes and writes the file, the index writer reads the walked entries and writes the index);
  - scans, each as one replay of a captured call: decompress (AsyncPagesDecompressor / AsyncFilesDecompressor), filter at 1 %
    (AsyncPagesFilter / AsyncFilesFilter, an interval holding 1 % of the rows), aggregate over the same interval (AsyncPagesAggregate /
    AsyncFilesAggregate) and take of a contiguous run of 1 % of the rows from n / 3 (AsyncPagesTake / AsyncFilesTake): pages_ms,
    files_ms, and scans_to_pay_off = ceil(transcode_graph_ms / (pages_ms - files_ms));
  - parity: the file and index equal standalone.compress_files' for the same chunks, the files decompress equals the input, and every scan
    of the file equals the same scan of the pages (values, positions, counts and aggregate totals).
Prints one JSON line; writes nothing.

    python bench_async_pages_to_file.py [--steps 10] [--chunks 1024]
"""
import argparse
import json
import math
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

    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec, _lib, datagen, standalone, wrapped

    L = _lib.lib()
    if not L.pco_b200_device_available():
        raise RuntimeError("libcpcodec.so found no usable CUDA device: " + L.pco_b200_last_error_message().decode())
    dev = torch.device("cuda", 0)
    steps = max(args.steps, 1)
    n_all = args.chunks * CHUNK_N
    h_np = np.empty(n_all, dtype=np.uint64)
    for c in range(args.chunks):
        h_np[c * CHUNK_N:(c + 1) * CHUNK_N] = datagen.c2_u64_cumsum_geometric(CHUNK_N, seed=c)
    nums_all = torch.from_numpy(h_np.view(np.int64)).to(dev)

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

    def timed_graph(fn):
        g = capture(fn)
        ms = events(g.replay)
        del g
        return ms

    legs = {"pages_1024_order1": (n_all, CHUNK_N, DeltaSpec.try_consecutive(1)), "pages_1024_order0": (n_all, CHUNK_N, DeltaSpec.no_op()),
            "pages_64x8192": (64 << 13, 1 << 13, DeltaSpec.try_consecutive(1))}
    res, parity = {}, {}
    for lname, (n, page_n, delta) in legs.items():
        nums = nums_all[:n]
        cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=delta, paging_spec=PagingSpec.equal_pages_up_to(page_n))
        metas, pages, refs = wrapped.compress_chunks(nums.view(torch.uint64), cfg)
        want_data, want_ref, want_idx = standalone.compress_files(nums.view(torch.uint64), np.array([n], np.uint64), cfg)
        torch.cuda.synchronize()
        want_file = want_data[: int(want_ref["len"][0])]
        want_index = want_idx[int(want_ref["index_offset"][0]): int(want_ref["index_offset"][0]) + int(want_ref["index_len"][0])]
        mp = len(refs)
        d_refs = torch.from_numpy(np.stack([refs[f].astype(np.int64) for f in wrapped.PAGE_REF.names], axis=1)).to(dev)
        d_n = torch.tensor([mp], dtype=torch.int64, device=dev)
        mcap, pcap = metas.numel(), pages.numel()
        dst_cap, index_cap = want_file.numel() + 64, want_index.numel() + 64
        t = wrapped.AsyncPagesToFile(np.uint64, mcap, pcap, mp, dst_cap, index_cap)
        call = lambda: t(metas, pages, d_refs, d_n)  # noqa: E731
        leg = {"pages": mp, "page_n": page_n, "metas_bytes": mcap, "pages_bytes": pcap, "workspace_bytes": t.workspace_bytes}
        leg["transcode_ms"] = events(call)
        fl, il = t.result()
        ok = fl == want_file.numel() and il == want_index.numel() and torch.equal(t.file[:fl], want_file) and torch.equal(t.index[:il], want_index)
        leg["transcode_graph_ms"] = timed_graph(call)
        ok = ok and t.result() == (fl, il)
        L.pco_b200_profile_enable(1)
        call()
        torch.cuda.synchronize()
        leg["kernel_ms"] = {k: round(v, 4) for k, v in parse_profile(L).items()}
        L.pco_b200_profile_enable(0)
        frames = int(sum((4 + int(r["meta_len"]) + int(r["page_len"]) + 15) // 16 * 16 for r in refs))
        walked = int(sum(2 * ((int(r["page_n"]) + 255) // 256) * 12 for r in refs))
        leg["read_mb"] = round((mcap + pcap + fl + walked) / 1e6, 3)
        leg["written_mb"] = round((frames + walked + fl + il) / 1e6, 3)
        leg["file_bytes"], leg["index_bytes"] = fl, il

        fa = t.files_args()
        srcs = {"pages": (metas, pages, d_refs, d_n), "files": (t.file, t.index, t.file_ref, t.n_files)}
        scans = {}
        # decompress
        d_out = torch.empty(n, dtype=torch.int64, device=dev)
        pd = wrapped.AsyncPagesDecompressor(np.uint64, mcap, pcap, mp, n)
        fd = standalone.AsyncFilesDecompressor(**fa, dst_cap=n)
        d_ns = torch.zeros(1, dtype=torch.int64, device=dev)
        s = {"pages_ms": timed_graph(lambda: pd(*srcs["pages"], d_out.view(torch.uint64)))}
        ok = ok and pd.result() == n and torch.equal(d_out, nums)
        d_out.fill_(-1)
        s["files_ms"] = timed_graph(lambda: fd(*srcs["files"], d_out.view(torch.uint64), d_ns))
        ok = ok and fd.result() == n and torch.equal(d_out, nums)
        scans["decompress"] = s
        del pd, fd
        # filter at 1 %
        srt = torch.sort(nums)[0]
        k1 = n // 100
        lo, hi = int(srt[n // 2]), int(srt[n // 2 + k1 - 1])
        iv = torch.tensor([lo, hi], dtype=torch.int64, device=dev)
        del srt
        outs = {}
        for kind in ("pages", "files"):
            vals = torch.empty(2 * k1 + 64, dtype=torch.int64, device=dev)
            pos = torch.empty(2 * k1 + 64, dtype=torch.int64, device=dev)
            nm = torch.zeros(1, dtype=torch.int64, device=dev)
            f = (wrapped.AsyncPagesFilter(np.uint64, mcap, pcap, mp, n, vals.numel()) if kind == "pages"
                 else standalone.AsyncFilesFilter(**fa, rows_cap=n, out_cap=vals.numel()))
            ms = timed_graph(lambda: f(*srcs[kind], iv, vals.view(torch.uint64), pos, nm))
            k = f.result()
            outs[kind] = (ms, k, vals[:k].clone(), pos[:k].clone())
            del f
        scans["filter_1%"] = {"pages_ms": outs["pages"][0], "files_ms": outs["files"][0], "matches": outs["files"][1]}
        ok = ok and outs["pages"][1] == outs["files"][1] and torch.equal(outs["pages"][2], outs["files"][2]) and torch.equal(outs["pages"][3], outs["files"][3])
        # aggregate over the same interval
        tots = {}
        for kind in ("pages", "files"):
            groups = mp if kind == "pages" else 1
            aggs = torch.zeros((groups, 6), dtype=torch.int64, device=dev)
            tot = torch.zeros(6, dtype=torch.int64, device=dev)
            a = (wrapped.AsyncPagesAggregate(np.uint64, mcap, pcap, mp, n) if kind == "pages" else standalone.AsyncFilesAggregate(**fa, rows_cap=n))
            ms = timed_graph(lambda: a(*srcs[kind], iv, aggs, tot))
            a.result()
            tots[kind] = (ms, tot.clone())
            del a
        scans["aggregate_1%"] = {"pages_ms": tots["pages"][0], "files_ms": tots["files"][0]}
        ok = ok and torch.equal(tots["pages"][1], tots["files"][1])
        # take of a contiguous 1 %
        d_pos = torch.arange(n // 3, n // 3 + k1, dtype=torch.int64, device=dev)
        d_np = torch.tensor([k1], dtype=torch.int64, device=dev)
        taken = {}
        for kind in ("pages", "files"):
            out = torch.empty(k1, dtype=torch.int64, device=dev)
            tk = (wrapped.AsyncPagesTake(np.uint64, mcap, pcap, mp, n, k1) if kind == "pages"
                  else standalone.AsyncFilesTake(**fa, rows_cap=n, max_positions=k1))
            ms = timed_graph(lambda: tk(*srcs[kind], d_pos, d_np, out.view(torch.uint64)))
            ok = ok and tk.result() == k1 and torch.equal(out, nums[n // 3: n // 3 + k1])
            taken[kind] = ms
            del tk
        scans["take_run_1%"] = {"pages_ms": taken["pages"], "files_ms": taken["files"]}
        for s in scans.values():
            gain = s["pages_ms"] - s["files_ms"]
            s["scans_to_pay_off"] = math.ceil(leg["transcode_graph_ms"] / gain) if gain > 0 else None
        leg["scans"] = scans
        leg["parity"] = bool(ok)
        parity[lname] = bool(ok)
        res[lname] = leg
        del t, metas, pages, want_data, want_idx, want_file, want_index, d_out
        torch.cuda.empty_cache()
    print(json.dumps({"workload": f"C2: {args.chunks} chunks x 2^18 u64 as {args.chunks} wrapped pages (order 1 and 0) and 64 pages of 2^13, "
                                  "transcoded into one indexed file, then scanned; device buffers",
                      "gpu": gpu_description(), "steps": steps, "results": res, "parity": parity}))


if __name__ == "__main__":
    main()
