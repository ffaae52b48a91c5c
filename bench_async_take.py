#!/usr/bin/env python
"""bench_async_take.py — the numbers at device-resident positions, decoding only the pages or chunks the positions touch
(pco_b200_take_pages_async / _files_async, wrapped.AsyncPagesTake, standalone.AsyncFilesTake), against decoding everything and indexing
afterwards (AsyncPagesDecompressor / AsyncFilesDecompressor, then index_select, captured in one graph).

Inputs: bench.py's array (1024 chunks of 2^18 u64, C2 data, chunk c = datagen.c2_u64_cumsum_geometric(seed = c)), every buffer in HBM:
  - file_order1 / file_order0: standalone.compress_files, one indexed file of 1024 chunks, consecutive delta order 1 (fused_narrow_kernel) /
    no_op (the general pair);
  - files_4096: bench_files.py's uniform cut, 4096 files of 2^16 numbers, delta order 1;
  - pages_1024: wrapped.compress_chunks, 1024 pages, delta order 1.
Position sets (seeded): uniform at 0.001 %, 0.1 %, 1 %, 10 % and 100 % of the rows; one contiguous run of 1 % and of 10 % from row n / 3;
and every 64th row of one chunk in 16 (chunks 0, 16, 32, ...).
Per leg: take_ms (one call) and take_graph_ms (one replay of the call captured once), baseline_graph_ms (one replay of the decompressor
and index_select captured in one graph), ranges_graph_ms (single-file legs with at most 4096 positions: AsyncRangeDecompressor with one
range per position, captured), CUDA events, median of --steps; enqueue_us (host time of one take call); kernel_ms (per-kernel split of one
profiled take call); records_decoded (the status field: pages or chunks decoded); written_mb (HBM bytes the store side writes, computed
from the counts: the take's slot runs of touched batches and its values; the baseline's decoded numbers and its values); parity (the
take's values, the baseline's and the ranges' equal torch's index_select over the input).
Graph leg filter_then_take: AsyncFilesFilter on column A (bench.py's array as file_order1) writes positions that AsyncFilesTake reads from
column B (datagen.c1_u32_lomax chunks of the same chunking), both captured in one graph, at 0.1 % and 1 % selectivity; parity against
B[(A >= lo) & (A <= hi)].
Prints one JSON line; writes nothing.

    python bench_async_take.py [--steps 10] [--chunks 1024]
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

UNIFORM = [0.00001, 0.001, 0.01, 0.1, 1.0]
RUNS = [0.01, 0.1]
RANGES_MAX = 4096


def position_sets(n, n_chunks, seed=0):
    rng = np.random.default_rng(seed)
    sets = {}
    for p in UNIFORM:
        sets[f"uniform_{p * 100:g}%"] = np.arange(n) if p == 1.0 else np.nonzero(rng.random(n) < p)[0]
    for p in RUNS:
        a = n // 3
        sets[f"run_{p * 100:g}%"] = np.arange(a, a + int(p * n))
    chunk = n // n_chunks
    sets["one_chunk_in_16"] = np.concatenate([np.arange(c * chunk, (c + 1) * chunk, 64) for c in range(0, n_chunks, 16)])
    return sets


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

    def refs_tensor(refs):
        return torch.from_numpy(np.stack([refs[f].astype(np.int64) for f in wrapped.PAGE_REF.names], axis=1)).to(dev)

    sets = position_sets(n, args.chunks)
    max_pos = n
    d_pos = torch.empty(max_pos, dtype=torch.int64, device=dev)
    d_npos = torch.zeros(1, dtype=torch.int64, device=dev)
    out = torch.empty(max_pos, dtype=torch.int64, device=dev)
    d_out = torch.empty(n, dtype=torch.int64, device=dev)

    inputs = {"file_order1": ("files", DeltaSpec.try_consecutive(1), [n]), "file_order0": ("files", DeltaSpec.no_op(), [n]),
              "files_4096": ("files", DeltaSpec.try_consecutive(1), [1 << 16] * (n >> 16)), "pages_1024": ("pages", DeltaSpec.try_consecutive(1), None)}
    res, parity = {}, {}
    for iname, (kind, delta, sizes) in inputs.items():
        cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=delta, paging_spec=PagingSpec.equal_pages_up_to(CHUNK_N))
        rng_obj = None
        if kind == "pages":
            metas, pages, refs = wrapped.compress_chunks(nums.view(torch.uint64), cfg)
            torch.cuda.synchronize()
            n_recs = len(refs)
            d_refs, d_n = refs_tensor(refs), torch.tensor([n_recs], dtype=torch.int64, device=dev)
            take = wrapped.AsyncPagesTake(np.uint64, metas.numel(), pages.numel(), n_recs, n, max_pos)
            dec = wrapped.AsyncPagesDecompressor(np.uint64, metas.numel(), pages.numel(), n_recs, n)
            call = lambda: take(metas, pages, d_refs, d_n, d_pos, d_npos, out.view(torch.uint64))  # noqa: E731
            decode = lambda: dec(metas, pages, d_refs, d_n, d_out.view(torch.uint64))  # noqa: E731
            legs = {"pages": n_recs, "pages_bytes": int(pages.numel())}
        else:
            d_data, files, d_index = standalone.compress_files(nums.view(torch.uint64), np.array(sizes, np.uint64), cfg)
            torch.cuda.synchronize()
            frefs = np.stack([files["offset"], files["len"], files["index_offset"], files["index_len"]], axis=1).astype(np.uint64)
            nf = len(frefs)
            n_recs = int(sum(-(-int(s) // CHUNK_N) for s in sizes))
            d_refs, d_n = torch.as_tensor(frefs.view(np.int64), device=dev), torch.tensor([nf], dtype=torch.int64, device=dev)
            head = d_data[:32]
            take = standalone.AsyncFilesTake(head, np.uint64, d_data.numel(), d_index.numel(), nf, n_recs, n, max_pos)
            dec = standalone.AsyncFilesDecompressor(head, np.uint64, d_data.numel(), d_index.numel(), nf, n_recs, n)
            d_ns = torch.zeros(nf, dtype=torch.int64, device=dev)
            call = lambda: take(d_data, d_index, d_refs, d_n, d_pos, d_npos, out.view(torch.uint64))  # noqa: E731
            decode = lambda: dec(d_data, d_index, d_refs, d_n, d_out.view(torch.uint64), d_ns)  # noqa: E731
            legs = {"files": nf, "chunks": n_recs, "file_bytes": int(d_data.numel())}
            if nf == 1:
                rng_obj = standalone.AsyncRangeDecompressor(head, np.uint64, d_data.numel(), d_index.numel(), n_recs, RANGES_MAX, RANGES_MAX, n)
                d_ranges = torch.zeros((RANGES_MAX, 2), dtype=torch.int64, device=dev)
                d_nr = torch.zeros(1, dtype=torch.int64, device=dev)
                r_out = torch.empty(RANGES_MAX, dtype=torch.int64, device=dev)
        legs["take_workspace_bytes"] = take.workspace_bytes
        legs["decompressor_workspace_bytes"] = dec.workspace_bytes
        d_npos.fill_(0)
        g_take = capture(call)
        ok_all = True
        for sname, pos in sets.items():
            k = int(pos.size)
            d_pos[:k].copy_(torch.from_numpy(pos.astype(np.int64)))
            d_npos.fill_(k)
            ref = nums.index_select(0, d_pos[:k])
            t = {"positions": k}
            t["take_ms"] = events(call)
            st = take.status_record()
            ok_t = take.result() == k and torch.equal(out[:k], ref)
            t["records_decoded"] = int(st.records_decoded)
            out.fill_(-1)
            t["take_graph_ms"] = events(g_take.replay)
            ok_tg = take.result() == k and torch.equal(out[:k], ref)
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
            res_b = {}

            def baseline():
                decode()
                res_b["vals"] = d_out.index_select(0, d_pos[:k])

            g_base = capture(baseline)
            t["baseline_graph_ms"] = events(g_base.replay)
            ok_b = torch.equal(res_b["vals"], ref)
            del g_base
            ok_r = True
            if rng_obj is not None and 0 < k <= RANGES_MAX:
                rr = np.stack([pos, np.ones_like(pos)], axis=1).astype(np.int64)
                d_ranges[:k].copy_(torch.from_numpy(rr))
                d_nr.fill_(k)
                g_r = capture(lambda: rng_obj(d_data, d_index, d_ranges, d_nr, r_out.view(torch.uint64)))
                t["ranges_graph_ms"] = events(g_r.replay)
                ok_r = rng_obj.result() == k and torch.equal(r_out[:k], ref)
                del g_r
            batches_hit = int(np.unique(pos // 256).size) if k else 0
            t["written_mb"] = {"take": round((16 * batches_hit + 8 * k) / 1e6, 3), "baseline": round((8 * n + 8 * k) / 1e6, 3)}
            t["parity"] = bool(ok_t and ok_tg and ok_b and ok_r)
            ok_all = ok_all and t["parity"]
            legs[sname] = t
        parity[iname] = ok_all
        res[iname] = legs
        del g_take, take, dec
        torch.cuda.empty_cache()

    # filter on column A, take from column B of the same chunking, in one graph
    b_np = np.concatenate([datagen.c1_u32_lomax(CHUNK_N, seed=c).astype(np.uint64) for c in range(args.chunks)])
    col_b = torch.from_numpy(b_np.view(np.int64)).to(dev)
    cfg1 = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(1), paging_spec=PagingSpec.equal_pages_up_to(CHUNK_N))
    a_data, a_files, a_index = standalone.compress_files(nums.view(torch.uint64), np.array([n], np.uint64), cfg1)
    b_data, b_files, b_index = standalone.compress_files(col_b.view(torch.uint64), np.array([n], np.uint64), cfg1)
    torch.cuda.synchronize()
    ref_of = lambda f: torch.as_tensor(np.stack([f["offset"], f["len"], f["index_offset"], f["index_len"]], axis=1).astype(np.int64), device=dev)  # noqa: E731
    a_refs, b_refs = ref_of(a_files), ref_of(b_files)
    one = torch.ones(1, dtype=torch.int64, device=dev)
    flt = standalone.AsyncFilesFilter(a_data[:32], np.uint64, a_data.numel(), a_index.numel(), 1, args.chunks, n, n)
    tk = standalone.AsyncFilesTake(b_data[:32], np.uint64, b_data.numel(), b_index.numel(), 1, args.chunks, n, n)
    iv = torch.zeros(2, dtype=torch.int64, device=dev)
    a_vals = torch.empty(n, dtype=torch.int64, device=dev)
    nm = torch.zeros(1, dtype=torch.int64, device=dev)

    def both():
        flt(a_data, a_index, a_refs, one, iv, a_vals.view(torch.uint64), d_pos, nm)
        tk(b_data, b_index, b_refs, one, d_pos, nm, out.view(torch.uint64))

    srt = torch.sort(nums)[0]
    g_both = capture(both)
    gleg = {}
    ok_g = True
    for s in (0.001, 0.01):
        kw = int(s * n)
        a0 = n // 2 - kw // 2
        lo, hi = int(srt[a0]), int(srt[a0 + kw - 1])
        iv.copy_(torch.tensor([lo, hi], dtype=torch.int64))
        t = {"graph_ms": events(g_both.replay)}
        want = col_b[(nums >= lo) & (nums <= hi)]
        k = int(want.numel())
        t["positions"] = k
        t["records_decoded"] = int(tk.status_record().records_decoded)
        t["parity"] = bool(flt.result() == k and tk.result() == k and torch.equal(out[:k], want))
        ok_g = ok_g and t["parity"]
        gleg[f"sel_{s * 100:g}%"] = t
    res["filter_then_take"] = gleg
    parity["filter_then_take"] = ok_g
    print(json.dumps({"workload": f"C2: {args.chunks} chunks x 2^18 u64 (one indexed file at order 1 and 0, {n >> 16} files of 2^16, "
                                  f"{args.chunks} wrapped pages), take at device positions, device buffers",
                      "gpu": gpu_description(), "steps": steps, "results": res, "parity": parity}))


if __name__ == "__main__":
    main()
