#!/usr/bin/env python
"""bench_async_pages.py — a batch of wrapped-format pages on the caller's stream (pco_b200_decompress_pages_async) against the blocking
call (pco_b200_decompress_pages).

Pages: bench.py's array (1024 chunks of 2^18 u64, C2 data, chunk c = datagen.c2_u64_cumsum_geometric(seed = c)) written by
wrapped.compress_chunks as 1024 wrapped chunks of one page each (classic mode, consecutive delta order 1), every buffer in HBM.
  - full: every page once in order.  sync_ms: the blocking call, refs in host memory; async_ms: one async call; graph_ms: one replay of the
    call captured once (CUDA events around each); enqueue_us: host time of the async call's enqueue; kernel_ms: per-kernel split of one
    profiled async call; parity: all three equal the input.
  - small: 64 pages of 2^13 numbers (the first 2^13 numbers of the first 64 chunks).  Wall time per call over `--steps` calls: the blocking
    call in a loop, back-to-back async calls, back-to-back graph replays (one synchronisation at the end for the last two).
  - pruned: a scan that keeps the pages whose stored max lies in a query range (a quarter of the pages' maxima, at a random quantile).
    A torch kernel tests the stats, compacts the kept refs and writes their count on the device, and the graph (predicate + decode) is replayed; against copying the mask to the host and
    making the blocking call.  Wall time per step, one synchronisation per step for both; parity against the input.
Prints one JSON line; writes nothing.

    python bench_async_pages.py [--steps 20] [--chunks 1024]
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
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--chunks", type=int, default=1024)
    args = ap.parse_args()

    import torch

    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec, _lib, datagen, wrapped

    L = wrapped._lib_batch()
    wrapped._lib_async_pages()
    if not L.pco_b200_device_available():
        raise RuntimeError("libcpcodec.so found no usable CUDA device: " + L.pco_b200_last_error_message().decode())
    dev = torch.device("cuda", 0)
    SRC, DST = 1, 2
    steps = max(args.steps, 1)
    n = args.chunks * CHUNK_N
    h_np = np.empty(n, dtype=np.uint64)
    for c in range(args.chunks):
        h_np[c * CHUNK_N:(c + 1) * CHUNK_N] = datagen.c2_u64_cumsum_geometric(CHUNK_N, seed=c)
    nums = torch.from_numpy(h_np.view(np.int64)).to(dev)

    def sync_call(d_metas, d_pages, refs, d_out):
        r = np.ascontiguousarray(refs.astype(wrapped.PAGE_REF))
        nw = C.c_size_t()
        _lib.check(L.pco_b200_decompress_pages(C.c_void_p(d_metas.data_ptr()), C.c_size_t(d_metas.numel()), C.c_void_p(d_pages.data_ptr()),
                                               C.c_size_t(d_pages.numel()), C.c_ubyte(2), r.ctypes.data_as(C.c_void_p), C.c_size_t(len(r)),
                                               C.c_void_p(d_out.data_ptr()), C.c_size_t(d_out.numel()), C.byref(nw), C.c_uint32(SRC | DST),
                                               C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        return nw.value

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

    def wall(fn, sync_each):
        fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            fn()
            if sync_each:
                torch.cuda.synchronize()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / steps * 1e3

    def refs_tensor(refs, rows):
        t = torch.zeros((rows, 5), dtype=torch.int64)
        t[: len(refs)] = torch.from_numpy(np.stack([refs[f].astype(np.int64) for f in wrapped.PAGE_REF.names], axis=1))
        return t.to(dev)

    res, parity = {}, {}
    cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(1), paging_spec=PagingSpec.equal_pages_up_to(CHUNK_N))

    # ---- full: bench.py's array as wrapped pages
    metas, pages, refs = wrapped.compress_chunks(nums.view(torch.uint64), cfg)
    torch.cuda.synchronize()
    npg = len(refs)
    dec = wrapped.AsyncPagesDecompressor(np.uint64, metas.numel(), pages.numel(), npg, n)
    d_refs = refs_tensor(refs, npg)
    d_n = torch.tensor([npg], dtype=torch.int64, device=dev)
    d_out = torch.empty(n, dtype=torch.int64, device=dev)
    d_sync = torch.empty(n, dtype=torch.int64, device=dev)
    call = lambda: dec(metas, pages, d_refs, d_n, d_out.view(torch.uint64))  # noqa: E731
    t = {"pages": npg, "metas_bytes": int(metas.numel()), "pages_bytes": int(pages.numel()), "workspace_bytes": dec.workspace_bytes}
    t["sync_ms"] = events(lambda: sync_call(metas, pages, refs, d_sync))
    ok_sync = torch.equal(d_sync, nums)
    t["async_ms"] = events(call)
    ok_async = dec.result() == n and torch.equal(d_out, nums)
    g = capture(call)
    d_out.fill_(0)
    t["graph_ms"] = events(g.replay)
    ok_graph = dec.result() == n and torch.equal(d_out, nums)
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
    t["kernel_ms"] = parse_profile(L)
    L.pco_b200_profile_enable(0)
    parity["full"] = bool(ok_sync and ok_async and ok_graph)
    res["full"] = t
    del g, d_sync
    torch.cuda.synchronize()

    # ---- small: 64 pages of 2^13 numbers
    sn, sp = 1 << 13, 64
    small = torch.cat([nums[c * CHUNK_N:c * CHUNK_N + sn] for c in range(sp)])
    s_metas, s_pages, s_refs = wrapped.compress_chunks(small.view(torch.uint64), ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(1),
                                                                                             paging_spec=PagingSpec.equal_pages_up_to(sn)))
    s_dec = wrapped.AsyncPagesDecompressor(np.uint64, s_metas.numel(), s_pages.numel(), sp, sp * sn)
    s_drefs = refs_tensor(s_refs, sp)
    s_n = torch.tensor([sp], dtype=torch.int64, device=dev)
    s_out = torch.empty(sp * sn, dtype=torch.int64, device=dev)
    s_sync = torch.empty(sp * sn, dtype=torch.int64, device=dev)
    s_call = lambda: s_dec(s_metas, s_pages, s_drefs, s_n, s_out.view(torch.uint64))  # noqa: E731
    sm = {"pages": sp, "page_n": sn}
    sm["sync_wall_ms"] = wall(lambda: sync_call(s_metas, s_pages, s_refs, s_sync), True)
    sm["async_wall_ms"] = wall(s_call, False)
    ok_async = s_dec.result() == sp * sn and torch.equal(s_out, small)
    g = capture(s_call)
    s_out.fill_(0)
    sm["graph_wall_ms"] = wall(g.replay, False)
    parity["small"] = bool(torch.equal(s_sync, small) and ok_async and s_dec.result() == sp * sn and torch.equal(s_out, small))
    res["small"] = sm
    del g, s_dec
    torch.cuda.synchronize()

    # ---- pruned: keep the pages whose max lies in a query range, decided on the device
    maxs = nums.view(npg, CHUNK_N).max(dim=1).values
    all_refs = refs_tensor(refs, npg)
    rng = np.random.default_rng(0)
    sorted_max = np.sort(maxs.cpu().numpy())
    lo_hi = []
    for _ in range(steps):
        q = int(rng.integers(0, npg - npg // 4))
        lo_hi.append((int(sorted_max[q]), int(sorted_max[q + npg // 4 - 1])))
    d_q = torch.zeros(2, dtype=torch.int64, device=dev)
    buf = torch.zeros((npg + 1, 5), dtype=torch.int64, device=dev)  # row npg takes the pages not kept
    p_refs = buf[:npg]
    p_n = torch.zeros(1, dtype=torch.int64, device=dev)
    p_out = torch.empty(n, dtype=torch.int64, device=dev)
    p_sync = torch.empty(n, dtype=torch.int64, device=dev)

    def prune_step():
        keep = (maxs >= d_q[0]) & (maxs <= d_q[1])
        pos = torch.where(keep, torch.cumsum(keep, 0) - 1, torch.full_like(maxs, npg))
        buf.index_copy_(0, pos, all_refs)
        p_n.copy_(keep.sum().reshape(1))
        dec(metas, pages, p_refs, p_n, p_out.view(torch.uint64))

    g = capture(prune_step)

    def run_graph():
        t0 = time.perf_counter()
        for a, b in lo_hi:
            d_q.copy_(torch.tensor([a, b], dtype=torch.int64), non_blocking=False)
            g.replay()
            torch.cuda.synchronize()
        return (time.perf_counter() - t0) / steps * 1e3

    def run_sync():
        t0 = time.perf_counter()
        for a, b in lo_hi:
            d_q.copy_(torch.tensor([a, b], dtype=torch.int64), non_blocking=False)
            keep = ((maxs >= d_q[0]) & (maxs <= d_q[1])).cpu().numpy()  # the mask goes through the host
            sync_call(metas, pages, refs[keep], p_sync)
            torch.cuda.synchronize()
        return (time.perf_counter() - t0) / steps * 1e3

    run_graph()
    run_sync()  # warm both
    pr = {"graph_wall_ms": run_graph(), "sync_wall_ms": run_sync()}
    keep = ((maxs >= lo_hi[-1][0]) & (maxs <= lo_hi[-1][1])).cpu().numpy()
    kept = np.nonzero(keep)[0]
    want = torch.cat([nums[int(i) * CHUNK_N:(int(i) + 1) * CHUNK_N] for i in kept]) if kept.size else nums[:0]
    m = want.numel()
    pr["pages_kept_last_step"] = int(kept.size)
    parity["pruned"] = bool(dec.result() == m and torch.equal(p_out[:m], want) and torch.equal(p_sync[:m], want))
    res["pruned"] = pr
    res["parity"] = {"all": all(parity.values()), **parity}
    print(json.dumps({"workload": f"C2: {args.chunks} chunks x 2^18 u64 as wrapped pages from compress_chunks, classic mode, order 1, device buffers; "
                                  "small: 64 pages of 2^13; pruned: a quarter of the pages, by their max, picked on the device",
                      "unit": "ms per call (enqueue: us; small and pruned: wall ms per call or step)", "steps": steps, "gpu": gpu_description(), **res}))


if __name__ == "__main__":
    main()
