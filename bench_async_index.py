#!/usr/bin/env python
"""bench_async_index.py — the side index of a standalone file without one, built on the caller's stream (pco_b200_build_index_async)
against the blocking pco_b200_build_index.

Legs (every buffer in HBM; every leg checks parity and reports it):
  - "bench": bench.py's array (--chunks chunks of 2^18 u64, C2 data, chunk c = datagen.c2_u64_cumsum_geometric(seed = c)), classic mode,
    consecutive delta order 1, as a file without an index: async_ms (CUDA events around one call), graph_ms (one replay of the call
    captured once), enqueue_us (host time of the call's enqueue), kernel_ms (per-kernel split of one profiled call); parity: the built
    index equals, byte for byte, the index pco_b200_compress_ex writes for the same file;
  - "build_index_scaled": the blocking pco_b200_build_index on a file of the first --prefix chunks (host clock around the call, which
    waits for its serial walk), and that time scaled by chunks / prefix - an estimate for the whole file, not a measurement of it;
  - "graph_vs_decompress_ex": a graph of "build index + pco_b200_decompress_async" replayed, against pco_b200_decompress_ex without an
    index (its speculative index-free walk); parity: both outputs equal the input;
  - "level12": 64 chunks of 2^16 lognormal u64 at compression level 12 (tables of up to 2^12 states): async_ms, serial_chunks, parity;
  - "exact_alternating": 256 chunks of Exact pages alternating 2^16 and 2^16 - 1000 numbers, the worst case for the serial walker (a
    round takes one chunk only): async_ms of one call, serial_chunks, parity.
Prints one JSON line with the card's name, power limit and SM clock; writes nothing.

    python bench_async_index.py [--steps 10] [--chunks 1024] [--prefix 8]
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
    ap.add_argument("--chunks", type=int, default=1024)
    ap.add_argument("--prefix", type=int, default=8)
    args = ap.parse_args()

    import torch

    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec, _lib, datagen, standalone

    L = _lib.lib()
    if not L.pco_b200_device_available():
        raise RuntimeError("libcpcodec.so found no usable CUDA device: " + L.pco_b200_last_error_message().decode())
    dev = torch.device("cuda", 0)
    steps = max(args.steps, 1)

    def events(fn, reps=steps):
        stream = torch.cuda.current_stream()
        fn()
        torch.cuda.synchronize()
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
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

    def u8(b):
        return torch.as_tensor(np.frombuffer(b, np.uint8).copy(), device=dev)

    class Leg:
        """One file on the device, an index builder for it and its buffers."""

        def __init__(self, data, dtype, max_chunks, index_cap):
            self.data, self.d_src = data, u8(data)
            self.d_len = torch.tensor([len(data)], dtype=torch.int64, device=dev)
            self.d_idx = torch.zeros(index_cap, dtype=torch.uint8, device=dev)
            self.b = standalone.AsyncIndexBuilder(data[:32], dtype, len(data), index_cap, max_chunks)

        def call(self):
            self.b(self.d_src, self.d_len, self.d_idx)

        def index(self):
            n = self.b.result()
            return self.d_idx[:n].cpu().numpy().tobytes()

    res, parity = {}, {}
    cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(1))
    n = args.chunks * CHUNK_N
    h_np = np.empty(n, dtype=np.uint64)
    for c in range(args.chunks):
        h_np[c * CHUNK_N:(c + 1) * CHUNK_N] = datagen.c2_u64_cumsum_geometric(CHUNK_N, seed=c)
    data, want_index = standalone.simple_compress_with_index(h_np, cfg)

    # ---- bench.py's array as a file without an index
    leg = Leg(data, np.uint64, args.chunks, len(want_index) + 4096)
    t = {"chunks": args.chunks, "compressed_bytes": len(data), "index_bytes": len(want_index), "workspace_bytes": leg.b.workspace_bytes}
    t["async_ms"] = events(leg.call)
    ok_async = leg.index() == want_index
    t["serial_chunks"] = int(leg.b.status_record().serial_chunks)
    g = capture(leg.call)
    leg.d_idx.zero_()
    t["graph_ms"] = events(g.replay)
    ok_graph = leg.index() == want_index
    enq = []
    for _ in range(steps):
        t0 = time.perf_counter()
        leg.call()
        enq.append(time.perf_counter() - t0)
        torch.cuda.synchronize()
    t["enqueue_us"] = float(np.median(enq) * 1e6)
    L.pco_b200_profile_enable(1)
    leg.call()
    t["kernel_ms"] = parse_profile(L)
    L.pco_b200_profile_enable(0)
    parity["bench"] = bool(ok_async and ok_graph)
    res["bench"] = t
    del g

    # ---- the blocking build_index on a prefix, scaled
    p = min(args.prefix, args.chunks)
    pdata, pindex = standalone.simple_compress_with_index(h_np[: p * CHUNK_N], cfg)
    d_p = u8(pdata)
    idx = np.zeros(len(pindex) + (1 << 20), np.uint8)
    il = C.c_size_t()

    def blocking():
        _lib.check(L.pco_b200_build_index(C.c_void_p(d_p.data_ptr()), C.c_size_t(len(pdata)), C.c_ubyte(2), idx.ctypes.data_as(C.c_void_p),
                                          C.c_size_t(idx.size), C.byref(il), C.c_uint32(1), C.c_void_p(torch.cuda.current_stream().cuda_stream)))

    blocking()
    times = []
    for _ in range(3):
        t0 = time.perf_counter()
        blocking()
        times.append((time.perf_counter() - t0) * 1e3)
    pleg = Leg(pdata, np.uint64, p, len(pindex) + 4096)
    pleg.call()
    ok_prefix = pleg.index() == pindex and il.value >= len(pindex)
    res["build_index_scaled"] = {"prefix_chunks": p, "prefix_ms": float(np.median(times)), "prefix_async_ms": events(pleg.call, 3),
                                 "scaled_ms_estimate": float(np.median(times)) * args.chunks / p,
                                 "note": "prefix time x chunks / prefix_chunks: an estimate for the whole file, not measured on it"}
    parity["build_index_prefix"] = bool(ok_prefix)

    # ---- graph of build + decompress_async against decompress_ex without an index
    dec = standalone.AsyncDecompressor(data[:32], np.uint64, len(data), leg.d_idx.numel(), n, args.chunks)
    d_out = torch.zeros(n, dtype=torch.int64, device=dev)
    d_ex = torch.zeros(n, dtype=torch.int64, device=dev)

    def both():
        leg.call()
        dec(leg.d_src, leg.d_idx, d_out.view(torch.uint64))

    def ex():
        prog = _lib._CProgress()
        _lib.check(L.pco_b200_decompress_ex(C.c_void_p(leg.d_src.data_ptr()), C.c_size_t(len(data)), C.c_ubyte(2), C.c_void_p(d_ex.data_ptr()),
                                            C.c_size_t(n), C.byref(prog), None, C.c_size_t(0), C.c_uint32(3),
                                            C.c_void_p(torch.cuda.current_stream().cuda_stream)))

    g = capture(both)
    nums = torch.from_numpy(h_np.view(np.int64)).to(dev)
    d_out.zero_()
    gv = {"graph_build_and_decode_ms": events(g.replay)}
    ok_g = dec.result().n_processed == n and torch.equal(d_out, nums)
    gv["decompress_ex_no_index_ms"] = events(ex)
    ok_ex = torch.equal(d_ex, nums)
    res["graph_vs_decompress_ex"] = gv
    parity["graph_vs_decompress_ex"] = bool(ok_g and ok_ex)
    del g, dec, d_out, d_ex, nums

    # ---- level 12 and the alternating Exact pages
    rng = np.random.default_rng(12)
    x12 = rng.lognormal(10, 2, size=64 << 16).astype(np.uint64)
    d12, i12 = standalone.simple_compress_with_index(x12, ChunkConfig(compression_level=12, mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.no_op(),
                                                                      paging_spec=PagingSpec.equal_pages_up_to(1 << 16)))
    l12 = Leg(d12, np.uint64, 64, len(i12) + 4096)
    t12 = {"chunks": 64, "async_ms": events(l12.call, 3)}
    parity["level12"] = l12.index() == i12
    t12["serial_chunks"] = int(l12.b.status_record().serial_chunks)
    res["level12"] = t12
    sizes = [(1 << 16) - (1000 if i % 2 else 0) for i in range(256)]
    xa = datagen.c2_u64_cumsum_geometric(sum(sizes), seed=12345)  # this leg's own data, whatever --chunks is
    da, ia = standalone.simple_compress_with_index(xa, ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(1),
                                                                   paging_spec=PagingSpec.exact_page_sizes(sizes)))
    la = Leg(da, np.uint64, len(sizes), len(ia) + 4096)
    ta = {"chunks": len(sizes), "async_ms": events(la.call, 1)}
    parity["exact_alternating"] = la.index() == ia
    ta["serial_chunks"] = int(la.b.status_record().serial_chunks)
    res["exact_alternating"] = ta

    res["parity"] = {"all": all(parity.values()), **parity}
    print(json.dumps({"workload": f"C2: {args.chunks} chunks x 2^18 u64, classic mode, order 1, as a standalone file without an index, device buffers",
                      "unit": "ms per call (enqueue: us)", "steps": steps, "gpu": gpu_description(), **res}))


if __name__ == "__main__":
    main()
