#!/usr/bin/env python
"""bench_async_ranges.py — ranges of an indexed standalone file on the caller's stream (pco_b200_decompress_ranges_async) against the
blocking call (pco_b200_decompress_ranges).

Files: those of bench_ranges.py, 1024 chunks of 2^18 u64 (C2 data, chunk c = datagen.c2_u64_cumsum_geometric(seed = c)), classic mode,
written by pco_b200_compress_ex with the side index, every buffer in HBM: order1 (consecutive delta order 1, bench.py's file) and order0
(DeltaSpec NoOp).  Legs, with bench_ranges.py's seeded positions: points_1, points_64, points_4096 (count 1), range_1m (one range of
2^20), ranges_4096 (4096 ranges of 256 to 65,536 numbers).  One AsyncRangeDecompressor per file (max_ranges 4096, window_cap the largest
window a leg needs), one CUDA graph per file captured once: each leg only rewrites the ranges and their count in device memory.
Per leg:
  - sync_ms: the blocking call, ranges in host memory (CUDA events around each call);
  - async_ms: one async call (CUDA events), graph_ms: one replay of the captured call (CUDA events);
  - enqueue_us: host time of the async call's enqueue (the call returns without waiting);
  - kernel_ms: per-kernel split of one profiled async call outside the capture;
  - parity: the async call and the replay equal the sync call and the input.
small: a file of 2^16 u64 (one chunk, order 1), 1 and 64 point lookups: wall time per call of a loop of blocking calls, of back-to-back async
calls and of back-to-back graph replays (one synchronisation at the end of each loop).  Prints one JSON line; writes nothing.

    python bench_async_ranges.py [--steps 20] [--chunks 1024]
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


def window_needed(pairs, chunk_n):
    """The documented window rule for chunks of chunk_n numbers."""
    hi = {}
    for s, c in pairs:
        a = s
        while a < s + c:
            k = a // chunk_n
            b = min(s + c, (k + 1) * chunk_n)
            hi[k] = max(hi.get(k, 0), b - k * chunk_n)
            a = b
    return sum((h + 255) // 256 * 256 for h in hi.values())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--chunks", type=int, default=1024)
    args = ap.parse_args()

    import torch

    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, _lib, datagen, standalone

    L = _lib.lib()
    if not L.pco_b200_device_available():
        raise RuntimeError("libcpcodec.so found no usable CUDA device: " + L.pco_b200_last_error_message().decode())
    dev = torch.device("cuda", 0)
    SRC, DST, IDX = 1, 2, 4
    steps = max(args.steps, 1)

    def compress(nums, n, order, n_chunks):
        ds = DeltaSpec.try_consecutive(1) if order else DeltaSpec.no_op()
        cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=ds)._to_c()
        cap = L.pco_standalone_guarantee_file_size(n, 2)
        icap = L.pco_b200_index_size_bound(n, n_chunks)
        d_file = torch.empty(cap, dtype=torch.uint8, device=dev)
        d_index = torch.empty(icap, dtype=torch.uint8, device=dev)
        written, ilen = C.c_size_t(), C.c_size_t()
        _lib.check(L.pco_b200_compress_ex(C.c_void_p(nums.data_ptr()), C.c_size_t(n), C.c_ubyte(2), C.byref(cfg), C.c_int(0), C.c_void_p(d_file.data_ptr()),
                                          C.c_size_t(cap), C.byref(written), C.c_void_p(d_index.data_ptr()), C.c_size_t(icap), C.byref(ilen),
                                          C.c_uint32(SRC | DST | IDX), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        torch.cuda.synchronize()
        return d_file[: written.value], d_index[: ilen.value]

    def setup(d_file, d_index, n_chunks, max_ranges, dst_cap, window_cap):
        dec = standalone.AsyncRangeDecompressor(d_file[:32], np.uint64, d_file.numel(), d_index.numel(), n_chunks, max_ranges, dst_cap, window_cap)
        d_ranges = torch.zeros((max_ranges, 2), dtype=torch.int64, device=dev)
        d_n = torch.zeros(1, dtype=torch.int64, device=dev)
        d_out = torch.empty(dst_cap, dtype=torch.int64, device=dev)
        call = lambda: dec(d_file, d_index, d_ranges, d_n, d_out.view(torch.uint64))  # noqa: E731
        call()  # warm-up outside the capture
        torch.cuda.synchronize()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side):
            call()
        torch.cuda.synchronize()
        return dec, d_ranges, d_n, d_out, call, g

    def load(d_ranges, d_n, pairs):
        r = np.zeros((d_ranges.shape[0], 2), np.int64)
        r[: len(pairs)] = np.array(pairs, np.int64).reshape(-1, 2)
        d_ranges.copy_(torch.as_tensor(r))
        d_n.fill_(len(pairs))
        torch.cuda.synchronize()

    def sync_call(d_file, d_index, pairs, d_sync):
        r = standalone._ranges_array(pairs)
        nw = C.c_size_t()
        _lib.check(L.pco_b200_decompress_ranges(C.c_void_p(d_file.data_ptr()), C.c_size_t(d_file.numel()), C.c_ubyte(2), C.c_void_p(d_index.data_ptr()),
                                                C.c_size_t(d_index.numel()), r.ctypes.data_as(C.c_void_p), C.c_size_t(r.size), C.c_void_p(d_sync.data_ptr()),
                                                C.c_size_t(d_sync.numel()), C.byref(nw), C.c_uint32(SRC | DST | IDX),
                                                C.c_void_p(torch.cuda.current_stream().cuda_stream)))

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
        ms = [a.elapsed_time(b) for a, b in evs]
        return float(np.median(ms))

    def wall(fn):
        fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / steps * 1e3

    # ---- the two large files
    n_chunks = args.chunks
    n = n_chunks * CHUNK_N
    h_np = np.empty(n, dtype=np.uint64)
    for c in range(n_chunks):
        h_np[c * CHUNK_N:(c + 1) * CHUNK_N] = datagen.c2_u64_cumsum_geometric(CHUNK_N, seed=c)
    nums = torch.from_numpy(h_np.view(np.int64)).to(dev)
    rng = np.random.default_rng(0)  # bench_ranges.py's positions
    legs = {"range_1m": [(int(rng.integers(0, n - (1 << 20))), 1 << 20)]}
    for m in (1, 64, 4096):
        legs[f"points_{m}"] = [(int(s), 1) for s in rng.integers(0, n, m)]
    starts = rng.integers(0, n - 65536, 4096)
    legs["ranges_4096"] = [(int(s), int(c)) for s, c in zip(starts, rng.integers(256, 65537, 4096))]
    max_total = max(sum(c for _, c in v) for v in legs.values())
    window_cap = max(window_needed(v, CHUNK_N) for v in legs.values())

    res, parity = {}, {}
    for name, order in (("order1", 1), ("order0", 0)):
        d_file, d_index = compress(nums, n, order, n_chunks)
        dec, d_ranges, d_n, d_out, call, g = setup(d_file, d_index, n_chunks, 4096, max_total, window_cap)
        d_sync = torch.empty(max_total, dtype=torch.int64, device=dev)
        out = {"compressed_bytes": int(d_file.numel()), "workspace_bytes": dec.workspace_bytes, "window_cap": window_cap}
        for leg, pairs in legs.items():
            total = sum(c for _, c in pairs)
            load(d_ranges, d_n, pairs)
            t = {"numbers": total, "window_needed": window_needed(pairs, CHUNK_N)}
            t["sync_ms"] = events(lambda: sync_call(d_file, d_index, pairs, d_sync[:total]))
            t["async_ms"] = events(call)
            ok_async = dec.result() == total and torch.equal(d_out[:total], d_sync[:total])
            d_out.fill_(0)
            t["graph_ms"] = events(g.replay)
            ok_graph = dec.result() == total and torch.equal(d_out[:total], d_sync[:total])
            torch.cuda.synchronize()
            enq = []
            for _ in range(steps):
                t0 = time.perf_counter()
                call()
                enq.append(time.perf_counter() - t0)
                torch.cuda.synchronize()
            t["enqueue_us"] = float(np.median(enq) * 1e6)
            L.pco_b200_profile_enable(1)
            call()
            t["kernel_ms"] = parse_profile(L)
            L.pco_b200_profile_enable(0)
            want = torch.cat([nums[s:s + c] for s, c in pairs])
            parity[f"{name}.{leg}"] = bool(ok_async and ok_graph and torch.equal(d_sync[:total], want))
            out[leg] = t
        res[name] = out
        del d_file, d_index, dec, d_ranges, d_n, d_out, g, d_sync
        torch.cuda.synchronize()

    # ---- a small file: fixed costs
    sn = 1 << 16
    snums = nums[:sn].clone()
    d_file, d_index = compress(snums, sn, 1, 1)
    srng = np.random.default_rng(1)
    small = {"numbers": sn}
    for m in (1, 64):
        pairs = [(int(s), 1) for s in srng.integers(0, sn, m)]
        dec, d_ranges, d_n, d_out, call, g = setup(d_file, d_index, 1, 64, 64, sn)
        load(d_ranges, d_n, pairs)
        d_sync = torch.empty(m, dtype=torch.int64, device=dev)
        t = {"sync_wall_ms": wall(lambda: sync_call(d_file, d_index, pairs, d_sync)), "async_wall_ms": wall(call), "graph_wall_ms": wall(g.replay)}
        want = torch.cat([snums[s:s + 1] for s, _ in pairs])
        parity[f"small.points_{m}"] = bool(dec.result() == m and torch.equal(d_out[:m], want) and torch.equal(d_sync, want))
        small[f"points_{m}"] = t
    res["small"] = small
    res["parity"] = {"all": all(parity.values()), **parity}
    print(json.dumps({"workload": f"C2: {n_chunks} chunks x 2^18 u64, classic mode, order 1 and order 0 (NoOp), side index from compress_ex, device buffers; "
                                  "small: 2^16 u64, order 1", "unit": "ms per call (enqueue: us)", "steps": steps, "gpu": gpu_description(), **res}))


if __name__ == "__main__":
    main()
