#!/usr/bin/env python
"""bench_async_files.py — a batch of indexed standalone files on the caller's stream (pco_b200_decompress_files_async) against the
blocking call (pco_b200_decompress_files).

Files: bench_files.py's two cuts of bench.py's array (1024 chunks of 2^18 u64, C2 data, chunk c = datagen.c2_u64_cumsum_geometric(seed =
c)), classic mode, consecutive delta order 1, written by pco_b200_compress_files with side indexes, every buffer in HBM:
  - "uniform": 4096 files of 2^16 numbers;  - "lognormal": bench_files.py's seeded lognormal sizes (1706 files).
Per cut, every file once in order:
  - sync_ms: the blocking call, refs in host memory (CUDA events around each call);
  - async_ms: one async call (CUDA events), graph_ms: one replay of the call captured once (CUDA events);
  - enqueue_us: host time of the async call's enqueue (the call returns without waiting);
  - kernel_ms: per-kernel split of one profiled async call outside the capture;
  - parity: the sync call, the async call and the replay equal the input, file_ns included.
loader: 256 of the 4096 uniform files, picked each step on the device by a torch gather of seeded random ids into the refs; the graph
(gather + decode) replayed against a step that copies the same refs to the host and makes the blocking call (wall time per step over
`--steps` steps, one synchronisation per step for both).  Prints one JSON line; writes nothing.

    python bench_async_files.py [--steps 20] [--chunks 1024]
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

from bench_files import file_sizes  # noqa: E402
from bench_levels import CHUNK_N, gpu_description, parse_profile  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--chunks", type=int, default=1024)
    args = ap.parse_args()

    import torch

    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, _lib, datagen, standalone

    L = standalone._lib_files()
    if not L.pco_b200_device_available():
        raise RuntimeError("libcpcodec.so found no usable CUDA device: " + L.pco_b200_last_error_message().decode())
    dev = torch.device("cuda", 0)
    SRC, DST, IDX = 1, 2, 4
    steps = max(args.steps, 1)
    n = args.chunks * CHUNK_N
    h_np = np.empty(n, dtype=np.uint64)
    for c in range(args.chunks):
        h_np[c * CHUNK_N:(c + 1) * CHUNK_N] = datagen.c2_u64_cumsum_geometric(CHUNK_N, seed=c)
    nums = torch.from_numpy(h_np.view(np.int64)).to(dev)
    cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(1))

    def refs_of(files):
        return np.stack([files["offset"], files["len"], files["index_offset"], files["index_len"]], axis=1).astype(np.uint64)

    def sync_call(d_data, d_index, refs, d_out, h_ns):
        r = np.zeros(len(refs), dtype=standalone.FILE_REF)
        r["offset"], r["len"], r["index_offset"], r["index_len"] = refs[:, 0], refs[:, 1], refs[:, 2], refs[:, 3]
        nw = C.c_size_t()
        _lib.check(L.pco_b200_decompress_files(C.c_void_p(d_data.data_ptr()), C.c_size_t(d_data.numel()), C.c_void_p(d_index.data_ptr()),
                                               C.c_size_t(d_index.numel()), C.c_ubyte(2), r.ctypes.data_as(C.c_void_p), C.c_size_t(len(refs)),
                                               C.c_void_p(d_out.data_ptr()), C.c_size_t(d_out.numel()), h_ns.ctypes.data_as(C.c_void_p), C.byref(nw),
                                               C.c_uint32(SRC | DST | IDX), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
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

    res, parity = {}, {}
    cuts = {}
    for cut in ("uniform", "lognormal"):
        sizes = file_sizes(cut, n)
        d_data, files, d_index = standalone.compress_files(nums.view(torch.uint64), sizes, cfg)
        torch.cuda.synchronize()
        refs = refs_of(files)
        cuts[cut] = (d_data, d_index, refs, sizes)
        nf = len(refs)
        n_chunks = int(sum(-(-int(s) // CHUNK_N) for s in sizes))
        dec = standalone.AsyncFilesDecompressor(d_data[int(refs[0, 0]):int(refs[0, 0]) + 32], np.uint64, d_data.numel(), d_index.numel(), nf, n_chunks, n)
        d_files = torch.as_tensor(refs.view(np.int64), device=dev)
        d_n = torch.tensor([nf], dtype=torch.int64, device=dev)
        d_out = torch.empty(n, dtype=torch.int64, device=dev)
        d_ns = torch.zeros(nf, dtype=torch.int64, device=dev)
        d_sync = torch.empty(n, dtype=torch.int64, device=dev)
        h_ns = np.zeros(nf, np.uint64)
        call = lambda: dec(d_data, d_index, d_files, d_n, d_out.view(torch.uint64), d_ns)  # noqa: E731
        t = {"files": nf, "chunks": n_chunks, "compressed_bytes": int(d_data.numel()), "index_bytes": int(d_index.numel()),
             "workspace_bytes": dec.workspace_bytes}
        t["sync_ms"] = events(lambda: sync_call(d_data, d_index, refs, d_sync, h_ns))
        ok_sync = torch.equal(d_sync, nums) and (h_ns == sizes).all()
        t["async_ms"] = events(call)
        ok_async = dec.result() == n and torch.equal(d_out, nums) and (d_ns.cpu().numpy() == sizes.astype(np.int64)).all()
        g = capture(call)
        d_out.fill_(0)
        d_ns.fill_(0)
        t["graph_ms"] = events(g.replay)
        ok_graph = dec.result() == n and torch.equal(d_out, nums) and (d_ns.cpu().numpy() == sizes.astype(np.int64)).all()
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
        parity[cut] = bool(ok_sync and ok_async and ok_graph)
        res[cut] = t
        del dec, d_out, d_sync, g
        torch.cuda.synchronize()

    # ---- loader: 256 uniform files picked on the device each step
    d_data, d_index, refs, sizes = cuts["uniform"]
    pick_n, fn = 256, 1 << 16
    dec = standalone.AsyncFilesDecompressor(d_data[:32], np.uint64, d_data.numel(), d_index.numel(), pick_n, pick_n, pick_n * fn)
    all_refs = torch.as_tensor(refs.view(np.int64), device=dev)
    d_pick = torch.zeros(pick_n, dtype=torch.int64, device=dev)
    d_files = torch.zeros((pick_n, 4), dtype=torch.int64, device=dev)
    d_n = torch.tensor([pick_n], dtype=torch.int64, device=dev)
    d_out = torch.empty(pick_n * fn, dtype=torch.int64, device=dev)
    d_ns = torch.zeros(pick_n, dtype=torch.int64, device=dev)
    d_sync = torch.empty(pick_n * fn, dtype=torch.int64, device=dev)
    h_ns = np.zeros(pick_n, np.uint64)

    def loader_step():
        torch.index_select(all_refs, 0, d_pick, out=d_files)
        dec(d_data, d_index, d_files, d_n, d_out.view(torch.uint64), d_ns)

    g = capture(loader_step)
    rng = np.random.default_rng(0)
    picks = [torch.as_tensor(rng.integers(0, len(refs), pick_n), device=dev) for _ in range(steps)]

    def run_graph():
        t0 = time.perf_counter()
        for p in picks:
            d_pick.copy_(p)
            g.replay()
            torch.cuda.synchronize()
        return (time.perf_counter() - t0) / steps * 1e3

    def run_sync():
        t0 = time.perf_counter()
        for p in picks:
            d_pick.copy_(p)
            h_refs = torch.index_select(all_refs, 0, d_pick).cpu().numpy().view(np.uint64)  # the refs go through the host
            sync_call(d_data, d_index, h_refs, d_sync, h_ns)
            torch.cuda.synchronize()
        return (time.perf_counter() - t0) / steps * 1e3

    run_graph()
    run_sync()  # warm both
    loader = {"files_per_step": pick_n, "numbers_per_step": pick_n * fn, "graph_wall_ms": run_graph(), "sync_wall_ms": run_sync()}
    # parity on the last step's pick: both against the input
    last = picks[-1].cpu().numpy()
    want = torch.cat([nums[int(i) * fn:(int(i) + 1) * fn] for i in last])
    ok = dec.result() == pick_n * fn and torch.equal(d_out, want) and torch.equal(d_sync, want) and (d_ns.cpu().numpy() == fn).all()
    parity["loader"] = bool(ok)
    res["loader"] = loader
    res["parity"] = {"all": all(parity.values()), **parity}
    print(json.dumps({"workload": f"C2: {args.chunks} chunks x 2^18 u64 cut into files (uniform 2^16, lognormal), classic mode, order 1, side indexes "
                                  "from compress_files, device buffers; loader: 256 of the uniform files picked on the device per step",
                      "unit": "ms per call (enqueue: us; loader: wall ms per step)", "steps": steps, "gpu": gpu_description(), **res}))


if __name__ == "__main__":
    main()
