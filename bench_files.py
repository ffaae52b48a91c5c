#!/usr/bin/env python
"""bench_files.py — the batched standalone-file calls against a loop of the one-file calls on the same files.

The array of bench.py (1024 chunks of 2^18 u64, C2 data, chunk c = datagen.c2_u64_cumsum_geometric(seed = c)), classic mode, consecutive
delta order 1, every buffer in HBM, cut into files two ways:
  - "uniform": 4096 files of 2^16 numbers;
  - "lognormal": seeded lognormal sizes (median 2^16) clipped to [1, 2^20], the last file taking what is left.
For each cut:
  - compress: pco_b200_compress_files (files + side indexes) against one pco_b200_compress_ex per file;
  - decompress: pco_b200_decompress_files with the side indexes and without them, against one pco_b200_decompress_ex per file each way.
One warm-up call each, then `--steps` batch calls and `--loop-steps` loops timed with CUDA events, with the per-kernel split the
library's profiler reports for the batch calls, and how many times the index-free batch launched walk_kernel.
`parity`: a seeded sample of files against oracle.simple_compress bytes, and the full decode (both ways) against the input.
Prints one JSON line; writes nothing.

    python bench_files.py [--steps 5] [--loop-steps 1] [--chunks 1024]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_levels import CHUNK_N, gpu_description, parse_profile  # noqa: E402


def file_sizes(kind, n, seed=1):
    if kind == "uniform":
        return np.full(n >> 16, 1 << 16, dtype=np.uint64)
    rng = np.random.default_rng(seed)
    out, left = [], n
    while left > 0:
        s = int(np.clip(rng.lognormal(np.log(1 << 16), 1.5), 1, 1 << 20))
        out.append(min(s, left))
        left -= out[-1]
    return np.array(out, dtype=np.uint64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--loop-steps", type=int, default=1)
    ap.add_argument("--chunks", type=int, default=1024)
    args = ap.parse_args()

    import torch

    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, _lib, datagen, standalone

    L = standalone._lib_files()
    if not L.pco_b200_device_available():
        raise RuntimeError("libcpcodec.so found no usable CUDA device: " + L.pco_b200_last_error_message().decode())
    dev = torch.device("cuda", 0)
    n = args.chunks * CHUNK_N
    U = n * 8
    h_np = np.empty(n, dtype=np.uint64)
    for c in range(args.chunks):
        h_np[c * CHUNK_N:(c + 1) * CHUNK_N] = datagen.c2_u64_cumsum_geometric(CHUNK_N, seed=c)
    nums = torch.from_numpy(h_np.view(np.int64)).to(dev)
    cfg_py = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(1))
    cfg = cfg_py._to_c()
    stream = torch.cuda.current_stream()
    sp = C.c_void_p(stream.cuda_stream)
    SRC, DST, IDX = 1, 2, 4
    d_out = torch.empty(n, dtype=torch.int64, device=dev)
    written, ilen = C.c_size_t(), C.c_size_t()

    def timed(fn, steps, profile=True):
        fn()  # warm-up (modules, scratch)
        torch.cuda.synchronize()
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(max(steps, 1))]
        profs = []
        L.pco_b200_profile_enable(1 if profile else 0)
        for a, b in evs:
            a.record(stream)
            fn()
            b.record(stream)
            if profile:
                profs.append(parse_profile(L))
        L.pco_b200_profile_enable(0)
        torch.cuda.synchronize()
        ms = [a.elapsed_time(b) for a, b in evs]
        spans = {}
        for p in profs:
            for k, v in p.items():
                spans.setdefault(k, []).append(v)
        m = float(np.mean(ms))
        out = {"ms": m, "ms_min": float(np.min(ms)), "ms_max": float(np.max(ms)), "gb_s": U / 1e9 / (m / 1e3)}
        if profile:
            out["kernel_ms"] = {k: float(np.mean(v)) for k, v in spans.items()}
        return out

    results = {}
    for kind in ("uniform", "lognormal"):
        ns = file_sizes(kind, n)
        nf = len(ns)
        at = np.concatenate([[0], np.cumsum(ns)]).astype(np.int64)
        cap = sum(L.pco_standalone_guarantee_file_size(int(k), 2) for k in ns)
        icap = sum(L.pco_b200_index_size_bound(int(k), -(-int(k) // CHUNK_N)) + 16 for k in ns)
        d_data = torch.empty(cap, dtype=torch.uint8, device=dev)
        d_index = torch.empty(icap, dtype=torch.uint8, device=dev)
        files = np.zeros(nf, dtype=standalone.FILE_REF)
        files_p = files.ctypes.data_as(C.c_void_p)
        ns_p = ns.ctypes.data_as(C.c_void_p)
        file_ns = np.zeros(nf, dtype=np.uint64)
        nw = C.c_size_t()

        def compress_files():
            _lib.check(L.pco_b200_compress_files(C.c_void_p(nums.data_ptr()), ns_p, C.c_size_t(nf), C.c_ubyte(2), C.byref(cfg), C.c_int(0),
                                                 C.c_void_p(d_data.data_ptr()), C.c_size_t(cap), C.c_void_p(d_index.data_ptr()), C.c_size_t(icap), files_p,
                                                 C.c_uint32(SRC | DST | IDX), sp))

        loop_data = torch.empty(cap, dtype=torch.uint8, device=dev)
        loop_index = torch.empty(icap, dtype=torch.uint8, device=dev)

        def compress_loop():
            for i in range(nf):
                f = files[i]
                _lib.check(L.pco_b200_compress_ex(C.c_void_p(nums.data_ptr() + int(at[i]) * 8), C.c_size_t(int(ns[i])), C.c_ubyte(2), C.byref(cfg), C.c_int(0),
                                                  C.c_void_p(loop_data.data_ptr() + int(f["offset"])), C.c_size_t(cap - int(f["offset"])), C.byref(written),
                                                  C.c_void_p(loop_index.data_ptr() + int(f["index_offset"])), C.c_size_t(icap - int(f["index_offset"])), C.byref(ilen),
                                                  C.c_uint32(SRC | DST | IDX), sp))

        no_index = files.copy()

        def decompress_files(with_index):
            refs = files if with_index else no_index
            _lib.check(L.pco_b200_decompress_files(C.c_void_p(d_data.data_ptr()), C.c_size_t(cap), C.c_void_p(d_index.data_ptr()), C.c_size_t(icap),
                                                   C.c_ubyte(2), refs.ctypes.data_as(C.c_void_p), C.c_size_t(nf), C.c_void_p(d_out.data_ptr()), C.c_size_t(n),
                                                   file_ns.ctypes.data_as(C.c_void_p), C.byref(nw), C.c_uint32(SRC | DST | IDX), sp))

        prog = _lib._CProgress()

        def decompress_loop(with_index):
            for i in range(nf):
                f = files[i]
                _lib.check(L.pco_b200_decompress_ex(C.c_void_p(d_data.data_ptr() + int(f["offset"])), C.c_size_t(int(f["len"])), C.c_ubyte(2),
                                                    C.c_void_p(d_out.data_ptr() + int(at[i]) * 8), C.c_size_t(int(ns[i])), C.byref(prog),
                                                    C.c_void_p(d_index.data_ptr() + int(f["index_offset"])) if with_index else None,
                                                    C.c_size_t(int(f["index_len"]) if with_index else 0), C.c_uint32(SRC | DST | IDX), sp))

        r = {"files": nf, "file_n_min": int(ns.min()), "file_n_median": int(np.median(ns)), "file_n_max": int(ns.max())}
        r["compress_files"] = timed(compress_files, args.steps)
        no_index[:] = files
        no_index["index_len"] = 0
        r["compress_ex_loop"] = timed(compress_loop, args.loop_steps, profile=False)
        same = bool(torch.equal(loop_data[: int(files[-1]["offset"] + files[-1]["len"])], d_data[: int(files[-1]["offset"] + files[-1]["len"])]))
        r["decompress_files_index"] = timed(lambda: decompress_files(True), args.steps)
        ok_index = bool(torch.equal(d_out, nums))
        d_out.zero_()
        r["decompress_files_no_index"] = timed(lambda: decompress_files(False), args.steps)
        ok_walk = bool(torch.equal(d_out, nums))
        walk_prof = r["decompress_files_no_index"]
        L.pco_b200_profile_enable(1)
        decompress_files(False)
        buf = C.create_string_buffer(1 << 20)
        L.pco_b200_profile_last(buf, C.c_size_t(len(buf)))
        L.pco_b200_profile_enable(0)
        walk_prof["walk_kernel_launches"] = buf.value.decode().count("walk_kernel=")
        r["decompress_ex_loop_index"] = timed(lambda: decompress_loop(True), args.loop_steps, profile=False)
        r["decompress_ex_loop_no_index"] = timed(lambda: decompress_loop(False), args.loop_steps, profile=False)
        ok_loop = bool(torch.equal(d_out, nums))
        used = int(files[-1]["offset"] + files[-1]["len"])
        r["ratio"] = U / used
        parity = {"files_equal_compress_ex_loop": same, "decoded_equals_input_index": ok_index, "decoded_equals_input_no_index": ok_walk,
                  "loop_decoded_equals_input": ok_loop, "checked_files": 0}
        try:
            from oracle import pyoracle

            h_data = d_data[:used].cpu().numpy()
            ocfg = pyoracle.make_config(mode=pyoracle.MODE_CLASSIC, delta=pyoracle.DELTA_CONSECUTIVE, delta_order=1)
            sample = sorted(set(np.random.default_rng(7).choice(nf, size=min(8, nf), replace=False).tolist()) | {0, nf - 1})
            for i in sample:
                f = files[i]
                want = pyoracle.simple_compress(h_np[at[i]:at[i + 1]], ocfg)
                assert h_data[int(f["offset"]):int(f["offset"] + f["len"])].tobytes() == want, f"file {i} differs from the oracle's"
                parity["checked_files"] += 1
            parity["files"] = sample
            parity["against"] = "oracle/ (C++ restatement of pco 1.0.3), same numbers and ChunkConfig"
        except ImportError as ex:
            parity["error"] = str(ex)
        r["parity"] = parity
        r["speedup_compress"] = r["compress_ex_loop"]["ms"] / r["compress_files"]["ms"]
        r["speedup_decompress_index"] = r["decompress_ex_loop_index"]["ms"] / r["decompress_files_index"]["ms"]
        r["speedup_decompress_no_index"] = r["decompress_ex_loop_no_index"]["ms"] / r["decompress_files_no_index"]["ms"]
        results[kind] = r
    print(json.dumps({"workload": f"C2: {args.chunks} x 2^18 u64 cut into files, classic mode, consecutive delta order 1, device buffers",
                      "unit": "GB/s (10^9 uncompressed bytes)", "steps": args.steps, "loop_steps": args.loop_steps, "gpu": gpu_description(), **results}))


if __name__ == "__main__":
    main()
