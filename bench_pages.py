#!/usr/bin/env python
"""bench_pages.py — the batched wrapped-format calls against their standalone counterparts on the same data.

The workload of bench.py's resident leg: 1024 chunks of 2^18 u64 (C2 data, chunk c = datagen.c2_u64_cumsum_geometric(seed = c)),
classic mode, consecutive delta order 1, every buffer in HBM.
  - compress: pco_b200_compress_wrapped (metas + pages + refs) against pco_b200_compress_ex with PCO_B200_CHUNKS_ONLY and the side
    index (the same pipeline without the split);
  - decompress: pco_b200_decompress_pages over the 1024 pages against pco_b200_decompress_chunks over the same chunks framed as a
    standalone file;
  - the per-page loop: pco_b200_page_decompress (host buffers, one page per call) over the first 32 pages, scaled to all of them.
One warm-up call each, then `--steps` calls timed with CUDA events, with the per-kernel split the library's profiler reports.
`parity`: six chunks' meta and page bytes against oracle.ChunkCompressor, and the decoded array against the input.
Prints one JSON line; writes nothing.

    python bench_pages.py [--steps 10] [--chunks 1024]
"""
import argparse
import ctypes as C
import json
import os
import struct
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

    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, _lib, datagen, wrapped

    L = wrapped._lib_batch()
    if not L.pco_b200_device_available():
        raise RuntimeError("libcpcodec.so found no usable CUDA device: " + L.pco_b200_last_error_message().decode())
    dev = torch.device("cuda", 0)
    n_chunks = args.chunks
    n = n_chunks * CHUNK_N
    U = n * 8
    h_np = np.empty(n, dtype=np.uint64)
    for c in range(n_chunks):
        h_np[c * CHUNK_N:(c + 1) * CHUNK_N] = datagen.c2_u64_cumsum_geometric(CHUNK_N, seed=c)
    nums = torch.from_numpy(h_np.view(np.int64)).to(dev)
    cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(1))._to_c()
    stream = torch.cuda.current_stream()
    sp = C.c_void_p(stream.cuda_stream)
    SRC, DST, IDX, CHUNKS_ONLY = 1, 2, 4, 8
    cap = L.pco_standalone_guarantee_file_size(n, 2)
    icap = L.pco_b200_index_size_bound(n, n_chunks)
    d_file = torch.empty(cap, dtype=torch.uint8, device=dev)
    d_index = torch.empty(icap, dtype=torch.uint8, device=dev)
    d_metas = torch.empty(n_chunks * 4096 + 64, dtype=torch.uint8, device=dev)
    d_pages = torch.empty(cap, dtype=torch.uint8, device=dev)
    d_out = torch.empty(n, dtype=torch.int64, device=dev)
    refs = np.zeros(n_chunks, dtype=wrapped.PAGE_REF)
    refs_p = refs.ctypes.data_as(C.c_void_p)
    written, ilen, ml, pl, nc, nw = (C.c_size_t() for _ in range(6))

    def compress_wrapped():
        _lib.check(L.pco_b200_compress_wrapped(C.c_void_p(nums.data_ptr()), C.c_size_t(n), C.c_ubyte(2), C.byref(cfg), C.c_void_p(d_metas.data_ptr()),
                                               C.c_size_t(d_metas.numel()), C.byref(ml), C.c_void_p(d_pages.data_ptr()), C.c_size_t(cap), C.byref(pl),
                                               refs_p, C.c_size_t(n_chunks), C.byref(nc), C.c_uint32(SRC | DST), sp))

    def compress_chunks_only():
        _lib.check(L.pco_b200_compress_ex(C.c_void_p(nums.data_ptr()), C.c_size_t(n), C.c_ubyte(2), C.byref(cfg), C.c_int(0), C.c_void_p(d_file.data_ptr()),
                                          C.c_size_t(cap), C.byref(written), C.c_void_p(d_index.data_ptr()), C.c_size_t(icap), C.byref(ilen),
                                          C.c_uint32(SRC | DST | IDX | CHUNKS_ONLY), sp))

    def decompress_pages():
        _lib.check(L.pco_b200_decompress_pages(C.c_void_p(d_metas.data_ptr()), C.c_size_t(ml.value), C.c_void_p(d_pages.data_ptr()), C.c_size_t(pl.value),
                                               C.c_ubyte(2), refs_p, C.c_size_t(n_chunks), C.c_void_p(d_out.data_ptr()), C.c_size_t(n), C.byref(nw),
                                               C.c_uint32(SRC | DST), sp))

    def timed(fn, steps):
        fn()  # warm-up (modules, scratch)
        torch.cuda.synchronize()
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(max(steps, 1))]
        profs = []
        for a, b in evs:
            a.record(stream)
            fn()
            b.record(stream)
            profs.append(parse_profile(L))
        torch.cuda.synchronize()
        ms = [a.elapsed_time(b) for a, b in evs]
        spans = {}
        for p in profs:
            for k, v in p.items():
                spans.setdefault(k, []).append(v)
        m = float(np.mean(ms))
        return {"ms": m, "ms_min": float(np.min(ms)), "ms_max": float(np.max(ms)), "gb_s": U / 1e9 / (m / 1e3),
                "kernel_ms": {k: float(np.mean(v)) for k, v in spans.items()}}

    L.pco_b200_profile_enable(1)
    res = {"compress_wrapped": timed(compress_wrapped, args.steps), "compress_ex_chunks_only": timed(compress_chunks_only, args.steps)}
    # the same chunks as a standalone file, with their offsets from its side index
    _lib.check(L.pco_b200_compress_ex(C.c_void_p(nums.data_ptr()), C.c_size_t(n), C.c_ubyte(2), C.byref(cfg), C.c_int(0), C.c_void_p(d_file.data_ptr()),
                                      C.c_size_t(cap), C.byref(written), C.c_void_p(d_index.data_ptr()), C.c_size_t(icap), C.byref(ilen),
                                      C.c_uint32(SRC | DST | IDX), sp))
    torch.cuda.synchronize()
    ih = bytes(d_index[:64].cpu().numpy())
    n_idx, chunks_off = struct.unpack_from("<Q", ih, 8)[0], struct.unpack_from("<Q", ih, 32)[0]
    recs = bytes(d_index[chunks_off:chunks_off + 32 * n_idx].cpu().numpy())
    offs = (C.c_uint64 * n_idx)(*[struct.unpack_from("<Q", recs, 32 * i)[0] for i in range(n_idx)])
    ns = (C.c_uint32 * n_idx)(*[struct.unpack_from("<I", recs, 32 * i + 8)[0] for i in range(n_idx)])

    def decompress_chunks():
        _lib.check(L.pco_b200_decompress_chunks(C.c_void_p(d_file.data_ptr()), C.c_size_t(written.value), C.c_ubyte(2), offs, ns, C.c_size_t(n_idx),
                                                C.c_void_p(d_out.data_ptr()), C.c_size_t(n), C.byref(nw), C.c_uint32(SRC | DST), sp))

    compress_wrapped()  # the refs and bytes the page decoder reads
    res["decompress_pages"] = timed(decompress_pages, args.steps)
    decoded_ok = bool(torch.equal(d_out, nums))
    res["decompress_chunks"] = timed(decompress_chunks, args.steps)
    L.pco_b200_profile_enable(0)

    # the per-page loop: one pco_b200_page_decompress per page, host buffers
    h_metas, h_pages = d_metas[:ml.value].cpu().numpy(), d_pages[:pl.value].cpu().numpy()
    k = min(32, n_chunks)
    page_dst = np.empty(CHUNK_N, dtype=np.uint64)
    prog, nread = _lib._CProgress(), C.c_size_t()
    L.pco_b200_page_decompress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_ubyte, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]

    def one_page(i):
        r = refs[i]
        _lib.check(L.pco_b200_page_decompress(h_metas.ctypes.data + int(r["meta_offset"]), int(r["meta_len"]), h_pages.ctypes.data + int(r["page_offset"]),
                                              int(r["page_len"]), int(r["page_n"]), 2, page_dst.ctypes.data, page_dst.size, C.byref(prog), C.byref(nread)))

    one_page(0)
    t0 = time.perf_counter()
    for i in range(k):
        one_page(i)
    per_page_ms = (time.perf_counter() - t0) * 1e3 / k
    res["page_decompress_loop"] = {"pages_timed": k, "ms_per_page": per_page_ms, "ms_scaled_to_all_pages": per_page_ms * n_chunks,
                                   "gb_s": U / 1e9 / (per_page_ms * n_chunks / 1e3), "buffers": "host (the call takes host memory only)"}

    parity = {"checked_chunks": 0, "decoded_equals_input": decoded_ok, "against": "oracle/ (C++ restatement of pco 1.0.3), same numbers and ChunkConfig"}
    try:
        from oracle import pyoracle

        sample = sorted({0, 1, n_chunks // 3, n_chunks // 2, n_chunks - 2, n_chunks - 1} & set(range(n_chunks)))
        for c in sample:
            occ = pyoracle.ChunkCompressor(h_np[c * CHUNK_N:(c + 1) * CHUNK_N],
                                           pyoracle.make_config(mode=pyoracle.MODE_CLASSIC, delta=pyoracle.DELTA_CONSECUTIVE, delta_order=1, exact_pages=[CHUNK_N]))
            r = refs[c]
            assert h_metas[r["meta_offset"]:r["meta_offset"] + r["meta_len"]].tobytes() == occ.write_meta(), f"chunk {c}: meta differs from the oracle's"
            assert h_pages[r["page_offset"]:r["page_offset"] + r["page_len"]].tobytes() == occ.write_page(0), f"chunk {c}: page differs from the oracle's"
            parity["checked_chunks"] += 1
        parity["chunks"] = sample
    except ImportError as ex:
        parity["error"] = str(ex)
    res["parity"] = parity
    res["ratio"] = U / (ml.value + pl.value)
    res["pages_vs_chunks"] = res["decompress_pages"]["ms"] / res["decompress_chunks"]["ms"]
    res["wrapped_vs_chunks_only"] = res["compress_wrapped"]["ms"] / res["compress_ex_chunks_only"]["ms"]
    print(json.dumps({"workload": f"C2: {n_chunks} chunks x 2^18 u64, classic mode, consecutive delta order 1, device buffers",
                      "unit": "GB/s (10^9 uncompressed bytes)", "steps": args.steps, "gpu": gpu_description(), **res}))


if __name__ == "__main__":
    main()
