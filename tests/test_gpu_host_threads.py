"""Calls from several host threads at once.  The library keeps one scratch context per calling thread (device buffers, readback bounce,
profiler spans, error message) and shares only a mutex-guarded cache of mode-search sample positions and the turns of big copies.  These
tests run the entry points on overlapping threads, each with its own stream, and compare every output with the oracle's bytes or with the
same call made alone on the main thread, computed before the workers start; every decode must give the input back bit for bit.  Each
scenario runs once: the tests check results under overlap, they are not stress loops.  The last test checks that a call failing with a
CUDA error (an allocation refused while another thread captures a CUDA graph in global mode) leaves its thread usable."""
import ctypes as C
import json
import os
import queue
import struct
import subprocess
import sys
import threading
import traceback

import numpy as np
import pytest

from tests.golden_generators import bits_view
from tests.test_gpu_async_files import Bufs, _batch, _cfg as _files_cfg
from tests.test_gpu_async_pages import _dev, _refs_dev
from tests.test_gpu_auto import _auto_cfgs
from tests.test_gpu_encode import _cfgs, _walk

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC_ON_DEVICE, DST_ON_DEVICE, INDEX_ON_DEVICE = 1, 2, 4
TIMEOUT = 240  # seconds a worker may take before the test fails


@pytest.fixture(scope="module")
def sa():
    from pcodec_b200 import standalone

    return standalone


def _L():
    from pcodec_b200 import _lib

    return _lib.lib()


def _run_workers(fns, timeout=TIMEOUT):
    """Runs fns[i](sync) on thread i, each thread with its own torch.cuda.Stream as the current stream.  All threads meet at one barrier
    before they start, and sync() meets it again, so their calls overlap.  Each worker records its exception and calls
    pco_b200_thread_release() before it returns; the main thread joins with a timeout and fails if a worker is still running.  Returns
    the workers' results."""
    import torch

    L = _L()
    barrier = threading.Barrier(len(fns))
    results, errors = [None] * len(fns), [None] * len(fns)

    def sync():
        barrier.wait(timeout)

    def run(i):
        try:
            with torch.cuda.stream(torch.cuda.Stream()):
                sync()
                results[i] = fns[i](sync)
                torch.cuda.current_stream().synchronize()
        except BaseException:  # noqa: BLE001
            errors[i] = traceback.format_exc()
            barrier.abort()  # the others stop waiting for this one
        finally:
            L.pco_b200_thread_release()

    threads = [threading.Thread(target=run, args=(i,), daemon=True) for i in range(len(fns))]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout)
    assert not any(t.is_alive() for t in threads), "a worker thread is still running"
    failed = [f"worker {i}:\n{e}" for i, e in enumerate(errors) if e is not None]
    assert not failed, "\n".join(failed)
    return results


def _stream():
    import torch

    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(a):
    return C.c_void_p(a.data_ptr()) if hasattr(a, "data_ptr") else a.ctypes.data_as(C.c_void_p)


def _caps(x, cfg):
    """Capacities of pco_b200_compress_ex for the numpy array x under cfg: (file bytes, side index bytes)."""
    from pcodec_b200 import _lib

    L = _L()
    ps = cfg.paging_spec
    pages = len(ps.sizes) if ps.sizes is not None else -(-x.size // (ps.n or (1 << 18)))
    cap = L.pco_standalone_guarantee_file_size(C.c_size_t(x.size), C.c_ubyte(_lib.dtype_byte(x.dtype)))
    return cap + 160 * pages + 64, L.pco_b200_index_size_bound(C.c_size_t(x.size), C.c_size_t(max(x.size >> 8, 64))) + 64 * pages


def _compress_ex(x, cfg, dst_cap=None):
    """pco_b200_compress_ex of host numbers on the calling thread's current stream: (rc, file bytes, side index bytes)."""
    from pcodec_b200 import _lib

    cap, icap = _caps(x, cfg)
    cap = cap if dst_cap is None else dst_cap
    dst, idx = np.empty(max(cap, 1), np.uint8), np.empty(icap, np.uint8)
    nw, il = C.c_size_t(), C.c_size_t()
    c = cfg._to_c()
    rc = _L().pco_b200_compress_ex(_ptr(x), C.c_size_t(x.size), C.c_ubyte(_lib.dtype_byte(x.dtype)), C.byref(c), C.c_int(0), _ptr(dst), C.c_size_t(cap),
                                   C.byref(nw), _ptr(idx), C.c_size_t(icap), C.byref(il), C.c_uint32(0), _stream())
    return rc, dst[: nw.value].tobytes(), idx[: il.value].tobytes()


def _decompress_ex(data, dtype, n, index=None):
    """pco_b200_decompress_ex of host bytes into a host array of n numbers on the calling thread's current stream."""
    from pcodec_b200 import _lib

    src = np.frombuffer(bytes(data) + b"\0", np.uint8)
    ix = np.frombuffer(bytes(index) + b"\0", np.uint8) if index is not None else None
    dst = np.empty(max(n, 1), dtype)
    prog = _lib._CProgress()
    _lib.check(_L().pco_b200_decompress_ex(_ptr(src), C.c_size_t(len(data)), C.c_ubyte(_lib.dtype_byte(dtype)), _ptr(dst), C.c_size_t(n), C.byref(prog),
                                           _ptr(ix) if ix is not None else None, C.c_size_t(len(index) if index is not None else 0), C.c_uint32(0), _stream()))
    assert prog.finished and prog.n_processed == n
    return dst[:n]


def _roundtrip_on_device(x, cfg):
    """pco_b200_compress_ex and pco_b200_decompress_ex with numbers, file and index in device memory, on the current stream: (file bytes,
    index bytes, decoded numbers)."""
    import torch

    from pcodec_b200 import _lib

    L = _L()
    dt = C.c_ubyte(_lib.dtype_byte(x.dtype))
    t = torch.from_numpy(x.view(np.uint8).copy()).cuda()
    cap, icap = _caps(x, cfg)
    dst, idx = torch.empty(cap, dtype=torch.uint8, device="cuda"), torch.empty(icap, dtype=torch.uint8, device="cuda")
    nw, il = C.c_size_t(), C.c_size_t()
    c = cfg._to_c()
    flags = C.c_uint32(SRC_ON_DEVICE | DST_ON_DEVICE | INDEX_ON_DEVICE)
    _lib.check(L.pco_b200_compress_ex(_ptr(t), C.c_size_t(x.size), dt, C.byref(c), C.c_int(0), _ptr(dst), C.c_size_t(cap), C.byref(nw), _ptr(idx),
                                      C.c_size_t(icap), C.byref(il), flags, _stream()))
    out = torch.empty(x.nbytes, dtype=torch.uint8, device="cuda")
    prog = _lib._CProgress()
    _lib.check(L.pco_b200_decompress_ex(_ptr(dst), nw, dt, _ptr(out), C.c_size_t(x.size), C.byref(prog), _ptr(idx), il, flags, _stream()))
    assert prog.finished and prog.n_processed == x.size
    return dst[: nw.value].cpu().numpy().tobytes(), idx[: il.value].cpu().numpy().tobytes(), out.cpu().numpy().view(x.dtype)


def _same(got, want, where):
    """Outputs of one call (a dict of bytes / arrays / tuples) equal, arrays bit for bit."""
    assert got.keys() == want.keys(), where
    for k in want:
        g, w = got[k], want[k]
        if isinstance(w, np.ndarray):
            assert g.dtype == w.dtype and g.shape == w.shape, (where, k)
            np.testing.assert_array_equal(bits_view(g) if g.dtype.kind == "f" else g, bits_view(w) if w.dtype.kind == "f" else w, err_msg=f"{where} {k}")
        else:
            assert g == w, f"{where} {k}: differs from the same call made alone"


def _split(x, ns):
    at = np.concatenate([[0], np.cumsum(ns)]).astype(np.int64)
    return [x[at[i]:at[i + 1]] for i in range(len(ns))]


def _pieces(data, files):
    return [bytes(data[int(f["offset"]):int(f["offset"] + f["len"])]) for f in files]


def _int_mult_walk(n, seed, dtype=np.int32):
    """Numbers the Auto mode search answers with IntMult(1000) (test_gpu_auto's inputs)."""
    rng = np.random.default_rng(seed)
    return (np.cumsum(rng.integers(-50, 50, size=n)) * 1000 + 10**6).astype(dtype)


def _decimals(n, seed, dtype=np.float64):
    """Numbers the Auto mode search answers with FloatMult(0.01) (test_gpu_auto's inputs)."""
    rng = np.random.default_rng(seed)
    return (rng.integers(-5000, 5000, size=n).astype(np.float64) / 100.0).astype(dtype)


# ---- 1. mixed entry points on four threads ------------------------------------------------------------------------------------------


def _w1(sa, oracle):
    """u64, Classic, delta order 1: compress_ex / decompress_ex with pageable host buffers, then with device-resident ones."""
    cfg, ocfg = _cfgs(oracle, mode="classic", order=1)
    xs = [_walk(np.uint64, n, seed=10 + r) for r, n in enumerate([30_000, 300_000, 1_200_000])]

    def work(r):
        x = xs[r]
        rc, data, idx = _compress_ex(x, cfg)
        assert rc == 0
        d_data, d_idx, d_out = _roundtrip_on_device(x, cfg)
        return {"host.file": data, "host.index": idx, "host.decoded": _decompress_ex(data, np.uint64, x.size, idx),
                "dev.file": d_data, "dev.index": d_idx, "dev.decoded": d_out}

    def check(r, out):
        assert out["host.file"] == out["dev.file"] == oracle.simple_compress(xs[r], ocfg), f"round {r}: bytes differ from the oracle's"
        for k in ("host.decoded", "dev.decoded"):
            np.testing.assert_array_equal(out[k], xs[r], err_msg=k)

    return work, check


def _w2(sa, oracle):
    """f32, FloatMult(0.01): compress_files over lognormal file sizes, decompress_files with and without the side index, then
    decompress_ranges on the batch's largest file."""
    cfg, ocfg = _cfgs(oracle, mode="float_mult", order=1)
    rounds = []
    for r in range(3):
        rng = np.random.default_rng(20 + r)
        ns = np.clip(rng.lognormal(np.log(3000 * 4**r), 1.0, size=12), 1, 400_000).astype(np.int64)
        x = (np.round(np.cumsum(rng.normal(size=int(ns.sum()))) * 100) * 0.01).astype(np.float32)
        big = int(np.argmax(ns))
        ranges = np.array([[0, 1], [ns[big] // 3, ns[big] // 4], [ns[big] - 5, 5], [7, ns[big] // 2]], dtype=np.int64).clip(0)
        rounds.append((x, ns, big, ranges, [oracle.simple_compress(nums, ocfg) for nums in _split(x, ns)]))

    def work(r):
        x, ns, big, ranges, _ = rounds[r]
        data, files, index = sa.compress_files(x, ns, cfg)
        with_idx, ns_a = sa.decompress_files(data, files, np.float32, index)
        refs = files.copy()
        refs["index_len"] = 0
        walked, ns_b = sa.decompress_files(data, refs, np.float32, None)
        f = files[big]
        one = data[int(f["offset"]):int(f["offset"] + f["len"])]
        one_idx = index[int(f["index_offset"]):int(f["index_offset"] + f["index_len"])]
        return {"data": data, "refs": files.tobytes(), "index": index, "indexed": with_idx, "indexed.ns": ns_a, "walked": walked, "walked.ns": ns_b,
                "ranges": sa.decompress_ranges(one, np.float32, one_idx, ranges)}

    def check(r, out):
        x, ns, big, ranges, want = rounds[r]
        got = _pieces(out["data"], np.frombuffer(out["refs"], sa.FILE_REF))
        assert got == want, f"round {r}: files {[i for i in range(len(want)) if got[i] != want[i]]} differ from the oracle's"
        for k in ("indexed", "walked"):
            np.testing.assert_array_equal(bits_view(out[k]), bits_view(x), err_msg=k)
            np.testing.assert_array_equal(out[k + ".ns"], ns.astype(np.uint64))
        piece = _split(x, ns)[big]
        want = np.concatenate([piece[s:s + c] for s, c in ranges])
        np.testing.assert_array_equal(bits_view(out["ranges"]), bits_view(want))

    return work, check


def _w3(sa, oracle):
    """i16, delta order 2: compress_chunks / decompress_pages, then build_index on an index-free file the oracle wrote and decompress_ex
    through that index."""
    from pcodec_b200 import wrapped

    cfg, ocfg = _cfgs(oracle, mode="classic", order=2, max_page_n=1 << 14)
    xs = [_walk(np.int16, n, seed=30 + r) for r, n in enumerate([20_000, 150_000, 600_000])]
    files = [oracle.simple_compress(x, ocfg) for x in xs]

    def work(r):
        x = xs[r]
        metas, pages, refs = wrapped.compress_chunks(x, cfg)
        idx = sa.build_index(files[r], np.int16)
        return {"metas": metas, "pages": pages, "refs": refs.tobytes(), "pages.decoded": wrapped.decompress_pages(metas, pages, refs, np.int16),
                "index": idx, "file.decoded": _decompress_ex(files[r], np.int16, x.size, idx)}

    def check(r, out):
        for k in ("pages.decoded", "file.decoded"):
            np.testing.assert_array_equal(out[k], xs[r], err_msg=k)
        # build_index returns its unused chunk record slots too: zeros, not what the thread's scratch held before
        idx = out["index"]
        n_chunks, first_entries = struct.unpack_from("<Q", idx, 8)[0], struct.unpack_from("<Q", idx, 64 + 16)[0]
        assert not any(idx[64 + 32 * n_chunks:first_entries]), f"round {r}: unused chunk records of the index are not zero"

    return work, check


def _w4(sa, oracle):
    """ModeSpec::Auto + DeltaSpec::Auto: compress_files over 70 distinct file sizes of int-mult-friendly i32 and decimal f64 numbers, and
    the drop-in pco_standalone_simple_compress_into / _decompress_into with a null config."""
    from pcodec_b200 import _lib

    cfg, ocfg = _auto_cfgs(oracle)
    rounds = []
    for r in range(3):
        ns = np.array([10 + 7 * k + 600 * r for k in range(70)], dtype=np.int64)
        xi, xf = _int_mult_walk(int(ns.sum()), seed=40 + r), _decimals(int(ns.sum()), seed=50 + r)
        want = {name: ([oracle.simple_compress(nums, ocfg) for nums in _split(x, ns)], oracle.simple_compress(x, ocfg, uniform_type=True))
                for name, x in (("i32", xi), ("f64", xf))}
        rounds.append((ns, xi, xf, want))

    def dropin(x):
        L = _L()
        dt = C.c_ubyte(_lib.dtype_byte(x.dtype))
        cap = L.pco_standalone_guarantee_file_size(C.c_size_t(x.size), dt)
        dst, nw = np.zeros(cap, np.uint8), C.c_size_t()
        assert L.pco_standalone_simple_compress_into(_ptr(x), C.c_size_t(x.size), dt, None, _ptr(dst), C.c_size_t(cap), C.byref(nw)) == 0
        back, nb = np.empty(x.size, x.dtype), C.c_size_t()
        assert L.pco_standalone_simple_decompress_into(_ptr(dst), nw, dt, _ptr(back), C.c_size_t(x.size), C.byref(nb)) == 0
        assert nb.value == x.size
        return dst[: nw.value].tobytes(), back

    def work(r):
        ns, xi, xf, _ = rounds[r]
        out = {}
        for name, x in (("i32", xi), ("f64", xf)):
            data, files, index = sa.compress_files(x, ns, cfg)
            vals, _ = sa.decompress_files(data, files, x.dtype, index)
            out.update({f"{name}.data": data, f"{name}.refs": files.tobytes(), f"{name}.decoded": vals})
            out[f"{name}.dropin"], out[f"{name}.dropin.decoded"] = dropin(x)
        return out

    def check(r, out):
        ns, xi, xf, want = rounds[r]
        for name, x in (("i32", xi), ("f64", xf)):
            got = _pieces(out[f"{name}.data"], np.frombuffer(out[f"{name}.refs"], sa.FILE_REF))
            bad = [i for i in range(len(ns)) if got[i] != want[name][0][i]]
            assert not bad, f"round {r} {name}: files {bad[:8]} (sizes {[int(ns[i]) for i in bad[:8]]}) differ from the oracle's"
            assert out[f"{name}.dropin"] == want[name][1], f"round {r} {name}: drop-in bytes differ from the oracle's"
            for k in ("decoded", "dropin.decoded"):
                np.testing.assert_array_equal(bits_view(out[f"{name}.{k}"]), bits_view(x), err_msg=f"{name}.{k}")

    return work, check


def test_mixed_entry_points_on_four_threads(sa, oracle):
    """Four threads, each with its own dtype, config and entry points, run three rounds whose inputs grow, so every thread frees and
    reallocates its scratch while the other threads' kernels run.  Every output equals the same call made alone (itself checked against
    the oracle and the input) and every decode gives the input back."""
    workers = [w(sa, oracle) for w in (_w1, _w2, _w3, _w4)]
    alone = [[work(r) for r in range(3)] for work, _ in workers]
    for (_, check), outs in zip(workers, alone):
        for r, out in enumerate(outs):
            check(r, out)

    def thread(work):
        def fn(sync):
            outs = []
            for r in range(3):
                outs.append(work(r))
                sync()  # every thread is in the same round
            return outs

        return fn

    got = _run_workers([thread(work) for work, _ in workers])
    for w, ((_, check), outs, want) in enumerate(zip(workers, got, alone)):
        for r in range(3):
            _same(outs[r], want[r], f"worker {w + 1} round {r}")
            check(r, outs[r])


# ---- 2. Auto mode on threads with disjoint size sets ----------------------------------------------------------------------------------


def test_auto_mode_on_threads_with_disjoint_size_sets(sa, oracle):
    """Four threads each compress one ModeSpec::Auto batch of 100 files.  Each thread's file sizes are distinct and differ from every other
    thread's, so the process-wide cache of mode-search sample positions (cleared once it holds more than 64 sizes) is cleared several times
    while the calls run.  Every file's bytes must equal the oracle's.

    This exercises the window in which a call that kept a reference into that cache would read freed memory after another thread cleared
    it; the cache now hands out copies.  The race is timing-dependent, so the test cannot be relied on to fail on code that keeps such a
    reference."""
    cfg, ocfg = _auto_cfgs(oracle)
    jobs = []
    for t, make in enumerate((lambda n, s: _int_mult_walk(n, s, np.int64), _decimals, _int_mult_walk, lambda n, s: _decimals(n, s, np.float32))):
        ns = np.array([200 + 4 * k + t for k in range(100)], dtype=np.int64)
        x = make(int(ns.sum()), 60 + t)
        want = [oracle.simple_compress(nums, ocfg) for nums in _split(x, ns)]
        jobs.append((x, ns, want))
    for x, ns, want in jobs:
        data, files, _ = sa.compress_files(x, ns, cfg)
        assert _pieces(data, files) == want, "the call made alone differs from the oracle"

    def thread(job):
        x, ns, _ = job
        return lambda sync: sa.compress_files(x, ns, cfg, with_index=False)

    for t, ((data, files), (x, ns, want)) in enumerate(zip(_run_workers([thread(j) for j in jobs]), jobs)):
        got = _pieces(data, files)
        bad = [i for i in range(len(want)) if got[i] != want[i]]
        assert not bad, f"thread {t}: files {bad[:8]} (sizes {[int(ns[i]) for i in bad[:8]]}) differ from the oracle's"


# ---- 3. streamed pipeline across dtypes -----------------------------------------------------------------------------------------------


class _Group:
    """One group of the streamed pipeline: its numbers, compressed bytes, side index and decoded numbers in page-locked host buffers."""

    def __init__(self, x, cfg):
        import torch

        from pcodec_b200 import _lib

        self.x, self.cfg, self.dt = x, cfg._to_c(), _lib.dtype_byte(x.dtype)
        self.cap, self.icap = _caps(x, cfg)
        self.nums = torch.empty(x.nbytes, dtype=torch.uint8, pin_memory=True)
        self.nums.copy_(torch.from_numpy(x.view(np.uint8)))
        self.comp = torch.empty(self.cap, dtype=torch.uint8, pin_memory=True)
        self.index = torch.empty(self.icap, dtype=torch.uint8, pin_memory=True)
        self.out = torch.empty(x.nbytes, dtype=torch.uint8, pin_memory=True)
        self.nw, self.il = C.c_size_t(), C.c_size_t()

    def compress(self):
        from pcodec_b200 import _lib

        _lib.check(_L().pco_b200_compress_ex(_ptr(self.nums), C.c_size_t(self.x.size), C.c_ubyte(self.dt), C.byref(self.cfg), C.c_int(0), _ptr(self.comp),
                                             C.c_size_t(self.cap), C.byref(self.nw), _ptr(self.index), C.c_size_t(self.icap), C.byref(self.il),
                                             C.c_uint32(0), _stream()))

    def decompress(self):
        from pcodec_b200 import _lib

        prog = _lib._CProgress()
        _lib.check(_L().pco_b200_decompress_ex(_ptr(self.comp), self.nw, C.c_ubyte(self.dt), _ptr(self.out), C.c_size_t(self.x.size), C.byref(prog),
                                               _ptr(self.index), self.il, C.c_uint32(0), _stream()))
        assert prog.finished and prog.n_processed == self.x.size

    def reset(self):
        self.comp.zero_()
        self.index.zero_()
        self.out.zero_()

    def results(self):
        return self.comp[: self.nw.value].numpy().tobytes(), self.index[: self.il.value].numpy().tobytes()


@pytest.fixture(scope="module")
def pipeline_groups(oracle):
    """Four groups of 2^24 u64 (each above copy_sliced's 64 MB threshold, so the sliced copies and the cross-thread turns run), then
    eight groups of 300 000 f64 and i32 numbers, each with the bytes and index of its compress made alone."""
    from pcodec_b200 import datagen

    cfg, _ = _cfgs(oracle, mode="classic", order=1)
    passes = [[_Group(datagen.c2_u64_cumsum_geometric(n=1 << 24, seed=g), cfg) for g in range(4)],
              [_Group(datagen.c3_f64_decimal_sinusoid(n=300_000, seed=g) if g % 2 == 0 else _walk(np.int32, 300_000, seed=g), cfg) for g in range(8)]]
    alone = []
    for groups in passes:
        want = []
        for g in groups:
            g.compress()
            want.append(g.results())
        alone.append(want)
    return passes, alone


def _stream_groups(groups, producers=2):
    """bench.py's streamed leg at small scale: producer p compresses groups p, p + P, ... and hands each to consumer p, which decompresses it."""
    handoffs = [queue.Queue() for _ in range(producers)]

    def produce(p):
        def fn(sync):
            try:
                for k in range(p, len(groups), producers):
                    groups[k].compress()
                    handoffs[p].put(k)
            finally:
                handoffs[p].put(None)

        return fn

    def consume(p):
        def fn(sync):
            while True:
                k = handoffs[p].get(timeout=TIMEOUT)
                if k is None:
                    return
                groups[k].decompress()

        return fn

    _run_workers([produce(p) for p in range(producers)] + [consume(p) for p in range(producers)])


@pytest.mark.parametrize("mask", [0, 7])
def test_streamed_pipeline_across_dtypes(pipeline_groups, mask):
    """Two producer threads run compress_ex and hand groups through queues to two consumer threads running decompress_ex, with page-locked
    host buffers, staged (mask 0) or read and written in place by the kernels (mask 7).  Every group's bytes and index equal the same call
    made alone, and every group decodes to its numbers."""
    passes, alone = pipeline_groups
    L = _L()
    before = L.pco_b200_zero_copy(mask)
    try:
        for groups, want in zip(passes, alone):
            for g in groups:
                g.reset()
            _stream_groups(groups)
            for k, (g, w) in enumerate(zip(groups, want)):
                assert g.results() == w, f"group {k} ({g.x.dtype}, n={g.x.size}): bytes or index differ from the call made alone"
                np.testing.assert_array_equal(g.out.numpy(), g.x.view(np.uint8), err_msg=f"group {k} does not decode to its numbers")
    finally:
        L.pco_b200_zero_copy(before)


# ---- 4. per-thread state --------------------------------------------------------------------------------------------------------------


def _profile_names():
    buf = C.create_string_buffer(1 << 16)
    _L().pco_b200_profile_last(buf, C.c_size_t(len(buf)))
    return [s.split("=")[0] for s in buf.value.decode().split(";") if s]


def _chunk_classes():
    counts = (C.c_uint * 8)()
    n = _L().pco_b200_profile_chunk_classes(counts)
    return n, list(counts)


def test_error_message_profile_and_chunk_classes_are_per_thread(sa, oracle):
    """Thread A decodes while thread B compresses, then A makes a compress the host refuses (a destination one byte too small: Io) while B
    decodes.  Each thread's last error message, kernel spans (profiling on for both) and chunk classes of its last decode are its own:
    what the same calls made alone on one thread give."""
    from pcodec_b200 import _lib

    cfg_a, ocfg_a = _cfgs(oracle, mode="classic", order=1, max_page_n=1 << 15)
    cfg_b, ocfg_b = _cfgs(oracle, mode="classic", order=0, max_page_n=1 << 13)
    x_a, x_b = _walk(np.uint64, 200_000, seed=71), _walk(np.uint32, 90_000, seed=72)
    file_a, file_b = oracle.simple_compress(x_a, ocfg_a), oracle.simple_compress(x_b, ocfg_b)
    _, _, idx_a = _compress_ex(x_a, cfg_a)
    _, _, idx_b = _compress_ex(x_b, cfg_b)
    L = _L()

    def a_decode():
        np.testing.assert_array_equal(_decompress_ex(file_a, np.uint64, x_a.size, idx_a), x_a)

    def a_refused():
        rc, _, _ = _compress_ex(x_a, cfg_a, dst_cap=len(file_a) - 1)
        assert rc == 4, _lib.ERROR_KINDS.get(rc, rc)
        return L.pco_b200_last_error_message().decode()

    def b_compress():
        rc, data, _ = _compress_ex(x_b, cfg_b)
        assert rc == 0 and data == file_b

    def b_decode():
        np.testing.assert_array_equal(_decompress_ex(file_b, np.uint32, x_b.size, idx_b), x_b)

    def b_unknown_dtype():
        nw = C.c_size_t()
        rc = L.pco_b200_compress_ex(_ptr(x_b), C.c_size_t(x_b.size), C.c_ubyte(99), None, C.c_int(0), None, C.c_size_t(0), C.byref(nw), None,
                                    C.c_size_t(0), None, C.c_uint32(0), None)
        assert rc == 5
        return L.pco_b200_last_error_message().decode()

    L.pco_b200_profile_enable(1)
    try:
        want = {}
        for name, fn in (("a_decode", a_decode), ("a_refused", a_refused), ("b_compress", b_compress), ("b_decode", b_decode)):
            msg = fn()
            want[name] = (_profile_names(), _chunk_classes() if "decode" in name else None, msg)
        assert want["a_refused"][2].startswith("failed to write whole buffer"), want["a_refused"][2]
        assert {"fused_narrow_kernel"} <= set(want["a_decode"][0]) and {"fused_narrow_kernel"} <= set(want["b_decode"][0])
        assert not {"fused_narrow_kernel"} & set(want["b_compress"][0] + want["a_refused"][0])
        assert want["a_decode"][1] != want["b_decode"][1], "the two decodes should differ in their chunk classes"

        def thread_a(sync):
            a_decode()
            seen = {"decode": (_profile_names(), _chunk_classes())}
            sync()
            msg = a_refused()
            sync()  # B's decode has finished too
            seen["refused"] = (_profile_names(), _chunk_classes(), msg, L.pco_b200_last_error_message().decode())
            return seen

        def thread_b(sync):
            own = b_unknown_dtype()
            b_compress()
            seen = {"compress": (_profile_names(), _chunk_classes())}
            sync()
            b_decode()
            sync()  # A's refused call has finished too
            seen["decode"] = (_profile_names(), _chunk_classes(), own, L.pco_b200_last_error_message().decode())
            return seen

        a, b = _run_workers([thread_a, thread_b])
    finally:
        L.pco_b200_profile_enable(0)
    assert a["decode"] == (want["a_decode"][0], want["a_decode"][1])
    assert b["compress"] == (want["b_compress"][0], (0, [0] * 8)), "a thread that has decoded nothing has no chunk classes"
    names, classes, msg, last = a["refused"]
    assert names == want["a_refused"][0], "A's spans are those of its own refused compress"
    assert classes == want["a_decode"][1], "A's chunk classes are those of its own last decode"
    assert msg == last == want["a_refused"][2]
    names, classes, own, last = b["decode"]
    assert names == want["b_decode"][0] and classes == want["b_decode"][1]
    assert own == last == "unknown number type byte: 99", f"B's message changed to {last!r}"


# ---- 5. plan, capture and replay on different threads ---------------------------------------------------------------------------------


def test_plan_capture_and_replay_on_different_threads(sa, oracle):
    """Thread A plans an AsyncFilesDecompressor and an AsyncPagesFilter, runs each once, releases its scratch and exits.  Thread B, which
    has never called the library, captures both calls into CUDA graphs (thread-local capture mode) while thread C makes its first blocking
    calls, so C's scratch is allocated during B's capture.  The main thread then replays both graphs twice with new refs and bounds written
    into the device tensors before each replay.  Every output equals the blocking decompress_files, and numpy's selection for the filter:
    a captured call refers to no memory of any thread's scratch."""
    import torch

    from pcodec_b200 import wrapped

    # files: two ref orders over one batch; pages: two page orders and two intervals
    xs = [_walk(np.uint32, 3000 * (i + 1) + 11, seed=80 + i) for i in range(6)]
    data, index, refs = _batch(sa, xs, _files_cfg(1, page=4096))
    orders = [[5, 0, 3, 1], [2, 2, 4, 0, 1, 5]]
    files_want = []
    for order in orders:
        r = np.zeros(len(order), sa.FILE_REF)
        rr = refs[order]
        r["offset"], r["len"], r["index_offset"], r["index_len"] = rr[:, 0], rr[:, 1], rr[:, 2], rr[:, 3]
        vals, ns = sa.decompress_files(data, r, np.uint32, index)
        np.testing.assert_array_equal(vals, np.concatenate([xs[i] for i in order]))
        files_want.append((vals, ns))
    xp = _walk(np.int64, 50_000, seed=90)
    pcfg, _ = _cfgs(oracle, mode="classic", order=1, max_page_n=6000)
    metas, pages, prefs = wrapped.compress_chunks(xp, pcfg)
    pieces = _split(xp, prefs["page_n"].astype(np.int64))
    page_orders = [list(range(len(prefs)))[::-1], [1, 0, 4, 4, 2]]
    s = np.sort(xp)
    intervals = [(int(s[len(s) // 5]), int(s[len(s) // 2])), (int(s[0]), int(s[len(s) // 10]))]
    filter_want = []
    for order, (lo, hi) in zip(page_orders, intervals):
        dec = np.concatenate([pieces[i] for i in order])
        sel = np.nonzero((dec >= lo) & (dec <= hi))[0]
        filter_want.append((sel, dec[sel]))
    # the blocking calls thread C makes, made alone
    c_x = _walk(np.uint64, 400_000, seed=91)
    c_cfg, c_ocfg = _cfgs(oracle, mode="classic", order=2)
    c_want = oracle.simple_compress(c_x, c_ocfg)

    max_pages, rows_cap = 12, int(sum(p.size for p in pieces)) * 2
    assert max(len(o) for o in page_orders) <= max_pages
    made, captured, c_started, c_done = {}, {}, threading.Event(), threading.Event()

    def thread_a(sync):
        b = Bufs(sa, data[:32], np.uint32, len(data) + 64, len(index) + 64, 8, 64, 1 << 16)
        b.load(data, index, refs[orders[0]])
        # frames for a batch that names a page twice
        f = wrapped.AsyncPagesFilter(np.int64, len(metas), len(pages), max_pages, rows_cap, rows_cap, 2 * (len(metas) + len(pages)) + 32 * max_pages)
        t = {"metas": _dev(metas), "pages": _dev(pages), "refs": _refs_dev(prefs[page_orders[0]], max_pages),
             "n": torch.tensor([len(page_orders[0])], dtype=torch.int64).cuda(),
             "iv": torch.from_numpy(wrapped.pack_interval(*intervals[0], np.int64)).cuda(),
             "vals": torch.zeros(rows_cap, dtype=torch.int64, device="cuda"), "pos": torch.zeros(rows_cap, dtype=torch.int64, device="cuda"),
             "nm": torch.zeros(1, dtype=torch.int64, device="cuda")}
        b.call()  # once outside any capture
        f(t["metas"], t["pages"], t["refs"], t["n"], t["iv"], t["vals"], t["pos"], t["nm"])
        torch.cuda.current_stream().synchronize()
        made.update(b=b, f=f, t=t)

    def filter_call():
        t = made["t"]
        made["f"](t["metas"], t["pages"], t["refs"], t["n"], t["iv"], t["vals"], t["pos"], t["nm"])

    def thread_b(sync):
        for name, call in (("files", made["b"].call), ("filter", filter_call)):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=torch.cuda.current_stream(), capture_error_mode="thread_local"):
                call()
                if name == "files":
                    c_started.set()
                    assert c_done.wait(TIMEOUT), "thread C did not finish"
            captured[name] = g

    def thread_c(sync):
        assert c_started.wait(TIMEOUT), "thread B did not start its capture"
        try:
            rc, got, idx = _compress_ex(c_x, c_cfg)
            assert rc == 0 and got == c_want
            np.testing.assert_array_equal(_decompress_ex(got, np.uint64, c_x.size, idx), c_x)
            np.testing.assert_array_equal(_decompress_ex(got, np.uint64, c_x.size), c_x)
        finally:
            c_done.set()

    _run_workers([thread_a])
    _run_workers([thread_b, thread_c])
    b, t = made["b"], made["t"]
    for step in range(2):
        b.load(data, index, refs[orders[step]])
        t["refs"].copy_(_refs_dev(prefs[page_orders[step]], max_pages))
        t["n"].fill_(len(page_orders[step]))
        t["iv"].copy_(torch.from_numpy(wrapped.pack_interval(*intervals[step], np.int64)))
        t["nm"].fill_(-1)
        t["pos"].fill_(-1)
        captured["files"].replay()
        captured["filter"].replay()
        torch.cuda.synchronize()
        got, err, st = b.outcome()
        assert err is None, err
        np.testing.assert_array_equal(got[0], files_want[step][0], err_msg=f"replay {step}: files")
        np.testing.assert_array_equal(got[1], files_want[step][1])
        assert made["f"].result() == len(filter_want[step][0])
        k = int(t["nm"].item())
        np.testing.assert_array_equal(t["pos"][:k].cpu().numpy(), filter_want[step][0], err_msg=f"replay {step}: filter positions")
        np.testing.assert_array_equal(t["vals"][:k].cpu().numpy(), filter_want[step][1], err_msg=f"replay {step}: filter values")


# ---- 6. a failed CUDA call leaves the thread usable -----------------------------------------------------------------------------------

_CHILD = r"""
import ctypes as C, json, os, sys, threading, traceback
sys.path.insert(0, os.getcwd())
import numpy as np
import torch
from oracle import pyoracle
from pcodec_b200 import _lib

WAIT = 60
L = _lib.lib()
small = np.cumsum(np.random.default_rng(1).geometric(0.01, size=3000)).astype(np.uint64)
big = np.cumsum(np.random.default_rng(2).geometric(0.01, size=2_000_000)).astype(np.uint64)
ocfg = pyoracle.make_config(mode=pyoracle.MODE_CLASSIC, delta=pyoracle.DELTA_CONSECUTIVE, delta_order=1)
want = {"small": pyoracle.simple_compress(small, ocfg), "big": pyoracle.simple_compress(big, ocfg)}
cfg = _lib.ChunkConfig(mode_spec=_lib.ModeSpec.classic(), delta_spec=_lib.DeltaSpec.try_consecutive(1))._to_c()
torch.zeros(1, device="cuda")
streams = {k: torch.cuda.Stream() for k in "ABD"}
out, ev = {}, {k: threading.Event() for k in ("d_ready", "capturing", "b_tried", "d_tried", "release", "ended")}

def call(name, x, stream):
    cap = L.pco_standalone_guarantee_file_size(C.c_size_t(x.size), C.c_ubyte(2))
    dst, nw = np.zeros(cap, np.uint8), C.c_size_t()
    rc = L.pco_b200_compress_ex(x.ctypes.data_as(C.c_void_p), C.c_size_t(x.size), C.c_ubyte(2), C.byref(cfg), C.c_int(0),
                                dst.ctypes.data_as(C.c_void_p), C.c_size_t(cap), C.byref(nw), None, C.c_size_t(0), None, C.c_uint32(0),
                                C.c_void_p(stream.cuda_stream))
    ok = rc == 0 and dst[: nw.value].tobytes() == want["small" if x is small else "big"]
    out[name] = {"kind": _lib.ERROR_KINDS.get(rc, "ok"), "message": L.pco_b200_last_error_message().decode() if rc else "", "equal": ok}

def guarded(fn):
    def run():
        try:
            fn()
        except BaseException:
            out.setdefault("errors", []).append(traceback.format_exc())
    return run

@guarded
def thread_a():
    g, x = torch.cuda.CUDAGraph(), torch.ones(1024, device="cuda")
    try:
        with torch.cuda.graph(g, stream=streams["A"]):  # global capture mode, torch's default
            y = x * 2
            ev["capturing"].set()
            ev["release"].wait(WAIT)
        out["capture"] = "ended without an error"
    except Exception as e:
        out["capture"] = f"{type(e).__name__}: {e}"

@guarded
def thread_b():
    ev["capturing"].wait(WAIT)
    try:
        call("b.during", small, streams["B"])
    finally:
        ev["b_tried"].set()
    ev["ended"].wait(WAIT)
    call("b.after", small, streams["B"])
    call("b.again", small, streams["B"])
    L.pco_b200_thread_release()
    call("b.released", small, streams["B"])
    L.pco_b200_thread_release()

@guarded
def thread_d():
    try:
        call("d.before", small, streams["D"])
    finally:
        ev["d_ready"].set()
    ev["capturing"].wait(WAIT)
    try:
        call("d.during", big, streams["D"])
    finally:
        ev["d_tried"].set()
    ev["ended"].wait(WAIT)
    call("d.after", small, streams["D"])
    L.pco_b200_thread_release()

threads = {k: threading.Thread(target=f, daemon=True) for k, f in (("D", thread_d), ("A", thread_a), ("B", thread_b))}
threads["D"].start()
ev["d_ready"].wait(WAIT)
threads["A"].start()
threads["B"].start()
ev["capturing"].wait(WAIT)
ev["b_tried"].wait(WAIT)
ev["d_tried"].wait(WAIT)
ev["release"].set()
threads["A"].join(WAIT)
ev["ended"].set()
for t in threads.values():
    t.join(WAIT)
out["alive"] = [k for k, t in threads.items() if t.is_alive()]
print("RESULT " + json.dumps(out), flush=True)
os._exit(0)
"""


def test_failed_cuda_call_leaves_the_thread_usable():
    """While thread A holds a global-mode CUDA graph capture open, the runtime refuses allocations on every other thread.  Thread B, which
    has never called the library, and thread D, whose call needs more scratch than its first call made, then fail with kind Cuda - never
    with wrong output.  Once A's capture has ended, B's next calls (with and without pco_b200_thread_release in between) and D's next call,
    which needs no growth, succeed with the oracle's bytes: the device set-up caches only permanent outcomes and a failed call clears the
    runtime's last error.  Runs in a child process so the capture cannot leak into the test session."""
    proc = subprocess.run([sys.executable, "-c", _CHILD], cwd=ROOT, capture_output=True, text=True, timeout=600)
    lines = [ln for ln in proc.stdout.splitlines() if ln.startswith("RESULT ")]
    assert proc.returncode == 0 and lines, f"child failed ({proc.returncode}):\n{proc.stdout[-4000:]}\n{proc.stderr[-4000:]}"
    out = json.loads(lines[-1][len("RESULT "):])
    assert not out.get("errors") and not out["alive"], out
    assert out["d.before"] == {"kind": "ok", "message": "", "equal": True}, out
    for name in ("b.during", "d.during"):
        assert out[name]["kind"] == "Cuda", (name, out)
    for name in ("b.after", "b.again", "b.released", "d.after"):
        assert out[name] == {"kind": "ok", "message": "", "equal": True}, (name, out)
