"""Mirror of `pcodec.standalone` (pco_python/src/standalone.rs:44-135) over libcpcodec.so."""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import ChunkConfig, PcoError, Progress  # noqa: F401


def _src_buf(data):
    mv = memoryview(data)
    n = mv.nbytes
    arr = np.frombuffer(mv, dtype=np.uint8) if n else np.zeros(1, dtype=np.uint8)
    return arr, n


def simple_decompress_into(src, dst):
    """pcodec.standalone.simple_decompress_into (pco_python/src/standalone.rs:90-118): decompresses into a
    numpy array, returning Progress; never errors on a too-short or too-long dst."""
    return decompress_into_with_index(src, dst, None)


def simple_decompress(src, dtype=None, index=None):
    """pcodec.standalone.simple_decompress (pco_python/src/standalone.rs:120-135).  The reference infers the
    dtype from the file; pass `dtype` to assert it.  `index` is an optional side index (bytes)."""
    if dtype is None:
        dtype = peek_dtype(src)
        if dtype is None:
            return None
    # size the destination from n_hint when present, growing if the file holds more.  n_hint is untrusted (a 20-byte file may claim 2^64
    # numbers): the first allocation is capped at 2^32 bytes like the reference's (pco/src/standalone/constants.rs:10-17, decompressor.rs:265-269)
    cap = max(min(n_hint(src), (1 << 32) // np.dtype(dtype).itemsize), 1)
    while True:
        dst = np.empty(cap, dtype=dtype)
        prog = decompress_into_with_index(src, dst, index)
        if prog.finished:
            return dst[: prog.n_processed]
        cap = max(cap * 2, 1 << 16)


def decompress_into_with_index(src, dst, index=None):
    L = _lib.lib()
    arr, n = _src_buf(src)
    prog = _lib._CProgress()
    if index is not None:
        iarr, ilen = _src_buf(index)
        iptr, ilen_c = iarr.ctypes.data_as(C.c_void_p), C.c_size_t(ilen)
    else:
        iptr, ilen_c = None, C.c_size_t(0)
    rc = L.pco_b200_decompress_ex(arr.ctypes.data_as(C.c_void_p), C.c_size_t(n), C.c_ubyte(_lib.dtype_byte(dst.dtype)),
                                  dst.ctypes.data_as(C.c_void_p), C.c_size_t(dst.size), C.byref(prog), iptr, ilen_c,
                                  C.c_uint32(0), None)
    _lib.check(rc)
    return Progress(prog.n_processed, bool(prog.finished))


def build_index(src, dtype, n_total_hint=None):
    """Builds the per-batch side index of a standalone file on the device (one serial tANS walk)."""
    L = _lib.lib()
    arr, n = _src_buf(src)
    hint = n_total_hint if n_total_hint is not None else max(n_hint(src), 1)
    cap = L.pco_b200_index_size_bound(hint, max(hint >> 8, 64))
    while True:
        buf = np.empty(cap, dtype=np.uint8)
        used = C.c_size_t()
        rc = L.pco_b200_build_index(arr.ctypes.data_as(C.c_void_p), C.c_size_t(n), C.c_ubyte(_lib.dtype_byte(dtype)),
                                    buf.ctypes.data_as(C.c_void_p), C.c_size_t(cap), C.byref(used), C.c_uint32(0), None)
        if rc == 4:  # Io: index buffer too small
            cap *= 4
            continue
        _lib.check(rc)
        return buf[: used.value].tobytes()


def _header(src):
    """(standalone_version, uniform_type, n_hint, first_chunk_byte) — docs/format.md:173-192."""
    b = bytes(memoryview(src)[:32])
    if len(b) < 5 or b[:4] != b"pco!":
        return None
    ver = b[4]
    if ver < 2:
        return ver, 0, 0, 4 + 1
    pos = 5
    uniform = 0
    if ver >= 3:
        uniform = b[pos] if pos < len(b) else 0
        pos += 1
    wide = int.from_bytes(b[pos:pos + 10].ljust(10, b"\0"), "little")
    power = 1 + (wide & 63)
    n = (wide >> 6) & ((1 << power) - 1)
    pos += (6 + power + 7) // 8
    major = b[pos] if pos < len(b) else 0
    pos += 2 if major >= 4 else 1
    return ver, uniform, n, pos


def n_hint(src):
    h = _header(src)
    return h[2] if h else 0


def peek_dtype(src):
    h = _header(src)
    if h is None:
        raise PcoError("Corruption", "magic header does not match")
    if h[1]:
        return _lib.BYTE_TO_NP[h[1]]
    mv = memoryview(src)
    if h[3] >= mv.nbytes:
        raise PcoError("InsufficientData", "unable to peek number type from empty bytes")
    t = mv[h[3]]
    if t == 0:
        return None
    if t not in _lib.BYTE_TO_NP:
        raise PcoError("Corruption", f"peeked unknown number type byte: {t}")
    return _lib.BYTE_TO_NP[t]


def _compress(nums, config, uniform_type, want_index):
    L = _lib.lib()
    arr = np.ascontiguousarray(nums)
    dt = _lib.dtype_byte(arr.dtype)
    cfg = (config or ChunkConfig())._to_c()
    cap = L.pco_standalone_guarantee_file_size(arr.size, dt)
    if cfg.paging_spec == 1 or (cfg.max_page_n and cfg.max_page_n < (1 << 18)):
        # the guarantee above assumes default paging; small pages add a per-chunk meta allowance
        n_pages = cfg.n_exact_pages if cfg.paging_spec == 1 else -(-arr.size // max(cfg.max_page_n, 1))
        cap += int(n_pages) * 160
    dst = np.empty(cap, dtype=np.uint8)
    n_written = C.c_size_t()
    if want_index:
        icap = L.pco_b200_index_size_bound(arr.size, max(arr.size >> 8, 64))
        if cfg.paging_spec == 1 or cfg.max_page_n:
            icap += 64 * (int(cfg.n_exact_pages) if cfg.paging_spec == 1 else -(-arr.size // max(cfg.max_page_n, 1)))
        idx = np.empty(icap, dtype=np.uint8)
        ilen = C.c_size_t()
        iptr, icap_c, ilen_p = idx.ctypes.data_as(C.c_void_p), C.c_size_t(icap), C.byref(ilen)
    else:
        idx, ilen, iptr, icap_c, ilen_p = None, None, None, C.c_size_t(0), None
    rc = L.pco_b200_compress_ex(arr.ctypes.data_as(C.c_void_p), C.c_size_t(arr.size), C.c_ubyte(dt), C.byref(cfg),
                                C.c_int(1 if uniform_type else 0), dst.ctypes.data_as(C.c_void_p), C.c_size_t(cap), C.byref(n_written),
                                iptr, icap_c, ilen_p, C.c_uint32(0), None)
    _lib.check(rc)
    out = dst[: n_written.value].tobytes()
    if want_index:
        return out, idx[: ilen.value].tobytes()
    return out


def simple_compress(nums, config=None):
    """pcodec.standalone.simple_compress (pco_python/src/standalone.rs:44-88; pco/src/standalone/simple.rs:58-91)."""
    return _compress(nums, config, False, False)


def simple_compress_into(nums, config=None):
    """pco::standalone::simple_compress_into flavour (uniform-type header, pco/src/standalone/simple.rs:22-48)."""
    return _compress(nums, config, True, False)


def simple_compress_with_index(nums, config=None, uniform_type=False):
    """simple_compress plus the per-batch side index the GPU decoder uses (metadata beside the .pco bytes)."""
    return _compress(nums, config, uniform_type, True)


def decompress_chunks(src, dtype, chunk_offsets, chunk_ns):
    """Batched, index-free decompress of chunks at known byte offsets (pco_b200_decompress_chunks): `src` is a standalone
    file or bare chunks back to back; chunk_offsets[i] = byte offset of chunk i's type byte, chunk_ns[i] = its count.
    The device walks every chunk's tANS stream in parallel to build the per-batch index, then decodes."""
    L = _lib.lib()
    arr, n = _src_buf(src)
    offs = np.ascontiguousarray(chunk_offsets, dtype=np.uint64)
    ns = np.ascontiguousarray(chunk_ns, dtype=np.uint32)
    if offs.size != ns.size:
        raise ValueError("chunk_offsets and chunk_ns differ in length")
    dst = np.empty(int(ns.sum(dtype=np.uint64)), dtype=dtype)
    n_written = C.c_size_t()
    rc = L.pco_b200_decompress_chunks(arr.ctypes.data_as(C.c_void_p), C.c_size_t(n), C.c_ubyte(_lib.dtype_byte(dst.dtype)),
                                      offs.ctypes.data_as(C.c_void_p), ns.ctypes.data_as(C.c_void_p), C.c_size_t(offs.size),
                                      dst.ctypes.data_as(C.c_void_p), C.c_size_t(dst.size), C.byref(n_written), C.c_uint32(0), None)
    _lib.check(rc)
    return dst[: n_written.value]


# PcoB200FileRef (include/pco_b200.h): one standalone file of a batch, and its side index (index_len 0 = none)
FILE_REF = np.dtype([("offset", "<u8"), ("len", "<u8"), ("index_offset", "<u8"), ("index_len", "<u8")])
_INDEX_ON_DEVICE = 4


def _lib_files():
    L = _lib.lib()
    if not getattr(L, "_files_ready", False):
        L.pco_b200_compress_files.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_ubyte, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p,
                                              C.c_size_t, C.c_void_p, C.c_uint32, C.c_void_p]
        L.pco_b200_decompress_files.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_ubyte, C.c_void_p, C.c_size_t, C.c_void_p,
                                                C.c_size_t, C.c_void_p, C.POINTER(C.c_size_t), C.c_uint32, C.c_void_p]
        L._files_ready = True
    return L


def _is_cuda(x):
    return getattr(x, "is_cuda", False)


def _stream_of(t):
    import torch

    return C.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


def compress_files(nums, file_ns, config=None, uniform_type=False, with_index=True):
    """Compresses many arrays of one number type in one call (pco_b200_compress_files): file i is the next file_ns[i] numbers of
    `nums`, written as its own standalone file, byte-identical to simple_compress (uniform_type=False) or simple_compress_into
    (True) of those numbers.  Returns (data, files[, index]): the files back to back, one FILE_REF record per file, and - with
    with_index - the files' side indexes at 16-byte aligned offsets.  A torch CUDA tensor gives uint8 CUDA tensors, computed on
    the current stream."""
    from .wrapped import _torch_dtypes

    ns = np.ascontiguousarray(file_ns, dtype=np.uint64).reshape(-1)
    cfg = (config or ChunkConfig())._to_c()
    L = _lib_files()
    if _is_cuda(nums):
        import torch

        t = nums.contiguous().reshape(-1)
        dt = next(k for k, v in _torch_dtypes().items() if v == t.dtype)
        src, flags, stream = C.c_void_p(t.data_ptr()), _lib.SRC_ON_DEVICE | _lib.DST_ON_DEVICE | _INDEX_ON_DEVICE, _stream_of(t)
        total_n = t.numel()

        def alloc(nbytes):
            return torch.empty(max(nbytes, 1), dtype=torch.uint8, device=t.device)

        def ptr(buf):
            return C.c_void_p(buf.data_ptr())
    else:
        arr = np.ascontiguousarray(nums).reshape(-1)
        dt, src, flags, stream, total_n = arr.dtype, arr.ctypes.data_as(C.c_void_p), 0, None, arr.size

        def alloc(nbytes):
            return np.empty(max(nbytes, 1), dtype=np.uint8)

        def ptr(buf):
            return buf.ctypes.data_as(C.c_void_p)
    if int(ns.sum()) != total_n:
        raise ValueError(f"file_ns add up to {int(ns.sum())} numbers, nums holds {total_n}")
    dtb = _lib.dtype_byte(dt)
    page_n = cfg.max_page_n or (1 << 18)
    chunks = [int(cfg.n_exact_pages) if cfg.paging_spec == 1 else -(-int(n) // page_n) for n in ns]
    cap = sum(L.pco_standalone_guarantee_file_size(int(n), dtb) + 160 * k for n, k in zip(ns, chunks))
    icap = sum(L.pco_b200_index_size_bound(int(n), k) + 64 * k + 16 for n, k in zip(ns, chunks)) if with_index else 0
    files = np.zeros(max(ns.size, 1), dtype=FILE_REF)
    for attempt in range(2):  # a first guess of the capacities, then what the call reported it needs
        data = alloc(cap)
        index = alloc(icap) if with_index else None
        rc = L.pco_b200_compress_files(src, ns.ctypes.data_as(C.c_void_p), C.c_size_t(ns.size), C.c_ubyte(dtb), C.byref(cfg), C.c_int(1 if uniform_type else 0),
                                       ptr(data), C.c_size_t(cap), ptr(index) if with_index else None, C.c_size_t(icap), files.ctypes.data_as(C.c_void_p),
                                       C.c_uint32(flags), stream)
        if rc == 4 and attempt == 0 and ns.size:  # PCO_B200_IO: the refs report the sizes needed
            last = files[ns.size - 1]
            cap = max(cap, int(last["offset"] + last["len"]))
            icap = max(icap, int(last["index_offset"] + last["index_len"]))
            continue
        _lib.check(rc)
        break
    files = files[: ns.size].copy()
    used = int(files[-1]["offset"] + files[-1]["len"]) if ns.size else 0
    iused = int(files[-1]["index_offset"] + files[-1]["index_len"]) if ns.size and with_index else 0
    if _is_cuda(nums):
        out = (data[:used], files)
        return out + (index[:iused],) if with_index else out
    out = (data[:used].tobytes(), files)
    return out + (index[:iused].tobytes(),) if with_index else out


def decompress_files(data, files, dtype, index=None):
    """Decodes every standalone file `files` (FILE_REF records) names into one array, file after file in `files` order
    (pco_b200_decompress_files).  Returns (values, file_ns).  Files with index_len > 0 are decoded through their side index in
    `index`.  `data` and `index` are bytes / numpy, or torch CUDA tensors (then `values` is a CUDA tensor, computed on the current
    stream)."""
    from .wrapped import _host_u8, _torch_dtypes

    dt = np.dtype(dtype)
    r = np.ascontiguousarray(np.asarray(files).astype(FILE_REF, copy=False)).reshape(-1)
    L = _lib_files()
    nf = r.size
    file_ns = np.zeros(max(nf, 1), dtype=np.uint64)
    nw = C.c_size_t()
    cuda = _is_cuda(data)
    if cuda:
        import torch

        d = data.contiguous().reshape(-1)
        ix = index.contiguous().reshape(-1) if index is not None else None
        # the headers' count hints size the destination (grown if the files hold more)
        pos = torch.as_tensor(r["offset"].astype(np.int64), device=d.device)[:, None] + torch.arange(32, device=d.device)[None, :]
        heads = d[pos.clamp_(max=max(d.numel() - 1, 0))].cpu().numpy() if nf and d.numel() else np.zeros((nf, 32), np.uint8)
        src_p, src_len = C.c_void_p(d.data_ptr()), d.numel()
        idx_p, idx_len = (C.c_void_p(ix.data_ptr()), ix.numel()) if ix is not None else (None, 0)
        flags, stream = _lib.SRC_ON_DEVICE | _lib.DST_ON_DEVICE | (_INDEX_ON_DEVICE if ix is not None else 0), _stream_of(d)

        def alloc(n):
            return torch.empty(max(n, 1), dtype=_torch_dtypes()[dt], device=d.device)

        def ptr(buf):
            return C.c_void_p(buf.data_ptr())
    else:
        d = _host_u8(data)
        ix = _host_u8(index) if index is not None else None
        heads = np.stack([np.frombuffer(d[int(o):int(o) + 32].tobytes().ljust(32, b"\0"), np.uint8) for o in r["offset"]]) if nf else np.zeros((0, 32), np.uint8)
        src_p, src_len = d.ctypes.data_as(C.c_void_p), d.size
        idx_p, idx_len = (ix.ctypes.data_as(C.c_void_p), ix.size) if ix is not None else (None, 0)
        flags, stream = 0, None

        def alloc(n):
            return np.empty(max(n, 1), dtype=dt)

        def ptr(buf):
            return buf.ctypes.data_as(C.c_void_p)
    cap = sum(n_hint(heads[k, : int(min(r["len"][k], 32))].tobytes()) for k in range(nf))
    while True:
        dst = alloc(cap)
        rc = L.pco_b200_decompress_files(src_p, C.c_size_t(src_len), idx_p, C.c_size_t(idx_len), C.c_ubyte(_lib.dtype_byte(dt)), r.ctypes.data_as(C.c_void_p),
                                         C.c_size_t(nf), ptr(dst), C.c_size_t(cap), file_ns.ctypes.data_as(C.c_void_p), C.byref(nw), C.c_uint32(flags), stream)
        if rc == 4 and "dst holds" in _lib.lib().pco_b200_last_error_message().decode():  # the hints were short
            cap = max(2 * cap, 1 << 16)
            continue
        _lib.check(rc)
        return dst[: nw.value], file_ns[:nf].copy()


# PcoB200Range (include/pco_b200.h): numbers [start, start + count) of a file
RANGE = np.dtype([("start", "<u8"), ("count", "<u8")])


def _ranges_array(ranges):
    a = np.asarray(ranges)
    if a.dtype.names:
        return np.ascontiguousarray(a.astype(RANGE, copy=False)).reshape(-1)
    a = a.reshape(-1, 2) if a.size else a.reshape(0, 2)
    if a.dtype.kind not in "iu":
        raise TypeError(f"ranges must be integers, got {a.dtype}")
    if a.dtype.kind == "i" and a.size and a.min() < 0:
        raise ValueError("ranges must not be negative")
    r = np.zeros(a.shape[0], dtype=RANGE)
    r["start"], r["count"] = a[:, 0], a[:, 1]
    return r


def decompress_ranges(data, dtype, index, ranges):
    """Decodes ranges of numbers of one standalone file (pco_b200_decompress_ranges): range i lands right behind range i - 1.  Only
    the chunks a range touches are decoded, and in chunks of delta order 0 only the batches it touches.  `ranges` is a numpy array of
    RANGE records or an (m, 2) integer array of (start, count); ranges may overlap, repeat and come in any order.  `index` is the
    file's side index; index=None builds it first with build_index, which walks the whole file serially on the device (keep the index
    from compress for repeated reads).  `data` and `index` are bytes / numpy, or torch CUDA tensors (then the result is a CUDA tensor,
    computed on the current stream)."""
    from .wrapped import _host_u8, _torch_dtypes

    dt = np.dtype(dtype)
    r = _ranges_array(ranges)
    total = int(r["count"].sum(dtype=np.uint64)) if r.size else 0
    L = _lib.lib()
    nw = C.c_size_t()
    if _is_cuda(data):
        import torch

        d = data.contiguous().reshape(-1)
        if index is None:
            index = torch.as_tensor(np.frombuffer(build_index(d.cpu().numpy().tobytes(), dt), np.uint8).copy(), device=d.device)
        ix = index.contiguous().reshape(-1) if _is_cuda(index) else torch.as_tensor(_host_u8(index).copy(), device=d.device)
        dst = torch.empty(max(total, 1), dtype=_torch_dtypes()[dt], device=d.device)
        flags = _lib.SRC_ON_DEVICE | _lib.DST_ON_DEVICE | _INDEX_ON_DEVICE
        rc = L.pco_b200_decompress_ranges(C.c_void_p(d.data_ptr()), C.c_size_t(d.numel()), C.c_ubyte(_lib.dtype_byte(dt)), C.c_void_p(ix.data_ptr()),
                                          C.c_size_t(ix.numel()), r.ctypes.data_as(C.c_void_p), C.c_size_t(r.size), C.c_void_p(dst.data_ptr()),
                                          C.c_size_t(total), C.byref(nw), C.c_uint32(flags), _stream_of(d))
        _lib.check(rc)
        return dst[: nw.value]
    d = _host_u8(data)
    if index is None:
        index = build_index(d.tobytes(), dt)
    ix = _host_u8(index)
    dst = np.empty(max(total, 1), dtype=dt)
    rc = L.pco_b200_decompress_ranges(d.ctypes.data_as(C.c_void_p), C.c_size_t(d.size), C.c_ubyte(_lib.dtype_byte(dt)), ix.ctypes.data_as(C.c_void_p),
                                      C.c_size_t(ix.size), r.ctypes.data_as(C.c_void_p), C.c_size_t(r.size), dst.ctypes.data_as(C.c_void_p),
                                      C.c_size_t(total), C.byref(nw), C.c_uint32(0), None)
    _lib.check(rc)
    return dst[: nw.value]


class _CAsyncPlan(C.Structure):  # PcoB200AsyncPlan (include/pco_b200.h)
    _fields_ = [("dtype", C.c_uint32), ("uniform_type", C.c_uint32), ("format_major", C.c_uint32), ("reserved", C.c_uint32),
                ("src_cap", C.c_uint64), ("index_cap", C.c_uint64), ("dst_cap", C.c_uint64), ("max_chunks", C.c_uint64),
                ("workspace_bytes", C.c_uint64)]


class _CAsyncStatus(C.Structure):  # PcoB200AsyncStatus (include/pco_b200.h)
    _fields_ = [("kind", C.c_uint32), ("device_status", C.c_uint32), ("chunk", C.c_uint64), ("n_processed", C.c_uint64),
                ("finished", C.c_uint32), ("n_chunks", C.c_uint32)]


def _lib_async():
    return _lib.bind("_async_ready",
                     pco_b200_decompress_async_plan=[C.c_void_p, C.c_size_t, C.c_ubyte, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p],
                     pco_b200_decompress_async=[C.c_void_p] * 7,
                     pco_b200_decompress_async_result=[C.c_void_p, C.c_void_p])


class AsyncDecompressor(_lib._AsyncCall):
    """Decodes indexed standalone files on the current CUDA stream without waiting for the device (pco_b200_decompress_async): a call
    only enqueues kernels, so it can run behind other GPU work while the host moves on, and it can be captured in a torch.cuda.CUDAGraph.

    The plan comes from `head`, the first bytes of a file (32 suffice; bytes, numpy or a tensor): it fixes the number type `dtype`, the
    header flavour (uniform type) and the format version of every file decoded with it.  src_cap, index_cap (bytes) and dst_cap (numbers)
    are the sizes of the buffers every call passes, max_chunks the most chunks a file may have.  The file length, chunk count and number
    count come from each file's side index on the device, so one captured call decodes whatever file its buffers hold on each replay.
    The decompressor owns a device workspace and a status word; it serves one call in flight at a time (calls on one stream queue up)."""

    _Plan, _Status = _CAsyncPlan, _CAsyncStatus

    def __init__(self, head, dtype, src_cap, index_cap, dst_cap, max_chunks, device=None):
        self.dtype = np.dtype(dtype)
        h = self._head(head)
        self._make_plan(device, lambda plan: _lib_async().pco_b200_decompress_async_plan(
            h.ctypes.data_as(C.c_void_p), C.c_size_t(h.size), C.c_ubyte(_lib.dtype_byte(self.dtype)), C.c_size_t(src_cap), C.c_size_t(index_cap),
            C.c_size_t(dst_cap), C.c_size_t(max_chunks), plan))
        self._alloc()

    def __call__(self, src, index, dst):
        """Enqueues the decode of the file in `src` (uint8 CUDA tensor of at least src_cap bytes) through its side index `index` (at least
        index_cap bytes) into `dst` (a CUDA tensor of the plan's dtype, at least dst_cap numbers) on torch.cuda.current_stream().  Returns
        nothing and does not wait; result() reports the outcome."""
        from .wrapped import _torch_dtypes

        p = self._plan
        self._check_tensors(src=src, index=index, dst=dst)
        if src.numel() * src.element_size() < p.src_cap or index.numel() * index.element_size() < p.index_cap:
            raise ValueError(f"src holds fewer than src_cap = {p.src_cap} bytes, or index fewer than index_cap = {p.index_cap}")
        if dst.dtype != _torch_dtypes()[self.dtype] or dst.numel() < p.dst_cap:
            raise ValueError(f"dst must hold at least dst_cap = {p.dst_cap} numbers of {self.dtype}")
        rc = _lib_async().pco_b200_decompress_async(C.byref(p), C.c_void_p(src.data_ptr()), C.c_void_p(index.data_ptr()), C.c_void_p(dst.data_ptr()),
                                                    C.c_void_p(self.workspace.data_ptr()), C.c_void_p(self.status.data_ptr()), self._stream())
        _lib.check(rc)

    def result(self):
        """Copies the status of the last call back (waiting for it on the current stream) and returns its Progress, or raises PcoError
        with the kind pco_b200_decompress_ex gives."""
        s = self.status_record()
        prog = _lib._CProgress()
        _lib.check(_lib_async().pco_b200_decompress_async_result(C.byref(s), C.byref(prog)))
        return Progress(prog.n_processed, bool(prog.finished))


class _CAsyncIndexPlan(C.Structure):  # PcoB200AsyncIndexPlan (include/pco_b200.h)
    _fields_ = [("dtype", C.c_uint32), ("uniform_type", C.c_uint32), ("format_major", C.c_uint32), ("reserved", C.c_uint32),
                ("src_cap", C.c_uint64), ("index_cap", C.c_uint64), ("max_chunks", C.c_uint64), ("workspace_bytes", C.c_uint64)]


class _CAsyncIndexStatus(C.Structure):  # PcoB200AsyncIndexStatus (include/pco_b200.h)
    _fields_ = [("kind", C.c_uint32), ("device_status", C.c_uint32), ("chunk", C.c_uint64), ("n_chunks", C.c_uint64), ("n_total", C.c_uint64),
                ("index_bytes", C.c_uint64), ("serial_chunks", C.c_uint64)]


def _lib_async_index():
    return _lib.bind("_async_index_ready",
                     pco_b200_build_index_async_plan=[C.c_void_p, C.c_size_t, C.c_ubyte, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p],
                     pco_b200_build_index_async=[C.c_void_p] * 7,
                     pco_b200_build_index_async_result=[C.c_void_p, C.POINTER(C.c_size_t)])


class AsyncIndexBuilder(_lib._AsyncCall):
    """Builds the side index of a standalone file without one (as pco writes them) on the current CUDA stream without waiting for the
    device (pco_b200_build_index_async): a file loaded into device memory can be indexed behind other GPU work, and "build the index, then
    AsyncDecompressor" can be captured in one torch.cuda.CUDAGraph.

    The plan comes from `head`, the first bytes of a file (as AsyncDecompressor).  src_cap and index_cap (bytes) are the sizes of the
    buffers every call passes, max_chunks the most chunks a file may have.  The file length is read from a device tensor, so one captured
    call indexes a different file on each replay.  The builder owns a device workspace and a status; it serves one call in flight."""

    _Plan, _Status = _CAsyncIndexPlan, _CAsyncIndexStatus

    def __init__(self, head, dtype, src_cap, index_cap, max_chunks, device=None):
        self.dtype = np.dtype(dtype)
        h = self._head(head)
        self._make_plan(device, lambda plan: _lib_async_index().pco_b200_build_index_async_plan(
            h.ctypes.data_as(C.c_void_p), C.c_size_t(h.size), C.c_ubyte(_lib.dtype_byte(self.dtype)), C.c_size_t(src_cap), C.c_size_t(index_cap),
            C.c_size_t(max_chunks), plan))
        self._alloc()

    def __call__(self, src, src_len, index):
        """Enqueues the indexing of the file of src_len[0] bytes in `src` (uint8 CUDA tensor of at least src_cap bytes) into `index` (a
        16-byte aligned uint8 CUDA tensor of at least index_cap bytes) on torch.cuda.current_stream(); `src_len` is a 1-element int64 CUDA
        tensor.  Returns nothing and does not wait; result() reports the outcome."""
        import torch

        p = self._plan
        self._check_tensors(src=src, src_len=src_len, index=index)
        if src.numel() * src.element_size() < p.src_cap or index.numel() * index.element_size() < p.index_cap:
            raise ValueError(f"src holds fewer than src_cap = {p.src_cap} bytes, or index fewer than index_cap = {p.index_cap}")
        if src_len.dtype != torch.int64 or src_len.numel() != 1:
            raise ValueError("src_len must be a 1-element int64 tensor")
        rc = _lib_async_index().pco_b200_build_index_async(C.byref(p), C.c_void_p(src.data_ptr()), C.c_void_p(src_len.data_ptr()),
                                                           C.c_void_p(index.data_ptr()), C.c_void_p(self.workspace.data_ptr()),
                                                           C.c_void_p(self.status.data_ptr()), self._stream())
        _lib.check(rc)

    def result(self):
        """Copies the status of the last call back (waiting for it on the current stream) and returns the index length in bytes, or raises
        PcoError with the kind build_index gives ("chunk 17: ...")."""
        s = self.status_record()
        n = C.c_size_t()
        _lib.check(_lib_async_index().pco_b200_build_index_async_result(C.byref(s), C.byref(n)))
        return int(n.value)


class _CAsyncRangesPlan(C.Structure):  # PcoB200AsyncRangesPlan (include/pco_b200.h)
    _fields_ = [("dtype", C.c_uint32), ("uniform_type", C.c_uint32), ("format_major", C.c_uint32), ("reserved", C.c_uint32),
                ("src_cap", C.c_uint64), ("index_cap", C.c_uint64), ("max_chunks", C.c_uint64), ("max_ranges", C.c_uint64),
                ("dst_cap", C.c_uint64), ("window_cap", C.c_uint64), ("workspace_bytes", C.c_uint64)]


class _CAsyncRangesStatus(C.Structure):  # PcoB200AsyncRangesStatus (include/pco_b200.h)
    _fields_ = [("kind", C.c_uint32), ("device_status", C.c_uint32), ("range", C.c_uint64), ("chunk", C.c_uint64), ("n_written", C.c_uint64),
                ("window_needed", C.c_uint64)]


def _lib_async_ranges():
    return _lib.bind("_async_ranges_ready",
                     pco_b200_decompress_ranges_async_plan=[C.c_void_p, C.c_size_t, C.c_ubyte, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t,
                                                            C.c_size_t, C.c_size_t, C.c_void_p],
                     pco_b200_decompress_ranges_async=[C.c_void_p] * 9,
                     pco_b200_decompress_ranges_async_result=[C.c_void_p, C.POINTER(C.c_size_t)])


class AsyncRangeDecompressor(_lib._AsyncCall):
    """Decodes ranges of indexed standalone files on the current CUDA stream with the ranges in device memory and without waiting for the
    device (pco_b200_decompress_ranges_async): positions a kernel produced need no trip to the host, and a call can be captured in a
    torch.cuda.CUDAGraph.

    The plan comes from `head`, the first bytes of a file (as AsyncDecompressor).  src_cap, index_cap (bytes) and dst_cap (numbers) are the
    sizes of the buffers every call passes, max_chunks the most chunks a file may have, max_ranges the most ranges of a call, and
    window_cap the most window numbers a call may need (include/pco_b200.h: the sum over touched chunks of the end of the last number
    wanted, rounded up to 256).  The number of ranges is read from a device tensor, so one captured call serves a different count, different
    ranges and a different file on each replay.  The decompressor owns a device workspace and a status; it serves one call in flight."""

    _Plan, _Status = _CAsyncRangesPlan, _CAsyncRangesStatus

    def __init__(self, head, dtype, src_cap, index_cap, max_chunks, max_ranges, dst_cap, window_cap, device=None):
        self.dtype = np.dtype(dtype)
        h = self._head(head)
        self._make_plan(device, lambda plan: _lib_async_ranges().pco_b200_decompress_ranges_async_plan(
            h.ctypes.data_as(C.c_void_p), C.c_size_t(h.size), C.c_ubyte(_lib.dtype_byte(self.dtype)), C.c_size_t(src_cap), C.c_size_t(index_cap),
            C.c_size_t(max_chunks), C.c_size_t(max_ranges), C.c_size_t(dst_cap), C.c_size_t(window_cap), plan))
        self._alloc()

    def __call__(self, src, index, ranges, n_ranges, dst):
        """Enqueues the decode of ranges[: n_ranges[0]] of the file in `src` (uint8 CUDA tensor of at least src_cap bytes) through its side
        index `index` (at least index_cap bytes) into `dst` (a CUDA tensor of the plan's dtype, at least dst_cap numbers) on
        torch.cuda.current_stream().  `ranges` is an int64 CUDA tensor of shape (max_ranges, 2) of (start, count), `n_ranges` a 1-element
        int64 CUDA tensor.  Returns nothing and does not wait; result() reports the outcome."""
        import torch

        from .wrapped import _torch_dtypes

        p = self._plan
        self._check_tensors(src=src, index=index, ranges=ranges, n_ranges=n_ranges, dst=dst)
        if src.numel() * src.element_size() < p.src_cap or index.numel() * index.element_size() < p.index_cap:
            raise ValueError(f"src holds fewer than src_cap = {p.src_cap} bytes, or index fewer than index_cap = {p.index_cap}")
        if ranges.dtype != torch.int64 or ranges.dim() != 2 or ranges.shape[1] != 2 or ranges.shape[0] < p.max_ranges:
            raise ValueError(f"ranges must be an int64 tensor of shape ({p.max_ranges}, 2)")
        if n_ranges.dtype != torch.int64 or n_ranges.numel() != 1:
            raise ValueError("n_ranges must be a 1-element int64 tensor")
        if dst.dtype != _torch_dtypes()[self.dtype] or dst.numel() < p.dst_cap:
            raise ValueError(f"dst must hold at least dst_cap = {p.dst_cap} numbers of {self.dtype}")
        rc = _lib_async_ranges().pco_b200_decompress_ranges_async(
            C.byref(p), C.c_void_p(src.data_ptr()), C.c_void_p(index.data_ptr()), C.c_void_p(ranges.data_ptr()), C.c_void_p(n_ranges.data_ptr()),
            C.c_void_p(dst.data_ptr()), C.c_void_p(self.workspace.data_ptr()), C.c_void_p(self.status.data_ptr()), self._stream())
        _lib.check(rc)

    def result(self):
        """Copies the status of the last call back (waiting for it on the current stream) and returns the number of numbers written, or
        raises PcoError with the kind pco_b200_decompress_ranges gives."""
        s = self.status_record()
        nw = C.c_size_t()
        _lib.check(_lib_async_ranges().pco_b200_decompress_ranges_async_result(C.byref(s), C.byref(nw)))
        return int(nw.value)


class _CAsyncCompressPlan(C.Structure):  # PcoB200AsyncCompressPlan (include/pco_b200.h)
    _fields_ = [("dtype", C.c_uint32), ("uniform_type_header", C.c_uint32), ("mode", C.c_uint32), ("order", C.c_uint32),
                ("n_vars", C.c_uint32), ("bins_log", C.c_uint32), ("mode_k", C.c_uint32), ("reserved", C.c_uint32),
                ("n", C.c_uint64), ("max_page_n", C.c_uint64), ("dst_cap", C.c_uint64), ("index_cap", C.c_uint64),
                ("mode_base", C.c_uint64), ("base_bits", C.c_uint64), ("inv_base_bits", C.c_uint64),
                ("index_bytes", C.c_uint64), ("workspace_bytes", C.c_uint64)]


class _CAsyncCompressStatus(C.Structure):  # PcoB200AsyncCompressStatus (include/pco_b200.h)
    _fields_ = [("kind", C.c_uint32), ("device_status", C.c_uint32), ("file_bytes", C.c_uint64), ("n_written", C.c_uint64),
                ("index_bytes", C.c_uint64)]


def _lib_async_compress():
    return _lib.bind("_async_compress_ready",
                     pco_b200_compress_async_plan=[C.c_size_t, C.c_ubyte, C.c_void_p, C.c_int, C.c_size_t, C.c_size_t, C.c_void_p],
                     pco_b200_compress_async=[C.c_void_p] * 7,
                     pco_b200_compress_async_result=[C.c_void_p, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)])


class AsyncCompressor(_lib._AsyncCall):
    """Compresses n numbers on the current CUDA stream without waiting for the device (pco_b200_compress_async): a call only enqueues
    kernels, so it can run behind other GPU work while the host moves on, and it can be captured in a torch.cuda.CUDAGraph.

    The plan fixes n, the number type `dtype`, the config (explicit mode and delta specs, levels up to 8, EqualPagesUpTo paging), the
    header flavour (uniform_type_header: as simple_compress_into) and the capacities: dst_cap bytes of file (default: the size guarantee
    pco_standalone_guarantee_file_size) and, with index=True, the exact size of the side index.  The numbers are read when the call runs,
    so a captured call compresses whatever its input tensor holds on each replay.  The bytes equal what compress_ex writes for the same
    numbers and config.  The compressor owns a device workspace and a status word; it serves one call in flight at a time (calls on one
    stream queue up)."""

    _Plan, _Status = _CAsyncCompressPlan, _CAsyncCompressStatus

    def __init__(self, n, dtype, config=None, dst_cap=None, index=True, uniform_type_header=False, device=None):
        self.dtype = np.dtype(dtype)
        self.n = int(n)
        dtb = _lib.dtype_byte(self.dtype)
        L = _lib_async_compress()
        if dst_cap is None:
            dst_cap = L.pco_standalone_guarantee_file_size(self.n, dtb)
        cfg = (config or ChunkConfig())._to_c()

        def plan_fn(index_cap):
            return lambda plan: L.pco_b200_compress_async_plan(C.c_size_t(self.n), C.c_ubyte(dtb), C.byref(cfg), C.c_int(1 if uniform_type_header else 0),
                                                               C.c_size_t(dst_cap), C.c_size_t(index_cap), plan)

        # the exact index size is known once the plan exists: a first plan without an index reports it
        self._make_plan(device, plan_fn(0))
        if index:
            self._replan(plan_fn(self._plan.index_bytes))
        self._alloc()

    @property
    def dst_cap(self):
        return int(self._plan.dst_cap)

    @property
    def index_bytes(self):
        """Bytes of the side index each call writes (0 without one)."""
        return int(self._plan.index_cap and self._plan.index_bytes)

    def __call__(self, nums, dst, index=None):
        """Enqueues the compress of `nums` (a CUDA tensor of the plan's dtype and n numbers) into `dst` (uint8 CUDA tensor of at least dst_cap
        bytes) and, when given, the side index into `index` (uint8 CUDA tensor of at least index_bytes bytes) on torch.cuda.current_stream().
        Returns nothing and does not wait; result() reports the outcome."""
        from .wrapped import _torch_dtypes

        p = self._plan
        self._check_tensors(nums=nums, dst=dst, **({"index": index} if index is not None else {}))
        if nums.dtype != _torch_dtypes()[self.dtype] or nums.numel() != self.n:
            raise ValueError(f"nums must hold n = {self.n} numbers of {self.dtype}")
        if dst.numel() * dst.element_size() < p.dst_cap:
            raise ValueError(f"dst holds fewer than dst_cap = {p.dst_cap} bytes")
        if index is not None and (not p.index_cap or index.numel() * index.element_size() < p.index_bytes):
            raise ValueError(f"index needs a compressor made with index=True and at least {p.index_bytes} bytes")
        rc = _lib_async_compress().pco_b200_compress_async(C.byref(p), C.c_void_p(nums.data_ptr()), C.c_void_p(dst.data_ptr()),
                                                          C.c_void_p(index.data_ptr()) if index is not None else None,
                                                          C.c_void_p(self.workspace.data_ptr()), C.c_void_p(self.status.data_ptr()), self._stream())
        _lib.check(rc)

    def result(self):
        """Copies the status of the last call back (waiting for it on the current stream) and returns (file_bytes, index_bytes), or raises
        PcoError (Io when the file does not fit dst_cap)."""
        s = self.status_record()
        nw, il = C.c_size_t(), C.c_size_t()
        _lib.check(_lib_async_compress().pco_b200_compress_async_result(C.byref(s), C.byref(nw), C.byref(il)))
        return int(nw.value), int(il.value)


class _CAsyncFilesPlan(C.Structure):  # PcoB200AsyncFilesPlan (include/pco_b200.h)
    _fields_ = [("dtype", C.c_uint32), ("uniform_type", C.c_uint32), ("format_major", C.c_uint32), ("reserved", C.c_uint32),
                ("src_cap", C.c_uint64), ("index_cap", C.c_uint64), ("max_files", C.c_uint64), ("max_chunks", C.c_uint64),
                ("dst_cap", C.c_uint64), ("workspace_bytes", C.c_uint64)]


class _CAsyncFilesStatus(C.Structure):  # PcoB200AsyncFilesStatus (include/pco_b200.h)
    _fields_ = [("kind", C.c_uint32), ("device_status", C.c_uint32), ("file", C.c_uint64), ("chunk", C.c_uint64), ("n_written", C.c_uint64),
                ("n_files", C.c_uint64)]


def _lib_async_files():
    return _lib.bind("_async_files_ready",
                     pco_b200_decompress_files_async_plan=[C.c_void_p, C.c_size_t, C.c_ubyte, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t,
                                                           C.c_size_t, C.c_void_p],
                     pco_b200_decompress_files_async=[C.c_void_p] * 10,
                     pco_b200_decompress_files_async_result=[C.c_void_p, C.POINTER(C.c_size_t)])


class AsyncFilesDecompressor(_lib._AsyncCall):
    """Decodes a batch of indexed standalone files on the current CUDA stream with the file list in device memory and without waiting for
    the device (pco_b200_decompress_files_async): refs a kernel picked (a sampler, a cache lookup) need no trip to the host, and a call can
    be captured in a torch.cuda.CUDAGraph.

    The plan comes from `head`, the first bytes of any file of the batch (as AsyncDecompressor): every file must share its number type and
    header flavour.  src_cap, index_cap (bytes) and dst_cap (numbers) are the sizes of the buffers every call passes, max_files the most
    files of a call and max_chunks the most chunks of a whole batch.  The number of files is read from a device tensor, so one captured call
    serves different refs, a different count and different files on each replay.  The decompressor owns a device workspace and a status;
    it serves one call in flight."""

    _Plan, _Status = _CAsyncFilesPlan, _CAsyncFilesStatus

    def __init__(self, head, dtype, src_cap, index_cap, max_files, max_chunks, dst_cap, device=None):
        self.dtype = np.dtype(dtype)
        h = self._head(head)
        self._make_plan(device, lambda plan: _lib_async_files().pco_b200_decompress_files_async_plan(
            h.ctypes.data_as(C.c_void_p), C.c_size_t(h.size), C.c_ubyte(_lib.dtype_byte(self.dtype)), C.c_size_t(src_cap), C.c_size_t(index_cap),
            C.c_size_t(max_files), C.c_size_t(max_chunks), C.c_size_t(dst_cap), plan))
        self._alloc()

    def __call__(self, src, index, files, n_files, dst, file_ns):
        """Enqueues the decode of files[: n_files[0]] into `dst` (a CUDA tensor of the plan's dtype, at least dst_cap numbers) on
        torch.cuda.current_stream(): file i lands right behind file i - 1 and file_ns[i] gets its count.  `src` and `index` are uint8 CUDA
        tensors of at least src_cap and index_cap bytes; `files` is an int64 CUDA tensor of shape (max_files, 4) holding the FILE_REF
        fields (offset, len, index_offset, index_len), `n_files` a 1-element int64 CUDA tensor, `file_ns` an int64 CUDA tensor of at least
        max_files elements.  Returns nothing and does not wait; result() reports the outcome."""
        import torch

        from .wrapped import _torch_dtypes

        p = self._plan
        self._check_tensors(src=src, index=index, files=files, n_files=n_files, dst=dst, file_ns=file_ns)
        if src.numel() * src.element_size() < p.src_cap or index.numel() * index.element_size() < p.index_cap:
            raise ValueError(f"src holds fewer than src_cap = {p.src_cap} bytes, or index fewer than index_cap = {p.index_cap}")
        if files.dtype != torch.int64 or files.dim() != 2 or files.shape[1] != 4 or files.shape[0] < p.max_files:
            raise ValueError(f"files must be an int64 tensor of shape ({p.max_files}, 4)")
        if n_files.dtype != torch.int64 or n_files.numel() != 1:
            raise ValueError("n_files must be a 1-element int64 tensor")
        if file_ns.dtype != torch.int64 or file_ns.numel() < p.max_files:
            raise ValueError(f"file_ns must be an int64 tensor of at least max_files = {p.max_files} elements")
        if dst.dtype != _torch_dtypes()[self.dtype] or dst.numel() < p.dst_cap:
            raise ValueError(f"dst must hold at least dst_cap = {p.dst_cap} numbers of {self.dtype}")
        rc = _lib_async_files().pco_b200_decompress_files_async(
            C.byref(p), C.c_void_p(src.data_ptr()), C.c_void_p(index.data_ptr()), C.c_void_p(files.data_ptr()), C.c_void_p(n_files.data_ptr()),
            C.c_void_p(dst.data_ptr()), C.c_void_p(file_ns.data_ptr()), C.c_void_p(self.workspace.data_ptr()), C.c_void_p(self.status.data_ptr()),
            self._stream())
        _lib.check(rc)

    def result(self):
        """Copies the status of the last call back (waiting for it on the current stream) and returns the number of numbers written, or
        raises PcoError with the kind pco_b200_decompress_files gives ("file 17: ...")."""
        s = self.status_record()
        nw = C.c_size_t()
        _lib.check(_lib_async_files().pco_b200_decompress_files_async_result(C.byref(s), C.byref(nw)))
        return int(nw.value)


class _CAsyncFilesFilterPlan(C.Structure):  # PcoB200AsyncFilesFilterPlan (include/pco_b200.h)
    _fields_ = [("dtype", C.c_uint32), ("uniform_type", C.c_uint32), ("format_major", C.c_uint32), ("reserved", C.c_uint32),
                ("src_cap", C.c_uint64), ("index_cap", C.c_uint64), ("max_files", C.c_uint64), ("max_chunks", C.c_uint64),
                ("rows_cap", C.c_uint64), ("out_cap", C.c_uint64), ("workspace_bytes", C.c_uint64)]


class _CAsyncFilesFilterStatus(C.Structure):  # PcoB200AsyncFilesFilterStatus (include/pco_b200.h)
    _fields_ = [("kind", C.c_uint32), ("device_status", C.c_uint32), ("file", C.c_uint64), ("chunk", C.c_uint64), ("n_written", C.c_uint64),
                ("n_files", C.c_uint64), ("n_matches", C.c_uint64), ("matches_needed", C.c_uint64)]


def _lib_async_filter_files():
    return _lib.bind("_async_filter_files_ready",
                     pco_b200_filter_files_async_plan=[C.c_void_p, C.c_size_t, C.c_ubyte, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t,
                                                       C.c_size_t, C.c_size_t, C.c_void_p],
                     pco_b200_filter_files_async=[C.c_void_p] * 13,
                     pco_b200_filter_files_async_result=[C.c_void_p, C.POINTER(C.c_size_t)])


class AsyncFilesFilter(_lib._AsyncCall):
    """Decodes a batch of indexed standalone files on the current CUDA stream and writes only the numbers inside a closed interval, in row
    order, with their positions in the files' concatenation (pco_b200_filter_files_async): the predicate runs inside the decoder, so the
    decoded files never reach HBM whole.  Refs, their count and the interval are read from device tensors, so one captured call serves new
    files and new bounds on each replay.

    The plan and capacities are AsyncFilesDecompressor's, with rows_cap (the most numbers of a call's files) in place of dst_cap, and
    out_cap the most matches a call writes.  The filter owns a device workspace (about rows_cap * (itemsize + 1) bytes beyond the
    decompressor's) and a status; it serves one call in flight."""

    _Plan, _Status = _CAsyncFilesFilterPlan, _CAsyncFilesFilterStatus

    def __init__(self, head, dtype, src_cap, index_cap, max_files, max_chunks, rows_cap, out_cap, device=None):
        self.dtype = np.dtype(dtype)
        h = self._head(head)
        self._make_plan(device, lambda plan: _lib_async_filter_files().pco_b200_filter_files_async_plan(
            h.ctypes.data_as(C.c_void_p), C.c_size_t(h.size), C.c_ubyte(_lib.dtype_byte(self.dtype)), C.c_size_t(src_cap), C.c_size_t(index_cap),
            C.c_size_t(max_files), C.c_size_t(max_chunks), C.c_size_t(rows_cap), C.c_size_t(out_cap), plan))
        self._alloc()

    def __call__(self, src, index, files, n_files, interval, values, positions, n_matches, file_ns=None):
        """Enqueues the filter of files[: n_files[0]] on torch.cuda.current_stream().  `src`, `index`, `files` and `n_files` are as
        AsyncFilesDecompressor takes them; `interval` is a 2-element int64 CUDA tensor (wrapped.pack_interval's bit patterns of lo and hi),
        `values` a CUDA tensor of the plan's dtype and `positions` an int64 CUDA tensor, each of at least out_cap elements, `n_matches` a
        1-element int64 CUDA tensor that receives the count, and `file_ns` (optional) an int64 CUDA tensor of at least max_files elements
        that receives each file's count.  Returns nothing and does not wait; result() reports the outcome."""
        import torch

        from .wrapped import _torch_dtypes

        p = self._plan
        self._check_tensors(src=src, index=index, files=files, n_files=n_files, interval=interval, values=values, positions=positions,
                            n_matches=n_matches, **({} if file_ns is None else {"file_ns": file_ns}))
        if src.numel() * src.element_size() < p.src_cap or index.numel() * index.element_size() < p.index_cap:
            raise ValueError(f"src holds fewer than src_cap = {p.src_cap} bytes, or index fewer than index_cap = {p.index_cap}")
        if files.dtype != torch.int64 or files.dim() != 2 or files.shape[1] != 4 or files.shape[0] < p.max_files:
            raise ValueError(f"files must be an int64 tensor of shape ({p.max_files}, 4)")
        for name, t in (("n_files", n_files), ("n_matches", n_matches)):
            if t.dtype != torch.int64 or t.numel() != 1:
                raise ValueError(f"{name} must be a 1-element int64 tensor")
        if interval.dtype != torch.int64 or interval.numel() != 2:
            raise ValueError("interval must be a 2-element int64 tensor")
        if values.dtype != _torch_dtypes()[self.dtype] or values.numel() < p.out_cap:
            raise ValueError(f"values must hold at least out_cap = {p.out_cap} numbers of {self.dtype}")
        if positions.dtype != torch.int64 or positions.numel() < p.out_cap:
            raise ValueError(f"positions must be an int64 tensor of at least out_cap = {p.out_cap} elements")
        if file_ns is not None and (file_ns.dtype != torch.int64 or file_ns.numel() < p.max_files):
            raise ValueError(f"file_ns must be an int64 tensor of at least max_files = {p.max_files} elements")
        rc = _lib_async_filter_files().pco_b200_filter_files_async(
            C.byref(p), C.c_void_p(src.data_ptr()), C.c_void_p(index.data_ptr()), C.c_void_p(files.data_ptr()), C.c_void_p(n_files.data_ptr()),
            C.c_void_p(interval.data_ptr()), C.c_void_p(values.data_ptr()), C.c_void_p(positions.data_ptr()), C.c_void_p(n_matches.data_ptr()),
            C.c_void_p(None if file_ns is None else file_ns.data_ptr()), C.c_void_p(self.workspace.data_ptr()),
            C.c_void_p(self.status.data_ptr()), self._stream())
        _lib.check(rc)

    def result(self):
        """Copies the status of the last call back (waiting for it on the current stream) and returns the number of matches, or raises
        PcoError with the kind pco_b200_decompress_files gives ("file 3: chunk 2: ..."), or Io when the matches outnumber out_cap."""
        s = self.status_record()
        nm = C.c_size_t()
        _lib.check(_lib_async_filter_files().pco_b200_filter_files_async_result(C.byref(s), C.byref(nm)))
        return int(nm.value)


class _CAsyncFilesAggregatePlan(C.Structure):  # PcoB200AsyncFilesAggregatePlan (include/pco_b200.h)
    _fields_ = [("dtype", C.c_uint32), ("uniform_type", C.c_uint32), ("format_major", C.c_uint32), ("reserved", C.c_uint32),
                ("src_cap", C.c_uint64), ("index_cap", C.c_uint64), ("max_files", C.c_uint64), ("max_chunks", C.c_uint64),
                ("rows_cap", C.c_uint64), ("workspace_bytes", C.c_uint64)]


class _CAsyncFilesAggregateStatus(C.Structure):  # PcoB200AsyncFilesAggregateStatus (include/pco_b200.h)
    _fields_ = [("kind", C.c_uint32), ("device_status", C.c_uint32), ("file", C.c_uint64), ("chunk", C.c_uint64), ("n_written", C.c_uint64),
                ("n_files", C.c_uint64), ("n_matches", C.c_uint64)]


def _lib_async_aggregate_files():
    return _lib.bind("_async_aggregate_files_ready",
                     pco_b200_aggregate_files_async_plan=[C.c_void_p, C.c_size_t, C.c_ubyte, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t,
                                                          C.c_size_t, C.c_void_p],
                     pco_b200_aggregate_files_async=[C.c_void_p] * 11,
                     pco_b200_aggregate_files_async_result=[C.c_void_p, C.POINTER(C.c_size_t)])


class AsyncFilesAggregate(_lib._AsyncCall):
    """Decodes a batch of indexed standalone files on the current CUDA stream and reduces the numbers inside a closed interval to count,
    min, max and sum, per file and in all (pco_b200_aggregate_files_async): each 256-number batch is reduced in the decoder's registers, so
    neither the decoded files nor the matches reach HBM.  Refs, their count and the interval are read from device tensors, so one captured
    call serves new files and new bounds on each replay.

    The plan and capacities are AsyncFilesDecompressor's, with rows_cap (the most numbers of a call's files) in place of dst_cap.  The call
    owns a device workspace (about rows_cap * (itemsize + 0.15) bytes beyond the decompressor's) and a status; it serves one call in
    flight.  wrapped.unpack_aggregates reads the records."""

    _Plan, _Status = _CAsyncFilesAggregatePlan, _CAsyncFilesAggregateStatus

    def __init__(self, head, dtype, src_cap, index_cap, max_files, max_chunks, rows_cap, device=None):
        self.dtype = np.dtype(dtype)
        h = self._head(head)
        self._make_plan(device, lambda plan: _lib_async_aggregate_files().pco_b200_aggregate_files_async_plan(
            h.ctypes.data_as(C.c_void_p), C.c_size_t(h.size), C.c_ubyte(_lib.dtype_byte(self.dtype)), C.c_size_t(src_cap), C.c_size_t(index_cap),
            C.c_size_t(max_files), C.c_size_t(max_chunks), C.c_size_t(rows_cap), plan))
        self._alloc()

    def __call__(self, src, index, files, n_files, interval, aggs, total):
        """Enqueues the aggregates of files[: n_files[0]] on torch.cuda.current_stream().  `src`, `index`, `files` and `n_files` are as
        AsyncFilesDecompressor takes them; `interval` is a 2-element int64 CUDA tensor (wrapped.pack_interval's bit patterns of lo and hi),
        `aggs` an int64 CUDA tensor of shape (max_files, 6) whose row i receives file i's PcoB200Aggregate, and `total` a 6-element int64
        CUDA tensor that receives the total.  Returns nothing and does not wait; result() reports the outcome."""
        import torch

        from .wrapped import _check_aggregate_outputs

        p = self._plan
        self._check_tensors(src=src, index=index, files=files, n_files=n_files, interval=interval, aggs=aggs, total=total)
        if src.numel() * src.element_size() < p.src_cap or index.numel() * index.element_size() < p.index_cap:
            raise ValueError(f"src holds fewer than src_cap = {p.src_cap} bytes, or index fewer than index_cap = {p.index_cap}")
        if files.dtype != torch.int64 or files.dim() != 2 or files.shape[1] != 4 or files.shape[0] < p.max_files:
            raise ValueError(f"files must be an int64 tensor of shape ({p.max_files}, 4)")
        if n_files.dtype != torch.int64 or n_files.numel() != 1:
            raise ValueError("n_files must be a 1-element int64 tensor")
        if interval.dtype != torch.int64 or interval.numel() != 2:
            raise ValueError("interval must be a 2-element int64 tensor")
        _check_aggregate_outputs(aggs, total, p.max_files)
        rc = _lib_async_aggregate_files().pco_b200_aggregate_files_async(
            C.byref(p), C.c_void_p(src.data_ptr()), C.c_void_p(index.data_ptr()), C.c_void_p(files.data_ptr()), C.c_void_p(n_files.data_ptr()),
            C.c_void_p(interval.data_ptr()), C.c_void_p(aggs.data_ptr()), C.c_void_p(total.data_ptr()), C.c_void_p(self.workspace.data_ptr()),
            C.c_void_p(self.status.data_ptr()), self._stream())
        _lib.check(rc)

    def result(self):
        """Copies the status of the last call back (waiting for it on the current stream) and returns the total match count, or raises
        PcoError with the kind pco_b200_decompress_files gives ("file 3: chunk 2: ...")."""
        s = self.status_record()
        nm = C.c_size_t()
        _lib.check(_lib_async_aggregate_files().pco_b200_aggregate_files_async_result(C.byref(s), C.byref(nm)))
        return int(nm.value)


class _CAsyncFilesHistogramPlan(C.Structure):  # PcoB200AsyncFilesHistogramPlan (include/pco_b200.h)
    _fields_ = [("dtype", C.c_uint32), ("uniform_type", C.c_uint32), ("format_major", C.c_uint32), ("reserved", C.c_uint32),
                ("src_cap", C.c_uint64), ("index_cap", C.c_uint64), ("max_files", C.c_uint64), ("max_chunks", C.c_uint64),
                ("rows_cap", C.c_uint64), ("n_buckets", C.c_uint64), ("workspace_bytes", C.c_uint64)]


class _CAsyncFilesHistogramStatus(C.Structure):  # PcoB200AsyncFilesHistogramStatus (include/pco_b200.h)
    _fields_ = [("kind", C.c_uint32), ("device_status", C.c_uint32), ("file", C.c_uint64), ("chunk", C.c_uint64), ("n_written", C.c_uint64),
                ("n_files", C.c_uint64), ("edge", C.c_uint64)]


def _lib_async_histogram_files():
    return _lib.bind("_async_histogram_files_ready",
                     pco_b200_histogram_files_async_plan=[C.c_void_p, C.c_size_t, C.c_ubyte, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t,
                                                          C.c_size_t, C.c_size_t, C.c_void_p],
                     pco_b200_histogram_files_async=[C.c_void_p] * 11,
                     pco_b200_histogram_files_async_result=[C.c_void_p, C.POINTER(C.c_size_t)])


class AsyncFilesHistogram(_lib._AsyncCall):
    """Decodes a batch of indexed standalone files on the current CUDA stream and counts how many numbers fall in each of n_buckets
    buckets, per file and in all (pco_b200_histogram_files_async): each decode CTA counts its numbers in shared memory, so the decoded
    files never reach HBM.  Refs, their count and the edges are read from device tensors, so one captured call serves new files and new
    edges on each replay.  Rows are wrapped.AsyncPagesHistogram's.

    The plan and capacities are AsyncFilesDecompressor's, with rows_cap (the most numbers of a call's files) in place of dst_cap, and
    n_buckets (1 .. 4096) fixed by the plan.  The call owns a device workspace (about rows_cap * itemsize + 8 * (n_buckets + 3) *
    max_files bytes beyond the decompressor's) and a status; it serves one call in flight."""

    _Plan, _Status = _CAsyncFilesHistogramPlan, _CAsyncFilesHistogramStatus

    def __init__(self, head, dtype, src_cap, index_cap, max_files, max_chunks, rows_cap, n_buckets, device=None):
        self.dtype = np.dtype(dtype)
        h = self._head(head)
        self._make_plan(device, lambda plan: _lib_async_histogram_files().pco_b200_histogram_files_async_plan(
            h.ctypes.data_as(C.c_void_p), C.c_size_t(h.size), C.c_ubyte(_lib.dtype_byte(self.dtype)), C.c_size_t(src_cap), C.c_size_t(index_cap),
            C.c_size_t(max_files), C.c_size_t(max_chunks), C.c_size_t(rows_cap), C.c_size_t(n_buckets), plan))
        self._alloc()

    def __call__(self, src, index, files, n_files, edges, hists, total):
        """Enqueues the histograms of files[: n_files[0]] on torch.cuda.current_stream().  `src`, `index`, `files` and `n_files` are as
        AsyncFilesDecompressor takes them; `edges`, `hists` (of shape (max_files, n_buckets + 3)) and `total` are as
        wrapped.AsyncPagesHistogram takes them, row i of hists receiving file i's counts.  Returns nothing and does not wait; result()
        reports the outcome."""
        import torch

        from .wrapped import _check_histogram_inputs

        p = self._plan
        self._check_tensors(src=src, index=index, files=files, n_files=n_files, edges=edges, hists=hists, total=total)
        if src.numel() * src.element_size() < p.src_cap or index.numel() * index.element_size() < p.index_cap:
            raise ValueError(f"src holds fewer than src_cap = {p.src_cap} bytes, or index fewer than index_cap = {p.index_cap}")
        if files.dtype != torch.int64 or files.dim() != 2 or files.shape[1] != 4 or files.shape[0] < p.max_files:
            raise ValueError(f"files must be an int64 tensor of shape ({p.max_files}, 4)")
        if n_files.dtype != torch.int64 or n_files.numel() != 1:
            raise ValueError("n_files must be a 1-element int64 tensor")
        _check_histogram_inputs(edges, hists, total, p.n_buckets, p.max_files)
        rc = _lib_async_histogram_files().pco_b200_histogram_files_async(
            C.byref(p), C.c_void_p(src.data_ptr()), C.c_void_p(index.data_ptr()), C.c_void_p(files.data_ptr()), C.c_void_p(n_files.data_ptr()),
            C.c_void_p(edges.data_ptr()), C.c_void_p(hists.data_ptr()), C.c_void_p(total.data_ptr()), C.c_void_p(self.workspace.data_ptr()),
            C.c_void_p(self.status.data_ptr()), self._stream())
        _lib.check(rc)

    def result(self):
        """Copies the status of the last call back (waiting for it on the current stream) and returns the numbers counted, or raises
        PcoError with the kind pco_b200_decompress_files gives ("file 3: chunk 2: ...") or naming the lowest bad edge ("edge 3: ...")."""
        s = self.status_record()
        n = C.c_size_t()
        _lib.check(_lib_async_histogram_files().pco_b200_histogram_files_async_result(C.byref(s), C.byref(n)))
        return int(n.value)


class _CAsyncFilesTopkPlan(C.Structure):  # PcoB200AsyncFilesTopkPlan (include/pco_b200.h)
    _fields_ = [("dtype", C.c_uint32), ("uniform_type", C.c_uint32), ("format_major", C.c_uint32), ("largest", C.c_uint32),
                ("src_cap", C.c_uint64), ("index_cap", C.c_uint64), ("max_files", C.c_uint64), ("max_chunks", C.c_uint64),
                ("rows_cap", C.c_uint64), ("k", C.c_uint64), ("workspace_bytes", C.c_uint64)]


class _CAsyncFilesTopkStatus(C.Structure):  # PcoB200AsyncFilesTopkStatus (include/pco_b200.h)
    _fields_ = [("kind", C.c_uint32), ("device_status", C.c_uint32), ("file", C.c_uint64), ("chunk", C.c_uint64), ("n_written", C.c_uint64),
                ("n_files", C.c_uint64), ("n_matches", C.c_uint64)]


def _lib_async_topk_files():
    return _lib.bind("_async_topk_files_ready",
                     pco_b200_topk_files_async_plan=[C.c_void_p, C.c_size_t, C.c_ubyte, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t,
                                                     C.c_size_t, C.c_size_t, C.c_int, C.c_void_p],
                     pco_b200_topk_files_async=[C.c_void_p] * 12,
                     pco_b200_topk_files_async_result=[C.c_void_p, C.POINTER(C.c_size_t)])


class AsyncFilesTopK(_lib._AsyncCall):
    """Decodes a batch of indexed standalone files on the current CUDA stream and returns the k smallest (largest=False) or k largest
    (largest=True) numbers inside a closed interval, with their positions in the files' concatenation (pco_b200_topk_files_async), as
    wrapped.AsyncPagesTopK does for pages.  Refs, their count and the interval are read from device tensors, so one captured call serves
    new files and a new interval on each replay.

    The plan and capacities are AsyncFilesDecompressor's, with rows_cap (the most numbers of a call's files) in place of dst_cap, and k
    (1 .. 1024) and the direction fixed by the plan.  The call owns a device workspace (about rows_cap * itemsize + 16 * k * max_chunks
    bytes beyond the decompressor's) and a status; it serves one call in flight."""

    _Plan, _Status = _CAsyncFilesTopkPlan, _CAsyncFilesTopkStatus

    def __init__(self, head, dtype, src_cap, index_cap, max_files, max_chunks, rows_cap, k, largest=False, device=None):
        self.dtype = np.dtype(dtype)
        h = self._head(head)
        self._make_plan(device, lambda plan: _lib_async_topk_files().pco_b200_topk_files_async_plan(
            h.ctypes.data_as(C.c_void_p), C.c_size_t(h.size), C.c_ubyte(_lib.dtype_byte(self.dtype)), C.c_size_t(src_cap), C.c_size_t(index_cap),
            C.c_size_t(max_files), C.c_size_t(max_chunks), C.c_size_t(rows_cap), C.c_size_t(k), C.c_int(int(largest)), plan))
        self._alloc()

    def __call__(self, src, index, files, n_files, interval, out_values, out_positions, n_out):
        """Enqueues the top-k of files[: n_files[0]] on torch.cuda.current_stream().  `src`, `index`, `files` and `n_files` are as
        AsyncFilesDecompressor takes them; `interval`, `out_values`, `out_positions` and `n_out` are as wrapped.AsyncPagesTopK takes them.
        Returns nothing and does not wait; result() reports the outcome."""
        import torch

        from .wrapped import _check_topk_inputs

        p = self._plan
        self._check_tensors(src=src, index=index, files=files, n_files=n_files, interval=interval, out_values=out_values,
                            out_positions=out_positions, n_out=n_out)
        if src.numel() * src.element_size() < p.src_cap or index.numel() * index.element_size() < p.index_cap:
            raise ValueError(f"src holds fewer than src_cap = {p.src_cap} bytes, or index fewer than index_cap = {p.index_cap}")
        if files.dtype != torch.int64 or files.dim() != 2 or files.shape[1] != 4 or files.shape[0] < p.max_files:
            raise ValueError(f"files must be an int64 tensor of shape ({p.max_files}, 4)")
        if n_files.dtype != torch.int64 or n_files.numel() != 1:
            raise ValueError("n_files must be a 1-element int64 tensor")
        _check_topk_inputs(interval, out_values, out_positions, n_out, p.k, self.dtype)
        rc = _lib_async_topk_files().pco_b200_topk_files_async(
            C.byref(p), C.c_void_p(src.data_ptr()), C.c_void_p(index.data_ptr()), C.c_void_p(files.data_ptr()), C.c_void_p(n_files.data_ptr()),
            C.c_void_p(interval.data_ptr()), C.c_void_p(out_values.data_ptr()), C.c_void_p(out_positions.data_ptr()), C.c_void_p(n_out.data_ptr()),
            C.c_void_p(self.workspace.data_ptr()), C.c_void_p(self.status.data_ptr()), self._stream())
        _lib.check(rc)

    def result(self):
        """Copies the status of the last call back (waiting for it on the current stream) and returns the numbers inside the interval, or
        raises PcoError with the kind pco_b200_decompress_files gives ("file 3: chunk 2: ...")."""
        s = self.status_record()
        n = C.c_size_t()
        _lib.check(_lib_async_topk_files().pco_b200_topk_files_async_result(C.byref(s), C.byref(n)))
        return int(n.value)


class _CAsyncFilesTakePlan(C.Structure):  # PcoB200AsyncFilesTakePlan (include/pco_b200.h)
    _fields_ = [("dtype", C.c_uint32), ("uniform_type", C.c_uint32), ("format_major", C.c_uint32), ("reserved", C.c_uint32),
                ("src_cap", C.c_uint64), ("index_cap", C.c_uint64), ("max_files", C.c_uint64), ("max_chunks", C.c_uint64),
                ("rows_cap", C.c_uint64), ("max_positions", C.c_uint64), ("workspace_bytes", C.c_uint64)]


class _CAsyncFilesTakeStatus(C.Structure):  # PcoB200AsyncFilesTakeStatus (include/pco_b200.h)
    _fields_ = [("kind", C.c_uint32), ("device_status", C.c_uint32), ("file", C.c_uint64), ("chunk", C.c_uint64), ("n_written", C.c_uint64),
                ("n_files", C.c_uint64), ("n_positions", C.c_uint64), ("position", C.c_uint64), ("records_decoded", C.c_uint64)]


def _lib_async_take_files():
    return _lib.bind("_async_take_files_ready",
                     pco_b200_take_files_async_plan=[C.c_void_p, C.c_size_t, C.c_ubyte, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t,
                                                     C.c_size_t, C.c_size_t, C.c_void_p],
                     pco_b200_take_files_async=[C.c_void_p] * 12,
                     pco_b200_take_files_async_result=[C.c_void_p, C.POINTER(C.c_size_t)])


class AsyncFilesTake(_lib._AsyncCall):
    """Takes the numbers at strictly ascending positions of a batch of indexed standalone files' concatenation on the current CUDA stream
    (pco_b200_take_files_async), decoding only the chunks the positions touch: each decoded batch writes its selected numbers straight to
    their final index.  Refs, their count, the positions and their count are read from device tensors, so one captured call serves new
    files and new positions on each replay, and AsyncFilesFilter's positions and count can be passed straight in.

    The plan and capacities are AsyncFilesDecompressor's, with rows_cap (the most numbers of a call's files) in place of dst_cap, and
    max_positions the most positions a call takes.  The call owns a device workspace (about rows_cap * (itemsize + 0.07) bytes beyond the
    decompressor's) and a status; it serves one call in flight."""

    _Plan, _Status = _CAsyncFilesTakePlan, _CAsyncFilesTakeStatus

    def __init__(self, head, dtype, src_cap, index_cap, max_files, max_chunks, rows_cap, max_positions, device=None):
        self.dtype = np.dtype(dtype)
        h = self._head(head)
        self._make_plan(device, lambda plan: _lib_async_take_files().pco_b200_take_files_async_plan(
            h.ctypes.data_as(C.c_void_p), C.c_size_t(h.size), C.c_ubyte(_lib.dtype_byte(self.dtype)), C.c_size_t(src_cap), C.c_size_t(index_cap),
            C.c_size_t(max_files), C.c_size_t(max_chunks), C.c_size_t(rows_cap), C.c_size_t(max_positions), plan))
        self._alloc()

    def __call__(self, src, index, files, n_files, positions, n_positions, values, file_ns=None):
        """Enqueues the take of positions[: n_positions[0]] from files[: n_files[0]] on torch.cuda.current_stream().  `src`, `index`,
        `files` and `n_files` are as AsyncFilesDecompressor takes them; `positions` is an int64 CUDA tensor of at least max_positions
        elements (strictly ascending indices into the files' concatenation), `n_positions` a 1-element int64 CUDA tensor, `values` a CUDA
        tensor of the plan's dtype of at least max_positions elements that receives the numbers, and `file_ns` (optional) an int64 CUDA
        tensor of at least max_files elements that receives each file's count.  Returns nothing and does not wait; result() reports the
        outcome."""
        import torch

        from .wrapped import _check_take_tensors

        p = self._plan
        self._check_tensors(src=src, index=index, files=files, n_files=n_files, positions=positions, n_positions=n_positions, values=values,
                            **({} if file_ns is None else {"file_ns": file_ns}))
        if src.numel() * src.element_size() < p.src_cap or index.numel() * index.element_size() < p.index_cap:
            raise ValueError(f"src holds fewer than src_cap = {p.src_cap} bytes, or index fewer than index_cap = {p.index_cap}")
        if files.dtype != torch.int64 or files.dim() != 2 or files.shape[1] != 4 or files.shape[0] < p.max_files:
            raise ValueError(f"files must be an int64 tensor of shape ({p.max_files}, 4)")
        if n_files.dtype != torch.int64 or n_files.numel() != 1:
            raise ValueError("n_files must be a 1-element int64 tensor")
        _check_take_tensors(positions, n_positions, values, self.dtype, p.max_positions)
        if file_ns is not None and (file_ns.dtype != torch.int64 or file_ns.numel() < p.max_files):
            raise ValueError(f"file_ns must be an int64 tensor of at least max_files = {p.max_files} elements")
        rc = _lib_async_take_files().pco_b200_take_files_async(
            C.byref(p), C.c_void_p(src.data_ptr()), C.c_void_p(index.data_ptr()), C.c_void_p(files.data_ptr()), C.c_void_p(n_files.data_ptr()),
            C.c_void_p(positions.data_ptr()), C.c_void_p(n_positions.data_ptr()), C.c_void_p(values.data_ptr()),
            C.c_void_p(None if file_ns is None else file_ns.data_ptr()), C.c_void_p(self.workspace.data_ptr()), C.c_void_p(self.status.data_ptr()),
            self._stream())
        _lib.check(rc)

    def result(self):
        """Copies the status of the last call back (waiting for it on the current stream) and returns the number of values written, or
        raises PcoError with the kind pco_b200_decompress_files gives ("file 3: chunk 2: ...") or, for the positions, InvalidArgument
        ("position 17: ...")."""
        s = self.status_record()
        nw = C.c_size_t()
        _lib.check(_lib_async_take_files().pco_b200_take_files_async_result(C.byref(s), C.byref(nw)))
        return int(nw.value)


class _CAsyncFilesSegmentAggregatePlan(C.Structure):  # PcoB200AsyncFilesSegmentAggregatePlan (include/pco_b200.h)
    _fields_ = [("dtype", C.c_uint32), ("uniform_type", C.c_uint32), ("format_major", C.c_uint32), ("reserved", C.c_uint32),
                ("src_cap", C.c_uint64), ("index_cap", C.c_uint64), ("max_files", C.c_uint64), ("max_chunks", C.c_uint64),
                ("rows_cap", C.c_uint64), ("max_segments", C.c_uint64), ("workspace_bytes", C.c_uint64)]


class _CAsyncFilesSegmentAggregateStatus(C.Structure):  # PcoB200AsyncFilesSegmentAggregateStatus (include/pco_b200.h)
    _fields_ = [("kind", C.c_uint32), ("device_status", C.c_uint32), ("file", C.c_uint64), ("chunk", C.c_uint64), ("n_written", C.c_uint64),
                ("n_files", C.c_uint64), ("n_segments", C.c_uint64), ("segment", C.c_uint64), ("records_decoded", C.c_uint64),
                ("n_matches", C.c_uint64)]


def _lib_async_segment_aggregate_files():
    return _lib.bind("_async_segment_aggregate_files_ready",
                     pco_b200_segment_aggregate_files_async_plan=[C.c_void_p, C.c_size_t, C.c_ubyte, C.c_size_t, C.c_size_t, C.c_size_t,
                                                                  C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p],
                     pco_b200_segment_aggregate_files_async=[C.c_void_p] * 13,
                     pco_b200_segment_aggregate_files_async_result=[C.c_void_p, C.POINTER(C.c_size_t)])


class AsyncFilesSegmentAggregate(_lib._AsyncCall):
    """Decodes a batch of indexed standalone files on the current CUDA stream and reduces the numbers inside a closed interval to count,
    min, max and sum per row segment [bounds[g], bounds[g + 1]) of the files' concatenation and in all
    (pco_b200_segment_aggregate_files_async), decoding only the chunks the segments cover.  Refs, their count, the bounds, their count and
    the interval are read from device tensors, so one captured call serves new files and new segments on each replay.

    The plan and capacities are AsyncFilesAggregate's, with max_segments the most segments a call reduces.  The call owns a device workspace
    (about rows_cap * (itemsize + 0.2) + 96 * max_segments bytes beyond the decompressor's) and a status; it serves one call in flight.
    wrapped.unpack_aggregates reads the records."""

    _Plan, _Status = _CAsyncFilesSegmentAggregatePlan, _CAsyncFilesSegmentAggregateStatus

    def __init__(self, head, dtype, src_cap, index_cap, max_files, max_chunks, rows_cap, max_segments, device=None):
        self.dtype = np.dtype(dtype)
        h = self._head(head)
        self._make_plan(device, lambda plan: _lib_async_segment_aggregate_files().pco_b200_segment_aggregate_files_async_plan(
            h.ctypes.data_as(C.c_void_p), C.c_size_t(h.size), C.c_ubyte(_lib.dtype_byte(self.dtype)), C.c_size_t(src_cap), C.c_size_t(index_cap),
            C.c_size_t(max_files), C.c_size_t(max_chunks), C.c_size_t(rows_cap), C.c_size_t(max_segments), plan))
        self._alloc()

    def __call__(self, src, index, files, n_files, bounds, n_segments, interval, aggs, total):
        """Enqueues the segment aggregates of files[: n_files[0]] on torch.cuda.current_stream().  `src`, `index`, `files` and `n_files`
        are as AsyncFilesDecompressor takes them; `bounds`, `n_segments`, `interval`, `aggs` and `total` are as
        wrapped.AsyncPagesSegmentAggregate takes them, the bounds indexing the files' concatenation.  Returns nothing and does not wait;
        result() reports the outcome."""
        import torch

        from .wrapped import _check_segment_tensors

        p = self._plan
        self._check_tensors(src=src, index=index, files=files, n_files=n_files, bounds=bounds, n_segments=n_segments, interval=interval,
                            aggs=aggs, total=total)
        if src.numel() * src.element_size() < p.src_cap or index.numel() * index.element_size() < p.index_cap:
            raise ValueError(f"src holds fewer than src_cap = {p.src_cap} bytes, or index fewer than index_cap = {p.index_cap}")
        if files.dtype != torch.int64 or files.dim() != 2 or files.shape[1] != 4 or files.shape[0] < p.max_files:
            raise ValueError(f"files must be an int64 tensor of shape ({p.max_files}, 4)")
        if n_files.dtype != torch.int64 or n_files.numel() != 1:
            raise ValueError("n_files must be a 1-element int64 tensor")
        _check_segment_tensors(bounds, n_segments, interval, aggs, total, p.max_segments)
        rc = _lib_async_segment_aggregate_files().pco_b200_segment_aggregate_files_async(
            C.byref(p), C.c_void_p(src.data_ptr()), C.c_void_p(index.data_ptr()), C.c_void_p(files.data_ptr()), C.c_void_p(n_files.data_ptr()),
            C.c_void_p(bounds.data_ptr()), C.c_void_p(n_segments.data_ptr()), C.c_void_p(interval.data_ptr()), C.c_void_p(aggs.data_ptr()),
            C.c_void_p(total.data_ptr()), C.c_void_p(self.workspace.data_ptr()), C.c_void_p(self.status.data_ptr()), self._stream())
        _lib.check(rc)

    def result(self):
        """Copies the status of the last call back (waiting for it on the current stream) and returns the total match count, or raises
        PcoError with the kind pco_b200_decompress_files gives ("file 3: chunk 2: ...") or, for the bounds, InvalidArgument
        ("segment 17: ...")."""
        s = self.status_record()
        nm = C.c_size_t()
        _lib.check(_lib_async_segment_aggregate_files().pco_b200_segment_aggregate_files_async_result(C.byref(s), C.byref(nm)))
        return int(nm.value)


class _CAsyncCompressFilesPlan(C.Structure):  # PcoB200AsyncCompressFilesPlan (include/pco_b200.h)
    _fields_ = [("dtype", C.c_uint32), ("uniform_type_header", C.c_uint32), ("mode", C.c_uint32), ("order", C.c_uint32),
                ("n_vars", C.c_uint32), ("level", C.c_uint32), ("mode_k", C.c_uint32), ("reserved", C.c_uint32),
                ("max_files", C.c_uint64), ("nums_cap", C.c_uint64), ("max_file_n", C.c_uint64), ("max_page_n", C.c_uint64),
                ("max_chunks", C.c_uint64), ("dst_cap", C.c_uint64), ("index_cap", C.c_uint64),
                ("mode_base", C.c_uint64), ("base_bits", C.c_uint64), ("inv_base_bits", C.c_uint64),
                ("dst_bound", C.c_uint64), ("index_bound", C.c_uint64), ("workspace_bytes", C.c_uint64)]


class _CAsyncCompressFilesStatus(C.Structure):  # PcoB200AsyncCompressFilesStatus (include/pco_b200.h)
    _fields_ = [("kind", C.c_uint32), ("device_status", C.c_uint32), ("file", C.c_uint64), ("n_files", C.c_uint64),
                ("dst_bytes", C.c_uint64), ("index_bytes", C.c_uint64), ("dst_written", C.c_uint64), ("index_written", C.c_uint64)]


def _lib_async_compress_files():
    return _lib.bind("_async_compress_files_ready",
                     pco_b200_compress_files_async_plan=[C.c_ubyte, C.c_void_p, C.c_int, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t,
                                                         C.c_size_t, C.c_void_p],
                     pco_b200_compress_files_async=[C.c_void_p] * 10,
                     pco_b200_compress_files_async_result=[C.c_void_p, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)])


class AsyncFilesCompressor(_lib._AsyncCall):
    """Compresses a batch of standalone files on the current CUDA stream, with the file sizes in device memory and without waiting for the
    device (pco_b200_compress_files_async): sizes a kernel decided (the tensors of a checkpoint, the blocks a step evicted) need no trip to
    the host, and a call can be captured in a torch.cuda.CUDAGraph.

    The plan fixes the number type `dtype`, the config (explicit mode and delta specs, EqualPagesUpTo paging), the header flavour
    (uniform_type_header: as simple_compress_into) and the capacities: at most max_files files, nums_cap numbers in all and max_file_n per
    file, dst_cap bytes of files (default: the plan's dst_bound, which every batch within the capacities fits in) and, with index=True,
    the plan's index_bound bytes of side indexes.  The sizes and their count are read when the call runs, so one captured call compresses
    a different count, different sizes and different numbers on each replay.  The bytes, the indexes and the refs equal what compress_files
    writes.  The compressor owns a device workspace and a status; it serves one call in flight."""

    _Plan, _Status = _CAsyncCompressFilesPlan, _CAsyncCompressFilesStatus

    def __init__(self, dtype, config, max_files, nums_cap, max_file_n, dst_cap=None, index=True, uniform_type_header=False, device=None):
        self.dtype = np.dtype(dtype)
        dtb = _lib.dtype_byte(self.dtype)
        L = _lib_async_compress_files()
        cfg = (config or ChunkConfig())._to_c()

        def plan_fn(dcap, icap):
            return lambda plan: L.pco_b200_compress_files_async_plan(C.c_ubyte(dtb), C.byref(cfg), C.c_int(1 if uniform_type_header else 0),
                                                                     C.c_size_t(max_files), C.c_size_t(nums_cap), C.c_size_t(max_file_n),
                                                                     C.c_size_t(dcap), C.c_size_t(icap), plan)

        # the bounds are known once a plan exists: a first plan reports them
        self._make_plan(device, plan_fn(dst_cap or 0, 0))
        if dst_cap is None or index:
            self._replan(plan_fn(self._plan.dst_bound if dst_cap is None else dst_cap, self._plan.index_bound if index else 0))
        self._alloc()

    @property
    def dst_cap(self):
        return int(self._plan.dst_cap)

    @property
    def index_cap(self):
        """Bytes of side indexes a call may write (0 without an index)."""
        return int(self._plan.index_cap)

    @property
    def max_files(self):
        return int(self._plan.max_files)

    def __call__(self, nums, file_ns, n_files, dst, index, files):
        """Enqueues the compress of the first n_files[0] files on torch.cuda.current_stream(): file i is the next file_ns[i] numbers of
        `nums` (a CUDA tensor of the plan's dtype, at least nums_cap numbers).  `file_ns` is an int64 CUDA tensor of at least max_files
        elements, `n_files` a 1-element int64 CUDA tensor, `dst` a uint8 CUDA tensor of at least dst_cap bytes, `index` one of at least
        index_cap bytes (or None), and `files` the int64 (max_files, 4) CUDA tensor of FILE_REF fields that AsyncFilesDecompressor takes.
        Returns nothing and does not wait; result() reports the outcome."""
        import torch

        from .wrapped import _torch_dtypes

        p = self._plan
        self._check_tensors(nums=nums, file_ns=file_ns, n_files=n_files, dst=dst, files=files, **({"index": index} if index is not None else {}))
        if nums.dtype != _torch_dtypes()[self.dtype] or nums.numel() < p.nums_cap:
            raise ValueError(f"nums must hold at least nums_cap = {p.nums_cap} numbers of {self.dtype}")
        if file_ns.dtype != torch.int64 or file_ns.numel() < p.max_files:
            raise ValueError(f"file_ns must be an int64 tensor of at least max_files = {p.max_files} elements")
        if n_files.dtype != torch.int64 or n_files.numel() != 1:
            raise ValueError("n_files must be a 1-element int64 tensor")
        if dst.numel() * dst.element_size() < p.dst_cap:
            raise ValueError(f"dst holds fewer than dst_cap = {p.dst_cap} bytes")
        if index is not None and (not p.index_cap or index.numel() * index.element_size() < p.index_cap):
            raise ValueError(f"index needs a compressor made with index=True and at least index_cap = {p.index_cap} bytes")
        if files.dtype != torch.int64 or files.dim() != 2 or files.shape[1] != 4 or files.shape[0] < p.max_files:
            raise ValueError(f"files must be an int64 tensor of shape ({p.max_files}, 4)")
        rc = _lib_async_compress_files().pco_b200_compress_files_async(
            C.byref(p), C.c_void_p(nums.data_ptr()), C.c_void_p(file_ns.data_ptr()), C.c_void_p(n_files.data_ptr()), C.c_void_p(dst.data_ptr()),
            C.c_void_p(index.data_ptr()) if index is not None else None, C.c_void_p(files.data_ptr()), C.c_void_p(self.workspace.data_ptr()),
            C.c_void_p(self.status.data_ptr()), self._stream())
        _lib.check(rc)

    def result(self):
        """Copies the status of the last call back (waiting for it on the current stream) and returns (dst_len, index_len), the bytes
        written, or raises PcoError with the kind pco_b200_compress_files gives ("file 17: ...")."""
        s = self.status_record()
        dl, il = C.c_size_t(), C.c_size_t()
        _lib.check(_lib_async_compress_files().pco_b200_compress_files_async_result(C.byref(s), C.byref(dl), C.byref(il)))
        return int(dl.value), int(il.value)


class _CModeChoice(C.Structure):
    _fields_ = [("mode_spec", C.c_uint32), ("float_quant_k", C.c_uint32), ("float_mult_base", C.c_double), ("float_mult_inv_base", C.c_double),
                ("int_mult_base", C.c_uint64), ("bits_saved_per_num", C.c_double)]


def choose_mode(nums):
    """What `ModeSpec.auto()` resolves to in the reference for this chunk of numbers (pco/src/data_types/unsigned.rs:28-35,
    float.rs:70-98): a ModeSpec to put into a ChunkConfig.  Host-side planner logic of libcpcodec.so (pco_b200_choose_mode); needs no
    device.  `.inv_base` on a FloatMult answer is the inverse the reference's splitter multiplies by."""
    arr = np.ascontiguousarray(nums)
    out = _CModeChoice()
    _lib.check(_lib.lib().pco_b200_choose_mode(C.c_void_p(arr.ctypes.data), C.c_size_t(arr.size), C.c_ubyte(_lib.dtype_byte(arr.dtype)), C.byref(out)))
    spec = _lib.ModeSpec(out.mode_spec, base=out.float_mult_base, k=out.float_quant_k, int_base=out.int_mult_base)
    spec.inv_base = out.float_mult_inv_base
    spec.bits_saved_per_num = out.bits_saved_per_num
    return spec
