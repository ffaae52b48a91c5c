"""Mirror of pcodec.wrapped (pco_python/src/wrapped/{compressor,decompressor}.rs) over the C-ABI of libcpcodec.so.

A chunk's PagingSpec may cut it into several pages that share the chunk's bins.  Classic mode takes any number of pages; the
two-var modes (IntMult / FloatMult / FloatQuant) take one page per chunk, and `FileCompressor.chunk_compressor` raises
PcoError("Unsupported") when their PagingSpec would give several (DESIGN.md section 8).

Batched forms for containers that keep chunk metas and pages themselves: `compress_chunks` writes a whole array as wrapped
chunks of one page each, `decompress_pages` decodes any number of pages in one call.  Both take host buffers (bytes / numpy)
or torch CUDA tensors; with CUDA tensors the work runs on torch.cuda.current_stream() and the outputs are CUDA tensors.
`AsyncChunksCompressor` and `AsyncPagesDecompressor` are their forms with the sizes or refs in device memory, which do not wait for the
device and can be captured in a CUDA graph; `AsyncPagesFilter` decodes such pages and keeps only the numbers inside an interval, and
`AsyncPagesToFile` writes them out as one indexed standalone file that the files calls of `standalone` scan without a walk."""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import ChunkConfig, Progress


def _lib_wrapped():
    L = _lib.lib()
    if not getattr(L, "_wrapped_ready", False):
        for name in ("pco_b200_chunk_compressor_n_pages", "pco_b200_chunk_compressor_meta_size"):
            getattr(L, name).restype = C.c_size_t
            getattr(L, name).argtypes = [C.c_void_p]
        for name in ("pco_b200_chunk_compressor_page_n", "pco_b200_chunk_compressor_page_size"):
            getattr(L, name).restype = C.c_size_t
            getattr(L, name).argtypes = [C.c_void_p, C.c_size_t]
        L.pco_b200_chunk_compressor_free.argtypes = [C.c_void_p]
        L.pco_b200_chunk_compressor_free.restype = None
        L._wrapped_ready = True
    return L


class ChunkCompressor:
    """pcodec.wrapped.ChunkCompressor (pco_python/src/wrapped/compressor.rs:22-115)."""

    def __init__(self, handle):
        self._h = handle

    def __del__(self):
        if getattr(self, "_h", None):
            _lib_wrapped().pco_b200_chunk_compressor_free(self._h)
            self._h = None

    def n_per_page(self):
        L = _lib_wrapped()
        return [L.pco_b200_chunk_compressor_page_n(self._h, i) for i in range(L.pco_b200_chunk_compressor_n_pages(self._h))]

    def write_meta(self):
        L = _lib_wrapped()
        buf = np.empty(L.pco_b200_chunk_compressor_meta_size(self._h), dtype=np.uint8)
        n = C.c_size_t()
        _lib.check(L.pco_b200_chunk_compressor_write_meta(self._h, buf.ctypes.data_as(C.c_void_p), C.c_size_t(buf.size), C.byref(n)))
        return buf[: n.value].tobytes()

    def write_page(self, page_idx):
        L = _lib_wrapped()
        buf = np.empty(max(L.pco_b200_chunk_compressor_page_size(self._h, page_idx), 1), dtype=np.uint8)
        n = C.c_size_t()
        _lib.check(L.pco_b200_chunk_compressor_write_page(self._h, C.c_size_t(page_idx), buf.ctypes.data_as(C.c_void_p), C.c_size_t(buf.size), C.byref(n)))
        return buf[: n.value].tobytes()


class FileCompressor:
    """pcodec.wrapped.FileCompressor (pco_python/src/wrapped/compressor.rs:15-91)."""

    def write_header(self):
        buf = np.empty(2, dtype=np.uint8)
        n = C.c_size_t()
        _lib.check(_lib_wrapped().pco_b200_file_compressor_write_header(buf.ctypes.data_as(C.c_void_p), C.c_size_t(2), C.byref(n)))
        return buf[: n.value].tobytes()

    def chunk_compressor(self, nums, config=None):
        arr = np.ascontiguousarray(nums)
        cfg = (config or ChunkConfig())._to_c()
        h = C.c_void_p()
        _lib.check(_lib_wrapped().pco_b200_chunk_compressor_new(arr.ctypes.data_as(C.c_void_p), C.c_size_t(arr.size), C.c_ubyte(_lib.dtype_byte(arr.dtype)),
                                                                 C.byref(cfg), C.byref(h)))
        return ChunkCompressor(h)


class ChunkDecompressor:
    """pcodec.wrapped.ChunkDecompressor (pco_python/src/wrapped/decompressor.rs:25-122): holds the chunk meta bytes."""

    def __init__(self, meta, dtype):
        self._meta, self._dtype = bytes(meta), np.dtype(dtype)

    def read_page_into(self, src, page_n, dst):
        """Decodes one page of `page_n` numbers from the head of `src` into `dst`; returns (Progress, bytes_read)."""
        if np.dtype(dst.dtype) != self._dtype:
            raise TypeError("dst dtype does not match the chunk's")
        sb = np.frombuffer(bytes(src), dtype=np.uint8)
        mb = np.frombuffer(self._meta, dtype=np.uint8)
        prog = _lib._CProgress()
        nread = C.c_size_t()
        _lib.check(_lib_wrapped().pco_b200_page_decompress(mb.ctypes.data_as(C.c_void_p), C.c_size_t(mb.size), sb.ctypes.data_as(C.c_void_p), C.c_size_t(sb.size),
                                                            C.c_size_t(page_n), C.c_ubyte(_lib.dtype_byte(self._dtype)), dst.ctypes.data_as(C.c_void_p),
                                                            C.c_size_t(dst.size), C.byref(prog), C.byref(nread)))
        return Progress(prog.n_processed, bool(prog.finished)), nread.value


class FileDecompressor:
    """pcodec.wrapped.FileDecompressor (pco_python/src/wrapped/decompressor.rs:16-95)."""

    @staticmethod
    def new(src):
        """Returns (FileDecompressor, bytes_read) from the wrapped header at the head of `src`."""
        sb = np.frombuffer(bytes(src), dtype=np.uint8)
        n = C.c_size_t()
        _lib.check(_lib_wrapped().pco_b200_file_decompressor_read_header(sb.ctypes.data_as(C.c_void_p), C.c_size_t(sb.size), C.byref(n)))
        return FileDecompressor(), n.value

    def chunk_decompressor(self, src, dtype):
        """Returns (ChunkDecompressor, bytes_read) from the chunk meta at the head of `src`."""
        sb = np.frombuffer(bytes(src), dtype=np.uint8)
        n = C.c_size_t()
        _lib.check(_lib_wrapped().pco_b200_chunk_meta_size(sb.ctypes.data_as(C.c_void_p), C.c_size_t(sb.size), C.c_ubyte(_lib.dtype_byte(np.dtype(dtype))), C.byref(n)))
        return ChunkDecompressor(sb[: n.value].tobytes(), dtype), n.value


# PcoB200PageRef (include/pco_b200.h): one page of a wrapped container
PAGE_REF = np.dtype([("meta_offset", "<u8"), ("meta_len", "<u8"), ("page_offset", "<u8"), ("page_len", "<u8"), ("page_n", "<u8")])


def _lib_batch():
    L = _lib_wrapped()
    if not getattr(L, "_batch_ready", False):
        L.pco_b200_decompress_pages.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_ubyte, C.c_void_p, C.c_size_t, C.c_void_p,
                                                C.c_size_t, C.POINTER(C.c_size_t), C.c_uint32, C.c_void_p]
        L.pco_b200_compress_wrapped.argtypes = [C.c_void_p, C.c_size_t, C.c_ubyte, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t),
                                                C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t),
                                                C.c_uint32, C.c_void_p]
        L._batch_ready = True
    return L


def _is_cuda(x):
    return getattr(x, "is_cuda", False)


def _torch_dtypes():
    import torch

    return {np.dtype(np.uint8): torch.uint8, np.dtype(np.int8): torch.int8, np.dtype(np.uint16): torch.uint16, np.dtype(np.int16): torch.int16,
            np.dtype(np.float16): torch.float16, np.dtype(np.uint32): torch.uint32, np.dtype(np.int32): torch.int32, np.dtype(np.float32): torch.float32,
            np.dtype(np.uint64): torch.uint64, np.dtype(np.int64): torch.int64, np.dtype(np.float64): torch.float64}


def _host_u8(x):
    if isinstance(x, np.ndarray):
        return np.ascontiguousarray(x).reshape(-1).view(np.uint8)
    return np.frombuffer(bytes(x), dtype=np.uint8)


def _stream_of(t):
    import torch

    return C.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


def compress_chunks(nums, config=None):
    """Compresses `nums` into wrapped chunks of one page each - the chunks pco_b200_simple_compress would write for `config`'s
    PagingSpec - in one call (pco_b200_compress_wrapped).  Returns (metas, pages, refs): the chunk metas back to back, the pages
    back to back, and one PAGE_REF record per chunk.  Host input gives bytes; a torch CUDA tensor gives uint8 CUDA tensors."""
    cfg = (config or ChunkConfig())._to_c()
    L = _lib_batch()
    ps = (config or ChunkConfig()).paging_spec
    if _is_cuda(nums):
        import torch

        t = nums.contiguous()
        dt = next(k for k, v in _torch_dtypes().items() if v == t.dtype)
        n, src, flags, stream = t.numel(), C.c_void_p(t.data_ptr()), _lib.SRC_ON_DEVICE | _lib.DST_ON_DEVICE, _stream_of(t)

        def alloc(nbytes):
            return torch.empty(max(nbytes, 1), dtype=torch.uint8, device=t.device)

        def ptr(buf):
            return C.c_void_p(buf.data_ptr())
    else:
        arr = np.ascontiguousarray(nums)
        dt, n, src, flags, stream = arr.dtype, arr.size, arr.ctypes.data_as(C.c_void_p), 0, None

        def alloc(nbytes):
            return np.empty(max(nbytes, 1), dtype=np.uint8)

        def ptr(buf):
            return buf.ctypes.data_as(C.c_void_p)
    dtb = _lib.dtype_byte(dt)
    n_chunks = len(ps.sizes) if ps.sizes is not None else -(-n // (ps.n or (1 << 18)))
    caps = [n_chunks * 4096 + 64, L.pco_standalone_guarantee_file_size(n, dtb), n_chunks + 1]
    ml, pl, nc = C.c_size_t(), C.c_size_t(), C.c_size_t()
    for attempt in range(2):  # a first guess of the capacities, then what the call reported it needs
        metas, pages, refs = alloc(caps[0]), alloc(caps[1]), np.zeros(max(caps[2], 1), dtype=PAGE_REF)
        rc = L.pco_b200_compress_wrapped(src, C.c_size_t(n), C.c_ubyte(dtb), C.byref(cfg), ptr(metas), C.c_size_t(caps[0]), C.byref(ml), ptr(pages),
                                         C.c_size_t(caps[1]), C.byref(pl), refs.ctypes.data_as(C.c_void_p), C.c_size_t(caps[2]), C.byref(nc),
                                         C.c_uint32(flags), stream)
        if rc == 4 and attempt == 0:  # PCO_B200_IO
            caps = [max(caps[0], ml.value), max(caps[1], pl.value), max(caps[2], nc.value)]
            continue
        _lib.check(rc)
        break
    refs = refs[: nc.value].copy()
    if _is_cuda(nums):
        return metas[: ml.value], pages[: pl.value], refs
    return metas[: ml.value].tobytes(), pages[: pl.value].tobytes(), refs


def decompress_pages(metas, pages, refs, dtype):
    """Decodes every page `refs` (PAGE_REF records, or anything with their five fields in that order) names into one array,
    page after page in refs order (pco_b200_decompress_pages).  `metas` and `pages` are bytes / numpy, or torch CUDA tensors
    (then the result is a CUDA tensor, computed on the current stream)."""
    dt = np.dtype(dtype)
    r = np.ascontiguousarray(np.asarray(refs).astype(PAGE_REF, copy=False))
    total = int(r["page_n"].sum()) if r.size else 0
    L = _lib_batch()
    nw = C.c_size_t()
    if _is_cuda(metas) or _is_cuda(pages):
        import torch

        if not (_is_cuda(metas) and _is_cuda(pages)):
            raise TypeError("metas and pages must both be CUDA tensors or both be host buffers")
        m, p = metas.contiguous(), pages.contiguous()
        dst = torch.empty(max(total, 1), dtype=_torch_dtypes()[dt], device=p.device)
        _lib.check(L.pco_b200_decompress_pages(C.c_void_p(m.data_ptr()), C.c_size_t(m.numel() * m.element_size()), C.c_void_p(p.data_ptr()),
                                               C.c_size_t(p.numel() * p.element_size()), C.c_ubyte(_lib.dtype_byte(dt)), r.ctypes.data_as(C.c_void_p),
                                               C.c_size_t(r.size), C.c_void_p(dst.data_ptr()), C.c_size_t(total), C.byref(nw),
                                               C.c_uint32(_lib.SRC_ON_DEVICE | _lib.DST_ON_DEVICE), _stream_of(p)))
        return dst[:total]
    mb, pb = _host_u8(metas), _host_u8(pages)
    dst = np.empty(max(total, 1), dtype=dt)
    _lib.check(L.pco_b200_decompress_pages(mb.ctypes.data_as(C.c_void_p), C.c_size_t(mb.size), pb.ctypes.data_as(C.c_void_p), C.c_size_t(pb.size),
                                           C.c_ubyte(_lib.dtype_byte(dt)), r.ctypes.data_as(C.c_void_p), C.c_size_t(r.size),
                                           dst.ctypes.data_as(C.c_void_p), C.c_size_t(total), C.byref(nw), C.c_uint32(0), None))
    return dst[:total]


class _CAsyncPagesPlan(C.Structure):  # PcoB200AsyncPagesPlan (include/pco_b200.h)
    _fields_ = [("dtype", C.c_uint32), ("reserved", C.c_uint32), ("metas_cap", C.c_uint64), ("pages_cap", C.c_uint64), ("max_pages", C.c_uint64),
                ("dst_cap", C.c_uint64), ("frame_cap", C.c_uint64), ("workspace_bytes", C.c_uint64)]


class _CAsyncPagesStatus(C.Structure):  # PcoB200AsyncPagesStatus (include/pco_b200.h)
    _fields_ = [("kind", C.c_uint32), ("device_status", C.c_uint32), ("page", C.c_uint64), ("n_written", C.c_uint64), ("n_pages", C.c_uint64),
                ("frames_needed", C.c_uint64)]


def _lib_async_pages():
    return _lib.bind("_async_pages_ready",
                     pco_b200_decompress_pages_async_plan=[C.c_ubyte, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p],
                     pco_b200_decompress_pages_async=[C.c_void_p] * 9,
                     pco_b200_decompress_pages_async_result=[C.c_void_p, C.POINTER(C.c_size_t)])


class AsyncPagesDecompressor(_lib._AsyncCall):
    """Decodes a batch of wrapped-format pages on the current CUDA stream with the page refs in device memory and without waiting for the
    device (pco_b200_decompress_pages_async): pages a kernel kept (a filter on page statistics, a row-group selection) need no trip to the
    host, and a call can be captured in a torch.cuda.CUDAGraph.

    metas_cap and pages_cap (bytes) and dst_cap (numbers) are the sizes of the buffers every call passes, max_pages the most pages of a
    call.  frame_cap bounds the workspace each page is framed in (ceil((4 + meta_len + page_len) / 16) * 16 bytes per page); the default,
    metas_cap + pages_cap + 20 * max_pages, fits every batch that names each page and each meta at most once, as compress_chunks writes
    them.  Batches whose pages share a meta or repeat need more; a batch above frame_cap is refused with Io.  The number of pages is read
    from a device tensor, so one captured call serves different refs, a different count and different bytes on each replay.  The
    decompressor owns a device workspace and a status; it serves one call in flight."""

    _Plan, _Status = _CAsyncPagesPlan, _CAsyncPagesStatus

    def __init__(self, dtype, metas_cap, pages_cap, max_pages, dst_cap, frame_cap=None, device=None):
        self.dtype = np.dtype(dtype)
        if frame_cap is None:
            frame_cap = metas_cap + pages_cap + 20 * max_pages
        self._make_plan(device, lambda plan: _lib_async_pages().pco_b200_decompress_pages_async_plan(
            C.c_ubyte(_lib.dtype_byte(self.dtype)), C.c_size_t(metas_cap), C.c_size_t(pages_cap), C.c_size_t(max_pages), C.c_size_t(dst_cap),
            C.c_size_t(frame_cap), plan))
        self._alloc()

    def __call__(self, metas, pages, refs, n_pages, dst):
        """Enqueues the decode of the pages refs[: n_pages[0]] names into `dst` (a CUDA tensor of the plan's dtype, at least dst_cap
        numbers) on torch.cuda.current_stream(): page i lands right behind page i - 1.  `metas` and `pages` are uint8 CUDA tensors of at
        least metas_cap and pages_cap bytes (they may be one tensor); `refs` is an int64 CUDA tensor of shape (max_pages, 5) holding the
        PAGE_REF fields in order (meta_offset, meta_len, page_offset, page_len, page_n), `n_pages` a 1-element int64 CUDA tensor.  Returns
        nothing and does not wait; result() reports the outcome."""
        import torch

        p = self._plan
        self._check_tensors(metas=metas, pages=pages, refs=refs, n_pages=n_pages, dst=dst)
        if metas.numel() * metas.element_size() < p.metas_cap or pages.numel() * pages.element_size() < p.pages_cap:
            raise ValueError(f"metas holds fewer than metas_cap = {p.metas_cap} bytes, or pages fewer than pages_cap = {p.pages_cap}")
        if refs.dtype != torch.int64 or refs.dim() != 2 or refs.shape[1] != 5 or refs.shape[0] < p.max_pages:
            raise ValueError(f"refs must be an int64 tensor of shape ({p.max_pages}, 5)")
        if n_pages.dtype != torch.int64 or n_pages.numel() != 1:
            raise ValueError("n_pages must be a 1-element int64 tensor")
        if dst.dtype != _torch_dtypes()[self.dtype] or dst.numel() < p.dst_cap:
            raise ValueError(f"dst must hold at least dst_cap = {p.dst_cap} numbers of {self.dtype}")
        rc = _lib_async_pages().pco_b200_decompress_pages_async(
            C.byref(p), C.c_void_p(metas.data_ptr()), C.c_void_p(pages.data_ptr()), C.c_void_p(refs.data_ptr()), C.c_void_p(n_pages.data_ptr()),
            C.c_void_p(dst.data_ptr()), C.c_void_p(self.workspace.data_ptr()), C.c_void_p(self.status.data_ptr()), self._stream())
        _lib.check(rc)

    def result(self):
        """Copies the status of the last call back (waiting for it on the current stream) and returns the number of numbers written, or
        raises PcoError with the kind decompress_pages gives ("page 17: ...")."""
        s = self.status_record()
        nw = C.c_size_t()
        _lib.check(_lib_async_pages().pco_b200_decompress_pages_async_result(C.byref(s), C.byref(nw)))
        return int(nw.value)


class _CAsyncCompressWrappedPlan(C.Structure):  # PcoB200AsyncCompressWrappedPlan (include/pco_b200.h)
    _fields_ = [("dtype", C.c_uint32), ("mode", C.c_uint32), ("order", C.c_uint32), ("n_vars", C.c_uint32),
                ("level", C.c_uint32), ("mode_k", C.c_uint32), ("reserved0", C.c_uint32), ("reserved1", C.c_uint32),
                ("max_arrays", C.c_uint64), ("nums_cap", C.c_uint64), ("max_array_n", C.c_uint64), ("max_page_n", C.c_uint64),
                ("max_chunks", C.c_uint64), ("metas_cap", C.c_uint64), ("pages_cap", C.c_uint64),
                ("mode_base", C.c_uint64), ("base_bits", C.c_uint64), ("inv_base_bits", C.c_uint64),
                ("metas_bound", C.c_uint64), ("pages_bound", C.c_uint64), ("workspace_bytes", C.c_uint64)]


class _CAsyncCompressWrappedStatus(C.Structure):  # PcoB200AsyncCompressWrappedStatus (include/pco_b200.h)
    _fields_ = [("kind", C.c_uint32), ("device_status", C.c_uint32), ("array", C.c_uint64), ("n_arrays", C.c_uint64), ("n_chunks", C.c_uint64),
                ("metas_bytes", C.c_uint64), ("pages_bytes", C.c_uint64), ("metas_written", C.c_uint64), ("pages_written", C.c_uint64)]


def _lib_async_compress_wrapped():
    return _lib.bind("_async_compress_wrapped_ready",
                     pco_b200_compress_wrapped_async_plan=[C.c_ubyte, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t,
                                                           C.c_void_p],
                     pco_b200_compress_wrapped_async=[C.c_void_p] * 11,
                     pco_b200_compress_wrapped_async_result=[C.c_void_p, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)])


class AsyncChunksCompressor(_lib._AsyncCall):
    """Compresses a batch of arrays into wrapped chunks of one page each on the current CUDA stream, with the array sizes in device memory
    and without waiting for the device (pco_b200_compress_wrapped_async): column chunks a kernel sized need no trip to the host, and a call
    can be captured in a torch.cuda.CUDAGraph.  Each array is cut into the chunks compress_chunks writes for it alone, and its metas, pages
    and refs equal compress_chunks's, placed behind the arrays before it.

    The plan fixes the number type `dtype`, the config (explicit mode and delta specs, EqualPagesUpTo paging) and the capacities: at most
    max_arrays arrays, nums_cap numbers in all and max_array_n per array, metas_cap bytes of metas and pages_cap bytes of pages (default:
    the plan's metas_bound and pages_bound, which every batch within the capacities fits in).  The refs come out as the int64
    (max_chunks, 5) tensor AsyncPagesDecompressor takes, so one graph can compress pages and decode them.  The compressor owns a device
    workspace and a status; it serves one call in flight."""

    _Plan, _Status = _CAsyncCompressWrappedPlan, _CAsyncCompressWrappedStatus

    def __init__(self, dtype, config, max_arrays, nums_cap, max_array_n, metas_cap=None, pages_cap=None, device=None):
        self.dtype = np.dtype(dtype)
        dtb = _lib.dtype_byte(self.dtype)
        L = _lib_async_compress_wrapped()
        cfg = (config or ChunkConfig())._to_c()

        def plan_fn(mcap, pcap):
            return lambda plan: L.pco_b200_compress_wrapped_async_plan(C.c_ubyte(dtb), C.byref(cfg), C.c_size_t(max_arrays), C.c_size_t(nums_cap),
                                                                       C.c_size_t(max_array_n), C.c_size_t(mcap), C.c_size_t(pcap), plan)

        # the bounds are known once a plan exists: a first plan reports them
        self._make_plan(device, plan_fn(metas_cap or 0, pages_cap or 0))
        if metas_cap is None or pages_cap is None:
            self._replan(plan_fn(self._plan.metas_bound if metas_cap is None else metas_cap, self._plan.pages_bound if pages_cap is None else pages_cap))
        self._alloc()

    @property
    def metas_cap(self):
        return int(self._plan.metas_cap)

    @property
    def pages_cap(self):
        return int(self._plan.pages_cap)

    @property
    def max_arrays(self):
        return int(self._plan.max_arrays)

    @property
    def max_chunks(self):
        """Rows of `refs` a call takes: the most chunks of any batch within the capacities."""
        return int(self._plan.max_chunks)

    def __call__(self, nums, array_ns, n_arrays, metas, pages, refs, first_chunk):
        """Enqueues the compress of the first n_arrays[0] arrays on torch.cuda.current_stream(): array i is the next array_ns[i] numbers of
        `nums` (a CUDA tensor of the plan's dtype, at least nums_cap numbers).  `array_ns` is an int64 CUDA tensor of at least max_arrays
        elements, `n_arrays` a 1-element int64 CUDA tensor, `metas` and `pages` uint8 CUDA tensors of at least metas_cap and pages_cap
        bytes, `refs` the int64 (max_chunks, 5) CUDA tensor of PAGE_REF fields that AsyncPagesDecompressor takes, and `first_chunk` an int64
        CUDA tensor of max_arrays + 1 elements: array i's chunks are refs[first_chunk[i] : first_chunk[i + 1]].  Returns nothing and does
        not wait; result() reports the outcome."""
        import torch

        p = self._plan
        self._check_tensors(nums=nums, array_ns=array_ns, n_arrays=n_arrays, metas=metas, pages=pages, refs=refs, first_chunk=first_chunk)
        if nums.dtype != _torch_dtypes()[self.dtype] or nums.numel() < p.nums_cap:
            raise ValueError(f"nums must hold at least nums_cap = {p.nums_cap} numbers of {self.dtype}")
        if array_ns.dtype != torch.int64 or array_ns.numel() < p.max_arrays:
            raise ValueError(f"array_ns must be an int64 tensor of at least max_arrays = {p.max_arrays} elements")
        if n_arrays.dtype != torch.int64 or n_arrays.numel() != 1:
            raise ValueError("n_arrays must be a 1-element int64 tensor")
        if metas.numel() * metas.element_size() < p.metas_cap or pages.numel() * pages.element_size() < p.pages_cap:
            raise ValueError(f"metas holds fewer than metas_cap = {p.metas_cap} bytes, or pages fewer than pages_cap = {p.pages_cap}")
        if refs.dtype != torch.int64 or refs.dim() != 2 or refs.shape[1] != 5 or refs.shape[0] < p.max_chunks:
            raise ValueError(f"refs must be an int64 tensor of shape ({p.max_chunks}, 5)")
        if first_chunk.dtype != torch.int64 or first_chunk.numel() < p.max_arrays + 1:
            raise ValueError(f"first_chunk must be an int64 tensor of at least max_arrays + 1 = {p.max_arrays + 1} elements")
        rc = _lib_async_compress_wrapped().pco_b200_compress_wrapped_async(
            C.byref(p), C.c_void_p(nums.data_ptr()), C.c_void_p(array_ns.data_ptr()), C.c_void_p(n_arrays.data_ptr()), C.c_void_p(metas.data_ptr()),
            C.c_void_p(pages.data_ptr()), C.c_void_p(refs.data_ptr()), C.c_void_p(first_chunk.data_ptr()), C.c_void_p(self.workspace.data_ptr()),
            C.c_void_p(self.status.data_ptr()), self._stream())
        _lib.check(rc)

    def result(self):
        """Copies the status of the last call back (waiting for it on the current stream) and returns (metas_len, pages_len, n_chunks), or
        raises PcoError with the kind compress_chunks gives ("array 17: ...")."""
        s = self.status_record()
        ml, pl, nc = C.c_size_t(), C.c_size_t(), C.c_size_t()
        _lib.check(_lib_async_compress_wrapped().pco_b200_compress_wrapped_async_result(C.byref(s), C.byref(ml), C.byref(pl), C.byref(nc)))
        return int(ml.value), int(pl.value), int(nc.value)


class _CAsyncFilterPlan(C.Structure):  # PcoB200AsyncFilterPlan (include/pco_b200.h)
    _fields_ = [("dtype", C.c_uint32), ("reserved", C.c_uint32), ("metas_cap", C.c_uint64), ("pages_cap", C.c_uint64), ("max_pages", C.c_uint64),
                ("rows_cap", C.c_uint64), ("frame_cap", C.c_uint64), ("out_cap", C.c_uint64), ("workspace_bytes", C.c_uint64)]


class _CAsyncFilterStatus(C.Structure):  # PcoB200AsyncFilterStatus (include/pco_b200.h)
    _fields_ = [("kind", C.c_uint32), ("device_status", C.c_uint32), ("page", C.c_uint64), ("n_written", C.c_uint64), ("n_pages", C.c_uint64),
                ("frames_needed", C.c_uint64), ("n_matches", C.c_uint64), ("matches_needed", C.c_uint64)]


def _lib_async_filter():
    return _lib.bind("_async_filter_ready",
                     pco_b200_filter_pages_async_plan=[C.c_ubyte, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p],
                     pco_b200_filter_pages_async=[C.c_void_p] * 12,
                     pco_b200_filter_pages_async_result=[C.c_void_p, C.POINTER(C.c_size_t)])


def pack_interval(lo, hi, dtype):
    """The PcoB200Interval of [lo, hi] for numbers of `dtype`: a 2-element int64 array holding each bound's bit pattern, zero-extended
    (copy it to a CUDA tensor for AsyncPagesFilter).  The bounds are Python or numpy numbers, converted to `dtype` (NaN and infinities
    included for floats); a bound outside an integer dtype's range raises OverflowError."""
    return _pack_values((lo, hi), dtype, "bound")


def _pack_values(values, dtype, what):
    """The zero-extended bit patterns of `values` as numbers of `dtype` (an int64 array): the per-value conversion pack_interval and
    pack_edges share.  `what` names a value in the errors."""
    dt = np.dtype(dtype)
    _lib.dtype_byte(dt)
    ut = np.dtype(f"u{dt.itemsize}")
    bits = []
    for x in values:
        if dt.kind in "iu":
            info = np.iinfo(dt)
            if isinstance(x, (float, np.floating)) and not float(x).is_integer():
                raise TypeError(f"{what} {x!r} is not an integer of {dt}")
            if not info.min <= int(x) <= info.max:
                raise OverflowError(f"{what} {x!r} lies outside {dt}")
            v = np.array([int(x)], dtype=dt)
        else:
            v = np.array([x], dtype=dt)
        bits.append(int(v.view(ut)[0]))
    return np.array(bits, dtype=np.uint64).view(np.int64)


def pack_edges(edges, dtype):
    """The B + 1 bucket edges `edges` (a sequence or array of Python or numpy numbers) for numbers of `dtype` as the int64 array of their
    zero-extended bit patterns that AsyncPagesHistogram and standalone.AsyncFilesHistogram read (copy it to a CUDA tensor), converted as
    pack_interval converts its bounds.  Whether the edges ascend is checked by the call, on the device."""
    return _pack_values(list(edges), dtype, "edge")


def unpack_aggregates(records, dtype):
    """The PcoB200Aggregate records `records` (an int64 array of shape (n, 6) or (6,), on the host) of numbers of `dtype` as a list of
    (n_rows, count, min, max, sum) tuples: min and max as numpy scalars of `dtype` (0 when count is 0), the sum as a Python int (the exact
    128-bit sum, signed for signed dtypes) or, for floats, a float (the f64 sum)."""
    dt = np.dtype(dtype)
    _lib.dtype_byte(dt)
    ut = np.dtype(f"u{dt.itemsize}")
    recs = np.asarray(records).reshape(-1, 6).view(np.uint64)
    out = []
    for n_rows, count, mn, mx, lo, hi in recs.tolist():
        as_dt = lambda bits: np.array([bits], dtype=np.uint64).astype(ut).view(dt)[0]  # noqa: E731
        if dt.kind == "f":
            total = float(np.array([lo], dtype=np.uint64).view(np.float64)[0])
        else:
            total = (hi << 64) | lo
            if dt.kind == "i" and hi >> 63:
                total -= 1 << 128
        out.append((int(n_rows), int(count), as_dt(mn), as_dt(mx), total))
    return out


class _CAsyncAggregatePlan(C.Structure):  # PcoB200AsyncAggregatePlan (include/pco_b200.h)
    _fields_ = [("dtype", C.c_uint32), ("reserved", C.c_uint32), ("metas_cap", C.c_uint64), ("pages_cap", C.c_uint64), ("max_pages", C.c_uint64),
                ("rows_cap", C.c_uint64), ("frame_cap", C.c_uint64), ("workspace_bytes", C.c_uint64)]


class _CAsyncAggregateStatus(C.Structure):  # PcoB200AsyncAggregateStatus (include/pco_b200.h)
    _fields_ = [("kind", C.c_uint32), ("device_status", C.c_uint32), ("page", C.c_uint64), ("n_written", C.c_uint64), ("n_pages", C.c_uint64),
                ("frames_needed", C.c_uint64), ("n_matches", C.c_uint64)]


def _lib_async_aggregate():
    return _lib.bind("_async_aggregate_ready",
                     pco_b200_aggregate_pages_async_plan=[C.c_ubyte, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p],
                     pco_b200_aggregate_pages_async=[C.c_void_p] * 11,
                     pco_b200_aggregate_pages_async_result=[C.c_void_p, C.POINTER(C.c_size_t)])


def _check_aggregate_outputs(aggs, total, max_groups):
    import torch

    if aggs.dtype != torch.int64 or aggs.dim() != 2 or aggs.shape[1] != 6 or aggs.shape[0] < max_groups or not aggs.is_contiguous():
        raise ValueError(f"aggs must be a contiguous int64 tensor of shape ({max_groups}, 6)")
    if total.dtype != torch.int64 or total.numel() != 6 or not total.is_contiguous():
        raise ValueError("total must be a contiguous 6-element int64 tensor")


class AsyncPagesAggregate(_lib._AsyncCall):
    """Decodes a batch of wrapped-format pages on the current CUDA stream and reduces the numbers inside a closed interval to count, min,
    max and sum, per page and in all (pco_b200_aggregate_pages_async): each 256-number batch is reduced in the decoder's registers, so
    neither the decoded pages nor the matches reach HBM.  Refs, their count and the interval are read from device tensors, so one captured
    call serves new pages and new bounds on each replay.

    The capacities are AsyncPagesDecompressor's, with rows_cap (the most numbers of a call's pages) in place of dst_cap; frame_cap defaults
    to metas_cap + pages_cap + 20 * max_pages as there.  The call owns a device workspace (about rows_cap * (itemsize + 0.15) bytes beyond
    the decompressor's) and a status; it serves one call in flight."""

    _Plan, _Status = _CAsyncAggregatePlan, _CAsyncAggregateStatus

    def __init__(self, dtype, metas_cap, pages_cap, max_pages, rows_cap, frame_cap=None, device=None):
        self.dtype = np.dtype(dtype)
        if frame_cap is None:
            frame_cap = metas_cap + pages_cap + 20 * max_pages
        self._make_plan(device, lambda plan: _lib_async_aggregate().pco_b200_aggregate_pages_async_plan(
            C.c_ubyte(_lib.dtype_byte(self.dtype)), C.c_size_t(metas_cap), C.c_size_t(pages_cap), C.c_size_t(max_pages), C.c_size_t(rows_cap),
            C.c_size_t(frame_cap), plan))
        self._alloc()

    def __call__(self, metas, pages, refs, n_pages, interval, aggs, total):
        """Enqueues the aggregates of the pages refs[: n_pages[0]] names on torch.cuda.current_stream().  `metas`, `pages`, `refs` and
        `n_pages` are as AsyncPagesDecompressor takes them; `interval` is a 2-element int64 CUDA tensor (pack_interval's bit patterns of lo
        and hi), `aggs` an int64 CUDA tensor of shape (max_pages, 6) whose row i receives page i's PcoB200Aggregate, and `total` a 6-element
        int64 CUDA tensor that receives the total (unpack_aggregates reads them).  Returns nothing and does not wait; result() reports the
        outcome."""
        import torch

        p = self._plan
        self._check_tensors(metas=metas, pages=pages, refs=refs, n_pages=n_pages, interval=interval, aggs=aggs, total=total)
        if metas.numel() * metas.element_size() < p.metas_cap or pages.numel() * pages.element_size() < p.pages_cap:
            raise ValueError(f"metas holds fewer than metas_cap = {p.metas_cap} bytes, or pages fewer than pages_cap = {p.pages_cap}")
        if refs.dtype != torch.int64 or refs.dim() != 2 or refs.shape[1] != 5 or refs.shape[0] < p.max_pages:
            raise ValueError(f"refs must be an int64 tensor of shape ({p.max_pages}, 5)")
        if n_pages.dtype != torch.int64 or n_pages.numel() != 1:
            raise ValueError("n_pages must be a 1-element int64 tensor")
        if interval.dtype != torch.int64 or interval.numel() != 2:
            raise ValueError("interval must be a 2-element int64 tensor")
        _check_aggregate_outputs(aggs, total, p.max_pages)
        rc = _lib_async_aggregate().pco_b200_aggregate_pages_async(
            C.byref(p), C.c_void_p(metas.data_ptr()), C.c_void_p(pages.data_ptr()), C.c_void_p(refs.data_ptr()), C.c_void_p(n_pages.data_ptr()),
            C.c_void_p(interval.data_ptr()), C.c_void_p(aggs.data_ptr()), C.c_void_p(total.data_ptr()), C.c_void_p(self.workspace.data_ptr()),
            C.c_void_p(self.status.data_ptr()), self._stream())
        _lib.check(rc)

    def result(self):
        """Copies the status of the last call back (waiting for it on the current stream) and returns the total match count, or raises
        PcoError with the kind decompress_pages gives ("page 17: ...")."""
        s = self.status_record()
        nm = C.c_size_t()
        _lib.check(_lib_async_aggregate().pco_b200_aggregate_pages_async_result(C.byref(s), C.byref(nm)))
        return int(nm.value)


class _CAsyncHistogramPlan(C.Structure):  # PcoB200AsyncHistogramPlan (include/pco_b200.h)
    _fields_ = [("dtype", C.c_uint32), ("reserved", C.c_uint32), ("metas_cap", C.c_uint64), ("pages_cap", C.c_uint64), ("max_pages", C.c_uint64),
                ("rows_cap", C.c_uint64), ("frame_cap", C.c_uint64), ("n_buckets", C.c_uint64), ("workspace_bytes", C.c_uint64)]


class _CAsyncHistogramStatus(C.Structure):  # PcoB200AsyncHistogramStatus (include/pco_b200.h)
    _fields_ = [("kind", C.c_uint32), ("device_status", C.c_uint32), ("page", C.c_uint64), ("n_written", C.c_uint64), ("n_pages", C.c_uint64),
                ("frames_needed", C.c_uint64), ("edge", C.c_uint64)]


def _lib_async_histogram():
    return _lib.bind("_async_histogram_ready",
                     pco_b200_histogram_pages_async_plan=[C.c_ubyte, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t,
                                                          C.c_void_p],
                     pco_b200_histogram_pages_async=[C.c_void_p] * 11,
                     pco_b200_histogram_pages_async_result=[C.c_void_p, C.POINTER(C.c_size_t)])


def _check_histogram_inputs(edges, hists, total, n_buckets, max_groups):
    import torch

    w = n_buckets + 3
    if edges.dtype != torch.int64 or edges.numel() != n_buckets + 1:
        raise ValueError(f"edges must be an int64 tensor of {n_buckets + 1} elements (pack_edges' bit patterns)")
    if hists.dtype != torch.int64 or hists.dim() != 2 or hists.shape[1] != w or hists.shape[0] < max_groups or not hists.is_contiguous():
        raise ValueError(f"hists must be a contiguous int64 tensor of shape ({max_groups}, {w})")
    if total.dtype != torch.int64 or total.numel() != w or not total.is_contiguous():
        raise ValueError(f"total must be a contiguous {w}-element int64 tensor")


class AsyncPagesHistogram(_lib._AsyncCall):
    """Decodes a batch of wrapped-format pages on the current CUDA stream and counts how many numbers fall in each of n_buckets buckets,
    per page and in all (pco_b200_histogram_pages_async): each decode CTA counts its numbers in shared memory, so the decoded pages never
    reach HBM.  Refs, their count and the edges are read from device tensors, so one captured call serves new pages and new edges on each
    replay.  A row holds n_buckets + 3 counts: below edge 0, the buckets (the last one closed, as numpy.histogram's), above the last edge,
    and NaNs.

    The capacities are AsyncPagesDecompressor's, with rows_cap (the most numbers of a call's pages) in place of dst_cap; frame_cap defaults
    to metas_cap + pages_cap + 20 * max_pages as there.  n_buckets (1 .. 4096) is fixed by the plan.  The call owns a device workspace
    (about rows_cap * itemsize + 8 * (n_buckets + 3) * max_pages bytes beyond the decompressor's) and a status; it serves one call in
    flight."""

    _Plan, _Status = _CAsyncHistogramPlan, _CAsyncHistogramStatus

    def __init__(self, dtype, metas_cap, pages_cap, max_pages, rows_cap, n_buckets, frame_cap=None, device=None):
        self.dtype = np.dtype(dtype)
        if frame_cap is None:
            frame_cap = metas_cap + pages_cap + 20 * max_pages
        self._make_plan(device, lambda plan: _lib_async_histogram().pco_b200_histogram_pages_async_plan(
            C.c_ubyte(_lib.dtype_byte(self.dtype)), C.c_size_t(metas_cap), C.c_size_t(pages_cap), C.c_size_t(max_pages), C.c_size_t(rows_cap),
            C.c_size_t(frame_cap), C.c_size_t(n_buckets), plan))
        self._alloc()

    def __call__(self, metas, pages, refs, n_pages, edges, hists, total):
        """Enqueues the histograms of the pages refs[: n_pages[0]] names on torch.cuda.current_stream().  `metas`, `pages`, `refs` and
        `n_pages` are as AsyncPagesDecompressor takes them; `edges` is an int64 CUDA tensor of n_buckets + 1 elements (pack_edges' bit
        patterns), `hists` an int64 CUDA tensor of shape (max_pages, n_buckets + 3) whose row i receives page i's counts, and `total` an
        int64 CUDA tensor of n_buckets + 3 elements that receives their column sums.  Returns nothing and does not wait; result() reports
        the outcome."""
        import torch

        p = self._plan
        self._check_tensors(metas=metas, pages=pages, refs=refs, n_pages=n_pages, edges=edges, hists=hists, total=total)
        if metas.numel() * metas.element_size() < p.metas_cap or pages.numel() * pages.element_size() < p.pages_cap:
            raise ValueError(f"metas holds fewer than metas_cap = {p.metas_cap} bytes, or pages fewer than pages_cap = {p.pages_cap}")
        if refs.dtype != torch.int64 or refs.dim() != 2 or refs.shape[1] != 5 or refs.shape[0] < p.max_pages:
            raise ValueError(f"refs must be an int64 tensor of shape ({p.max_pages}, 5)")
        if n_pages.dtype != torch.int64 or n_pages.numel() != 1:
            raise ValueError("n_pages must be a 1-element int64 tensor")
        _check_histogram_inputs(edges, hists, total, p.n_buckets, p.max_pages)
        rc = _lib_async_histogram().pco_b200_histogram_pages_async(
            C.byref(p), C.c_void_p(metas.data_ptr()), C.c_void_p(pages.data_ptr()), C.c_void_p(refs.data_ptr()), C.c_void_p(n_pages.data_ptr()),
            C.c_void_p(edges.data_ptr()), C.c_void_p(hists.data_ptr()), C.c_void_p(total.data_ptr()), C.c_void_p(self.workspace.data_ptr()),
            C.c_void_p(self.status.data_ptr()), self._stream())
        _lib.check(rc)

    def result(self):
        """Copies the status of the last call back (waiting for it on the current stream) and returns the numbers counted, or raises
        PcoError with the kind decompress_pages gives ("page 17: ...") or naming the lowest bad edge ("edge 3: ...")."""
        s = self.status_record()
        n = C.c_size_t()
        _lib.check(_lib_async_histogram().pco_b200_histogram_pages_async_result(C.byref(s), C.byref(n)))
        return int(n.value)


class _CAsyncTopkPlan(C.Structure):  # PcoB200AsyncTopkPlan (include/pco_b200.h)
    _fields_ = [("dtype", C.c_uint32), ("largest", C.c_uint32), ("metas_cap", C.c_uint64), ("pages_cap", C.c_uint64), ("max_pages", C.c_uint64),
                ("rows_cap", C.c_uint64), ("frame_cap", C.c_uint64), ("k", C.c_uint64), ("workspace_bytes", C.c_uint64)]


class _CAsyncTopkStatus(C.Structure):  # PcoB200AsyncTopkStatus (include/pco_b200.h)
    _fields_ = [("kind", C.c_uint32), ("device_status", C.c_uint32), ("page", C.c_uint64), ("n_written", C.c_uint64), ("n_pages", C.c_uint64),
                ("frames_needed", C.c_uint64), ("n_matches", C.c_uint64)]


def _lib_async_topk():
    return _lib.bind("_async_topk_ready",
                     pco_b200_topk_pages_async_plan=[C.c_ubyte, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int,
                                                     C.c_void_p],
                     pco_b200_topk_pages_async=[C.c_void_p] * 12,
                     pco_b200_topk_pages_async_result=[C.c_void_p, C.POINTER(C.c_size_t)])


def _check_topk_inputs(interval, out_values, out_positions, n_out, k, dtype):
    import torch

    if interval.dtype != torch.int64 or interval.numel() != 2:
        raise ValueError("interval must be a 2-element int64 tensor (pack_interval's bit patterns)")
    if out_values.dtype != _torch_dtypes()[np.dtype(dtype)] or out_values.numel() < k or not out_values.is_contiguous():
        raise ValueError(f"out_values must be a contiguous tensor of at least k = {k} numbers of {np.dtype(dtype)}")
    if out_positions.dtype != torch.int64 or out_positions.numel() < k or not out_positions.is_contiguous():
        raise ValueError(f"out_positions must be a contiguous int64 tensor of at least k = {k} elements")
    if n_out.dtype != torch.int64 or n_out.numel() != 1:
        raise ValueError("n_out must be a 1-element int64 tensor")


class AsyncPagesTopK(_lib._AsyncCall):
    """Decodes a batch of wrapped-format pages on the current CUDA stream and returns the k smallest (largest=False) or k largest
    (largest=True) numbers inside a closed interval, with their positions in the pages' concatenation (pco_b200_topk_pages_async): each
    decode CTA keeps its best matches in shared memory, so the decoded pages never reach HBM.  Numbers compare as AsyncPagesFilter compares
    them; ties go to the lower position, so the output is a unique function of the numbers.  Refs, their count and the interval are read
    from device tensors, so one captured call serves new pages and a new interval on each replay.

    The capacities are AsyncPagesDecompressor's, with rows_cap (the most numbers of a call's pages) in place of dst_cap; frame_cap defaults
    to metas_cap + pages_cap + 20 * max_pages as there.  k (1 .. 1024) and the direction are fixed by the plan.  The call owns a device
    workspace (about rows_cap * itemsize + 16 * k * max_pages bytes beyond the decompressor's) and a status; it serves one call in
    flight."""

    _Plan, _Status = _CAsyncTopkPlan, _CAsyncTopkStatus

    def __init__(self, dtype, metas_cap, pages_cap, max_pages, rows_cap, k, largest=False, frame_cap=None, device=None):
        self.dtype = np.dtype(dtype)
        if frame_cap is None:
            frame_cap = metas_cap + pages_cap + 20 * max_pages
        self._make_plan(device, lambda plan: _lib_async_topk().pco_b200_topk_pages_async_plan(
            C.c_ubyte(_lib.dtype_byte(self.dtype)), C.c_size_t(metas_cap), C.c_size_t(pages_cap), C.c_size_t(max_pages), C.c_size_t(rows_cap),
            C.c_size_t(frame_cap), C.c_size_t(k), C.c_int(int(largest)), plan))
        self._alloc()

    def __call__(self, metas, pages, refs, n_pages, interval, out_values, out_positions, n_out):
        """Enqueues the top-k of the pages refs[: n_pages[0]] names on torch.cuda.current_stream().  `metas`, `pages`, `refs` and
        `n_pages` are as AsyncPagesDecompressor takes them and `interval` as AsyncPagesFilter takes it (pack_interval(lo, hi, dtype) on the
        device; the full range of the dtype for every number).  The best numbers, best first, go to out_values (a CUDA tensor of at least
        k numbers of the dtype, each with its own bits), their positions to out_positions (an int64 CUDA tensor of at least k elements) and
        their count, min(k, matches), to n_out (a 1-element int64 CUDA tensor; 0 on a failure).  Returns nothing and does not wait;
        result() reports the outcome."""
        import torch

        p = self._plan
        self._check_tensors(metas=metas, pages=pages, refs=refs, n_pages=n_pages, interval=interval, out_values=out_values,
                            out_positions=out_positions, n_out=n_out)
        if metas.numel() * metas.element_size() < p.metas_cap or pages.numel() * pages.element_size() < p.pages_cap:
            raise ValueError(f"metas holds fewer than metas_cap = {p.metas_cap} bytes, or pages fewer than pages_cap = {p.pages_cap}")
        if refs.dtype != torch.int64 or refs.dim() != 2 or refs.shape[1] != 5 or refs.shape[0] < p.max_pages:
            raise ValueError(f"refs must be an int64 tensor of shape ({p.max_pages}, 5)")
        if n_pages.dtype != torch.int64 or n_pages.numel() != 1:
            raise ValueError("n_pages must be a 1-element int64 tensor")
        _check_topk_inputs(interval, out_values, out_positions, n_out, p.k, self.dtype)
        rc = _lib_async_topk().pco_b200_topk_pages_async(
            C.byref(p), C.c_void_p(metas.data_ptr()), C.c_void_p(pages.data_ptr()), C.c_void_p(refs.data_ptr()), C.c_void_p(n_pages.data_ptr()),
            C.c_void_p(interval.data_ptr()), C.c_void_p(out_values.data_ptr()), C.c_void_p(out_positions.data_ptr()), C.c_void_p(n_out.data_ptr()),
            C.c_void_p(self.workspace.data_ptr()), C.c_void_p(self.status.data_ptr()), self._stream())
        _lib.check(rc)

    def result(self):
        """Copies the status of the last call back (waiting for it on the current stream) and returns the numbers inside the interval, or
        raises PcoError with the kind decompress_pages gives ("page 17: ...")."""
        s = self.status_record()
        n = C.c_size_t()
        _lib.check(_lib_async_topk().pco_b200_topk_pages_async_result(C.byref(s), C.byref(n)))
        return int(n.value)


class _CAsyncTakePlan(C.Structure):  # PcoB200AsyncTakePlan (include/pco_b200.h)
    _fields_ = [("dtype", C.c_uint32), ("reserved", C.c_uint32), ("metas_cap", C.c_uint64), ("pages_cap", C.c_uint64), ("max_pages", C.c_uint64),
                ("rows_cap", C.c_uint64), ("frame_cap", C.c_uint64), ("max_positions", C.c_uint64), ("workspace_bytes", C.c_uint64)]


class _CAsyncTakeStatus(C.Structure):  # PcoB200AsyncTakeStatus (include/pco_b200.h)
    _fields_ = [("kind", C.c_uint32), ("device_status", C.c_uint32), ("page", C.c_uint64), ("n_written", C.c_uint64), ("n_pages", C.c_uint64),
                ("frames_needed", C.c_uint64), ("n_positions", C.c_uint64), ("position", C.c_uint64), ("records_decoded", C.c_uint64)]


def _lib_async_take():
    return _lib.bind("_async_take_ready",
                     pco_b200_take_pages_async_plan=[C.c_ubyte, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p],
                     pco_b200_take_pages_async=[C.c_void_p] * 11,
                     pco_b200_take_pages_async_result=[C.c_void_p, C.POINTER(C.c_size_t)])


def _check_take_tensors(positions, n_positions, values, dtype, max_positions):
    import torch

    if positions.dtype != torch.int64 or positions.numel() < max_positions:
        raise ValueError(f"positions must be an int64 tensor of at least max_positions = {max_positions} elements")
    if n_positions.dtype != torch.int64 or n_positions.numel() != 1:
        raise ValueError("n_positions must be a 1-element int64 tensor")
    if values.dtype != _torch_dtypes()[dtype] or values.numel() < max_positions:
        raise ValueError(f"values must hold at least max_positions = {max_positions} numbers of {dtype}")


class AsyncPagesTake(_lib._AsyncCall):
    """Takes the numbers at strictly ascending positions of a batch of wrapped-format pages' concatenation on the current CUDA stream
    (pco_b200_take_pages_async), decoding only the pages the positions touch: each decoded batch writes its selected numbers straight to
    their final index.  Refs, their count, the positions and their count are read from device tensors, so one captured call serves new
    pages and new positions on each replay, and AsyncPagesFilter's positions and count can be passed straight in.

    The capacities are AsyncPagesDecompressor's, with rows_cap (the most numbers of a call's pages) in place of dst_cap, and max_positions
    the most positions a call takes; frame_cap defaults to metas_cap + pages_cap + 20 * max_pages as there.  The call owns a device
    workspace (about rows_cap * (itemsize + 0.07) bytes beyond the decompressor's) and a status; it serves one call in flight."""

    _Plan, _Status = _CAsyncTakePlan, _CAsyncTakeStatus

    def __init__(self, dtype, metas_cap, pages_cap, max_pages, rows_cap, max_positions, frame_cap=None, device=None):
        self.dtype = np.dtype(dtype)
        if frame_cap is None:
            frame_cap = metas_cap + pages_cap + 20 * max_pages
        self._make_plan(device, lambda plan: _lib_async_take().pco_b200_take_pages_async_plan(
            C.c_ubyte(_lib.dtype_byte(self.dtype)), C.c_size_t(metas_cap), C.c_size_t(pages_cap), C.c_size_t(max_pages), C.c_size_t(rows_cap),
            C.c_size_t(frame_cap), C.c_size_t(max_positions), plan))
        self._alloc()

    def __call__(self, metas, pages, refs, n_pages, positions, n_positions, values):
        """Enqueues the take of positions[: n_positions[0]] from the pages refs[: n_pages[0]] names on torch.cuda.current_stream().
        `metas`, `pages`, `refs` and `n_pages` are as AsyncPagesDecompressor takes them; `positions` is an int64 CUDA tensor of at least
        max_positions elements (strictly ascending indices into the pages' concatenation), `n_positions` a 1-element int64 CUDA tensor, and
        `values` a CUDA tensor of the plan's dtype of at least max_positions elements that receives the numbers.  Returns nothing and does
        not wait; result() reports the outcome."""
        import torch

        p = self._plan
        self._check_tensors(metas=metas, pages=pages, refs=refs, n_pages=n_pages, positions=positions, n_positions=n_positions, values=values)
        if metas.numel() * metas.element_size() < p.metas_cap or pages.numel() * pages.element_size() < p.pages_cap:
            raise ValueError(f"metas holds fewer than metas_cap = {p.metas_cap} bytes, or pages fewer than pages_cap = {p.pages_cap}")
        if refs.dtype != torch.int64 or refs.dim() != 2 or refs.shape[1] != 5 or refs.shape[0] < p.max_pages:
            raise ValueError(f"refs must be an int64 tensor of shape ({p.max_pages}, 5)")
        if n_pages.dtype != torch.int64 or n_pages.numel() != 1:
            raise ValueError("n_pages must be a 1-element int64 tensor")
        _check_take_tensors(positions, n_positions, values, self.dtype, p.max_positions)
        rc = _lib_async_take().pco_b200_take_pages_async(
            C.byref(p), C.c_void_p(metas.data_ptr()), C.c_void_p(pages.data_ptr()), C.c_void_p(refs.data_ptr()), C.c_void_p(n_pages.data_ptr()),
            C.c_void_p(positions.data_ptr()), C.c_void_p(n_positions.data_ptr()), C.c_void_p(values.data_ptr()),
            C.c_void_p(self.workspace.data_ptr()), C.c_void_p(self.status.data_ptr()), self._stream())
        _lib.check(rc)

    def result(self):
        """Copies the status of the last call back (waiting for it on the current stream) and returns the number of values written, or
        raises PcoError with the kind decompress_pages gives ("page 17: ...") or, for the positions, InvalidArgument ("position 17: ...")."""
        s = self.status_record()
        nw = C.c_size_t()
        _lib.check(_lib_async_take().pco_b200_take_pages_async_result(C.byref(s), C.byref(nw)))
        return int(nw.value)


class _CAsyncSegmentAggregatePlan(C.Structure):  # PcoB200AsyncSegmentAggregatePlan (include/pco_b200.h)
    _fields_ = [("dtype", C.c_uint32), ("reserved", C.c_uint32), ("metas_cap", C.c_uint64), ("pages_cap", C.c_uint64), ("max_pages", C.c_uint64),
                ("rows_cap", C.c_uint64), ("frame_cap", C.c_uint64), ("max_segments", C.c_uint64), ("workspace_bytes", C.c_uint64)]


class _CAsyncSegmentAggregateStatus(C.Structure):  # PcoB200AsyncSegmentAggregateStatus (include/pco_b200.h)
    _fields_ = [("kind", C.c_uint32), ("device_status", C.c_uint32), ("page", C.c_uint64), ("n_written", C.c_uint64), ("n_pages", C.c_uint64),
                ("frames_needed", C.c_uint64), ("n_segments", C.c_uint64), ("segment", C.c_uint64), ("records_decoded", C.c_uint64),
                ("n_matches", C.c_uint64)]


def _lib_async_segment_aggregate():
    return _lib.bind("_async_segment_aggregate_ready",
                     pco_b200_segment_aggregate_pages_async_plan=[C.c_ubyte, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t,
                                                                  C.c_size_t, C.c_void_p],
                     pco_b200_segment_aggregate_pages_async=[C.c_void_p] * 13,
                     pco_b200_segment_aggregate_pages_async_result=[C.c_void_p, C.POINTER(C.c_size_t)])


def _check_segment_tensors(bounds, n_segments, interval, aggs, total, max_segments):
    import torch

    if bounds.dtype != torch.int64 or bounds.numel() < max_segments + 1:
        raise ValueError(f"bounds must be an int64 tensor of at least max_segments + 1 = {max_segments + 1} elements")
    if n_segments.dtype != torch.int64 or n_segments.numel() != 1:
        raise ValueError("n_segments must be a 1-element int64 tensor")
    if interval.dtype != torch.int64 or interval.numel() != 2:
        raise ValueError("interval must be a 2-element int64 tensor")
    _check_aggregate_outputs(aggs, total, max_segments)


class AsyncPagesSegmentAggregate(_lib._AsyncCall):
    """Decodes a batch of wrapped-format pages on the current CUDA stream and reduces the numbers inside a closed interval to count, min,
    max and sum per row segment [bounds[g], bounds[g + 1]) of the pages' concatenation and in all (pco_b200_segment_aggregate_pages_async):
    time buckets, per-session ranges or a window's rows, with only the pages the segments cover decoded and each 256-number batch reduced
    in the decoder's registers.  Refs, their count, the bounds, their count and the interval are read from device tensors, so one captured
    call serves new pages and new segments on each replay, and torch.searchsorted's output can be passed straight in.

    The capacities are AsyncPagesAggregate's, with max_segments the most segments a call reduces.  The call owns a device workspace (about
    rows_cap * (itemsize + 0.2) + 96 * max_segments bytes beyond the decompressor's) and a status; it serves one call in flight.
    unpack_aggregates reads the records."""

    _Plan, _Status = _CAsyncSegmentAggregatePlan, _CAsyncSegmentAggregateStatus

    def __init__(self, dtype, metas_cap, pages_cap, max_pages, rows_cap, max_segments, frame_cap=None, device=None):
        self.dtype = np.dtype(dtype)
        if frame_cap is None:
            frame_cap = metas_cap + pages_cap + 20 * max_pages
        self._make_plan(device, lambda plan: _lib_async_segment_aggregate().pco_b200_segment_aggregate_pages_async_plan(
            C.c_ubyte(_lib.dtype_byte(self.dtype)), C.c_size_t(metas_cap), C.c_size_t(pages_cap), C.c_size_t(max_pages), C.c_size_t(rows_cap),
            C.c_size_t(frame_cap), C.c_size_t(max_segments), plan))
        self._alloc()

    def __call__(self, metas, pages, refs, n_pages, bounds, n_segments, interval, aggs, total):
        """Enqueues the segment aggregates of the pages refs[: n_pages[0]] names on torch.cuda.current_stream().  `metas`, `pages`, `refs`
        and `n_pages` are as AsyncPagesDecompressor takes them; `bounds` is an int64 CUDA tensor of at least max_segments + 1 elements
        (non-decreasing row indices into the pages' concatenation), `n_segments` a 1-element int64 CUDA tensor, `interval` a 2-element
        int64 CUDA tensor (pack_interval's bit patterns of lo and hi), `aggs` an int64 CUDA tensor of shape (max_segments, 6) whose row g
        receives segment g's PcoB200Aggregate, and `total` a 6-element int64 CUDA tensor that receives the total.  Returns nothing and
        does not wait; result() reports the outcome."""
        import torch

        p = self._plan
        self._check_tensors(metas=metas, pages=pages, refs=refs, n_pages=n_pages, bounds=bounds, n_segments=n_segments, interval=interval,
                            aggs=aggs, total=total)
        if metas.numel() * metas.element_size() < p.metas_cap or pages.numel() * pages.element_size() < p.pages_cap:
            raise ValueError(f"metas holds fewer than metas_cap = {p.metas_cap} bytes, or pages fewer than pages_cap = {p.pages_cap}")
        if refs.dtype != torch.int64 or refs.dim() != 2 or refs.shape[1] != 5 or refs.shape[0] < p.max_pages:
            raise ValueError(f"refs must be an int64 tensor of shape ({p.max_pages}, 5)")
        if n_pages.dtype != torch.int64 or n_pages.numel() != 1:
            raise ValueError("n_pages must be a 1-element int64 tensor")
        _check_segment_tensors(bounds, n_segments, interval, aggs, total, p.max_segments)
        rc = _lib_async_segment_aggregate().pco_b200_segment_aggregate_pages_async(
            C.byref(p), C.c_void_p(metas.data_ptr()), C.c_void_p(pages.data_ptr()), C.c_void_p(refs.data_ptr()), C.c_void_p(n_pages.data_ptr()),
            C.c_void_p(bounds.data_ptr()), C.c_void_p(n_segments.data_ptr()), C.c_void_p(interval.data_ptr()), C.c_void_p(aggs.data_ptr()),
            C.c_void_p(total.data_ptr()), C.c_void_p(self.workspace.data_ptr()), C.c_void_p(self.status.data_ptr()), self._stream())
        _lib.check(rc)

    def result(self):
        """Copies the status of the last call back (waiting for it on the current stream) and returns the total match count, or raises
        PcoError with the kind decompress_pages gives ("page 17: ...") or, for the bounds, InvalidArgument ("segment 17: ...")."""
        s = self.status_record()
        nm = C.c_size_t()
        _lib.check(_lib_async_segment_aggregate().pco_b200_segment_aggregate_pages_async_result(C.byref(s), C.byref(nm)))
        return int(nm.value)


class AsyncPagesFilter(_lib._AsyncCall):
    """Decodes a batch of wrapped-format pages on the current CUDA stream and writes only the numbers inside a closed interval, in row order,
    with their positions in the pages' concatenation (pco_b200_filter_pages_async): the predicate runs inside the decoder, so the decoded
    pages never reach HBM whole.  Refs, their count and the interval are read from device tensors, so one captured call serves new pages
    and new bounds on each replay.

    The capacities are AsyncPagesDecompressor's, with rows_cap (the most numbers of a call's pages) in place of dst_cap, and out_cap the
    most matches a call writes; frame_cap defaults to metas_cap + pages_cap + 20 * max_pages as there.  The filter owns a device workspace
    (about rows_cap * (itemsize + 1) bytes beyond the decompressor's) and a status; it serves one call in flight."""

    _Plan, _Status = _CAsyncFilterPlan, _CAsyncFilterStatus

    def __init__(self, dtype, metas_cap, pages_cap, max_pages, rows_cap, out_cap, frame_cap=None, device=None):
        self.dtype = np.dtype(dtype)
        if frame_cap is None:
            frame_cap = metas_cap + pages_cap + 20 * max_pages
        self._make_plan(device, lambda plan: _lib_async_filter().pco_b200_filter_pages_async_plan(
            C.c_ubyte(_lib.dtype_byte(self.dtype)), C.c_size_t(metas_cap), C.c_size_t(pages_cap), C.c_size_t(max_pages), C.c_size_t(rows_cap),
            C.c_size_t(frame_cap), C.c_size_t(out_cap), plan))
        self._alloc()

    def __call__(self, metas, pages, refs, n_pages, interval, values, positions, n_matches):
        """Enqueues the filter of the pages refs[: n_pages[0]] names on torch.cuda.current_stream().  `metas`, `pages`, `refs` and `n_pages`
        are as AsyncPagesDecompressor takes them; `interval` is a 2-element int64 CUDA tensor (pack_interval's bit patterns of lo and hi),
        `values` a CUDA tensor of the plan's dtype and `positions` an int64 CUDA tensor, each of at least out_cap elements, and `n_matches` a
        1-element int64 CUDA tensor that receives the count.  Returns nothing and does not wait; result() reports the outcome."""
        import torch

        p = self._plan
        self._check_tensors(metas=metas, pages=pages, refs=refs, n_pages=n_pages, interval=interval, values=values, positions=positions,
                            n_matches=n_matches)
        if metas.numel() * metas.element_size() < p.metas_cap or pages.numel() * pages.element_size() < p.pages_cap:
            raise ValueError(f"metas holds fewer than metas_cap = {p.metas_cap} bytes, or pages fewer than pages_cap = {p.pages_cap}")
        if refs.dtype != torch.int64 or refs.dim() != 2 or refs.shape[1] != 5 or refs.shape[0] < p.max_pages:
            raise ValueError(f"refs must be an int64 tensor of shape ({p.max_pages}, 5)")
        for name, t in (("n_pages", n_pages), ("n_matches", n_matches)):
            if t.dtype != torch.int64 or t.numel() != 1:
                raise ValueError(f"{name} must be a 1-element int64 tensor")
        if interval.dtype != torch.int64 or interval.numel() != 2:
            raise ValueError("interval must be a 2-element int64 tensor")
        if values.dtype != _torch_dtypes()[self.dtype] or values.numel() < p.out_cap:
            raise ValueError(f"values must hold at least out_cap = {p.out_cap} numbers of {self.dtype}")
        if positions.dtype != torch.int64 or positions.numel() < p.out_cap:
            raise ValueError(f"positions must be an int64 tensor of at least out_cap = {p.out_cap} elements")
        rc = _lib_async_filter().pco_b200_filter_pages_async(
            C.byref(p), C.c_void_p(metas.data_ptr()), C.c_void_p(pages.data_ptr()), C.c_void_p(refs.data_ptr()), C.c_void_p(n_pages.data_ptr()),
            C.c_void_p(interval.data_ptr()), C.c_void_p(values.data_ptr()), C.c_void_p(positions.data_ptr()), C.c_void_p(n_matches.data_ptr()),
            C.c_void_p(self.workspace.data_ptr()), C.c_void_p(self.status.data_ptr()), self._stream())
        _lib.check(rc)

    def result(self):
        """Copies the status of the last call back (waiting for it on the current stream) and returns the number of matches, or raises
        PcoError with the kind decompress_pages gives ("page 17: ..."), or Io when the matches outnumber out_cap."""
        s = self.status_record()
        nm = C.c_size_t()
        _lib.check(_lib_async_filter().pco_b200_filter_pages_async_result(C.byref(s), C.byref(nm)))
        return int(nm.value)


class _CAsyncPagesToFilePlan(C.Structure):  # PcoB200AsyncPagesToFilePlan (include/pco_b200.h)
    _fields_ = [("dtype", C.c_uint32), ("uniform_type", C.c_uint32), ("metas_cap", C.c_uint64), ("pages_cap", C.c_uint64), ("max_pages", C.c_uint64),
                ("frame_cap", C.c_uint64), ("dst_cap", C.c_uint64), ("index_cap", C.c_uint64), ("workspace_bytes", C.c_uint64)]


class _CAsyncPagesToFileStatus(C.Structure):  # PcoB200AsyncPagesToFileStatus (include/pco_b200.h)
    _fields_ = [("kind", C.c_uint32), ("device_status", C.c_uint32), ("page", C.c_uint64), ("n_pages", C.c_uint64), ("n_total", C.c_uint64),
                ("file_len", C.c_uint64), ("index_len", C.c_uint64), ("frames_needed", C.c_uint64), ("file_needed", C.c_uint64),
                ("index_needed", C.c_uint64)]


def _lib_async_pages_to_file():
    return _lib.bind("_async_pages_to_file_ready",
                     pco_b200_pages_to_file_async_plan=[C.c_ubyte, C.c_int, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t,
                                                        C.c_void_p],
                     pco_b200_pages_to_file_async=[C.c_void_p] * 11,
                     pco_b200_pages_to_file_async_result=[C.c_void_p, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)])


class AsyncPagesToFile(_lib._AsyncCall):
    """Writes a batch of wrapped-format pages out as one indexed standalone file on the current CUDA stream, without waiting for the device
    (pco_b200_pages_to_file_async): page i becomes chunk i, its bytes copied and not re-encoded, and the file's side index is written beside
    it.  Every pages call walks each page serially before it decodes; the files calls of `standalone` read the walk's result from the side
    index, so a reader that scans the same pages more than once pays the walk once.  Refs and their count are read from device tensors, so
    one captured call serves different pages on each replay.

    metas_cap, pages_cap, max_pages and frame_cap are AsyncPagesDecompressor's (frame_cap has the same default); dst_cap and index_cap are
    the bytes of the file and of its index (index_cap: at least 64 + 32 max_pages + 12 per 256 numbers and latent var, rounded up to 16
    bytes per page).  uniform_type_header picks the header flavour, as simple_compress_into.  The call owns the output tensors `file`,
    `index` and `file_ref` (an int64 (1, 4) FILE_REF row, zeroed when the call fails), plus a workspace and a status; it serves one call in
    flight.  files_args() gives the first arguments of standalone.AsyncFilesDecompressor, AsyncFilesFilter, AsyncFilesAggregate and
    AsyncFilesTake for the output, so their plans need no readback, and file_ref with n_files (a 1-element int64 tensor holding 1) is
    their `files` and `n_files`."""

    _Plan, _Status = _CAsyncPagesToFilePlan, _CAsyncPagesToFileStatus

    def __init__(self, dtype, metas_cap, pages_cap, max_pages, dst_cap, index_cap, frame_cap=None, uniform_type_header=False, device=None):
        import torch

        self.dtype = np.dtype(dtype)
        if frame_cap is None:
            frame_cap = metas_cap + pages_cap + 20 * max_pages
        self._make_plan(device, lambda plan: _lib_async_pages_to_file().pco_b200_pages_to_file_async_plan(
            C.c_ubyte(_lib.dtype_byte(self.dtype)), C.c_int(1 if uniform_type_header else 0), C.c_size_t(metas_cap), C.c_size_t(pages_cap),
            C.c_size_t(max_pages), C.c_size_t(frame_cap), C.c_size_t(dst_cap), C.c_size_t(index_cap), plan))
        self._alloc()
        p = self._plan
        self.file = torch.empty(max(p.dst_cap, 1), dtype=torch.uint8, device=self.device)
        self.index = torch.empty(max(p.index_cap, 1), dtype=torch.uint8, device=self.device)
        self.file_ref = torch.zeros((1, 4), dtype=torch.int64, device=self.device)
        self.n_files = torch.ones(1, dtype=torch.int64, device=self.device)

    @property
    def head(self):
        """A whole empty standalone file of the output's header flavour (header with a size hint of 0, then the terminator): what the files
        plans read of a header, so it stands for any output of this call."""
        return bytes([112, 99, 111, 33, 3, self._plan.uniform_type, 0, 4, 1, 0])

    def files_args(self):
        """The arguments (head, dtype, src_cap, index_cap, max_files, max_chunks) of a standalone files call's plan for this call's output."""
        p = self._plan
        return dict(head=self.head, dtype=self.dtype, src_cap=int(p.dst_cap), index_cap=int(p.index_cap), max_files=1, max_chunks=int(p.max_pages))

    def __call__(self, metas, pages, refs, n_pages):
        """Enqueues the transcode of the pages refs[: n_pages[0]] names on torch.cuda.current_stream() into `file`, `index` and `file_ref`,
        and returns those three tensors.  `metas`, `pages`, `refs` and `n_pages` are as AsyncPagesDecompressor takes them.  Does not wait;
        result() reports the outcome."""
        import torch

        p = self._plan
        self._check_tensors(metas=metas, pages=pages, refs=refs, n_pages=n_pages)
        if metas.numel() * metas.element_size() < p.metas_cap or pages.numel() * pages.element_size() < p.pages_cap:
            raise ValueError(f"metas holds fewer than metas_cap = {p.metas_cap} bytes, or pages fewer than pages_cap = {p.pages_cap}")
        if refs.dtype != torch.int64 or refs.dim() != 2 or refs.shape[1] != 5 or refs.shape[0] < p.max_pages:
            raise ValueError(f"refs must be an int64 tensor of shape ({p.max_pages}, 5)")
        if n_pages.dtype != torch.int64 or n_pages.numel() != 1:
            raise ValueError("n_pages must be a 1-element int64 tensor")
        rc = _lib_async_pages_to_file().pco_b200_pages_to_file_async(
            C.byref(p), C.c_void_p(metas.data_ptr()), C.c_void_p(pages.data_ptr()), C.c_void_p(refs.data_ptr()), C.c_void_p(n_pages.data_ptr()),
            C.c_void_p(self.file.data_ptr()), C.c_void_p(self.index.data_ptr()), C.c_void_p(self.file_ref.data_ptr()),
            C.c_void_p(self.workspace.data_ptr()), C.c_void_p(self.status.data_ptr()), self._stream())
        _lib.check(rc)
        return self.file, self.index, self.file_ref

    def result(self):
        """Copies the status of the last call back (waiting for it on the current stream) and returns (file_len, index_len), or raises
        PcoError with the kind decompress_pages gives ("page 17: ..."), Unsupported for a page no walker takes, or Io when the file or the
        index does not fit."""
        s = self.status_record()
        fl, il = C.c_size_t(), C.c_size_t()
        _lib.check(_lib_async_pages_to_file().pco_b200_pages_to_file_async_result(C.byref(s), C.byref(fl), C.byref(il)))
        return int(fl.value), int(il.value)
