"""ctypes binding of libcpcodec.so (include/cpcodec.h + include/pco_b200.h)."""
import ctypes as C
import os

import numpy as np

from . import _build

# dtype bytes: pco_c/include/cpcodec.h:10-20
NP_TO_BYTE = {
    np.dtype(np.uint32): 1, np.dtype(np.uint64): 2, np.dtype(np.int32): 3, np.dtype(np.int64): 4,
    np.dtype(np.float32): 5, np.dtype(np.float64): 6, np.dtype(np.uint16): 7, np.dtype(np.int16): 8,
    np.dtype(np.float16): 9, np.dtype(np.uint8): 10, np.dtype(np.int8): 11,
}
BYTE_TO_NP = {v: k for k, v in NP_TO_BYTE.items()}

ERROR_KINDS = {1: "Corruption", 2: "InsufficientData", 3: "InvalidArgument", 4: "Io", 5: "InvalidType", 6: "Cuda", 7: "Unsupported"}
SRC_ON_DEVICE, DST_ON_DEVICE = 1, 2


class PcoError(RuntimeError):
    """pco::errors::PcoError (pco/src/errors.rs:26-31): kind + message."""

    def __init__(self, kind, message):
        super().__init__(f"pco {kind} error: {message}")
        self.kind = kind
        self.message = message


class ModeSpec:
    """pco::ModeSpec (pco/src/chunk_config.rs:15-51; pco_python/src/config.rs:20-60)."""

    def __init__(self, kind, base=0.0, k=0, int_base=0):
        self.kind, self.base, self.k, self.int_base = kind, base, k, int_base

    @staticmethod
    def auto():
        return ModeSpec(0)

    @staticmethod
    def classic():
        return ModeSpec(1)

    @staticmethod
    def try_float_mult(base):
        return ModeSpec(2, base=float(base))

    @staticmethod
    def try_float_quant(k):
        return ModeSpec(3, k=int(k))

    @staticmethod
    def try_int_mult(base):
        return ModeSpec(4, int_base=int(base))

    @staticmethod
    def try_dict():
        return ModeSpec(5)


class DeltaSpec:
    """pco::DeltaSpec (pco/src/chunk_config.rs:63-109; pco_python/src/config.rs:62-100)."""

    def __init__(self, kind, order=0):
        self.kind, self.order = kind, order

    @staticmethod
    def auto():
        return DeltaSpec(0)

    @staticmethod
    def no_op():
        return DeltaSpec(1)

    @staticmethod
    def try_consecutive(order):
        return DeltaSpec(2, int(order))

    @staticmethod
    def try_lookback():
        return DeltaSpec(3)

    @staticmethod
    def try_conv1(order):
        return DeltaSpec(4, int(order))


class PagingSpec:
    """pco::PagingSpec (pco/src/chunk_config.rs:114-125)."""

    def __init__(self, kind, n=0, sizes=None):
        self.kind, self.n, self.sizes = kind, n, sizes

    @staticmethod
    def equal_pages_up_to(n):
        return PagingSpec(0, n=int(n))

    @staticmethod
    def exact_page_sizes(sizes):
        return PagingSpec(1, sizes=[int(s) for s in sizes])


class _CConfig(C.Structure):
    _fields_ = [
        ("compression_level", C.c_uint32), ("mode_spec", C.c_uint32), ("float_mult_base", C.c_double),
        ("int_mult_base", C.c_uint64), ("float_quant_k", C.c_uint32), ("delta_spec", C.c_uint32),
        ("delta_order", C.c_uint32), ("paging_spec", C.c_uint32), ("max_page_n", C.c_uint64),
        ("exact_page_ns", C.POINTER(C.c_uint64)), ("n_exact_pages", C.c_uint64), ("enable_8_bit", C.c_uint32),
        ("reserved", C.c_uint32),
    ]


class ChunkConfig:
    """pco::ChunkConfig (pco/src/chunk_config.rs:193-236; pco_python/src/config.rs:108-169)."""

    def __init__(self, compression_level=8, mode_spec=None, delta_spec=None, paging_spec=None, enable_8_bit=False):
        self.compression_level = compression_level
        self.mode_spec = mode_spec or ModeSpec.auto()
        self.delta_spec = delta_spec or DeltaSpec.auto()
        self.paging_spec = paging_spec or PagingSpec.equal_pages_up_to(1 << 18)
        self.enable_8_bit = enable_8_bit

    def _to_c(self):
        c = _CConfig()
        c.compression_level = self.compression_level
        c.mode_spec = self.mode_spec.kind
        c.float_mult_base = self.mode_spec.base
        c.int_mult_base = self.mode_spec.int_base
        c.float_quant_k = self.mode_spec.k
        c.delta_spec = self.delta_spec.kind
        c.delta_order = self.delta_spec.order
        c.paging_spec = self.paging_spec.kind
        c.max_page_n = self.paging_spec.n
        if self.paging_spec.sizes is not None:
            arr = (C.c_uint64 * len(self.paging_spec.sizes))(*self.paging_spec.sizes)
            c._keep = arr
            c.exact_page_ns = C.cast(arr, C.POINTER(C.c_uint64))
            c.n_exact_pages = len(self.paging_spec.sizes)
        c.enable_8_bit = 1 if self.enable_8_bit else 0
        return c


class _CProgress(C.Structure):
    _fields_ = [("n_processed", C.c_size_t), ("finished", C.c_int)]


class Progress:
    """pco::Progress (pco/src/progress.rs:3-11)."""

    def __init__(self, n_processed, finished):
        self.n_processed, self.finished = n_processed, finished

    def __repr__(self):
        return f"Progress(n_processed={self.n_processed}, finished={self.finished})"


_lib = None


def lib():
    """Loads libcpcodec.so, building it in-tree if needed.  Never falls back to anything else."""
    global _lib
    if _lib is None:
        path = os.environ.get("PCOB200_LIB") or _build.LIB  # PCOB200_LIB: experiment builds of the same library
        if not os.path.exists(path):
            path = _build.build()
        L = C.CDLL(path)
        L.pco_b200_last_error_message.restype = C.c_char_p
        L.pco_standalone_guarantee_file_size.restype = C.c_size_t
        L.pco_standalone_guarantee_file_size.argtypes = [C.c_size_t, C.c_ubyte]
        L.pco_b200_index_size_bound.restype = C.c_size_t
        L.pco_b200_index_size_bound.argtypes = [C.c_size_t, C.c_size_t]
        L.pco_b200_decompress_ranges.argtypes = [C.c_void_p, C.c_size_t, C.c_ubyte, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                                 C.c_size_t, C.POINTER(C.c_size_t), C.c_uint32, C.c_void_p]
        L.pco_b200_debug_plan_ranges.argtypes = [C.c_void_p, C.c_size_t, C.c_uint64, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                                 C.POINTER(C.c_size_t), C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        _lib = L
    return _lib


def check(rc):
    if rc != 0:
        raise PcoError(ERROR_KINDS.get(rc, f"code {rc}"), lib().pco_b200_last_error_message().decode())


def dtype_byte(dtype):
    dt = np.dtype(dtype)
    if dt not in NP_TO_BYTE:
        raise TypeError(f"unsupported dtype {dt}")
    return NP_TO_BYTE[dt]


def bind(flag, **argtypes):
    """The library, with the argtypes of the named functions set the first time a binder asks (the library attribute `flag` marks it)."""
    L = lib()
    if not getattr(L, flag, False):
        for name, types in argtypes.items():
            getattr(L, name).argtypes = types
        setattr(L, flag, True)
    return L


class _AsyncCall:
    """What the wrappers of the asynchronous calls share: the device, the plan (a ctypes struct of class _Plan, made under that device),
    the device workspace and the status (of class _Status) a call writes, the checks of the tensors a call takes and the stream it runs
    on.  One call in flight at a time; calls on one stream queue up."""

    _Plan = _Status = None

    def _make_plan(self, device, plan_fn):
        """Resolves the device and fills the plan with plan_fn(pointer to the plan), which returns the library's error code."""
        import torch

        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self._plan = self._Plan()
        self._replan(plan_fn)

    def _replan(self, plan_fn):
        import torch

        with torch.cuda.device(self.device):
            rc = plan_fn(C.byref(self._plan))
        check(rc)

    def _alloc(self):
        import torch

        self.workspace = torch.empty(max(self._plan.workspace_bytes, 1), dtype=torch.uint8, device=self.device)
        self.status = torch.zeros(C.sizeof(self._Status), dtype=torch.uint8, device=self.device)

    @staticmethod
    def _head(head):
        """The first 32 bytes of a file (bytes, numpy or a tensor) as host memory."""
        from .wrapped import _host_u8

        if getattr(head, "is_cuda", False):
            head = head.reshape(-1)[:32].cpu().numpy()
        return _host_u8(head)[:32].copy()

    def _check_tensors(self, **tensors):
        for name, t in tensors.items():
            if not getattr(t, "is_cuda", False) or t.device != self.device or not t.is_contiguous():
                raise ValueError(f"{name} must be a contiguous CUDA tensor on {self.device}")

    def _stream(self):
        import torch

        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    @property
    def workspace_bytes(self):
        return int(self._plan.workspace_bytes)

    def status_record(self):
        """The last call's status struct, copied back (waiting for it on the current stream)."""
        return self._Status.from_buffer_copy(self.status.cpu().numpy().tobytes())
