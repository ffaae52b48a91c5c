"""Host side of the asynchronous transcode of wrapped pages into an indexed standalone file (pco_b200_pages_to_file_async_plan / _async /
_result, wrapped.AsyncPagesToFile) without a GPU: the plan's argument checks, its workspace size against the formula include/pco_b200.h
documents, how a status written by the device becomes a kind and a message, the call's host-side refusals, the wrapper's argument checks,
and the standalone header the device writes against the oracle's."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from tests.test_async_files_host import HEAD, HEAD_U64
from tests.test_async_take_host import _bare, _FakeTensor

U64, U32 = 2, 1
NONE = (1 << 64) - 1
DTYPES = list(range(1, 12))
FILES_DST_FULL, FILES_INDEX_FULL = 0x118, 0x119
al = lambda x: (x + 255) // 256 * 256  # noqa: E731
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def L():
    from pcodec_b200 import wrapped

    return wrapped._lib_async_pages_to_file()


def _plan(L, dtype=U64, uniform=0, metas_cap=1 << 12, pages_cap=1 << 20, max_pages=64, frame_cap=1 << 21, dst_cap=1 << 21, index_cap=1 << 16,
          plan=True):
    from pcodec_b200 import wrapped

    p = wrapped._CAsyncPagesToFilePlan()
    rc = L.pco_b200_pages_to_file_async_plan(C.c_ubyte(dtype), C.c_int(uniform), C.c_size_t(metas_cap), C.c_size_t(pages_cap), C.c_size_t(max_pages),
                                             C.c_size_t(frame_cap), C.c_size_t(dst_cap), C.c_size_t(index_cap), C.byref(p) if plan else None)
    return rc, p, L.pco_b200_last_error_message().decode()


def _header_doc():
    text = open(os.path.join(ROOT, "include", "pco_b200.h")).read()
    doc = re.search(r"/\*((?:(?!\*/).)*?)\*/\s*PcoB200Error pco_b200_pages_to_file_async_plan\(", text, flags=re.S).group(1)
    return " ".join(line.strip(" *") for line in doc.splitlines())


def _expected_workspace(max_pages, frame_cap, index_cap):
    """The regions the header lists, each rounded up to 256 bytes, with m = max_pages and E = 24 floor(index_cap / 12)."""
    m, e = max_pages, 24 * (index_cap // 12)
    regions = [1880, 136, 48 * m, 32 * (m + 1) + e + 32 * m, (frame_cap + 15) // 16 * 16 + 64, 4 * m, 4 * m, 8 * m, 56 * ((m + 255) // 256),
               32 * m, 4 * m, 4 * m, 32, 4 * m, 8 * m, 8 * m, 8 * m]
    return sum(al(r) for r in regions)


def test_header_lists_the_regions():
    doc = _header_doc()
    tail = doc.split("workspace_bytes is the sum of these regions")[1]
    names = [x for x in re.findall(r"\(([A-Za-z][^()]*?)\)", tail.split("E is room")[0]) if not re.search(r"[/+]", x)]
    assert names == ["the binomial table", "state", "page table", "walked records and batch entries", "frames and a pad frame",
                     "meta statuses, walk statuses, walk ends", "CTA sums", "decode table", "its pages", "cold list", "transcode state",
                     "wide walk statuses and ends", "chunk and entries offsets"], names
    assert "E = 24 floor(index_cap / 12)" in tail and "32 (m + 1) + E + 32 m" in tail and "ceil(frame_cap / 16) * 16 + 64" in tail


def test_argument_checks_come_before_the_device(L):
    rc, _, msg = _plan(L, dtype=99)
    assert rc == 5 and "type" in msg, msg
    rc, _, msg = _plan(L, dtype=0)
    assert rc == 5, msg
    for mp in (0, 1 << 31):
        rc, _, msg = _plan(L, max_pages=mp)
        assert rc == 3 and "max_pages" in msg, msg
    for name in ("frame_cap", "dst_cap", "index_cap"):
        rc, _, msg = _plan(L, **{name: (1 << 56) + 1})
        assert rc == 3 and name in msg, msg
    rc, _, _ = _plan(L, plan=False)
    assert rc == 3


def test_limits_are_accepted_up_to_the_device(L):
    """The largest capacities pass the checks: without a device the plan then stops at the device (PCO_B200_CUDA), not at an argument."""
    import torch

    rc, p, msg = _plan(L, max_pages=(1 << 31) - 1, frame_cap=1 << 56, dst_cap=1 << 56, index_cap=1 << 56)
    assert rc in (0, 6), msg
    if not torch.cuda.is_available():
        assert rc == 6, msg
    assert p.workspace_bytes == _expected_workspace((1 << 31) - 1, 1 << 56, 1 << 56)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mp,fc,ic", [(1, 0, 0), (3, 17, 11), (255, 4096, 12), (256, 1 << 20, 1 << 20), (257, 999, 12345), (4096, 1 << 30, 1 << 24)])
def test_workspace_matches_the_formula(L, dtype, mp, fc, ic):
    for uniform in (0, 1):
        _, p, _ = _plan(L, dtype=dtype, uniform=uniform, max_pages=mp, frame_cap=fc, index_cap=ic)
        assert (p.dtype, p.uniform_type, p.max_pages, p.frame_cap, p.index_cap) == (dtype, dtype if uniform else 0, mp, fc, ic)
        assert p.workspace_bytes == _expected_workspace(mp, fc, ic)


def test_workspace_does_not_depend_on_the_buffers_or_the_file(L):
    ws = lambda **kw: _plan(L, **kw)[1].workspace_bytes  # noqa: E731
    assert ws(metas_cap=1 << 30, pages_cap=1 << 30) == ws() == ws(dst_cap=1 << 40) == ws(dst_cap=0) == ws(uniform=1)
    assert ws(index_cap=1 << 20) > ws()


def _result(L, **fields):
    from pcodec_b200 import wrapped

    s = wrapped._CAsyncPagesToFileStatus(**fields)
    fl, il = C.c_size_t(12345), C.c_size_t(678)
    rc = L.pco_b200_pages_to_file_async_result(C.byref(s), C.byref(fl), C.byref(il))
    return rc, L.pco_b200_last_error_message().decode(), fl.value, il.value


def test_result_of_success_is_the_lengths(L):
    assert _result(L, kind=0, page=NONE, file_len=1000, index_len=96)[::2] == (0, 1000)
    assert _result(L, kind=0, page=NONE, file_len=1000, index_len=96)[3] == 96
    from pcodec_b200 import wrapped

    s = wrapped._CAsyncPagesToFileStatus(kind=0, page=NONE, file_len=10, index_len=64)
    assert L.pco_b200_pages_to_file_async_result(C.byref(s), None, None) == 0
    assert L.pco_b200_pages_to_file_async_result(None, None, None) == 3


def test_result_names_the_page(L):
    rc, msg, fl, il = _result(L, kind=7, device_status=7, page=17)
    assert rc == 7 and msg.startswith("page 17: ") and "walker" in msg and (fl, il) == (12345, 678), msg
    rc, msg, _, _ = _result(L, kind=2, device_status=2, page=4)
    assert rc == 2 and msg.startswith("page 4: ") and "insufficient data" in msg, msg
    rc, msg, _, _ = _result(L, kind=1, device_status=1, page=0)
    assert rc == 1 and msg.startswith("page 0: "), msg
    rc, msg, _, _ = _result(L, kind=3, device_status=3, page=9)
    assert rc == 3 and msg.startswith("page 9: "), msg


def test_result_of_front_end_refusals_is_the_pages_calls(L):
    rc, msg, _, _ = _result(L, kind=3, device_status=0x11a, page=NONE, n_pages=99)
    assert rc == 3 and msg == "*n_pages is 99, above the plan's max_pages", msg
    for code, words in [(0x11b, "outside metas"), (0x11c, "outside pages"), (0x11d, "page n")]:
        rc, msg, _, _ = _result(L, kind=3, device_status=code, page=5)
        assert rc == 3 and msg.startswith("page 5: ") and words in msg, msg
    rc, msg, _, _ = _result(L, kind=4, device_status=0x11f, page=NONE, frames_needed=4096)
    assert rc == 4 and "4096" in msg and "frame_cap" in msg, msg


def test_result_of_capacities_reports_the_bytes_needed(L):
    rc, msg, _, _ = _result(L, kind=4, device_status=FILES_DST_FULL, page=NONE, file_needed=123456, index_needed=999)
    assert rc == 4 and "123456" in msg and "dst_cap" in msg, msg
    rc, msg, _, _ = _result(L, kind=4, device_status=FILES_INDEX_FULL, page=NONE, file_needed=10, index_needed=4160)
    assert rc == 4 and "4160" in msg and "index_cap" in msg, msg
    rc, msg, _, _ = _result(L, kind=4, device_status=FILES_INDEX_FULL, page=NONE)
    assert rc == 4 and "twice" in msg and "index_cap" in msg, msg


def test_status_kinds_come_from_the_shared_table():
    from pcodec_b200 import _lib

    k = _lib.lib().pco_b200_debug_async_kind
    assert k(FILES_DST_FULL) == 4 and k(FILES_INDEX_FULL) == 4 and k(7) == 7 and k(0x11a) == 3 and k(0x11f) == 4


def test_call_refuses_missing_buffers_without_a_device(L):
    from pcodec_b200 import wrapped

    _, p, _ = _plan(L)
    nz = C.c_void_p(256)
    s = wrapped._CAsyncPagesToFileStatus()
    args = [nz] * 9  # metas, pages, refs, n_pages, dst, index, file_ref, workspace
    for i in range(8):
        a = list(args[:8])
        a[i] = None
        assert L.pco_b200_pages_to_file_async(C.byref(p), *a, C.byref(s), None) == 3
        assert "null buffer" in L.pco_b200_last_error_message().decode()
    assert L.pco_b200_pages_to_file_async(C.byref(p), *args[:8], None, None) == 3  # null status
    assert L.pco_b200_pages_to_file_async(None, *args[:8], C.byref(s), None) == 3
    a = list(args[:8])
    a[7] = C.c_void_p(257)
    assert L.pco_b200_pages_to_file_async(C.byref(p), *a, C.byref(s), None) == 3
    assert "workspace is not 256-byte aligned" in L.pco_b200_last_error_message().decode()
    a = list(args[:8])
    a[5] = C.c_void_p(264)
    assert L.pco_b200_pages_to_file_async(C.byref(p), *a, C.byref(s), None) == 3
    assert "index is not 16-byte aligned" in L.pco_b200_last_error_message().decode()
    for field, delta in (("workspace_bytes", 1), ("uniform_type", 1), ("index_cap", 1 << 20)):
        bad = wrapped._CAsyncPagesToFilePlan.from_buffer_copy(bytes(p))
        setattr(bad, field, getattr(bad, field) + delta)
        assert L.pco_b200_pages_to_file_async(C.byref(bad), *args[:8], C.byref(s), None) == 3
        assert "not made by" in L.pco_b200_last_error_message().decode()
    assert L.pco_b200_pages_to_file_async(C.byref(wrapped._CAsyncPagesToFilePlan()), *args[:8], C.byref(s), None) == 3
    assert "not made by" in L.pco_b200_last_error_message().decode()


def test_structs_match_the_header():
    from pcodec_b200 import wrapped

    assert C.sizeof(wrapped._CAsyncPagesToFilePlan) == 64 and C.sizeof(wrapped._CAsyncPagesToFileStatus) == 72
    text = open(os.path.join(ROOT, "include", "pco_b200.h")).read()
    body = re.search(r"typedef struct PcoB200AsyncPagesToFileStatus \{(.*?)\}", text, flags=re.S).group(1)
    names = re.findall(r"\b(\w+);", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert names == [f[0] for f in wrapped._CAsyncPagesToFileStatus._fields_]


def _header_bytes(n, uniform_type):
    from pcodec_b200 import _lib

    L = _lib.lib()
    L.pco_b200_debug_standalone_header.restype = C.c_size_t
    L.pco_b200_debug_standalone_header.argtypes = [C.c_uint64, C.c_ubyte, C.c_void_p]
    buf = (C.c_ubyte * 32)()
    k = L.pco_b200_debug_standalone_header(C.c_uint64(n), C.c_ubyte(uniform_type), buf)
    return bytes(buf[:k])


def _size_hints():
    out = {0, 1}
    for k in range(1, 57):
        out |= {(1 << k) - 1, 1 << k}
    return sorted(out)


@pytest.mark.parametrize("uniform", [False, True])
def test_header_bytes_match_the_format_and_the_oracle(oracle, uniform):
    """The header the file writer builds (standalone_header_into, which pco_b200_debug_standalone_header calls) for size hints at every
    power boundary up to 2^56, against the format's varint; and, for the counts the oracle can write, its own header."""
    for n in _size_hints():
        p = max(1, n.bit_length())
        nbytes = (6 + p + 7) // 8
        val = (p - 1) | (n << 6)
        want = bytes([112, 99, 111, 33, 3, 2 if uniform else 0]) + val.to_bytes(nbytes + 1, "little")[:nbytes] + bytes([4, 1])
        assert _header_bytes(n, 2 if uniform else 0) == want, n
    for n in [0, 1, 2, 3, 4, 7, 8, 255, 256, 1023, 1024, (1 << 16) - 1, 1 << 16]:
        data = oracle.simple_compress(np.zeros(n, dtype=np.uint64), uniform_type=uniform)
        want = _header_bytes(n, 2 if uniform else 0)
        assert data[: len(want)] == want, n


def test_wrapper_head_is_an_empty_file_of_the_flavour():
    from pcodec_b200 import wrapped

    for dtype, uniform, head in ((np.uint32, False, HEAD), (np.uint64, True, HEAD_U64)):
        p = wrapped._CAsyncPagesToFilePlan(dtype=2 if dtype == np.uint64 else 1, uniform_type=2 if uniform else 0, max_pages=7, dst_cap=100,
                                           index_cap=300)
        t = _bare(wrapped.AsyncPagesToFile, p, dtype)
        assert t.head == head == _header_bytes(0, p.uniform_type) + b"\0"
        args = t.files_args()
        assert args == dict(head=head, dtype=np.dtype(dtype), src_cap=100, index_cap=300, max_files=1, max_chunks=7)


def test_wrapper_checks_its_arguments():
    import torch

    from pcodec_b200 import wrapped

    p = wrapped._CAsyncPagesToFilePlan(dtype=U64, metas_cap=64, pages_cap=64, max_pages=4, frame_cap=256, dst_cap=1000, index_cap=1000)
    t = _bare(wrapped.AsyncPagesToFile, p, np.uint64)
    dev = t.device
    T = lambda dt, *shape: _FakeTensor(dt, shape, dev)  # noqa: E731
    good = dict(metas=T(torch.uint8, 64), pages=T(torch.uint8, 64), refs=T(torch.int64, 4, 5), n_pages=T(torch.int64, 1))
    for name, bad, words in [("refs", T(torch.int64, 3, 5), "refs"), ("refs", T(torch.int32, 4, 5), "refs"), ("refs", T(torch.int64, 4, 4), "refs"),
                             ("n_pages", T(torch.int64, 2), "n_pages"), ("n_pages", T(torch.int32, 1), "n_pages"),
                             ("metas", T(torch.uint8, 63), "metas_cap"), ("pages", T(torch.uint8, 63), "pages_cap")]:
        kw = dict(good, **{name: bad})
        with pytest.raises(ValueError, match=words):
            t(**kw)
    with pytest.raises(ValueError, match="refs must be a contiguous CUDA tensor"):
        t(**dict(good, refs=object()))


def test_new_symbols_are_exported(L):
    for name in ("pco_b200_pages_to_file_async_plan", "pco_b200_pages_to_file_async", "pco_b200_pages_to_file_async_result"):
        assert hasattr(L, name), name
