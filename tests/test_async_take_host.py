"""Host side of the asynchronous takes (pco_b200_take_pages_async_plan / _files_async_plan / _result, wrapped.AsyncPagesTake,
standalone.AsyncFilesTake) without a GPU: the plans' argument checks, their workspace sizes against the formulas include/pco_b200.h
documents, how a status written by the device becomes a kind and a message, the calls' host-side refusals, and the wrappers' argument
checks."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from tests.test_async_files_host import HEAD
from tests.test_async_files_host import _expected_workspace as _files_workspace
from tests.test_async_pages_host import _expected_workspace as _pages_workspace

U64, U32 = 2, 1
NONE = (1 << 64) - 1
ELEM = {1: 4, 2: 8, 3: 4, 4: 8, 5: 4, 6: 8, 7: 2, 8: 2, 9: 2, 10: 1, 11: 1}
TOO_MANY, ORDER, PAST = 0x301, 0x302, 0x303
al = lambda x: (x + 255) // 256 * 256  # noqa: E731
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def L():
    from pcodec_b200 import wrapped

    return wrapped._lib_async_take()


@pytest.fixture(scope="module")
def LF():
    from pcodec_b200 import standalone

    return standalone._lib_async_take_files()


def _plan(L, dtype=U64, metas_cap=1 << 12, pages_cap=1 << 20, max_pages=64, rows_cap=1 << 18, frame_cap=1 << 21, max_positions=1 << 10,
          plan=True):
    from pcodec_b200 import wrapped

    p = wrapped._CAsyncTakePlan()
    rc = L.pco_b200_take_pages_async_plan(C.c_ubyte(dtype), C.c_size_t(metas_cap), C.c_size_t(pages_cap), C.c_size_t(max_pages),
                                          C.c_size_t(rows_cap), C.c_size_t(frame_cap), C.c_size_t(max_positions), C.byref(p) if plan else None)
    return rc, p, L.pco_b200_last_error_message().decode()


def _files_plan(LF, head, dtype=U32, max_files=8, max_chunks=16, rows_cap=1 << 16, max_positions=1 << 10, plan=True):
    from pcodec_b200 import standalone

    p = standalone._CAsyncFilesTakePlan()
    buf = C.create_string_buffer(head, len(head))
    rc = LF.pco_b200_take_files_async_plan(buf, C.c_size_t(len(head)), C.c_ubyte(dtype), C.c_size_t(1 << 20), C.c_size_t(1 << 16),
                                           C.c_size_t(max_files), C.c_size_t(max_chunks), C.c_size_t(rows_cap), C.c_size_t(max_positions),
                                           C.byref(p) if plan else None)
    return rc, p, LF.pco_b200_last_error_message().decode()


def _header_regions(call):
    """The regions the header's workspace paragraph of `call`'s plan lists, as (coefficient, term, name): a region is written as
    `<coefficient> [<term>] (<name>)`."""
    text = open(os.path.join(ROOT, "include", "pco_b200.h")).read()
    doc = re.search(r"/\*((?:(?!\*/).)*?)\*/\s*PcoB200Error " + call + r"\(", text, flags=re.S).group(1)
    doc = " ".join(line.strip(" *") for line in doc.splitlines())
    tail = doc.split("E the bytes of a number of dtype:")[1]
    return re.findall(r"(\d+|E)(?: (S|max_pages|max_chunks|rows_cap|\(max_chunks \+ 1\)))? \(([^)]*)\)", tail)


def _formula(call, s, elem, rows_cap, m):
    """The take's regions of `call`'s plan as the header states them, for S = s, E = elem and max_pages / max_chunks = m."""
    terms = {"": 1, "S": s, "rows_cap": rows_cap, "max_pages": m, "max_chunks": m, "(max_chunks + 1)": m + 1}
    return sum(al((elem if coef == "E" else int(coef)) * terms[term]) for coef, term, _ in _header_regions(call))


def test_header_lists_the_regions():
    assert [r[2] for r in _header_regions("pco_b200_take_pages_async_plan")] == [
        "the pages status", "the take's state", "each slot's run of positions", "touched flags", "the cold pages' values"]
    assert [r[2] for r in _header_regions("pco_b200_take_files_async_plan")] == [
        "the files status", "the take's state", "each slot's run of positions", "touched flags", "the cold chunks' values", "slot map",
        "cold list"]


def _expected_pages(dtype, max_pages, rows_cap, frame_cap):
    """The pages call's formula with dst_cap = rows_cap, then the take's regions: the pages status, the take's state, the slot runs, the
    touched flags and the value staging; the header's text states the same."""
    s = rows_cap // 256 + max_pages
    own = sum(al(r) for r in [40, 56, 16 * s, 4 * max_pages, ELEM[dtype] * rows_cap])
    assert own == _formula("pco_b200_take_pages_async_plan", s, ELEM[dtype], rows_cap, max_pages)
    return _pages_workspace(max_pages, rows_cap, frame_cap) + own


def _expected_files(dtype, max_files, max_chunks, rows_cap):
    s = rows_cap // 256 + max_chunks
    own = sum(al(r) for r in [40, 56, 16 * s, 4 * max_chunks, ELEM[dtype] * rows_cap, 4 * max_chunks, 4 * (max_chunks + 1)])
    assert own == _formula("pco_b200_take_files_async_plan", s, ELEM[dtype], rows_cap, max_chunks)
    return _files_workspace(max_files, max_chunks, rows_cap) + own


def test_argument_checks_come_before_the_device(L):
    rc, _, msg = _plan(L, dtype=99)
    assert rc == 5 and "type" in msg, msg
    for mp in (0, 1 << 31):
        rc, _, msg = _plan(L, max_pages=mp)
        assert rc == 3 and "max_pages" in msg, msg
    for name in ("rows_cap", "frame_cap"):
        rc, _, msg = _plan(L, **{name: (1 << 56) + 1})
        assert rc == 3 and name in msg, msg
    for mpos in (0, (1 << 56) + 1, 1 << 63):
        rc, _, msg = _plan(L, max_positions=mpos)
        assert rc == 3 and "max_positions" in msg, msg
    rc, _, _ = _plan(L, plan=False)
    assert rc == 3


def test_max_positions_range_is_accepted_up_to_the_device(L, LF):
    """1 and 2^56 pass the checks: without a device the plan then stops at the device (PCO_B200_CUDA), not at the argument."""
    import torch

    for mpos in (1, 2, 1 << 20, 1 << 56):
        rc, p, msg = _plan(L, max_positions=mpos)
        assert rc in (0, 6) and "max_positions" not in msg, msg
        if not torch.cuda.is_available():
            assert rc == 6, msg
        assert p.max_positions == mpos
        rc, p, msg = _files_plan(LF, HEAD, max_positions=mpos)
        assert rc in (0, 6) and "max_positions" not in msg, msg
        assert p.max_positions == mpos


@pytest.mark.parametrize("dtype", sorted(ELEM))
@pytest.mark.parametrize("mp,rc_,fc", [(1, 0, 0), (3, 255, 17), (257, 12345, 999), (4096, 1 << 24, 1 << 30)])
def test_pages_workspace_matches_the_formula(L, dtype, mp, rc_, fc):
    _, p, _ = _plan(L, dtype=dtype, max_pages=mp, rows_cap=rc_, frame_cap=fc)
    assert (p.dtype, p.max_pages, p.rows_cap, p.frame_cap) == (dtype, mp, rc_, fc)
    assert p.workspace_bytes == _expected_pages(dtype, mp, rc_, fc)


def test_workspace_does_not_depend_on_the_buffers_or_positions(L):
    ws = lambda **kw: _plan(L, **kw)[1].workspace_bytes  # noqa: E731
    assert ws(metas_cap=1 << 30, pages_cap=1 << 30) == ws()
    assert ws(max_positions=1) == ws(max_positions=1 << 56)


def test_files_plan_checks(LF):
    for kw, words in [({"max_files": 0}, "max_files"), ({"max_chunks": 0}, "max_chunks"), ({"rows_cap": (1 << 56) + 1}, "rows_cap"),
                      ({"max_positions": 0}, "max_positions"), ({"max_positions": (1 << 56) + 1}, "max_positions")]:
        rc, _, msg = _files_plan(LF, HEAD, **kw)
        assert rc == 3 and words in msg, msg
    rc, _, msg = _files_plan(LF, HEAD, dtype=99)
    assert rc == 5


@pytest.mark.parametrize("dtype", sorted(ELEM))
@pytest.mark.parametrize("mf,mc,rows", [(1, 1, 0), (8, 16, 1 << 16), (4096, 5000, 12345), (3, 1 << 20, 1 << 28)])
def test_files_workspace_matches_the_formula(LF, dtype, mf, mc, rows):
    _, p, _ = _files_plan(LF, HEAD, dtype=dtype, max_files=mf, max_chunks=mc, rows_cap=rows)
    assert (p.dtype, p.max_files, p.max_chunks, p.rows_cap) == (dtype, mf, mc, rows)
    assert p.workspace_bytes == _expected_files(dtype, mf, mc, rows)


def _result(L, **fields):
    from pcodec_b200 import wrapped

    s = wrapped._CAsyncTakeStatus(**fields)
    nw = C.c_size_t(12345)
    rc = L.pco_b200_take_pages_async_result(C.byref(s), C.byref(nw))
    return rc, L.pco_b200_last_error_message().decode(), nw.value


def _files_result(LF, **fields):
    from pcodec_b200 import standalone

    s = standalone._CAsyncFilesTakeStatus(**fields)
    nw = C.c_size_t(12345)
    rc = LF.pco_b200_take_files_async_result(C.byref(s), C.byref(nw))
    return rc, LF.pco_b200_last_error_message().decode(), nw.value


def test_result_of_success_is_the_count(L, LF):
    assert _result(L, kind=0, n_positions=1000, page=NONE, position=NONE)[::2] == (0, 1000)
    assert _files_result(LF, kind=0, n_positions=77, file=NONE, chunk=NONE, position=NONE)[::2] == (0, 77)
    assert L.pco_b200_take_pages_async_result(None, None) == 3
    assert LF.pco_b200_take_files_async_result(None, None) == 3


@pytest.mark.parametrize("res", ["_result", "_files_result"])
def test_result_names_the_position(L, LF, res):
    f = (lambda **kw: _result(L, **kw)) if res == "_result" else (lambda **kw: _files_result(LF, **kw))
    rc, msg, nw = f(kind=3, device_status=TOO_MANY, n_positions=99, position=NONE)
    assert rc == 3 and msg == "*n_positions is 99, above the plan's max_positions" and nw == 12345, msg
    rc, msg, _ = f(kind=3, device_status=ORDER, n_positions=99, position=17)
    assert rc == 3 and msg.startswith("position 17: ") and "ascending" in msg, msg
    rc, msg, _ = f(kind=3, device_status=PAST, n_positions=99, position=5, n_written=1000)
    assert rc == 3 and msg.startswith("position 5: ") and "1000 rows" in msg, msg


def test_result_of_upstream_statuses_is_the_decompress_calls(L, LF):
    rc, msg, _ = _result(L, kind=2, device_status=2, page=17)
    assert rc == 2 and msg.startswith("page 17: ") and "insufficient data" in msg, msg
    rc, msg, _ = _result(L, kind=3, device_status=0x11e, page=4)
    assert rc == 3 and msg.startswith("page 4: ") and "rows_cap" in msg, msg
    rc, msg, _ = _result(L, kind=3, device_status=0x11a, page=NONE, n_pages=99)
    assert rc == 3 and "*n_pages is 99" in msg, msg
    rc, msg, _ = _result(L, kind=4, device_status=0x11f, page=NONE, frames_needed=5000)
    assert rc == 4 and "5000 bytes" in msg, msg
    rc, msg, _ = _files_result(LF, kind=1, device_status=1, file=3, chunk=2)
    assert rc == 1 and msg == "file 3: corrupt data in chunk 2", msg
    rc, msg, _ = _files_result(LF, kind=7, device_status=7, file=0, chunk=5)
    assert rc == 7 and msg.startswith("file 0: "), msg


def test_every_take_code_is_documented_with_its_kind():
    text = open(os.path.join(ROOT, "include", "pco_b200.h")).read()
    codes = dict((name, int(v, 16)) for name, v in re.findall(r"(PCO_B200_TAKE_\w+)\s*=\s*(0x[0-9a-f]+)", text))
    assert codes == {"PCO_B200_TAKE_TOO_MANY": TOO_MANY, "PCO_B200_TAKE_ORDER": ORDER, "PCO_B200_TAKE_PAST": PAST}
    for name in codes:
        assert re.search(name + r"\s*=\s*0x[0-9a-f]+,?\s*/\*(?:(?!\*/).)*\(PCO_B200_INVALID_ARGUMENT\) \*/", text), name


def test_calls_refuse_missing_buffers_without_a_device(L, LF):
    from pcodec_b200 import standalone, wrapped

    _, p, _ = _plan(L)
    nz = C.c_void_p(256)
    s = wrapped._CAsyncTakeStatus()
    args = [nz] * 8  # metas, pages, refs, n_pages, positions, n_positions, out_values, workspace
    for i in range(8):
        a = list(args)
        a[i] = None
        assert L.pco_b200_take_pages_async(C.byref(p), *a, C.byref(s), None) == 3
        assert "null buffer" in L.pco_b200_last_error_message().decode()
    assert L.pco_b200_take_pages_async(C.byref(p), *args[:7], nz, None, None) == 3  # null status
    assert L.pco_b200_take_pages_async(C.byref(p), *args[:7], C.c_void_p(257), C.byref(s), None) == 3
    assert "aligned" in L.pco_b200_last_error_message().decode()
    bad = wrapped._CAsyncTakePlan.from_buffer_copy(bytes(p))
    bad.workspace_bytes += 1
    assert L.pco_b200_take_pages_async(C.byref(bad), *args, C.byref(s), None) == 3
    assert "not made by" in L.pco_b200_last_error_message().decode()
    assert L.pco_b200_take_pages_async(C.byref(wrapped._CAsyncTakePlan()), *args, C.byref(s), None) == 3
    assert "not made by" in L.pco_b200_last_error_message().decode()

    _, fp, _ = _files_plan(LF, HEAD)
    fs = standalone._CAsyncFilesTakeStatus()
    fargs = [nz] * 7  # src, index, files, n_files, positions, n_positions, out_values
    for i in range(7):
        a = list(fargs)
        a[i] = None
        assert LF.pco_b200_take_files_async(C.byref(fp), *a, None, nz, C.byref(fs), None) == 3
        assert "null buffer" in LF.pco_b200_last_error_message().decode()
    assert LF.pco_b200_take_files_async(C.byref(fp), *fargs, None, C.c_void_p(257), C.byref(fs), None) == 3
    assert "aligned" in LF.pco_b200_last_error_message().decode()
    assert LF.pco_b200_take_files_async(C.byref(standalone._CAsyncFilesTakePlan()), *fargs, None, nz, C.byref(fs), None) == 3
    assert "not made by" in LF.pco_b200_last_error_message().decode()


def test_new_symbols_are_exported(L, LF):
    for name in ("pco_b200_take_pages_async_plan", "pco_b200_take_pages_async", "pco_b200_take_pages_async_result"):
        assert hasattr(L, name), name
    for name in ("pco_b200_take_files_async_plan", "pco_b200_take_files_async", "pco_b200_take_files_async_result"):
        assert hasattr(LF, name), name


def test_status_structs_match_the_header():
    from pcodec_b200 import standalone, wrapped

    assert C.sizeof(wrapped._CAsyncTakeStatus) == 64 and C.sizeof(standalone._CAsyncFilesTakeStatus) == 64
    assert C.sizeof(wrapped._CAsyncTakePlan) == 64 and C.sizeof(standalone._CAsyncFilesTakePlan) == 72


class _FakeTensor:
    """Enough of a CUDA tensor for the wrappers' argument checks, which run before any device call."""

    def __init__(self, dtype, shape, device):
        self.dtype, self.shape, self.device, self.is_cuda = dtype, tuple(shape), device, True

    def numel(self):
        return int(np.prod(self.shape))

    def dim(self):
        return len(self.shape)

    def element_size(self):
        import torch

        return torch.empty((), dtype=self.dtype).element_size()

    def is_contiguous(self):
        return True


def _bare(cls, plan, dtype):
    import torch

    obj = cls.__new__(cls)
    obj.dtype = np.dtype(dtype)
    obj.device = torch.device("cuda", 0)
    obj._plan = plan
    return obj


def test_pages_wrapper_checks_its_arguments():
    import torch

    from pcodec_b200 import wrapped

    p = wrapped._CAsyncTakePlan(dtype=U64, metas_cap=64, pages_cap=64, max_pages=4, rows_cap=1024, frame_cap=256, max_positions=10)
    t = _bare(wrapped.AsyncPagesTake, p, np.uint64)
    dev = t.device
    T = lambda dt, *shape: _FakeTensor(dt, shape, dev)  # noqa: E731
    good = dict(metas=T(torch.uint8, 64), pages=T(torch.uint8, 64), refs=T(torch.int64, 4, 5), n_pages=T(torch.int64, 1),
                positions=T(torch.int64, 10), n_positions=T(torch.int64, 1), values=T(torch.uint64, 10))
    for name, bad, words in [("positions", T(torch.int64, 9), "positions"), ("positions", T(torch.int32, 10), "positions"),
                             ("n_positions", T(torch.int64, 2), "n_positions"), ("values", T(torch.int64, 10), "values"),
                             ("values", T(torch.uint64, 9), "values"), ("refs", T(torch.int64, 3, 5), "refs"),
                             ("metas", T(torch.uint8, 63), "metas_cap")]:
        kw = dict(good, **{name: bad})
        with pytest.raises(ValueError, match=words):
            t(**kw)
    kw = dict(good, values=object())
    with pytest.raises(ValueError, match="values must be a contiguous CUDA tensor"):
        t(**kw)


def test_files_wrapper_checks_its_arguments():
    import torch

    from pcodec_b200 import standalone

    p = standalone._CAsyncFilesTakePlan(dtype=U32, src_cap=64, index_cap=64, max_files=2, max_chunks=4, rows_cap=1024, max_positions=10)
    t = _bare(standalone.AsyncFilesTake, p, np.uint32)
    dev = t.device
    T = lambda dt, *shape: _FakeTensor(dt, shape, dev)  # noqa: E731
    good = dict(src=T(torch.uint8, 64), index=T(torch.uint8, 64), files=T(torch.int64, 2, 4), n_files=T(torch.int64, 1),
                positions=T(torch.int64, 10), n_positions=T(torch.int64, 1), values=T(torch.uint32, 10))
    for name, bad, words in [("positions", T(torch.int64, 9), "positions"), ("n_positions", T(torch.int32, 1), "n_positions"),
                             ("values", T(torch.int32, 10), "values"), ("files", T(torch.int64, 2, 5), "files"),
                             ("file_ns", T(torch.int64, 1), "file_ns"), ("n_files", T(torch.int64, 2), "n_files")]:
        kw = dict(good, **{name: bad})
        with pytest.raises(ValueError, match=words):
            t(**kw)
