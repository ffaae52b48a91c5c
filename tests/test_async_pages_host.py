"""Host side of the asynchronous batch-of-pages call (pco_b200_decompress_pages_async_plan / _result) without a GPU: the plan's argument
checks, its workspace size against the formula include/pco_b200.h documents, how a status written by the device becomes a kind and a
"page <i>: " message, and the call's host-side argument checks."""
import ctypes as C
import os
import re

import pytest

U64, U32, F16 = 2, 1, 9
NONE = (1 << 64) - 1


@pytest.fixture(scope="module")
def L():
    from pcodec_b200 import wrapped

    return wrapped._lib_async_pages()


def _plan(L, dtype=U64, metas_cap=1 << 12, pages_cap=1 << 20, max_pages=64, dst_cap=1 << 18, frame_cap=1 << 21, plan=True):
    from pcodec_b200 import wrapped

    p = wrapped._CAsyncPagesPlan()
    rc = L.pco_b200_decompress_pages_async_plan(C.c_ubyte(dtype), C.c_size_t(metas_cap), C.c_size_t(pages_cap), C.c_size_t(max_pages),
                                                C.c_size_t(dst_cap), C.c_size_t(frame_cap), C.byref(p) if plan else None)
    return rc, p, L.pco_b200_last_error_message().decode()


def _expected_workspace(max_pages, dst_cap, frame_cap):
    """The formula of include/pco_b200.h, each region rounded up to 256 bytes."""
    al = lambda x: (x + 255) // 256 * 256  # noqa: E731
    ctas = lambda n: (n + 255) // 256  # noqa: E731
    per_var = (1 << 14) * 6 + (1 << 15) * 13 + 288 * 8 + 256 * 4 + 64
    cold = 3 * per_var + 2 * (2 * (1 << 16) * 8) + 8192
    rows = 2 * (dst_cap // 256 + max_pages + 1)
    m = max_pages
    regions = [32 + 33 * 7 * 8, 136, 48 * m, 32 * (m + 1) + 24 * (dst_cap // 256) + 32 * m, (frame_cap + 15) // 16 * 16 + 64, 4 * m, 4 * m, 8 * m,
               56 * ctas(m), 32 * m, 4 * m, 4 * m, 4 * m, m, rows * 256, rows * 4, cold]
    return sum(al(r) for r in regions)


def test_argument_checks_come_before_the_device(L):
    rc, _, msg = _plan(L, dtype=99)
    assert rc == 5 and "type" in msg, msg
    for mp in (0, 1 << 31):
        rc, _, msg = _plan(L, max_pages=mp)
        assert rc == 3 and "max_pages" in msg, msg
    rc, _, msg = _plan(L, dst_cap=(1 << 56) + 1)
    assert rc == 3 and "dst_cap" in msg, msg
    rc, _, msg = _plan(L, frame_cap=(1 << 56) + 1)
    assert rc == 3 and "frame_cap" in msg, msg
    rc, _, _ = _plan(L, plan=False)
    assert rc == 3


def test_valid_plan_fills_the_plan_or_needs_a_device(L):
    rc, p, msg = _plan(L, dtype=F16, metas_cap=1000, pages_cap=2000, max_pages=5, dst_cap=3000, frame_cap=4000)
    # without a device the set-up fails with Cuda, after the plan is filled
    assert rc == (0 if L.pco_b200_device_available() else 6), msg
    if rc == 6:
        assert "CUDA" in msg or "device" in msg, msg
    assert (p.dtype, p.metas_cap, p.pages_cap, p.max_pages, p.dst_cap, p.frame_cap) == (F16, 1000, 2000, 5, 3000, 4000)
    assert p.workspace_bytes == _expected_workspace(5, 3000, 4000)
    _, p, _ = _plan(L, max_pages=(1 << 31) - 1, dst_cap=1 << 56, frame_cap=1 << 56)
    assert p.workspace_bytes == _expected_workspace((1 << 31) - 1, 1 << 56, 1 << 56)


@pytest.mark.parametrize("mp,dc,fc", [(1, 0, 0), (3, 255, 17), (255, 256, 4096), (256, 1 << 20, 1 << 20), (257, 12345, 999), (4096, 1 << 24, 1 << 30)])
def test_workspace_matches_the_formula(L, mp, dc, fc):
    _, p, _ = _plan(L, max_pages=mp, dst_cap=dc, frame_cap=fc)
    assert p.workspace_bytes == _expected_workspace(mp, dc, fc)


def test_workspace_grows_with_every_capacity(L):
    ws = lambda **kw: _plan(L, **kw)[1].workspace_bytes  # noqa: E731
    base = ws(max_pages=1000, dst_cap=1 << 20, frame_cap=1 << 20)
    assert ws(max_pages=2000, dst_cap=1 << 20, frame_cap=1 << 20) - base == _expected_workspace(2000, 1 << 20, 1 << 20) - _expected_workspace(1000, 1 << 20, 1 << 20) > 0
    assert ws(max_pages=1000, dst_cap=1 << 21, frame_cap=1 << 20) > base
    assert ws(max_pages=1000, dst_cap=1 << 20, frame_cap=1 << 21) > base
    # metas_cap and pages_cap only bound the refs
    assert ws(max_pages=1000, dst_cap=1 << 20, frame_cap=1 << 20, metas_cap=1 << 30, pages_cap=1 << 30) == base


def _result(L, **fields):
    from pcodec_b200 import wrapped

    s = wrapped._CAsyncPagesStatus(**fields)
    nw = C.c_size_t(12345)
    rc = L.pco_b200_decompress_pages_async_result(C.byref(s), C.byref(nw))
    return rc, L.pco_b200_last_error_message().decode(), nw.value


def test_result_maps_statuses_to_kinds_and_messages(L):
    assert _result(L, kind=0, n_written=1000, page=NONE)[::2] == (0, 1000)
    # page failures on the device: "page P: <kind words> in the page", as pco_b200_decompress_pages words them
    for kind, st, words in [(1, 1, "corrupt data"), (2, 2, "insufficient data"), (3, 3, "invalid argument"), (7, 7, "valid pco outside")]:
        rc, msg, nw = _result(L, kind=kind, device_status=st, page=17)
        assert rc == kind and msg.startswith("page 17: ") and words in msg, msg
        assert nw == 12345  # left alone on an error
    cases = [(0x11b, 3, "chunk meta lies outside metas"), (0x11c, 3, "page lies outside pages"), (0x11d, 3, "page n must be 1..2^24"),
             (0x11e, 3, "dst holds fewer numbers")]
    for st, kind, words in cases:
        rc, msg, _ = _result(L, kind=kind, device_status=st, page=4, n_pages=9)
        assert rc == kind and msg.startswith("page 4: ") and words in msg, (st, msg)
    rc, msg, _ = _result(L, kind=3, device_status=0x11a, page=NONE, n_pages=99)
    assert rc == 3 and "*n_pages is 99" in msg and "max_pages" in msg and not msg.startswith("page"), msg
    rc, msg, _ = _result(L, kind=4, device_status=0x11f, page=NONE, n_pages=3, frames_needed=123456)
    assert rc == 4 and "123456 bytes" in msg and "frame_cap" in msg, msg
    rc, _, _ = _result(L, kind=99, device_status=1, page=0)
    assert rc == 1
    assert L.pco_b200_decompress_pages_async_result(None, None) == 3


def test_status_codes_continue_the_sequence():
    text = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "pco_b200.h")).read()
    codes = {name: int(v, 16) for name, v in re.findall(r"(PCO_B200_ASYNC_[A-Z_]+) = (0x[0-9a-f]+)", text)}
    assert len(set(codes.values())) == len(codes)
    new = ["TOO_MANY_PAGES", "META_OUTSIDE", "PAGE_OUTSIDE", "PAGE_N", "PAGES_DST", "FRAMES"]
    assert [codes["PCO_B200_ASYNC_" + n] for n in new] == list(range(0x11a, 0x120))
    assert max(v for k, v in codes.items() if k[len("PCO_B200_ASYNC_"):] not in new) == 0x119


def test_call_refuses_missing_buffers_without_a_device(L):
    from pcodec_b200 import wrapped

    _, p, _ = _plan(L)
    s = wrapped._CAsyncPagesStatus()
    nz = C.c_void_p(256)

    def call(plan, metas=nz, pages=nz, refs=nz, n=nz, dst=nz, ws=nz, status=C.byref(s)):
        return L.pco_b200_decompress_pages_async(plan, metas, pages, refs, n, dst, ws, status, None)

    assert call(None) == 3
    for kw in ("metas", "pages", "refs", "n", "dst", "ws", "status"):
        assert call(C.byref(p), **{kw: None}) == 3, kw
        assert "null buffer" in L.pco_b200_last_error_message().decode()
    bad = wrapped._CAsyncPagesPlan.from_buffer_copy(bytes(p))
    bad.workspace_bytes += 1
    assert call(C.byref(bad)) == 3
    assert "not made by" in L.pco_b200_last_error_message().decode()
    bad = wrapped._CAsyncPagesPlan.from_buffer_copy(bytes(p))
    bad.max_pages = 0
    assert call(C.byref(bad)) == 3
    assert call(C.byref(wrapped._CAsyncPagesPlan())) == 3  # a plan that was never filled
    assert call(C.byref(p), ws=C.c_void_p(257)) == 3
    assert "256-byte aligned" in L.pco_b200_last_error_message().decode()


def test_plan_needs_a_device(L):
    if L.pco_b200_device_available():
        pytest.skip("a CUDA device is present")
    rc, _, msg = _plan(L)
    assert rc == 6 and "no CPU fallback" in msg, msg


def test_new_symbols_are_exported(L):
    for name in ("pco_b200_decompress_pages_async_plan", "pco_b200_decompress_pages_async", "pco_b200_decompress_pages_async_result"):
        assert hasattr(L, name), name
