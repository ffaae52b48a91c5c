"""Host side of the asynchronous page filter (pco_b200_filter_pages_async_plan / _result, wrapped.pack_interval) without a GPU: the plan's
argument checks, its workspace size against the formula include/pco_b200.h documents, how a status written by the device becomes a kind
and a message, the call's host-side argument checks, and the bit patterns the interval packing gives for every number type."""
import ctypes as C
import math

import numpy as np
import pytest

from tests.test_async_pages_host import _expected_workspace as _pages_workspace

U64, U32, F16, U8 = 2, 1, 9, 10
NONE = (1 << 64) - 1
ELEM = {1: 4, 2: 8, 3: 4, 4: 8, 5: 4, 6: 8, 7: 2, 8: 2, 9: 2, 10: 1, 11: 1}
DTYPES = [np.uint8, np.int8, np.uint16, np.int16, np.float16, np.uint32, np.int32, np.float32, np.uint64, np.int64, np.float64]


@pytest.fixture(scope="module")
def L():
    from pcodec_b200 import wrapped

    return wrapped._lib_async_filter()


def _plan(L, dtype=U64, metas_cap=1 << 12, pages_cap=1 << 20, max_pages=64, rows_cap=1 << 18, frame_cap=1 << 21, out_cap=1 << 10, plan=True):
    from pcodec_b200 import wrapped

    p = wrapped._CAsyncFilterPlan()
    rc = L.pco_b200_filter_pages_async_plan(C.c_ubyte(dtype), C.c_size_t(metas_cap), C.c_size_t(pages_cap), C.c_size_t(max_pages),
                                            C.c_size_t(rows_cap), C.c_size_t(frame_cap), C.c_size_t(out_cap), C.byref(p) if plan else None)
    return rc, p, L.pco_b200_last_error_message().decode()


def _expected_workspace(dtype, max_pages, rows_cap, frame_cap):
    """The formula of include/pco_b200.h: the pages plan's with dst_cap = rows_cap, then these regions, each rounded up to 256 bytes."""
    al = lambda x: (x + 255) // 256 * 256  # noqa: E731
    s = rows_cap // 256 + max_pages
    regions = [40, 16, 4 * s, 8 * s, 8 * ((s + 255) // 256), ELEM[dtype] * rows_cap, rows_cap]
    return _pages_workspace(max_pages, rows_cap, frame_cap) + sum(al(r) for r in regions)


def test_argument_checks_come_before_the_device(L):
    rc, _, msg = _plan(L, dtype=99)
    assert rc == 5 and "type" in msg, msg
    rc, _, msg = _plan(L, dtype=0)
    assert rc == 5, msg
    for mp in (0, 1 << 31):
        rc, _, msg = _plan(L, max_pages=mp)
        assert rc == 3 and "max_pages" in msg, msg
    for name in ("rows_cap", "frame_cap", "out_cap"):
        rc, _, msg = _plan(L, **{name: (1 << 56) + 1})
        assert rc == 3 and name in msg, msg
    rc, _, _ = _plan(L, plan=False)
    assert rc == 3


def test_valid_plan_fills_the_plan_or_needs_a_device(L):
    rc, p, msg = _plan(L, dtype=F16, metas_cap=1000, pages_cap=2000, max_pages=5, rows_cap=3000, frame_cap=4000, out_cap=77)
    assert rc == (0 if L.pco_b200_device_available() else 6), msg
    if rc == 6:
        assert "CUDA" in msg or "device" in msg, msg
    assert (p.dtype, p.metas_cap, p.pages_cap, p.max_pages, p.rows_cap, p.frame_cap, p.out_cap) == (F16, 1000, 2000, 5, 3000, 4000, 77)
    assert p.workspace_bytes == _expected_workspace(F16, 5, 3000, 4000)
    _, p, _ = _plan(L, dtype=U8, max_pages=(1 << 31) - 1, rows_cap=1 << 56, frame_cap=1 << 56, out_cap=1 << 56)
    assert p.workspace_bytes == _expected_workspace(U8, (1 << 31) - 1, 1 << 56, 1 << 56)


@pytest.mark.parametrize("dtype", sorted(ELEM))
@pytest.mark.parametrize("mp,rc_,fc", [(1, 0, 0), (3, 255, 17), (255, 256, 4096), (257, 12345, 999), (4096, 1 << 24, 1 << 30)])
def test_workspace_matches_the_formula(L, dtype, mp, rc_, fc):
    _, p, _ = _plan(L, dtype=dtype, max_pages=mp, rows_cap=rc_, frame_cap=fc)
    assert p.workspace_bytes == _expected_workspace(dtype, mp, rc_, fc)


def test_workspace_does_not_depend_on_out_cap_or_the_buffers(L):
    ws = lambda **kw: _plan(L, **kw)[1].workspace_bytes  # noqa: E731
    base = ws()
    assert ws(out_cap=1 << 40) == base
    assert ws(metas_cap=1 << 30, pages_cap=1 << 30) == base
    assert ws(rows_cap=(1 << 18) + 256) - base == _expected_workspace(U64, 64, (1 << 18) + 256, 1 << 21) - _expected_workspace(U64, 64, 1 << 18, 1 << 21) > 0


def _result(L, **fields):
    from pcodec_b200 import wrapped

    s = wrapped._CAsyncFilterStatus(**fields)
    nm = C.c_size_t(12345)
    rc = L.pco_b200_filter_pages_async_result(C.byref(s), C.byref(nm))
    return rc, L.pco_b200_last_error_message().decode(), nm.value


def test_result_maps_statuses_to_kinds_and_messages(L):
    assert _result(L, kind=0, n_matches=1000, matches_needed=1000, page=NONE)[::2] == (0, 1000)
    for kind, st, words in [(1, 1, "corrupt data"), (2, 2, "insufficient data"), (3, 3, "invalid argument"), (7, 7, "valid pco outside")]:
        rc, msg, nm = _result(L, kind=kind, device_status=st, page=17)
        assert rc == kind and msg.startswith("page 17: ") and words in msg, msg
        assert nm == 12345  # left alone on an error
    cases = [(0x11b, 3, "chunk meta lies outside metas"), (0x11c, 3, "page lies outside pages"), (0x11d, 3, "page n must be 1..2^24"),
             (0x11e, 3, "more numbers than rows_cap")]
    for st, kind, words in cases:
        rc, msg, _ = _result(L, kind=kind, device_status=st, page=4, n_pages=9)
        assert rc == kind and msg.startswith("page 4: ") and words in msg, (st, msg)
    rc, msg, _ = _result(L, kind=3, device_status=0x11a, page=NONE, n_pages=99)
    assert rc == 3 and "*n_pages is 99" in msg and "max_pages" in msg, msg
    rc, msg, _ = _result(L, kind=4, device_status=0x11f, page=NONE, frames_needed=123456)
    assert rc == 4 and "123456 bytes" in msg and "frame_cap" in msg, msg
    rc, msg, nm = _result(L, kind=4, device_status=0x201, page=NONE, n_matches=10, matches_needed=987654)
    assert rc == 4 and "987654 matches" in msg and "out_cap" in msg and nm == 12345, msg
    rc, _, _ = _result(L, kind=99, device_status=1, page=0)
    assert rc == 1
    assert L.pco_b200_filter_pages_async_result(None, None) == 3


def test_call_refuses_missing_buffers_without_a_device(L):
    from pcodec_b200 import wrapped

    _, p, _ = _plan(L)
    s = wrapped._CAsyncFilterStatus()
    nz = C.c_void_p(256)

    def call(plan, metas=nz, pages=nz, refs=nz, n=nz, iv=nz, vals=nz, pos=nz, nm=nz, ws=nz, status=C.byref(s)):
        return L.pco_b200_filter_pages_async(plan, metas, pages, refs, n, iv, vals, pos, nm, ws, status, None)

    assert call(None) == 3
    for kw in ("metas", "pages", "refs", "n", "iv", "vals", "pos", "nm", "ws", "status"):
        assert call(C.byref(p), **{kw: None}) == 3, kw
        assert "null buffer" in L.pco_b200_last_error_message().decode()
    bad = wrapped._CAsyncFilterPlan.from_buffer_copy(bytes(p))
    bad.workspace_bytes += 1
    assert call(C.byref(bad)) == 3
    assert "not made by" in L.pco_b200_last_error_message().decode()
    bad = wrapped._CAsyncFilterPlan.from_buffer_copy(bytes(p))
    bad.out_cap = (1 << 56) + 1
    assert call(C.byref(bad)) == 3
    assert call(C.byref(wrapped._CAsyncFilterPlan())) == 3
    assert call(C.byref(p), ws=C.c_void_p(257)) == 3
    assert "256-byte aligned" in L.pco_b200_last_error_message().decode()


def test_plan_needs_a_device(L):
    if L.pco_b200_device_available():
        pytest.skip("a CUDA device is present")
    rc, _, msg = _plan(L)
    assert rc == 6 and "no CPU fallback" in msg, msg


def test_new_symbols_are_exported(L):
    for name in ("pco_b200_filter_pages_async_plan", "pco_b200_filter_pages_async", "pco_b200_filter_pages_async_result"):
        assert hasattr(L, name), name


def _bits(x, dtype):
    dt = np.dtype(dtype)
    return int(np.array([x], dtype=dt).view(f"u{dt.itemsize}")[0])


@pytest.mark.parametrize("dtype", DTYPES)
def test_pack_interval_gives_zero_extended_bit_patterns(dtype):
    from pcodec_b200 import wrapped

    dt = np.dtype(dtype)
    if dt.kind == "f":
        info = np.finfo(dt)
        cases = [(0.0, -0.0), (-0.0, 0.0), (-math.inf, math.inf), (math.nan, 1.0), (float(info.min), float(info.max)), (-1.5, 2.25),
                 (np.array(3.0, dtype=dt)[()], np.float64(-7.0))]
    else:
        info = np.iinfo(dt)
        cases = [(int(info.min), int(info.max)), (0, 0), (info.max, info.min), (np.array(5, dtype=dt)[()], 7)]
        if dt.kind == "i":
            cases.append((-1, -2))
    for lo, hi in cases:
        got = wrapped.pack_interval(lo, hi, dt)
        assert got.dtype == np.int64 and got.shape == (2,)
        want = [_bits(lo, dt), _bits(hi, dt)]
        assert [int(v) for v in got.view(np.uint64)] == want, (lo, hi)
        assert all(w < (1 << (8 * dt.itemsize)) for w in want)  # zero-extended
    if dt.kind == "f":
        nan = wrapped.pack_interval(math.nan, 0.0, dt).view(np.uint64)
        assert np.isnan(np.array([int(nan[0])], dtype=f"u{dt.itemsize}").view(dt)[0])
        assert int(wrapped.pack_interval(-0.0, 0.0, dt).view(np.uint64)[0]) == 1 << (8 * dt.itemsize - 1)
    else:
        with pytest.raises(OverflowError):
            wrapped.pack_interval(int(info.max) + 1, 0, dt)
        with pytest.raises(OverflowError):
            wrapped.pack_interval(int(info.min) - 1, 0, dt)
        with pytest.raises(TypeError):
            wrapped.pack_interval(0.5, 1, dt)


def test_pack_interval_refuses_other_types():
    from pcodec_b200 import wrapped

    with pytest.raises(TypeError):
        wrapped.pack_interval(0, 1, np.complex64)
