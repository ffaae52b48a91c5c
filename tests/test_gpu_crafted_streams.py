"""GPU decode of valid streams the encoder never writes (tests/crafted_streams.py): bins out of order, duplicated and overlapping,
lowers whose `lower + offset` wraps past the top of the type, full-width offsets in many-bin tables, all-weight-1 tables up to 2^14
states, moments at the wrap, IntMult adjustments at or above the base, FloatMult adjustments that land on NaN payloads and infinities,
FloatQuant at k = 1 and k = precision, and chunks of 1 to 2^18 numbers - through every decode entry point.

Every decode must equal the numpy restatement of the decode and the oracle's decode bit for bit, and every family asserts the decoder
that served it: the chunk classes of pco_b200_profile_chunk_classes for fused_narrow_kernel (classes 3, 4, 5) and the general pair
(1, 2), the profiler's cold_decode_kernel span for the catch-all decoder.  Files with a chunk
that the side index paths (build_index, decompress_ranges, decompress_chunks) cannot walk are refused by them as Unsupported, as
documented; every other call must decode them."""
import ctypes as C

import numpy as np
import pytest

from tests import crafted_streams as cs

pytestmark = pytest.mark.gpu

FAMILIES = cs.all_families()
FAST = [f for f in FAMILIES if not cs.is_cold(f)]
COLD = [f for f in FAMILIES if cs.is_cold(f)]
BY_DTYPE = sorted({f["dtype"].name for f in FAMILIES})
GUARD = 1024


def _ids(fams):
    return [f["name"] for f in fams]


def _bits(x, dtype):
    return np.asarray(x).view(cs._u(dtype))


def _same(got, want, dtype, what):
    g, w = _bits(got, dtype), _bits(want, dtype)
    if g.shape != w.shape or not np.array_equal(g, w):
        bad = np.flatnonzero(g != w) if g.shape == w.shape else []
        i = int(bad[0]) if len(bad) else -1
        raise AssertionError(f"{what}: {len(bad)} of {w.size} numbers differ; first at {i}: got {g[i] if i >= 0 else g.shape}, want {w[i] if i >= 0 else w.shape}")


@pytest.fixture(scope="module")
def crafted(oracle):
    """name -> (file, [(meta, page) per chunk], expected numbers), checked against the oracle's decode once."""
    out = {}
    for f in FAMILIES:
        data, parts = cs.write(oracle, f)
        want = cs.expected(f)
        _same(oracle.simple_decompress(data, f["dtype"]), want, f["dtype"], f"{f['name']}: oracle")
        out[f["name"]] = (data, parts, want)
    return out


def _profiled(fn):
    """fn()'s result, the kernel names of the call's profiler spans and the chunk classes of its last decode launch."""
    from pcodec_b200 import _lib

    L = _lib.lib()
    L.pco_b200_profile_enable(1)
    try:
        out = fn()
        buf = C.create_string_buffer(1 << 16)
        L.pco_b200_profile_last(buf, C.c_size_t(len(buf)))
        counts = (C.c_uint * 8)()
        L.pco_b200_profile_chunk_classes(counts)
    finally:
        L.pco_b200_profile_enable(0)
    return out, {kv.split("=")[0] for kv in buf.value.decode().split(";") if kv}, list(counts)


def _assert_route(f, spans, classes):
    if cs.is_cold(f):
        assert "cold_decode_kernel" in spans, (f["name"], sorted(spans))
    else:
        assert "cold_decode_kernel" not in spans, (f["name"], sorted(spans))
        assert classes == cs.class_counts(f), (f["name"], classes, cs.class_counts(f))


def _index(fam, data):
    """The file's side index from build_index, or None when build_index refuses it - as Unsupported, and only for a file with a chunk
    the catch-all decoder serves (build_index walks tables of up to 2^12 states; Lookback, Dict, Conv1 and larger tables it declines)."""
    from pcodec_b200 import PcoError
    from pcodec_b200 import standalone as sa

    try:
        return sa.build_index(data, fam["dtype"])
    except PcoError as e:
        assert e.kind == "Unsupported" and cs.is_cold(fam), (fam["name"], e)
        return None


def _offsets(oracle, data, dtype):
    info = oracle.inspect(data, dtype)
    return [c["chunk_start"] for c in info["chunks"]], [c["n"] for c in info["chunks"]]


def _tdtype(dtype):
    from pcodec_b200.wrapped import _torch_dtypes

    return _torch_dtypes()[np.dtype(dtype)]


def _dev_bytes(b, cap=None):
    import torch

    t = torch.zeros(max(cap or len(b), 1), dtype=torch.uint8, device="cuda")
    if len(b):
        t[: len(b)] = torch.as_tensor(np.frombuffer(bytes(b), np.uint8).copy())
    return t


def _dev_numbers(n, dtype):
    """A device buffer of n numbers with GUARD sentinel numbers (0xA5 bytes) on both sides: (whole buffer, dst view)."""
    import torch

    item = np.dtype(dtype).itemsize
    buf = torch.full(((2 * GUARD + max(n, 1)) * item,), 0xA5, dtype=torch.uint8, device="cuda")
    return buf, buf[GUARD * item:(GUARD + max(n, 1)) * item].view(_tdtype(dtype))


def _host(buf, dtype, n):
    """(numbers in dst, untouched guards?) of a _dev_numbers buffer."""
    item = np.dtype(dtype).itemsize
    b = buf.cpu().numpy()
    lo, hi = GUARD * item, (GUARD + n) * item
    return b[lo:hi].view(dtype), bool((b[:lo] == 0xA5).all() and (b[(GUARD + max(n, 1)) * item:] == 0xA5).all())


# ---- whole files -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fam", FAMILIES, ids=_ids(FAMILIES))
def test_simple_decompress(crafted, fam):
    """The index-free path: the speculative walk plus walk_kernel builds the index, then the decoder the family was built for."""
    from pcodec_b200 import standalone as sa

    data, _, want = crafted[fam["name"]]
    got, spans, classes = _profiled(lambda: sa.simple_decompress(data, fam["dtype"]))
    _same(got, want, fam["dtype"], "simple_decompress")
    _assert_route(fam, spans, classes)


@pytest.mark.parametrize("fam", FAMILIES, ids=_ids(FAMILIES))
def test_decompress_ex_device_buffers(crafted, fam):
    """pco_b200_decompress_ex with the file and dst in device memory and guard zones around dst, through the side index build_index
    made (without one where build_index declines the file)."""
    import torch

    from pcodec_b200 import _lib

    data, _, want = crafted[fam["name"]]
    dt = fam["dtype"]
    index = _index(fam, data)
    L = _lib.lib()
    src = _dev_bytes(data)
    idx = np.frombuffer(index, np.uint8) if index is not None else None
    buf, dst = _dev_numbers(want.size, dt)
    prog = _lib._CProgress()

    def call():
        rc = L.pco_b200_decompress_ex(C.c_void_p(src.data_ptr()), C.c_size_t(len(data)), C.c_ubyte(_lib.dtype_byte(dt)), C.c_void_p(dst.data_ptr()),
                                      C.c_size_t(want.size), C.byref(prog), idx.ctypes.data_as(C.c_void_p) if idx is not None else None,
                                      C.c_size_t(len(index) if index is not None else 0),
                                      C.c_uint32(_lib.SRC_ON_DEVICE | _lib.DST_ON_DEVICE),
                                      C.c_void_p(torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        return rc

    rc, spans, classes = _profiled(call)
    assert rc == 0, _lib.lib().pco_b200_last_error_message()
    assert (prog.n_processed, bool(prog.finished)) == (want.size, True)
    got, guards = _host(buf, dt, want.size)
    assert guards, "a write outside dst"
    _same(got, want, dt, "decompress_ex")
    _assert_route(fam, spans, classes)


@pytest.mark.parametrize("fam", FAMILIES, ids=_ids(FAMILIES))
def test_decompress_chunks_at_known_offsets(oracle, crafted, fam):
    from pcodec_b200 import PcoError
    from pcodec_b200 import standalone as sa

    data, _, want = crafted[fam["name"]]
    offs, ns = _offsets(oracle, data, fam["dtype"])
    try:
        got, spans, classes = _profiled(lambda: sa.decompress_chunks(data, fam["dtype"], offs, ns))
    except PcoError as e:  # the walk declines chunks of the catch-all decoder: Unsupported, never numbers
        assert e.kind == "Unsupported" and cs.is_cold(fam), (fam["name"], e)
        return
    _same(got, want, fam["dtype"], "decompress_chunks")
    if not cs.is_cold(fam):
        _assert_route(fam, spans, classes)
    last = len(offs) - 1  # the last chunk alone, as bare bytes
    got = sa.decompress_chunks(data[offs[last]:], fam["dtype"], [0], [ns[last]])
    _same(got, want[want.size - ns[last]:], fam["dtype"], "decompress_chunks, last chunk alone")


@pytest.mark.parametrize("fam", FAMILIES, ids=_ids(FAMILIES))
def test_async_decompressor(crafted, fam):
    import torch

    from pcodec_b200 import standalone as sa

    data, _, want = crafted[fam["name"]]
    dt = fam["dtype"]
    index = _index(fam, data)
    if index is None:
        return
    dec = sa.AsyncDecompressor(data[:32], dt, len(data), len(index), want.size, len(fam["chunks"]))
    buf, dst = _dev_numbers(want.size, dt)
    dec(_dev_bytes(data), _dev_bytes(index), dst)
    prog = dec.result()
    torch.cuda.synchronize()
    assert (prog.n_processed, prog.finished) == (want.size, True)
    got, guards = _host(buf, dt, want.size)
    assert guards, "a write outside dst"
    _same(got, want, dt, "AsyncDecompressor")


def _ranges(n):
    r = [(0, n), (n // 2, min(300, n - n // 2)), (n - 1, 1), (n // 3, 1)]
    if n > 600:
        r.append((257, n - 600))
    return r


@pytest.mark.parametrize("fam", FAMILIES, ids=_ids(FAMILIES))
def test_decompress_ranges(crafted, fam):
    """decompress_ranges (index from build_index) and its asynchronous form; files build_index declines are refused as Unsupported."""
    import torch

    from pcodec_b200 import PcoError
    from pcodec_b200 import standalone as sa

    data, _, want = crafted[fam["name"]]
    dt = fam["dtype"]
    ranges = _ranges(want.size)
    index = _index(fam, data)
    if index is None:
        with pytest.raises(PcoError) as e:
            sa.decompress_ranges(data, dt, None, ranges)
        assert e.value.kind == "Unsupported", e.value
        return
    expect = np.concatenate([want[s:s + c] for s, c in ranges])
    _same(sa.decompress_ranges(data, dt, index, ranges), expect, dt, "decompress_ranges")
    total = expect.size
    window_cap = len(ranges) * (want.size + 256 * len(fam["chunks"]))
    dec = sa.AsyncRangeDecompressor(data[:32], dt, len(data), len(index), len(fam["chunks"]), len(ranges), total, window_cap)
    r = torch.as_tensor(np.array(ranges, dtype=np.int64), device="cuda")
    n = torch.tensor([len(ranges)], dtype=torch.int64, device="cuda")
    buf, dst = _dev_numbers(total, dt)
    dec(_dev_bytes(data), _dev_bytes(index), r, n, dst)
    nw = dec.result()
    torch.cuda.synchronize()
    assert nw == total
    got, guards = _host(buf, dt, total)
    assert guards, "a write outside dst"
    _same(got, expect, dt, "AsyncRangeDecompressor")


# ---- batches that mix families ---------------------------------------------------------------------------------------------------
def _batch(crafted, dtype_str):
    fams = [f for f in FAMILIES if f["dtype"].name == dtype_str]
    return np.dtype(dtype_str), fams, [crafted[f["name"]] for f in fams]


@pytest.mark.parametrize("dtype_str", BY_DTYPE)
def test_decompress_files_mixing_families(crafted, dtype_str):
    """One pco_b200_decompress_files call per number type over every family of that type, fast files with their side indexes and
    without, catch-all files without."""
    from pcodec_b200 import standalone as sa

    dt, fams, items = _batch(crafted, dtype_str)
    want = np.concatenate([w for _, _, w in items])
    for with_index in (True, False):
        data, index, refs = bytearray(), bytearray(), []
        for f, (blob, _, _) in zip(fams, items):
            io = il = 0
            ix = _index(f, blob) if with_index else None
            if ix is not None:
                index += b"\0" * (-len(index) % 16)
                io, il = len(index), len(ix)
                index += ix
            refs.append((len(data), len(blob), io, il))
            data += blob + b"\x5a"
        files = np.array(refs, dtype=sa.FILE_REF)
        (vals, ns), spans, _ = _profiled(lambda: sa.decompress_files(bytes(data), files, dt, bytes(index) if with_index else None))
        np.testing.assert_array_equal(ns, [w.size for _, _, w in items])
        _same(vals, want, dt, f"decompress_files (index: {with_index})")
        assert ("cold_decode_kernel" in spans) == any(cs.is_cold(f) for f in fams), sorted(spans)


@pytest.mark.parametrize("dtype_str", BY_DTYPE)
def test_async_files_decompressor_mixing_families(crafted, dtype_str):
    import torch

    from pcodec_b200 import standalone as sa

    dt, fams, items = _batch(crafted, dtype_str)
    indexes = [_index(f, it[0]) for f, it in zip(fams, items)]
    keep = [i for i, ix in enumerate(indexes) if ix is not None]
    data, index, refs = bytearray(), bytearray(), []
    for i in keep:
        blob, ix = items[i][0], indexes[i]
        index += b"\0" * (-len(index) % 16)
        refs.append((len(data), len(blob), len(index), len(ix)))
        index += ix
        data += blob
    want = np.concatenate([items[i][2] for i in keep])
    n_chunks = sum(len(fams[i]["chunks"]) for i in keep)
    dec = sa.AsyncFilesDecompressor(bytes(data[:32]), dt, len(data), len(index), len(refs), n_chunks, want.size)
    files = torch.as_tensor(np.array(refs, dtype=np.int64), device="cuda")
    n = torch.tensor([len(refs)], dtype=torch.int64, device="cuda")
    ns = torch.zeros(len(refs), dtype=torch.int64, device="cuda")
    buf, dst = _dev_numbers(want.size, dt)
    dec(_dev_bytes(data), _dev_bytes(index), files, n, dst, ns)
    nw = dec.result()
    torch.cuda.synchronize()
    assert nw == want.size
    np.testing.assert_array_equal(ns.cpu().numpy(), [items[i][2].size for i in keep])
    got, guards = _host(buf, dt, want.size)
    assert guards, "a write outside dst"
    _same(got, want, dt, "AsyncFilesDecompressor")


@pytest.mark.parametrize("dtype_str", BY_DTYPE)
def test_decompress_pages_mixing_families(oracle, crafted, dtype_str):
    """Every chunk of every family of a type as a wrapped meta and page: decompress_pages (the catch-all pages through
    cold_decode_kernel, one launch per page) and AsyncPagesDecompressor."""
    import torch

    from pcodec_b200 import wrapped

    dt, fams, items = _batch(crafted, dtype_str)
    metas, pages, refs, pieces = bytearray(), bytearray(), [], []
    n_cold = 0
    for f, (_, parts, want) in zip(fams, items):
        at = 0
        for (meta, page), c in zip(parts, f["chunks"]):
            refs.append((len(metas), len(meta), len(pages), len(page), c["n"]))
            metas += meta
            pages += page
            pieces.append(want[at:at + c["n"]])
            at += c["n"]
            n_cold += c["route"] == "cold"
    want = np.concatenate(pieces)
    r = np.array(refs, dtype=wrapped.PAGE_REF)
    got, spans, _ = _profiled(lambda: wrapped.decompress_pages(bytes(metas), bytes(pages), r, dt))
    _same(got, want, dt, "decompress_pages")
    assert ("cold_decode_kernel" in spans) == (n_cold > 0), sorted(spans)
    frame_cap = 2 * (len(metas) + len(pages)) + 64 * len(refs)
    dec = wrapped.AsyncPagesDecompressor(dt, len(metas), len(pages), len(refs), want.size, frame_cap)
    rt = torch.as_tensor(np.array(refs, dtype=np.int64), device="cuda")
    n = torch.tensor([len(refs)], dtype=torch.int64, device="cuda")
    buf, dst = _dev_numbers(want.size, dt)
    dec(_dev_bytes(metas), _dev_bytes(pages), rt, n, dst)
    nw = dec.result()
    torch.cuda.synchronize()
    assert nw == want.size
    got, guards = _host(buf, dt, want.size)
    assert guards, "a write outside dst"
    _same(got, want, dt, "AsyncPagesDecompressor")
