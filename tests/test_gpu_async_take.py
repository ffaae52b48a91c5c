"""The asynchronous take on the GPU (pco_b200_take_pages_async / pco_b200_take_files_async, wrapped.AsyncPagesTake, standalone.AsyncFilesTake):
every output is compared bit for bit with the matching decompress call's output indexed at the positions, with the values buffer filled
with a sentinel first so that a write past *n_positions or on a refusal is caught; records_decoded with the pages or chunks the positions
touch; every refusal with the decompress call's kind and naming, or the take's own code and position."""
import ctypes as C
import math
import struct

import numpy as np
import pytest

from tests.golden_generators import GENERATORS, bits_view, load_assets
from tests.test_gpu_async_files import INDEXED_ASSETS, _batch, _cfg, _expect, _n_chunks, _run as _files_run, _walk
from tests.test_gpu_async_filter_pages import _routes
from tests.test_gpu_async_pages import _dev, _refs_dev, _run as _pages_run
from tests.test_gpu_wrapped_batch import _container, _mixed_chunks, _shuffled, _six_pages

pytestmark = pytest.mark.gpu

DTYPES = [np.uint8, np.int8, np.uint16, np.int16, np.float16, np.uint32, np.int32, np.float32, np.uint64, np.int64, np.float64]
SENTINEL = 0x5A
NONE = (1 << 64) - 1
TOO_MANY, ORDER, PAST = 0x301, 0x302, 0x303


@pytest.fixture(scope="module")
def sa():
    from pcodec_b200 import standalone

    return standalone


def _chunk_sizes(index, ref):
    """The numbers of each chunk of one indexed file, from its side index's chunk records (32 bytes each, n at +8)."""
    base = int(ref[2])
    k, co = _n_chunks(index, ref), struct.unpack_from("<Q", index, base + 32)[0]
    return [struct.unpack_from("<I", index, base + co + 32 * i + 8)[0] for i in range(k)]


def _touched(sizes, pos):
    """How many of the records of these sizes (in row order) hold a position."""
    ends = np.cumsum(np.asarray(sizes, np.int64))
    starts = ends - np.asarray(sizes, np.int64)
    pos = np.asarray(pos, np.int64)
    return int(np.sum(np.searchsorted(pos, starts) < np.searchsorted(pos, ends)))


def _position_sets(n, edges, seed=0):
    """Named strictly ascending position sets over n rows: empty, the first, the last, every row, 255 / 256 / 257 around each batch edge
    and each record edge, uniform at three densities and a contiguous run."""
    rng = np.random.default_rng(seed)
    out = {"empty": np.zeros(0, np.int64)}
    if n == 0:
        return out
    out["first"] = np.array([0])
    out["last"] = np.array([n - 1])
    out["every"] = np.arange(n)
    near = set()
    for e in list(edges) + list(range(0, n, 256)):
        for d in (-257, -256, -255, -1, 0, 1, 255, 256, 257):
            if 0 <= e + d < n:
                near.add(e + d)
    out["edges"] = np.array(sorted(near))
    for name, p in (("sparse", 0.001), ("medium", 0.05), ("dense", 0.7)):
        out[name] = np.nonzero(rng.random(n) < p)[0]
    a = int(rng.integers(0, n))
    out["run"] = np.arange(a, min(n, a + max(1, n // 10)))
    return out


class _Out:
    """values of max_positions + 64 numbers, filled with SENTINEL bytes"""

    def __init__(self, dtype, max_positions):
        import torch

        from pcodec_b200.wrapped import _torch_dtypes

        self.dtype = np.dtype(dtype)
        self.t = torch.full(((max_positions + 64) * self.dtype.itemsize,), SENTINEL, dtype=torch.uint8, device="cuda")
        self.vals = self.t.view(_torch_dtypes()[self.dtype])

    def reset(self):
        self.t.fill_(SENTINEL)

    def read(self, k, limit=None):
        """The first k values; asserts nothing was written behind the first `limit` (default k)."""
        v = self.vals.cpu().numpy()
        limit = k if limit is None else limit
        assert (v.view(np.uint8)[limit * self.dtype.itemsize:] == SENTINEL).all(), "written past the taken numbers"
        return v[:k]


def _read_out(out, k, err, st, n_pos):
    """A refusal with a code of the front end or of the take writes nothing; a chunk status (a decode failure, or a page's walk failure)
    may leave positions of rows the decompress call would write, never past *n_positions; a success writes exactly *n_positions."""
    if err is None:
        return out.read(k)
    return out.read(0, limit=n_pos if st.device_status < 0x100 else 0)


def _pos_dev(pos, max_positions):
    import torch

    t = torch.full((max(max_positions, 1),), -1, dtype=torch.int64)
    t[: len(pos)] = torch.as_tensor(np.asarray(pos, np.uint64).view(np.int64))
    return t.cuda()


def _profiled(fn, profile):
    from pcodec_b200 import _lib

    L = _lib.lib()
    if not profile:
        fn()
        return ""
    L.pco_b200_profile_enable(1)
    try:
        fn()
        buf = C.create_string_buffer(1 << 16)
        L.pco_b200_profile_last(buf, C.c_size_t(len(buf)))
        return buf.value.decode()
    finally:
        L.pco_b200_profile_enable(0)


def _outcome(t):
    from pcodec_b200 import PcoError

    st = t.status_record()
    try:
        k, err = t.result(), None
    except PcoError as e:
        k, err = 0, e
    return k, err, st


def _take_files(sa, data, index, dtype, refs, pos, rows_cap=None, max_positions=None, n=None, max_files=None, max_chunks=None, profile=False):
    """(values, PcoError or None, status, spans, file_ns) of one take over host bytes."""
    import torch

    nc = sum(_n_chunks(index, r) for r in refs)
    if rows_cap is None:
        rows_cap = sum(int(struct.unpack_from("<Q", index, int(r[2]) + 16)[0]) for r in refs)
    mpos = max_positions or max(len(pos), 1)
    mf = max_files or max(len(refs), 1)
    head = data[int(refs[0][0]):int(refs[0][0]) + 32] if len(refs) else data[:32]
    t = sa.AsyncFilesTake(head, dtype, len(data), len(index), mf, max_chunks or max(nc, 1), rows_cap, mpos)
    out = _Out(dtype, mpos)
    files = torch.zeros((mf, 4), dtype=torch.int64)
    if len(refs):
        files[: len(refs)] = torch.as_tensor(np.asarray(refs, np.uint64).view(np.int64))
    nf = torch.tensor([len(refs)], dtype=torch.int64).cuda()
    npos = torch.tensor([len(pos) if n is None else n], dtype=torch.int64).cuda()
    ns = torch.full((mf + 8,), -3, dtype=torch.int64, device="cuda")
    args = (_dev(data), _dev(index), files.cuda(), nf, _pos_dev(pos, mpos), npos, out.vals, ns[:mf])
    spans = _profiled(lambda: t(*args), profile)
    k, err, st = _outcome(t)
    vals = _read_out(out, k, err, st, len(pos) if n is None else min(n, mpos))
    file_ns = ns.cpu().numpy()
    assert (file_ns[mf:] == -3).all()
    if err is not None:
        assert (file_ns == -3).all(), "file_ns written on a failure"
    return vals, err, st, spans, file_ns[: len(refs)]


def _take_pages(metas, pages, refs, dtype, pos, rows_cap=None, max_positions=None, n=None, max_pages=None, profile=False):
    import torch

    from pcodec_b200 import wrapped

    total = int(np.asarray(refs)["page_n"].sum()) if len(refs) else 0
    rows_cap = total if rows_cap is None else rows_cap
    mpos = max_positions or max(len(pos), 1)
    mp = max_pages or max(len(refs), 1)
    t = wrapped.AsyncPagesTake(dtype, len(metas), len(pages), mp, rows_cap, mpos, 2 * (len(metas) + len(pages)) + 32 * mp)
    out = _Out(dtype, mpos)
    npg = torch.tensor([len(refs)], dtype=torch.int64).cuda()
    npos = torch.tensor([len(pos) if n is None else n], dtype=torch.int64).cuda()
    args = (_dev(metas), _dev(pages), _refs_dev(refs, mp), npg, _pos_dev(pos, mpos), npos, out.vals)
    spans = _profiled(lambda: t(*args), profile)
    k, err, st = _outcome(t)
    return _read_out(out, k, err, st, len(pos) if n is None else min(n, mpos)), err, st, spans


def _check_files(sa, data, index, refs, dtype, sets=None, x=None, **kw):
    """Each position set taken equals the files call's output (checked against x when given) at those positions, with the touched
    chunks as records_decoded."""
    dec, err, _ = _files_run(sa, data, index, dtype, refs, dst_cap=kw.get("rows_cap"))
    assert err is None, err
    dec = dec[0]
    if x is not None:
        np.testing.assert_array_equal(bits_view(dec), bits_view(np.asarray(x, dtype=dtype)))
    sizes = [s for r in refs for s in _chunk_sizes(index, r)]
    edges = np.cumsum(sizes)[:-1] if sizes else []
    for name, pos in (sets or _position_sets(len(dec), edges)).items():
        vals, err, st, _, ns = _take_files(sa, data, index, dtype, refs, pos, **kw)
        assert err is None, (name, err)
        np.testing.assert_array_equal(bits_view(vals), bits_view(dec[pos]), err_msg=name)
        assert st.n_positions == len(pos) and st.n_written == len(dec) and st.records_decoded == _touched(sizes, pos), (name, st.records_decoded)
        assert st.position == NONE
    return dec


def _check_pages(metas, pages, refs, dtype, sets=None, x=None, **kw):
    got, nw, err, _ = _pages_run(metas, pages, refs, dtype)
    assert err is None, err
    dec = got[:nw]
    if x is not None:
        np.testing.assert_array_equal(bits_view(dec), bits_view(np.asarray(x, dtype=dtype)))
    sizes = np.asarray(refs)["page_n"].astype(np.int64)
    for name, pos in (sets or _position_sets(nw, np.cumsum(sizes)[:-1])).items():
        vals, err, st, _ = _take_pages(metas, pages, refs, dtype, pos, **kw)
        assert err is None, (name, err)
        np.testing.assert_array_equal(bits_view(vals), bits_view(dec[pos]), err_msg=name)
        assert st.n_positions == len(pos) and st.n_written == nw and st.records_decoded == _touched(sizes, pos), (name, st.records_decoded)
    return dec


@pytest.mark.parametrize("dtype", DTYPES)
def test_every_dtype_on_mixed_batches_of_files(sa, dtype):
    """several chunks per file, a 1-number file, an empty file, files repeated and out of order"""
    xs = [_walk(dtype, m, seed=int(np.dtype(dtype).num) + i) for i, m in enumerate([3 * (1 << 14) + 777, 1, 0, 5000, 1 << 14, 257])]
    data, index, refs = _batch(sa, xs, _cfg(1))
    order = [4, 0, 0, 2, 5, 1, 3, 0]
    _check_files(sa, data, index, refs[order], dtype, x=_expect(xs, order))


@pytest.mark.parametrize("dtype", DTYPES)
def test_every_dtype_on_mixed_batches_of_pages(oracle, dtype):
    metas, pages, refs, pieces = _container(_mixed_chunks(oracle, dtype))
    refs, pieces = _shuffled(refs, pieces, seed=int(np.dtype(dtype).num))
    _check_pages(metas, pages, refs, dtype, x=np.concatenate(pieces))


@pytest.mark.parametrize("dtype", [np.float16, np.float32, np.float64])
def test_floats_keep_nan_payloads_zeros_and_infinities(sa, oracle, dtype):
    dt = np.dtype(dtype)
    ut = np.dtype(f"u{dt.itemsize}")
    rng = np.random.default_rng(7)
    x = (rng.normal(size=20000) * 10).astype(dt)
    special = np.array([math.inf, -math.inf, 0.0, -0.0, math.nan], dtype=dt)
    x[rng.integers(0, x.size, size=800)] = special[rng.integers(0, special.size, size=800)]
    xb = x.view(ut).copy()
    exp = {2: 0x7C00, 4: 0x7F800000, 8: 0x7FF0000000000000}[dt.itemsize]
    nan_ix = rng.integers(0, x.size, size=100)
    xb[nan_ix] = (exp | rng.integers(1, 1 << 9, size=100)).astype(ut) | (rng.integers(0, 2, size=100).astype(ut) << (8 * dt.itemsize - 1))
    x = xb.view(dt)
    special_rows = {"specials": np.nonzero(np.isnan(x) | np.isinf(x) | (x == 0))[0]}
    for order in (0, 1):
        data, index, refs = _batch(sa, [x[:7000], x[7000:]], _cfg(order, page=4096))
        _check_files(sa, data, index, refs, dtype, sets=special_rows, x=x)
    O = oracle
    metas, pages, refs, _ = _container([(x[:9000], O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_NOOP)),
                                        (x[9000:], O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=1))])
    _check_pages(metas, pages, refs, dtype, sets=special_rows, x=x)


FILE_ROUTES = {
    # name: (dtype, arrays, config, the kernel that decodes them)
    "fused_order1": (np.int64, lambda: [_walk(np.int64, m, seed=m) for m in (70000, 300)], lambda: _cfg(1, page=1 << 15), "fused_narrow_kernel"),
    "general_order0": (np.uint64, lambda: [np.random.default_rng(5).integers(0, 1 << 40, size=m).astype(np.uint64) for m in (70000, 999)],
                       lambda: _cfg(0, page=1 << 15), "decode_kernel"),
    "cold_level12": (np.uint64, lambda: [np.random.default_rng(12).lognormal(10, 2, size=m).astype(np.uint64) for m in ((1 << 16) + 1, 1000)],
                     lambda: _cfg(0, page=1 << 16, level=12), "tk_cold_files_kernel"),
}
FILE_ORDER = ["ff_map_kernel", "af_files_kernel", "merge_index_kernel", "tk_front_files_kernel", "tk_check_kernel", "tk_mark_kernel",
              "fused_narrow_kernel", "symwalk_kernel", "decode_kernel", "ff_cold_list_kernel", "cold_chunks_kernel", "af_finish_kernel",
              "tk_cold_files_kernel", "tk_finish_files_kernel"]


@pytest.mark.parametrize("name", sorted(FILE_ROUTES))
def test_every_file_route_with_spans(sa, name):
    dtype, arrays, cfg, _ = FILE_ROUTES[name]
    xs = [np.asarray(a, dtype=dtype) for a in arrays()]
    data, index, refs = _batch(sa, xs, cfg())
    order = [1, 0, 1]
    dec = _check_files(sa, data, index, refs[order], dtype, x=_expect(xs, order))
    pos = np.arange(0, len(dec), 97)
    vals, err, st, spans, _ = _take_files(sa, data, index, dtype, refs[order], pos, profile=True)
    assert err is None and st.records_decoded > 0
    np.testing.assert_array_equal(bits_view(vals), bits_view(dec[pos]))
    at = [spans.find(k) for k in FILE_ORDER]
    assert all(a >= 0 for a in at) and at == sorted(at), spans


def test_cold_chunks_are_decoded_only_when_touched(sa):
    """level-12 chunks go through the catch-all decoder; a position set that touches one of them decodes one chunk"""
    dtype, arrays, cfg, _ = FILE_ROUTES["cold_level12"]
    xs = [np.asarray(a, dtype=dtype) for a in arrays()]
    data, index, refs = _batch(sa, xs, cfg())
    x = _expect(xs, [0, 1])
    for pos in (np.array([5, 100, 7000]), np.array([len(x) - 1]), np.array([(1 << 16) - 1, 1 << 16])):
        vals, err, st, _, _ = _take_files(sa, data, index, dtype, refs, pos)
        assert err is None
        np.testing.assert_array_equal(vals, x[pos])
        sizes = [s for r in refs for s in _chunk_sizes(index, r)]
        assert st.records_decoded == _touched(sizes, pos)


def test_f16_float_mult_chunks_take_the_cold_route(sa, oracle):
    """f16 FloatMult chunks (written by the oracle: the GPU encoder leaves them out) are decoded by the catch-all decoder only when a
    position touches them"""
    O = oracle
    x = (np.round(np.random.default_rng(3).normal(size=9000) * 50) * 0.25).astype(np.float16)
    y = _walk(np.float16, 3000, seed=1)
    d1 = O.simple_compress(x, O.make_config(mode=O.MODE_FLOAT_MULT, float_mult_base=0.25, delta=O.DELTA_CONSECUTIVE, delta_order=1))
    d2 = O.simple_compress(y, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=1))
    i1, i2 = sa.build_index(d1, np.float16), sa.build_index(d2, np.float16)
    pad = (-len(i1)) % 16
    data, index = d1 + d2, i1 + b"\0" * pad + i2
    refs = np.array([[0, len(d1), 0, len(i1)], [len(d1), len(d2), len(i1) + pad, len(i2)]], np.uint64)
    _check_files(sa, data, index, refs, np.float16, x=np.concatenate([x, y]))
    pos = np.array([3, 4000, 8999, 9000])
    vals, err, st, spans, _ = _take_files(sa, data, index, np.float16, refs, pos, profile=True)
    assert err is None and st.records_decoded == 2 and "tk_cold_files_kernel" in spans and "cold_chunks_kernel" in spans
    np.testing.assert_array_equal(bits_view(vals), bits_view(np.concatenate([x, y])[pos]))
    pos = np.array([x.size, x.size + 2999])
    vals, err, st, _, _ = _take_files(sa, data, index, np.float16, refs, pos)
    assert err is None and st.records_decoded == 1
    np.testing.assert_array_equal(bits_view(vals), bits_view(y[pos - x.size]))


def test_every_page_route_with_spans(oracle):
    """fused, the general pair, level 12 and cold Lookback / Dict / Conv1 pages"""
    metas, pages, refs, x = _routes(oracle)
    refs2, _ = _shuffled(refs, [None] * len(refs), seed=3)
    for r in (refs, refs2):
        dec = _check_pages(metas, pages, r, np.int32)
    pos = np.arange(0, len(dec), 31)
    vals, err, st, spans = _take_pages(metas, pages, refs2, np.int32, pos, profile=True)
    assert err is None and st.records_decoded == len(refs2)
    order = ["ap_pages_kernel", "walk_kernel", "ap_rewalk_kernel", "tk_front_pages_kernel", "tk_check_kernel", "tk_mark_kernel",
             "tk_cold_list_kernel", "fused_narrow_kernel", "symwalk_kernel", "decode_kernel", "ap_cold_kernel", "ap_finish_kernel",
             "tk_cold_pages_kernel", "tk_finish_pages_kernel"]
    at = [spans.find(k) for k in order]
    assert all(a >= 0 for a in at) and at == sorted(at), spans


@pytest.mark.parametrize("name", INDEXED_ASSETS)
def test_golden_assets(sa, name):
    x = GENERATORS[name]()
    one = load_assets()[name]
    idx = sa.build_index(one, x.dtype)
    pad = (-len(idx)) % 16
    data, index = one + one, idx + b"\0" * pad + idx
    refs = np.array([[0, len(one), 0, len(idx)], [len(one), len(one), len(idx) + pad, len(idx)]], np.uint64)
    _check_files(sa, data, index, refs[[0, 1, 1]], x.dtype, x=np.concatenate([x, x, x]))


def test_a_2_24_chunk_and_a_2_24_page(sa, oracle):
    x = _walk(np.int64, 1 << 24, seed=24)
    data, index, refs = _batch(sa, [x[:300], x], _cfg(1, page=1 << 24))
    n = 300 + x.size
    rng = np.random.default_rng(3)
    sets = {"sparse": np.sort(rng.choice(n, 5000, replace=False)), "every": np.arange(n), "tail": np.arange(n - 1000, n)}
    _check_files(sa, data, index, refs, np.int64, sets=sets)
    O = oracle
    metas, pages, prefs, _ = _container([(x, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=1, max_page_n=1 << 24))])
    _check_pages(metas, pages, prefs, np.int64, sets={"sparse": sets["sparse"][sets["sparse"] < x.size], "every": np.arange(x.size)}, x=x)


def test_more_than_1000_small_files_and_pages(sa, oracle):
    xs = [_walk(np.uint16, int(m), seed=i) for i, m in enumerate(np.random.default_rng(2).integers(1, 600, 1100))]
    data, index, refs = _batch(sa, xs, _cfg(0, page=256))
    x = _expect(xs, range(len(xs)))
    sizes = [x_.size for x_ in xs]
    one_in_16 = np.concatenate([np.arange(s, s + min(n, 3)) for s, n in zip(np.cumsum([0] + sizes[:-1])[::16], sizes[::16])])
    _check_files(sa, data, index, refs, np.uint16, sets={"one_in_16": one_in_16, "every": np.arange(x.size)}, x=x)
    O = oracle
    metas, pages, prefs, pieces = _container([(x, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_NOOP, max_page_n=256))])
    assert len(prefs) > 1000
    _check_pages(metas, pages, prefs, np.uint16, x=x)


def test_the_position_sets_of_the_edges(sa, oracle):
    """batch, chunk and page edges at 255 / 256 / 257 with pages and chunks of those sizes"""
    sizes = [1, 255, 256, 257, 511, 512, 513, 4096 + 1]
    xs = [_walk(np.int32, m, seed=m) for m in sizes]
    data, index, refs = _batch(sa, xs, _cfg(1, page=256))
    _check_files(sa, data, index, refs, np.int32, x=_expect(xs, range(len(xs))))
    O = oracle
    metas, pages, prefs, pieces = _container([(a, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=1, max_page_n=256))
                                              for a in xs])
    _check_pages(metas, pages, prefs, np.int32, x=np.concatenate(pieces))


def test_records_decoded_counts_the_touched_chunks(sa):
    xs = [_walk(np.uint32, 1 << 16, seed=s) for s in range(4)]
    data, index, refs = _batch(sa, xs, _cfg(1, page=4096))
    sizes = [s for r in refs for s in _chunk_sizes(index, r)]
    assert len(sizes) == 64
    starts = np.cumsum([0] + sizes[:-1])
    for pick in ([0], [5, 6], list(range(0, 64, 16)), list(range(64))):
        pos = np.concatenate([np.arange(starts[c] + 7, starts[c] + 4000, 1000) for c in pick])
        _, err, st, _, _ = _take_files(sa, data, index, np.uint32, refs, pos)
        assert err is None and st.records_decoded == len(pick)
    _, err, st, _, _ = _take_files(sa, data, index, np.uint32, refs, np.zeros(0, np.int64))
    assert err is None and st.records_decoded == 0


def test_bit_flips_in_untouched_chunks_do_not_fail(sa):
    xs = [_walk(np.uint64, 1 << 16, seed=s) for s in range(2)]
    data, index, refs = _batch(sa, xs, _cfg(1, page=4096))
    x = _expect(xs, [0, 1])
    sizes = [s for r in refs for s in _chunk_sizes(index, r)]
    starts = np.cumsum([0] + sizes[:-1])
    base, co = int(refs[1, 2]), struct.unpack_from("<Q", index, int(refs[1, 2]) + 32)[0]
    c_in_file = 3
    chunk_off = struct.unpack_from("<Q", index, base + co + 32 * c_in_file)[0]
    chunk_len = struct.unpack_from("<Q", index, base + co + 32 * (c_in_file + 1))[0] - chunk_off
    c = len(_chunk_sizes(index, refs[0])) + c_in_file  # that chunk in the concatenation
    rng = np.random.default_rng(5)
    for _ in range(40):  # a flip inside the chunk that the files call reports for this chunk
        bad = bytearray(data)
        at = int(refs[1, 0]) + chunk_off + int(rng.integers(0, chunk_len))
        bad[at] ^= 1 << int(rng.integers(0, 8))
        bad = bytes(bad)
        _, werr, wst = _files_run(sa, bad, index, np.uint64, refs, dst_cap=len(x))
        if werr is not None:
            break
    assert werr is not None and wst.file == 1 and wst.chunk == c_in_file
    away = np.array([5, int(starts[c]) - 1, int(starts[c] + sizes[c]), len(x) - 1])
    vals, err, st, _, _ = _take_files(sa, bad, index, np.uint64, refs, away)
    assert err is None and st.records_decoded == 4
    np.testing.assert_array_equal(vals, x[away])
    on = np.array([5, int(starts[c]) + 10])
    vals, err, st, _, _ = _take_files(sa, bad, index, np.uint64, refs, on)
    assert err is not None and err.kind == werr[0] and (st.device_status, st.file, st.chunk) == (wst.device_status, wst.file, wst.chunk)
    assert len(vals) == 0


def test_page_meta_and_walk_failures_are_reported_even_when_untouched(oracle):
    metas, pages, refs, pieces = _six_pages(oracle)
    bad = refs.copy()
    bad[5]["meta_len"] = int(bad[5]["meta_len"]) + 1  # the walk of page 5 fails
    _, _, perr, pst = _pages_run(metas, pages, bad, np.uint64)
    assert perr is not None
    vals, err, st, _ = _take_pages(metas, pages, bad, np.uint64, np.array([0, 1]))
    assert err is not None and (err.kind, st.device_status, st.page) == (perr.kind, pst.device_status, pst.page) and len(vals) == 0
    buf = bytearray(metas)
    buf[int(refs[4]["meta_offset"])] = (buf[int(refs[4]["meta_offset"])] & 0xF0) | 0xE
    _, _, perr, pst = _pages_run(bytes(buf), pages, refs, np.uint64)
    vals, err, st, _ = _take_pages(bytes(buf), pages, refs, np.uint64, np.array([0]))
    assert perr is not None and err is not None and (err.kind, st.device_status, st.page) == (perr.kind, pst.device_status, pst.page)


def test_bit_flips_in_pages_fail_only_when_touched(oracle):
    metas, pages, refs, pieces = _six_pages(oracle)
    x = np.concatenate(pieces)
    ends = np.cumsum(refs["page_n"].astype(np.int64))
    rng = np.random.default_rng(1)
    for trial in range(12):
        k = int(rng.integers(0, len(refs)))
        buf = bytearray(pages)
        buf[int(refs[k]["page_offset"] + rng.integers(0, refs[k]["page_len"]))] ^= 1 << int(rng.integers(0, 8))
        got, nw, perr, pst = _pages_run(metas, bytes(buf), refs, np.uint64)
        other = np.array([0 if k else int(ends[0])])  # a page other than k
        vals, err, st, _ = _take_pages(metas, bytes(buf), refs, np.uint64, np.arange(int(ends[k]) - int(refs[k]["page_n"]), int(ends[k])))
        if perr is None:
            assert err is None, err
            np.testing.assert_array_equal(vals, got[int(ends[k]) - int(refs[k]["page_n"]):int(ends[k])])
        elif pst.page == k:
            assert err is not None and (err.kind, st.page) == (perr.kind, pst.page), (trial, err, perr)
            # a take that does not touch page k: a decode failure of page k is not met, a walk failure is a refusal
            vals, err, st, _ = _take_pages(metas, bytes(buf), refs, np.uint64, other)
            if err is None:
                assert st.records_decoded == 1
                np.testing.assert_array_equal(vals, x[other])
            else:
                assert (err.kind, st.device_status, st.page) == (perr.kind, pst.device_status, pst.page) and len(vals) == 0


def test_take_refusals_name_the_position_and_write_nothing(sa, oracle):
    xs = [_walk(np.int32, m, seed=m) for m in (5000, 3000)]
    data, index, refs = _batch(sa, xs, _cfg(1, page=1024))
    n = 8000
    metas, pages, prefs, _ = _six_pages(oracle)
    pn = int(prefs["page_n"].sum())
    cases = [  # (positions, n_positions override, max_positions, code, position)
        (np.arange(9), 10, 9, TOO_MANY, NONE),
        (np.array([1, 5, 5, 9]), None, None, ORDER, 2),
        (np.array([1, 9, 5, 3]), None, None, ORDER, 2),
        (np.array([0, 1, n]), None, None, PAST, 2),
        (np.array([0, 1, 1 << 63], np.uint64), None, None, PAST, 2),
        (np.array([7, 3, n + 5]), None, None, ORDER, 1),  # the order refusal comes first
    ]
    for pos, nn, mpos, code, at in cases:
        vals, err, st, _, ns = _take_files(sa, data, index, np.int32, refs, pos, max_positions=mpos or len(pos), n=nn)
        assert err is not None and err.kind == "InvalidArgument" and st.device_status == code and st.position == at, (pos, err, st.device_status)
        assert len(vals) == 0 and st.records_decoded == 0 and st.n_positions == (nn or len(pos))
        if code != TOO_MANY:
            assert err.message.startswith(f"position {at}: "), err.message
        ppos = np.where(pos.astype(np.uint64) == n, pn, pos)
        vals, err, st, _ = _take_pages(metas, pages, prefs, np.uint64, ppos, max_positions=mpos or len(pos), n=nn)
        assert err is not None and err.kind == "InvalidArgument" and st.device_status == code and st.position == at, (pos, err)
        assert len(vals) == 0 and st.records_decoded == 0


def test_upstream_refusals_come_first_with_the_decompress_calls_naming(sa, oracle):
    u = np.uint32
    xs = [_walk(u, m, seed=m) for m in (3 * (1 << 14), 5000, 20000, 7)]
    data, index, refs = _batch(sa, xs, _cfg(1))
    total = sum(x.size for x in xs)
    bad_pos = np.array([3, 2])  # refused by the take too, but later
    for r, cap in ((lambda r: (r.__setitem__((1, 2), r[1, 2] + 16), r)[1])(refs.copy()), total), (refs, total - 1):
        _, werr, wst = _files_run(sa, data, index, u, r, dst_cap=cap)
        vals, err, st, _, _ = _take_files(sa, data, index, u, r, bad_pos, rows_cap=cap)
        assert werr is not None and err is not None and err.kind == werr[0], (err, werr)
        assert (st.device_status, st.file, st.chunk) == (wst.device_status, wst.file, wst.chunk) and len(vals) == 0
    metas, pages, prefs, pieces = _six_pages(oracle)
    pn = int(prefs["page_n"].sum())
    for rows_cap in (pn - 1,):
        _, _, perr, pst = _pages_run(metas, pages, prefs, np.uint64, dst_cap=rows_cap)
        vals, err, st, _ = _take_pages(metas, pages, prefs, np.uint64, bad_pos, rows_cap=rows_cap)
        assert perr is not None and err is not None and (err.kind, st.device_status, st.page) == (perr.kind, pst.device_status, pst.page)
        assert "rows_cap" in err.message and len(vals) == 0
    bad = prefs.copy()
    bad[2]["page_n"] = 0
    _, _, perr, pst = _pages_run(metas, pages, bad, np.uint64)
    vals, err, st, _ = _take_pages(metas, pages, bad, np.uint64, bad_pos, rows_cap=pn)
    assert err is not None and (err.kind, st.device_status, st.page) == (perr.kind, pst.device_status, pst.page) and len(vals) == 0


class _FilesGraph:
    """An AsyncFilesTake with device buffers for graph capture."""

    def __init__(self, sa, head, dtype, src_cap, index_cap, max_files, max_chunks, rows_cap, max_positions):
        import torch

        self.t = sa.AsyncFilesTake(head, dtype, src_cap, index_cap, max_files, max_chunks, rows_cap, max_positions)
        self.src = torch.zeros(src_cap, dtype=torch.uint8, device="cuda")
        self.index = torch.zeros(index_cap, dtype=torch.uint8, device="cuda")
        self.files = torch.zeros((max_files, 4), dtype=torch.int64, device="cuda")
        self.nf = torch.zeros(1, dtype=torch.int64, device="cuda")
        self.pos = torch.zeros(max_positions, dtype=torch.int64, device="cuda")
        self.npos = torch.zeros(1, dtype=torch.int64, device="cuda")
        self.out = _Out(dtype, max_positions)
        self.max_files = max_files

    def load(self, data, index, refs, pos):
        import torch

        self.src.zero_()
        self.index.zero_()
        self.src[: len(data)] = torch.as_tensor(np.frombuffer(data, np.uint8).copy())
        self.index[: len(index)] = torch.as_tensor(np.frombuffer(index, np.uint8).copy())
        f = np.zeros((self.max_files, 4), np.uint64)
        f[: len(refs)] = np.asarray(refs, np.uint64).reshape(-1, 4)
        self.files.copy_(torch.as_tensor(f.view(np.int64)))
        self.nf.fill_(len(refs))
        self.pos[: len(pos)] = torch.as_tensor(np.asarray(pos, np.int64))
        self.npos.fill_(len(pos))
        self.out.reset()

    def call(self):
        self.t(self.src, self.index, self.files, self.nf, self.pos, self.npos, self.out.vals)


def _capture(step):
    import torch

    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    return g


def test_graph_replays_new_refs_counts_and_positions(sa):
    import torch

    from pcodec_b200 import _lib

    batches = []
    for s in (1, 2):
        xs = [_walk(np.uint32, 4000 * (i + 1) + s, seed=10 * s + i) for i in range(6)]
        batches.append((xs,) + _batch(sa, xs, _cfg(s - 1, page=4096)))
    src_cap = max(len(b[1]) for b in batches) + 64
    index_cap = max(len(b[2]) for b in batches) + 64
    fg = _FilesGraph(sa, batches[0][1][:32], np.uint32, src_cap, index_cap, 8, 64, 1 << 18, 1 << 17)
    fg.load(*batches[0][1:], [0])
    g = _capture(fg.call)
    rng = np.random.default_rng(0)
    plans = [(0, [0, 1, 2, 3, 4, 5], 0.3), (1, [5, 5, 0], 0.01), (0, [], 0.0), (1, [3], 1.0), (0, [2, 0, 4, 1, 3, 5, 0], 0.001), (1, [1, 2], 0.0)]
    for step, (k, order, dens) in enumerate(plans):
        xs, data, index, refs = batches[k]
        x = _expect(xs, order) if order else np.zeros(0, np.uint32)
        pos = np.nonzero(rng.random(x.size) < dens)[0]
        fg.load(data, index, refs[order] if order else refs[:0], pos)
        if step == 3:
            _lib.lib().pco_b200_thread_release()
        g.replay()
        torch.cuda.synchronize()
        assert fg.t.result() == len(pos)
        np.testing.assert_array_equal(fg.out.read(len(pos)), x[pos])
    # a repeated replay writes identical bytes
    fg.load(batches[1][1], batches[1][2], batches[1][3], np.arange(0, 20000, 3))
    g.replay()
    first = fg.out.t.cpu().numpy().copy()
    fg.out.reset()
    g.replay()
    torch.cuda.synchronize()
    np.testing.assert_array_equal(fg.out.t.cpu().numpy(), first)


def test_graph_of_filter_then_take(sa):
    """AsyncFilesFilter on column A writes the positions AsyncFilesTake reads from column B of the same chunking, in one graph replayed
    with new bounds: B[(A >= lo) & (A <= hi)]."""
    import torch

    from pcodec_b200 import wrapped

    rng = np.random.default_rng(9)
    a_cols = [_walk(np.int64, m, seed=m) for m in (40000, 25000, 3)]
    b_cols = [rng.normal(size=a.size).astype(np.float32) for a in a_cols]
    da, ia, ra = _batch(sa, a_cols, _cfg(1, page=4096))
    db, ib, rb = _batch(sa, b_cols, _cfg(0, page=4096))
    a, b = np.concatenate(a_cols), np.concatenate(b_cols)
    n = a.size
    flt = sa.AsyncFilesFilter(da[:32], np.int64, len(da), len(ia), 3, 64, n, n)
    tk = _FilesGraph(sa, db[:32], np.float32, len(db), len(ib), 3, 64, n, n)
    tk.load(db, ib, rb, [])
    src = torch.as_tensor(np.frombuffer(da, np.uint8).copy()).cuda()
    idx = torch.as_tensor(np.frombuffer(ia, np.uint8).copy()).cuda()
    files = torch.as_tensor(ra.astype(np.int64)).cuda()
    nf = torch.tensor([3], dtype=torch.int64).cuda()
    iv = torch.zeros(2, dtype=torch.int64, device="cuda")
    avals = torch.zeros(n, dtype=torch.int64, device="cuda")
    nm = torch.zeros(1, dtype=torch.int64, device="cuda")

    def step():
        flt(src, idx, files, nf, iv, avals, tk.pos, nm)
        tk.t(tk.src, tk.index, tk.files, tk.nf, tk.pos, nm, tk.out.vals)

    g = _capture(step)
    for qlo, qhi in ((0.1, 0.2), (0.0, 1.0), (0.5, 0.5), (0.9, 0.1), (0.33, 0.9)):
        lo, hi = np.quantile(a, qlo).astype(np.int64), np.quantile(a, qhi).astype(np.int64)
        iv.copy_(torch.from_numpy(wrapped.pack_interval(lo, hi, np.int64)))
        tk.out.reset()
        g.replay()
        torch.cuda.synchronize()
        want = b[(a >= lo) & (a <= hi)]
        assert flt.result() == tk.t.result() == want.size
        np.testing.assert_array_equal(bits_view(tk.out.read(want.size)), bits_view(want))


def test_graph_of_files_compress_then_take(sa):
    import torch

    cfg = _cfg(1, page=4096)
    n_files, max_n = 6, 6000
    comp = sa.AsyncFilesCompressor(np.int32, cfg, n_files, n_files * max_n, max_n, index=True)
    fg = _FilesGraph(sa, sa.simple_compress(np.zeros(10, np.int32), cfg)[:32], np.int32, comp.dst_cap, comp.index_cap, n_files, 64,
                     n_files * max_n, n_files * max_n)
    nums = torch.zeros(n_files * max_n, dtype=torch.int32, device="cuda")
    file_ns = torch.zeros(n_files, dtype=torch.int64, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")

    def step():
        comp(nums, file_ns, cnt, fg.src[: comp.dst_cap], fg.index[: comp.index_cap], fg.files)
        fg.nf.copy_(cnt)
        fg.call()

    g = _capture(step)
    rng = np.random.default_rng(4)
    for m in (6, 2, 1):
        sz = rng.integers(1, max_n + 1, m)
        x = np.concatenate([_walk(np.int32, int(s), seed=int(s)) for s in sz])
        nums[: x.size] = torch.as_tensor(x)
        file_ns[:m] = torch.as_tensor(sz)
        cnt.fill_(m)
        pos = np.nonzero(rng.random(x.size) < 0.02)[0]
        fg.pos[: pos.size] = torch.as_tensor(pos)
        fg.npos.fill_(pos.size)
        fg.out.reset()
        g.replay()
        torch.cuda.synchronize()
        comp.result()
        assert fg.t.result() == pos.size
        np.testing.assert_array_equal(fg.out.read(pos.size), x[pos])


def test_graph_of_chunks_compress_then_pages_take():
    import torch

    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec, wrapped

    cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(1), paging_spec=PagingSpec.equal_pages_up_to(1 << 14))
    n_cap = 1 << 17
    comp = wrapped.AsyncChunksCompressor(np.int32, cfg, 4, n_cap, n_cap)
    t = wrapped.AsyncPagesTake(np.int32, comp.metas_cap, comp.pages_cap, comp.max_chunks, n_cap, n_cap)
    nums = torch.zeros(n_cap, dtype=torch.int32, device="cuda")
    array_ns = torch.zeros(4, dtype=torch.int64, device="cuda")
    n_arrays = torch.ones(1, dtype=torch.int64, device="cuda")
    metas = torch.zeros(comp.metas_cap, dtype=torch.uint8, device="cuda")
    pages = torch.zeros(comp.pages_cap, dtype=torch.uint8, device="cuda")
    refs = torch.zeros((comp.max_chunks, 5), dtype=torch.int64, device="cuda")
    first = torch.zeros(5, dtype=torch.int64, device="cuda")
    pos = torch.zeros(n_cap, dtype=torch.int64, device="cuda")
    npos = torch.zeros(1, dtype=torch.int64, device="cuda")
    out = _Out(np.int32, n_cap)

    def step():
        comp(nums, array_ns, n_arrays, metas, pages, refs, first)
        t(metas, pages, refs, first[1:2], pos, npos, out.vals)

    g = _capture(step)
    rng = np.random.default_rng(8)
    for n in (100000, 5000, 1):
        x = _walk(np.int32, n, seed=n)
        nums[:n] = torch.as_tensor(x)
        array_ns[0] = n
        p = np.nonzero(rng.random(n) < 0.05)[0] if n > 1 else np.array([0])
        pos[: p.size] = torch.as_tensor(p)
        npos.fill_(p.size)
        out.reset()
        g.replay()
        torch.cuda.synchronize()
        comp.result()
        assert t.result() == p.size
        np.testing.assert_array_equal(out.read(p.size), x[p])
