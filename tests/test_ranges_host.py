"""pco_b200_decompress_ranges refuses bad arguments before any device work, and its host logic (splitting ranges at chunk
boundaries, grouping the pieces into one decode task per chunk) is exposed through pco_b200_debug_plan_ranges, so these run without
a GPU."""
import ctypes as C

import numpy as np
import pytest

OK, INVALID_ARGUMENT, IO, INVALID_TYPE = 0, 3, 4, 5
INDEX_MAGIC = 0x58444950
CHUNK = np.dtype([("chunk_offset", "<u8"), ("n", "<u4"), ("n_vars", "<u4"), ("entries_offset", "<u8"), ("out_offset", "<u8")])
HEADER = np.dtype([("magic", "<u4"), ("version", "<u4"), ("n_chunks", "<u8"), ("n_total", "<u8"), ("file_len", "<u8"), ("chunks_offset", "<u8"),
                   ("end_byte", "<u8"), ("reserved", "<u8", 2)])
# a standalone header (version 3, no uniform type, size hint 0, format 4.0) and room behind it; no device ever reads the chunks
FILE = b"pco!\x03\x00\x00\x04\x00" + bytes(55)


@pytest.fixture(scope="module")
def L():
    from pcodec_b200 import _lib

    return _lib.lib()


def _chunks(ns, out_offsets=None):
    recs = np.zeros(len(ns), dtype=CHUNK)
    recs["n"] = ns
    recs["chunk_offset"] = 9 + np.arange(len(ns))
    recs["out_offset"] = np.concatenate([[0], np.cumsum(ns)[:-1]]).astype(np.uint64) if out_offsets is None else out_offsets
    return recs


def _ranges(*pairs):
    from pcodec_b200 import standalone

    return standalone._ranges_array(np.array(pairs, dtype=np.uint64).reshape(-1, 2))


def _plan(L, recs, ranges, n_total=None):
    n_total = int(recs["n"].sum()) if n_total is None else n_total
    cap = len(ranges) * (len(recs) + 1) + 4
    pieces = np.zeros((cap, 6), dtype=np.uint64)
    tasks = np.zeros((cap, 6), dtype=np.uint64)
    npc, nt = C.c_size_t(), C.c_size_t()
    rc = L.pco_b200_debug_plan_ranges(recs.ctypes.data_as(C.c_void_p) if len(recs) else None, C.c_size_t(len(recs)), C.c_uint64(n_total),
                                      ranges.ctypes.data_as(C.c_void_p), C.c_size_t(len(ranges)), pieces.ctypes.data_as(C.c_void_p), C.c_size_t(cap),
                                      C.byref(npc), tasks.ctypes.data_as(C.c_void_p), C.c_size_t(cap), C.byref(nt))
    if rc != OK:
        return rc, None, None
    return rc, [tuple(int(x) for x in r) for r in pieces[: npc.value]], [tuple(int(x) for x in r) for r in tasks[: nt.value]]


def _index(recs, n_total=None, file_len=len(FILE), magic=INDEX_MAGIC):
    h = np.zeros(1, dtype=HEADER)
    h["magic"], h["version"], h["n_chunks"] = magic, 1, len(recs)
    h["n_total"] = int(recs["n"].sum()) if n_total is None else n_total
    h["file_len"], h["chunks_offset"] = file_len, HEADER.itemsize
    return h.tobytes() + recs.tobytes()


def _call(L, ranges, index=None, dtype=2, dst_len=1 << 12, null_ranges=False, n_ranges=None):
    src = np.frombuffer(FILE, dtype=np.uint8).copy()
    ix = np.frombuffer(index, dtype=np.uint8).copy() if index is not None else None
    dst = np.zeros(max(dst_len, 1), dtype=np.uint64)
    nw = C.c_size_t(12345)
    rng = None if null_ranges else ranges.ctypes.data_as(C.c_void_p)
    rc = L.pco_b200_decompress_ranges(src.ctypes.data_as(C.c_void_p), C.c_size_t(src.size), C.c_ubyte(dtype),
                                      ix.ctypes.data_as(C.c_void_p) if ix is not None else None, C.c_size_t(ix.size if ix is not None else 0), rng,
                                      C.c_size_t(len(ranges) if n_ranges is None else n_ranges), dst.ctypes.data_as(C.c_void_p), C.c_size_t(dst_len),
                                      C.byref(nw), C.c_uint32(0), None)
    return rc, nw.value


def _message(L):
    return L.pco_b200_last_error_message().decode()


# ---- arguments refused before any device work


def test_unknown_dtype_and_missing_arguments(L):
    recs = _chunks([1000])
    assert _call(L, _ranges((0, 5)), _index(recs), dtype=99)[0] == INVALID_TYPE
    assert _call(L, _ranges((0, 5)), None)[0] == INVALID_ARGUMENT
    assert "side index is required" in _message(L)
    assert _call(L, _ranges((0, 5)), _index(recs), null_ranges=True)[0] == INVALID_ARGUMENT
    assert "ranges are required" in _message(L)


def test_no_ranges_is_ok(L):
    recs = _chunks([1000])
    assert _call(L, _ranges(), _index(recs)) == (OK, 0)
    assert _call(L, _ranges(), _index(recs), null_ranges=True) == (OK, 0)


@pytest.mark.parametrize("bad", [(0, 1001), (1000, 1), (1 << 63, 1 << 63), ((1 << 64) - 1, 2), (5, (1 << 64) - 1)])
def test_range_past_the_file_names_the_range(L, bad):
    rc, nw = _call(L, _ranges((0, 10), bad, (3, 4)), _index(_chunks([600, 400])))
    assert (rc, nw) == (INVALID_ARGUMENT, 0)
    assert _message(L).startswith("range 1: ")


def test_dst_shorter_than_the_ranges(L):
    rc, _ = _call(L, _ranges((0, 600), (100, 600)), _index(_chunks([600, 400])), dst_len=1199)
    assert rc == INVALID_ARGUMENT
    assert "dst holds 1199 numbers, the ranges 1200" in _message(L)


def test_index_of_another_file(L):
    recs = _chunks([600, 400])
    assert _call(L, _ranges((0, 5)), _index(recs, file_len=len(FILE) + 1))[0] == INVALID_ARGUMENT
    assert "does not belong to this file" in _message(L)
    assert _call(L, _ranges((0, 5)), _index(recs, magic=0))[0] == INVALID_ARGUMENT
    assert _call(L, _ranges((0, 5)), _index(recs)[:40])[0] == INVALID_ARGUMENT
    assert _call(L, _ranges((0, 5)), _index(recs)[:-1])[0] == INVALID_ARGUMENT  # the chunk table runs past the index


@pytest.mark.parametrize("out_offsets, ns, what", [
    ([0, 500], [600, 400], "overlap"),
    ([0, 700], [600, 400], "gap"),
    ([400, 0], [600, 400], "out of order"),
    ([0, 600, 600], [600, 0, 400], "empty chunk"),
])
def test_chunk_tables_that_do_not_tile_are_refused(L, out_offsets, ns, what):
    recs = _chunks(ns, np.array(out_offsets, dtype=np.uint64))
    assert _plan(L, recs, _ranges((0, 5)), n_total=1000)[0] == INVALID_ARGUMENT, what
    assert "side index" in _message(L)
    assert _call(L, _ranges((0, 5)), _index(recs, n_total=1000))[0] == INVALID_ARGUMENT, what


def test_chunk_counts_must_add_up_to_the_header(L):
    recs = _chunks([600, 400])
    assert _plan(L, recs, _ranges((0, 5)), n_total=1001)[0] == INVALID_ARGUMENT
    assert _call(L, _ranges((0, 5)), _index(recs, n_total=999))[0] == INVALID_ARGUMENT


# ---- pieces and tasks


@pytest.mark.parametrize("k", [1, 2, 3])
def test_split_at_chunk_boundaries(L, k):
    n = 1000
    recs = _chunks([n] * 4)
    for start, count in [(k * n - 1, 1), (k * n, 1), (k * n + 1, 1), (k * n - 1, 2), (k * n - 1, 3)]:
        rc, pieces, tasks = _plan(L, recs, _ranges((start, count)))
        assert rc == OK
        want, s, left, off = [], start, count, 0
        while left:
            c = s // n
            take = min(left, n - s % n)
            want.append((c, s % n, s % n + take, off, 0))
            s, left, off = s + take, left - take, off + take
        assert [p[:5] for p in pieces] == want
        assert [(t[0], t[1], t[2], t[3], t[5]) for t in tasks] == [(w[0], w[1], w[2], 1, 0) for w in want]  # one piece each: direct


def test_short_last_chunk_and_whole_file(L):
    recs = _chunks([256, 256, 7])
    rc, pieces, tasks = _plan(L, recs, _ranges((0, 519)))
    assert rc == OK
    assert [p[:4] for p in pieces] == [(0, 0, 256, 0), (1, 0, 256, 256), (2, 0, 7, 512)]
    rc, pieces, _ = _plan(L, recs, _ranges((518, 1)))
    assert [p[:4] for p in pieces] == [(2, 6, 7, 0)]  # the last number


def _ref_plan(ns, pairs):
    """What the plan must be: pieces (chunk, lo, hi, dst_off, range) in range order; tasks (chunk, lo, hi, n_pieces, lowest range, staged)."""
    starts = np.concatenate([[0], np.cumsum(ns)]).tolist()
    pieces, off = [], 0
    for i, (s, left) in enumerate(pairs):
        while left:
            c = max(k for k in range(len(ns)) if starts[k] <= s)
            take = min(left, starts[c + 1] - s)
            pieces.append((c, s - starts[c], s - starts[c] + take, off, i))
            s, left, off = s + take, left - take, off + take
    tasks = []
    for c in sorted({p[0] for p in pieces}):
        mine = [p for p in pieces if p[0] == c]
        tasks.append((c, min(p[1] for p in mine), max(p[2] for p in mine), len(mine), min(p[4] for p in mine), int(len(mine) > 1)))
    return pieces, tasks


def test_exact_paging_chunks_of_unequal_size(L):
    ns = [3, 1000, 1, 257, 65536]
    starts = np.concatenate([[0], np.cumsum(ns)]).tolist()
    pairs = [(2, 1002), (starts[2], 258), (starts[4] + 255, 2), (starts[3] + 256, 1)]
    rc, pieces, tasks = _plan(L, _chunks(ns), _ranges(*pairs))
    assert rc == OK
    want_pieces, want_tasks = _ref_plan(ns, pairs)
    assert [p[:5] for p in pieces] == want_pieces
    assert tasks == want_tasks
    # chunks 2 and 3 are touched by two ranges each: staged tasks over their windows; the others are direct
    assert [t[5] for t in tasks] == [0, 0, 1, 1, 0]


def test_random_plans_match_the_reference_split(L):
    rng = np.random.default_rng(3)
    for _ in range(20):
        ns = rng.integers(1, 3000, rng.integers(1, 12)).tolist()
        total = sum(ns)
        pairs = []
        for _ in range(int(rng.integers(1, 30))):
            s = int(rng.integers(0, total + 1))
            pairs.append((s, int(rng.integers(0, total - s + 1))))
        rc, pieces, tasks = _plan(L, _chunks(ns), _ranges(*pairs))
        assert rc == OK
        want_pieces, want_tasks = _ref_plan(ns, pairs)
        assert [p[:5] for p in pieces] == want_pieces
        assert tasks == want_tasks
        assert all(tasks[p[5]][0] == p[0] for p in pieces)


def test_empty_and_repeated_ranges(L):
    recs = _chunks([1000, 1000])
    rc, pieces, tasks = _plan(L, recs, _ranges((5, 0), (1500, 10), (2000, 0), (1500, 10), (0, 0)))
    assert rc == OK
    assert [p[:5] for p in pieces] == [(1, 500, 510, 0, 1), (1, 500, 510, 10, 3)]
    assert [t[:6] for t in tasks] == [(1, 500, 510, 2, 1, 1)]
    rc, pieces, tasks = _plan(L, recs, _ranges((0, 0), (2000, 0)))
    assert (rc, pieces, tasks) == (OK, [], [])


def test_many_pieces_in_one_chunk_make_one_staged_task(L):
    rng = np.random.default_rng(7)
    n = 1 << 16
    recs = _chunks([n, n, n])
    starts = rng.integers(n, 2 * n - 64, 500)
    counts = rng.integers(1, 64, 500)
    pairs = list(zip(starts[::-1].tolist(), counts[::-1].tolist()))  # descending, overlapping
    pairs.insert(250, (0, 3))
    rc, pieces, tasks = _plan(L, recs, _ranges(*pairs))
    assert rc == OK
    assert len(pieces) == 501
    assert [t[0] for t in tasks] == [0, 1]
    t1 = tasks[1]
    assert (t1[1], t1[2], t1[3], t1[5]) == (int(starts.min()) - n, int((starts + counts).max()) - n, 500, 1)
    assert t1[4] == 0 and tasks[0][4] == 250  # lowest range with numbers in each chunk
    assert all(p[5] == (0 if p[0] == 0 else 1) for p in pieces)
    off = np.concatenate([[0], np.cumsum([c for _, c in pairs])[:-1]])
    assert [p[3] for p in pieces] == off.tolist()


def test_plan_reports_sizes_when_tables_are_short(L):
    recs = _chunks([10, 10])
    ranges = _ranges((0, 20))
    npc, nt = C.c_size_t(), C.c_size_t()
    out = np.zeros(6, dtype=np.uint64)
    rc = L.pco_b200_debug_plan_ranges(recs.ctypes.data_as(C.c_void_p), C.c_size_t(2), C.c_uint64(20), ranges.ctypes.data_as(C.c_void_p), C.c_size_t(1),
                                      out.ctypes.data_as(C.c_void_p), C.c_size_t(1), C.byref(npc), out.ctypes.data_as(C.c_void_p), C.c_size_t(1), C.byref(nt))
    assert rc == IO
    assert (npc.value, nt.value) == (2, 2)


def test_python_ranges_argument(L):
    from pcodec_b200 import standalone

    r = standalone._ranges_array([[1, 2], [3, 4]])
    assert r.dtype == standalone.RANGE and r["start"].tolist() == [1, 3] and r["count"].tolist() == [2, 4]
    rec = np.array([(5, 6)], dtype=standalone.RANGE)
    assert standalone._ranges_array(rec).tolist() == [(5, 6)]
    assert standalone._ranges_array(np.zeros((0, 2), np.int64)).size == 0
    with pytest.raises(ValueError):
        standalone._ranges_array([[-1, 2]])
