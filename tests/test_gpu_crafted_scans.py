"""The scan calls on valid streams the encoder never writes (tests/crafted_streams.py): the filter, aggregate, segment aggregate,
histogram and take calls over wrapped pages and over indexed files, the pages-to-file transcode and the asynchronous index builder, one
batch per number type of every crafted family of that type (bins out of order, `lower + offset` past the top of the type, full-width
offsets, all-weight-1 tables, moments at the wrap, IntMult and FloatMult adjustments that land on NaN payloads, infinities and -0.0,
FloatQuant at its edges, chunks of 1 to 2^18 numbers).

Every expected answer comes from the numpy restatement of the decode (cs.expected, itself checked against the oracle's decode by the
`crafted` fixture) and never from another GPU call: selections from IEEE comparisons, aggregates from tests/aggregate_reference.py,
segment records from tests/segment_reference.py, histogram rows from tests/histogram_reference.py, takes from indexing.  The files calls
get the families build_index indexes - decided here, by build_index, and refused by it only as Unsupported and only for families the
catch-all decoder serves; the indexed ones among those (tables of 2^11 or 2^12 states, 257 bins, FloatMult on f16, a secondary latent
with delta) reach the files calls' catch-all path.  The asynchronous calls launch their catch-all kernels on every call (a fixed launch
sequence, so that a call can be captured), so the profiler's spans show the launches; that a cold family was served by them is shown by
its numbers, which the fast decoders decline (tests/test_gpu_crafted_streams.py asserts their routes)."""
import numpy as np
import pytest

from tests import aggregate_reference as ar
from tests import crafted_streams as cs
from tests import segment_reference as sr
from tests.test_gpu_async_aggregate import UNTOUCHED, _outcome as _agg_outcome
from tests.test_gpu_async_histogram import _check_rows, _outcome as _hist_outcome
from tests.test_gpu_async_index import _blocking, _build, _fields
from tests.test_gpu_async_pages import _dev, _refs_dev
from tests.test_gpu_async_pages_to_file import _files_decode, _ok, _refused, _transcode
from tests.test_gpu_async_segment_aggregate import _check as _seg_check
from tests.test_gpu_crafted_streams import BY_DTYPE, _batch, _index, _profiled, _same, _tdtype, crafted  # noqa: F401

pytestmark = pytest.mark.gpu

SENTINEL = 0x5A
TAIL = 64  # sentinel elements past every output's capacity
TAIL_ROWS = 4  # sentinel rows past every segment or histogram output's count
# the catch-all launches of each call (the span names its own tests assert)
CATCH_ALL = {"pages": {"filter": ("ap_cold_kernel", "fl_cold_kernel"), "aggregate": ("ap_cold_kernel", "fl_cold_kernel"),
                       "take": ("ap_cold_kernel", "tk_cold_pages_kernel"), "segment": ("ap_cold_kernel", "sg_cold_pages_kernel"),
                       "histogram": ("ap_cold_kernel", "hg_cold_pages_kernel")},
             "files": {"filter": ("cold_chunks_kernel", "ff_cold_kernel"), "aggregate": ("cold_chunks_kernel", "ff_cold_kernel"),
                       "take": ("cold_chunks_kernel", "tk_cold_files_kernel"), "segment": ("cold_chunks_kernel", "sg_cold_files_kernel"),
                       "histogram": ("cold_chunks_kernel", "hg_cold_files_kernel")}}


class _Scan:
    """One number type's families as a scan batch: every chunk as a wrapped page (all families), and every family build_index indexes as
    an indexed file.  `groups` are the pages or the files, `records` the pages or the chunks, each side with its expected numbers."""

    def __init__(self, crafted, dtype_str):
        from pcodec_b200 import wrapped

        self.dt, self.fams, items = _batch(crafted, dtype_str)
        self.want = np.concatenate([w for _, _, w in items])
        metas, pages, refs, cold = bytearray(), bytearray(), [], []
        for f, (_, parts, _) in zip(self.fams, items):
            for (meta, page), c in zip(parts, f["chunks"]):
                refs.append((len(metas), len(meta), len(pages), len(page), c["n"]))
                metas += meta
                pages += page
                cold.append(c["route"] == "cold")
        self.metas, self.pages = bytes(metas), bytes(pages)
        self.refs = np.array(refs, dtype=wrapped.PAGE_REF)
        self.page_ns = [int(r[4]) for r in refs]
        self.page_cold = cold
        self.pages_cold = any(cold)
        self.indexes = [_index(f, it[0]) for f, it in zip(self.fams, items)]
        self.kept = [i for i, ix in enumerate(self.indexes) if ix is not None]
        data, index, frefs = bytearray(), bytearray(), []
        for i in self.kept:
            blob, ix = items[i][0], self.indexes[i]
            index += b"\0" * (-len(index) % 16)
            frefs.append((len(data), len(blob), len(index), len(ix)))
            index += ix
            data += blob
        self.data, self.index = bytes(data), bytes(index)
        self.file_refs = np.array(frefs, dtype=np.int64).reshape(-1, 4)
        self.files_want = np.concatenate([items[i][2] for i in self.kept]) if self.kept else self.want[:0]
        self.file_ns = [items[i][2].size for i in self.kept]
        self.file_chunk_ns = [[c["n"] for c in self.fams[i]["chunks"]] for i in self.kept]
        self.file_chunk_cold = [c["route"] == "cold" for i in self.kept for c in self.fams[i]["chunks"]]
        self.files_cold = [self.fams[i]["name"] for i in self.kept if cs.is_cold(self.fams[i])]

    # the two sides, as (groups' numbers, each group's record lengths, the device arguments in front of a call's own); `reps` names
    # every page or file that many times over, one copy after another
    def side(self, kind, reps=1):
        import torch

        if kind == "pages":
            refs = np.concatenate([self.refs] * reps)
            args = (_dev(self.metas), _dev(self.pages), _refs_dev(refs, len(refs)), torch.tensor([len(refs)], dtype=torch.int64, device="cuda"))
            return np.tile(self.want, reps), [[n] for n in self.page_ns] * reps, args
        refs = np.tile(self.file_refs, (reps, 1))
        args = (_dev(self.data), _dev(self.index), torch.as_tensor(refs, device="cuda"), torch.tensor([len(refs)], dtype=torch.int64, device="cuda"))
        return np.tile(self.files_want, reps), self.file_chunk_ns * reps, args

    def record_cold(self, kind):
        """Per record of the side (page or chunk), whether the catch-all decoder serves it."""
        return self.page_cold if kind == "pages" else self.file_chunk_cold

    def plan_args(self, kind, reps=1):
        """The leading plan arguments of the pages or files form of a scan call."""
        if kind == "pages":
            frames = reps * int(sum((4 + int(r["meta_len"]) + int(r["page_len"]) + 15) // 16 * 16 for r in self.refs))
            return dict(metas_cap=len(self.metas), pages_cap=len(self.pages), max_pages=reps * len(self.refs), frame_cap=2 * frames + 64)
        return dict(head=self.data[:32], src_cap=len(self.data), index_cap=len(self.index), max_files=reps * len(self.kept),
                    max_chunks=reps * sum(len(ns) for ns in self.file_chunk_ns))


@pytest.fixture(scope="module")
def scans(crafted):
    return {d: _Scan(crafted, d) for d in BY_DTYPE}


def _make(kind, call, s, reps=1, **caps):
    from pcodec_b200 import standalone, wrapped

    cls = {("pages", "filter"): wrapped.AsyncPagesFilter, ("files", "filter"): standalone.AsyncFilesFilter,
           ("pages", "aggregate"): wrapped.AsyncPagesAggregate, ("files", "aggregate"): standalone.AsyncFilesAggregate,
           ("pages", "segment"): wrapped.AsyncPagesSegmentAggregate, ("files", "segment"): standalone.AsyncFilesSegmentAggregate,
           ("pages", "histogram"): wrapped.AsyncPagesHistogram, ("files", "histogram"): standalone.AsyncFilesHistogram,
           ("pages", "take"): wrapped.AsyncPagesTake, ("files", "take"): standalone.AsyncFilesTake}[(kind, call)]
    return cls(dtype=s.dt, **s.plan_args(kind, reps), **caps)


def _sentinels(n, dtype):
    import torch

    return torch.full(((n + TAIL) * np.dtype(dtype).itemsize,), SENTINEL, dtype=torch.uint8, device="cuda").view(_tdtype(dtype))


def _assert_routes(s, kind, call, spans):
    """The call launched its catch-all pass behind its decode stage, and the batch gave that pass cold families to serve."""
    names = CATCH_ALL[kind][call]
    if isinstance(spans, str):  # the profiler's "name=...;" list, as the _outcome helpers return it
        spans = {kv.split("=")[0] for kv in spans.split(";") if kv}
    assert all(n in spans for n in names), (call, kind, sorted(spans))
    assert s.pages_cold if kind == "pages" else s.files_cold, "a batch without a cold family leaves the catch-all path untested"


def _interval(lo, hi, dtype):
    import torch

    from pcodec_b200 import wrapped

    return torch.from_numpy(wrapped.pack_interval(lo, hi, dtype)).cuda()


# ---- filter ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["pages", "files"])
@pytest.mark.parametrize("dtype_str", BY_DTYPE)
def test_filter(scans, dtype_str, kind):
    """Values, positions and counts of every interval equal numpy's selection over the expected numbers, nothing is written past the
    matches, the files call's file_ns are the files' sizes, and an out_cap one below the matches is refused as Io with the count."""
    import torch

    from pcodec_b200 import PcoError

    s = scans[dtype_str]
    want, groups, args = s.side(kind)
    total, item = want.size, s.dt.itemsize
    f = _make(kind, "filter", s, rows_cap=total, out_cap=total)
    vals, pos = _sentinels(total, s.dt), torch.empty(total + TAIL, dtype=torch.int64, device="cuda")
    nm = torch.empty(1, dtype=torch.int64, device="cuda")
    ns = torch.empty(len(groups) + TAIL, dtype=torch.int64, device="cuda")
    extra = (ns[: len(groups)],) if kind == "files" else ()
    for k, (name, (lo, hi)) in enumerate(cs.intervals(want, s.dt).items()):
        vals.view(torch.uint8).fill_(SENTINEL)
        pos.fill_(-1)
        nm.fill_(-7)
        ns.fill_(-3)
        iv = _interval(lo, hi, s.dt)
        if k == 0:
            _, spans, _ = _profiled(lambda: (f(*args, iv, vals, pos, nm, *extra), f.status_record()))
            _assert_routes(s, kind, "filter", spans)
        else:
            f(*args, iv, vals, pos, nm, *extra)
        st = f.status_record()
        got_n = f.result()
        sel = np.flatnonzero(ar.matches(want, lo, hi))
        assert got_n == sel.size == st.n_matches == st.matches_needed == int(nm.item()), (name, got_n, sel.size)
        p, v = pos.cpu().numpy(), vals.cpu().numpy()
        np.testing.assert_array_equal(p[: sel.size], sel, err_msg=name)
        _same(v[: sel.size], want[sel], s.dt, f"filter {kind} {name}")
        assert (p[sel.size:] == -1).all() and (v.view(np.uint8)[sel.size * item:] == SENTINEL).all(), f"{name}: written past the matches"
        if kind == "files":
            h = ns.cpu().numpy()
            np.testing.assert_array_equal(h[: len(groups)], s.file_ns, err_msg=name)
            assert (h[len(groups):] == -3).all(), "written past file_ns"
    # one match more than out_cap: refused as Io, with the count it needs
    lo, hi = cs.intervals(want, s.dt)["all"]
    sel = np.flatnonzero(ar.matches(want, lo, hi))
    short = _make(kind, "filter", s, rows_cap=total, out_cap=sel.size - 1)
    vals.view(torch.uint8).fill_(SENTINEL)
    pos.fill_(-1)
    short(*args, _interval(lo, hi, s.dt), vals, pos, nm, *extra)
    st = short.status_record()
    with pytest.raises(PcoError) as e:
        short.result()
    assert e.value.kind == "Io" and st.matches_needed == sel.size and str(sel.size) in e.value.message, e.value
    p = pos.cpu().numpy()
    np.testing.assert_array_equal(p[: sel.size - 1], sel[:-1])
    assert (p[sel.size - 1:] == -1).all(), "written past out_cap"


# ---- aggregate -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["pages", "files"])
@pytest.mark.parametrize("dtype_str", BY_DTYPE)
def test_aggregate(scans, dtype_str, kind):
    """Each page's (file's) record and the total equal aggregate_reference's over the expected numbers, float sums bit for bit in the
    order include/pco_b200.h gives (any NaN matching any NaN) - the FloatMult families' NaN and infinite sums and the 64-bit types' sums
    that need the high word included."""
    import torch

    s = scans[dtype_str]
    want, groups, args = s.side(kind)
    floats = s.dt.kind == "f"
    a = _make(kind, "aggregate", s, rows_cap=want.size)
    aggs = torch.empty((len(groups), 6), dtype=torch.int64, device="cuda")
    tot = torch.empty(6, dtype=torch.int64, device="cuda")
    bounds = np.cumsum([0] + [sum(g) for g in groups])
    high = False
    for k, (name, (lo, hi)) in enumerate(cs.intervals(want, s.dt).items()):
        aggs.fill_(-1)
        tot.fill_(-1)
        iv = _interval(lo, hi, s.dt)
        if k == 0:
            _, spans, _ = _profiled(lambda: (a(*args, iv, aggs, tot), a.status_record()))
            _assert_routes(s, kind, "aggregate", spans)
        else:
            a(*args, iv, aggs, tot)
        got_n = a.result()
        recs = [ar.record(want[bounds[g]:bounds[g + 1]], groups[g], lo, hi) for g in range(len(groups))]
        rows = aggs.cpu().numpy()
        for g, (rec, _) in enumerate(recs):
            assert ar.same(rows[g].tolist(), rec, floats), (name, kind, g, rows[g].tolist(), rec)
        want_total = ar.total(recs, s.dt)
        assert ar.same(tot.cpu().numpy().tolist(), want_total, floats), (name, tot.cpu().numpy().tolist(), want_total)
        assert got_n == want_total[1]
        high |= not floats and want_total[5] not in (0, (1 << 64) - 1)
    if s.dt.itemsize == 8 and not floats:
        assert high, "no interval's sum needed the high word"


# ---- segment aggregate -----------------------------------------------------------------------------------------------------------
def _records_met(record_ns, bounds):
    """The records sg_mark_kernel marks touched: those whose rows [o, o + n) have o < bounds[M] and o + n > bounds[0].  An empty set
    [k, k] with k inside a record marks that record (it is decoded, and adds nothing)."""
    ns = np.asarray(record_ns, dtype=np.int64)
    starts = np.concatenate([[0], np.cumsum(ns)[:-1]])
    return int(((starts < bounds[-1]) & (starts + ns > bounds[0])).sum())


def _segment_plan(ivs, bound_names):
    """The intervals each bound set runs: "all" and a half (the halves alternating), and every other interval dealt out in turn, so that
    each interval runs at least once."""
    plan = {b: ["all"] + [h for h in (("lower_half", "upper_half")[i % 2],) if h in ivs] for i, b in enumerate(bound_names)}
    rest = [n for n in ivs if n not in ("all", "lower_half", "upper_half")]
    for i, n in enumerate(rest):
        plan[bound_names[i % len(bound_names)]].append(n)
    return plan


def _segments(a, args, s, kind, record_ns, want, bound_sets, plan, ms):
    """Runs every (bound set, interval) pair of `plan` through the segment aggregate `a` and checks its records against
    segment_reference over the expected numbers, and records_decoded against _records_met; the first call under the profiler."""
    import torch

    d_b = torch.zeros(ms + 1, dtype=torch.int64, device="cuda")
    ns = torch.zeros(1, dtype=torch.int64, device="cuda")
    ivs = cs.intervals(want, s.dt)
    first = True
    for bname, names in plan.items():
        b = np.asarray(bound_sets[bname], dtype=np.int64)
        m = b.size - 1
        d_b.zero_()
        d_b[: b.size] = torch.from_numpy(b).cuda()
        ns.fill_(m)
        for name in names:
            lo, hi = ivs[name]
            iv = _interval(lo, hi, s.dt)
            aggs, tot, k, err, st, spans = _agg_outcome(lambda out, total: a(*args, d_b, ns, iv, out, total), a, ms + TAIL_ROWS, first)
            if first:
                _assert_routes(s, kind, "segment", spans)
                first = False
            assert err is None, (bname, name, err)
            if s.dt.kind in "iu" and s.dt.itemsize <= 4 and m > 1024 and (np.diff(b) > 0).all():  # u32 every_batch: thousands of segments
                recs, wt = sr.segment_records_int(want, b, lo, hi)
                assert np.array_equal(aggs[:m].view(np.uint64), np.array(recs, dtype=np.uint64).reshape(m, 6)), (bname, name)
                assert (aggs[m:].view(np.uint64) == UNTOUCHED).all(), "records past the count written"
                assert [int(v) & ar.MASK64 for v in tot] == wt and k == wt[1] == st.n_matches and st.n_segments == m, (bname, name)
            else:
                _seg_check(aggs, tot, k, st, want, record_ns, b, s.dt, lo, hi)
            assert st.records_decoded == _records_met(record_ns, b), (bname, name, st.records_decoded, _records_met(record_ns, b))


@pytest.mark.parametrize("kind", ["pages", "files"])
@pytest.mark.parametrize("dtype_str", BY_DTYPE)
def test_segment_aggregate(scans, dtype_str, kind):
    """Every cs.bounds set (segments on and around the record starts and their rows 255-257, every batch, empty and one-row segments,
    windows into the cold records, segments of more than 2^18 rows on u32) gives, with every cs.intervals interval somewhere, the records
    and total segment_reference gives over the expected numbers (float sums bit for bit, any NaN matching any NaN), n_matches and
    n_segments, nothing past M, and records_decoded counting the pages (chunks) under [bounds[0], bounds[M])."""
    s = scans[dtype_str]
    want, groups, args = s.side(kind)
    record_ns = [n for g in groups for n in g]
    sets = cs.bounds(record_ns, seed=int(s.dt.num), cold=s.record_cold(kind))
    ms = max(b.size - 1 for b in sets.values())
    a = _make(kind, "segment", s, rows_cap=want.size, max_segments=ms)
    _segments(a, args, s, kind, record_ns, want, sets, _segment_plan(cs.intervals(want, s.dt), list(sets)), ms)


@pytest.mark.parametrize("kind", ["pages", "files"])
@pytest.mark.parametrize("dtype_str", ["float16", "float32", "float64"])
def test_long_float_segments(scans, dtype_str, kind):
    """The f64 chain of segments longer than 2^18 rows over the FloatMult specials and the cold records: the batch's refs repeated past
    2^19 rows, one segment over all of them, one inside them, and two long segments around a short one, each with the sums of every number
    but NaN (NaN or infinite), of the finite numbers and of +inf alone."""
    s = scans[dtype_str]
    reps = ((1 << 19) + 1024) // (s.want if kind == "pages" else s.files_want).size + 1
    want, groups, args = s.side(kind, reps)
    rows = want.size
    record_ns = [n for g in groups for n in g]
    cut = (1 << 18) + 77
    sets = {"all": [0, rows], "inside": [100, rows - 100], "long_short_long": [0, cut, cut + 300, rows]}
    assert all(np.diff(b).max() > 1 << 18 for b in sets.values()) and np.diff(sets["long_short_long"])[[0, 2]].min() > 1 << 18
    a = _make(kind, "segment", s, reps=reps, rows_cap=rows, max_segments=3)
    _segments(a, args, s, kind, record_ns, want, sets, {b: ["all", "finite", "pos_inf"] for b in sets}, 3)


# ---- histogram -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["pages", "files"])
@pytest.mark.parametrize("dtype_str", BY_DTYPE)
def test_histogram(scans, dtype_str, kind):
    """Every cs.edges set (the type's extremes and the numbers inside them, a closed top edge on the type's max, the signed key's flip,
    the signed zeros, subnormals and infinities, edges on and between present numbers, 1 to 4096 quantile buckets) gives each page's
    (file's) row histogram_reference gives over its expected numbers, their column sum as the total, rows summing to the groups' sizes,
    the rows past the count untouched, and no edge refused."""
    import torch

    from pcodec_b200 import wrapped

    s = scans[dtype_str]
    want, groups, args = s.side(kind)
    parts = np.split(want, np.cumsum([sum(g) for g in groups])[:-1])
    for k, (name, e) in enumerate(cs.edges(want, s.dt).items()):
        h = _make(kind, "histogram", s, rows_cap=want.size, n_buckets=e.size - 1)
        ed = torch.from_numpy(wrapped.pack_edges(e, s.dt)).cuda()
        hists, tot, n, err, st, spans = _hist_outcome(lambda rows, total: h(*args, ed, rows, total), h, len(groups) + TAIL_ROWS, e.size + 2,
                                                      k == 0)
        if k == 0:
            _assert_routes(s, kind, "histogram", spans)
        assert err is None, (name, err)
        _check_rows(hists, tot, n, parts, e)
        assert st.edge == (1 << 64) - 1 and st.n_written == want.size, (name, st.edge, st.n_written)


# ---- take ------------------------------------------------------------------------------------------------------------------------
def _touched(record_ns, p):
    starts = np.cumsum([0] + list(record_ns))[:-1]
    return int(np.unique(np.searchsorted(starts, p, side="right") - 1).size)


@pytest.mark.parametrize("kind", ["pages", "files"])
@pytest.mark.parametrize("dtype_str", BY_DTYPE)
def test_take(scans, dtype_str, kind):
    """Every position set's values equal the expected numbers at those positions bit for bit, nothing is written past them, and
    records_decoded counts the pages (chunks) the set touches."""
    import torch

    s = scans[dtype_str]
    want, groups, args = s.side(kind)
    record_ns = [n for g in groups for n in g]
    total, item = want.size, s.dt.itemsize
    t = _make(kind, "take", s, rows_cap=total, max_positions=max(total, 1))
    vals = _sentinels(total, s.dt)
    pos = torch.zeros(max(total, 1), dtype=torch.int64, device="cuda")
    npos = torch.zeros(1, dtype=torch.int64, device="cuda")
    for k, (name, p) in enumerate(cs.positions(record_ns, seed=int(s.dt.num)).items()):
        vals.view(torch.uint8).fill_(SENTINEL)
        if p.size:
            pos[: p.size] = torch.from_numpy(p).cuda()
        npos.fill_(p.size)
        if k == 0:
            _, spans, _ = _profiled(lambda: (t(*args, pos, npos, vals), t.status_record()))
            _assert_routes(s, kind, "take", spans)
        else:
            t(*args, pos, npos, vals)
        st = t.status_record()
        assert t.result() == p.size == st.n_positions, name
        v = vals.cpu().numpy()
        _same(v[: p.size], want[p], s.dt, f"take {kind} {name}")
        assert (v.view(np.uint8)[p.size * item:] == SENTINEL).all(), f"{name}: written past the positions"
        assert st.records_decoded == _touched(record_ns, p), (name, st.records_decoded, _touched(record_ns, p))


# ---- pages to file ---------------------------------------------------------------------------------------------------------------
def _page_refs(parts_list):
    """metas, pages and PAGE_REF records of [(meta, page) per chunk] lists, back to back."""
    from pcodec_b200 import wrapped

    metas, pages, refs = bytearray(), bytearray(), []
    for parts, ns in parts_list:
        for (meta, page), n in zip(parts, ns):
            refs.append((len(metas), len(meta), len(pages), len(page), n))
            metas += meta
            pages += page
    return bytes(metas), bytes(pages), np.array(refs, dtype=wrapped.PAGE_REF)


@pytest.mark.parametrize("dtype_str", BY_DTYPE)
def test_pages_to_file(oracle, crafted, scans, dtype_str):
    """The pages of every family build_index indexes, transcoded together, are the file the oracle's explicit writer makes of the same
    chunks in the same order, byte for byte (both write the non-uniform header with the total as its size hint), with the index
    build_index makes of that file (record by record and entry by entry: build_index reserves room for more chunk records than the file
    has, so its entries lie further on), and AsyncFilesDecompressor reads the numbers back.  A family build_index refuses, between walkable pages, is refused
    with build_index's kind, naming its first page, and nothing is written."""
    from pcodec_b200 import PcoError
    from pcodec_b200 import standalone as sa

    s = scans[dtype_str]
    items = [crafted[f["name"]] for f in s.fams]
    kept = [s.fams[i] for i in s.kept]
    metas, pages, refs = _page_refs([(items[i][1], [c["n"] for c in s.fams[i]["chunks"]]) for i in s.kept])
    o = _ok(_transcode(metas, pages, refs, s.dt))
    want_file, _ = oracle.write_explicit_file(s.dt, [{k: v for k, v in c.items() if k != "route"} for f in kept for c in f["chunks"]])
    assert o.file == want_file
    assert _fields(o.index) == _fields(sa.build_index(o.file, s.dt))
    assert o.st.n_pages == len(refs) and o.st.n_total == s.files_want.size
    got, err, _ = _files_decode(o, s.dt, s.files_want.size)
    assert err is None, err
    _same(got, s.files_want, s.dt, "AsyncFilesDecompressor on the transcoded file")
    # the refused families, each between a walkable page before and after it
    first = items[s.kept[0]][1][0]
    for i, f in enumerate(s.fams):
        if s.indexes[i] is not None:
            continue
        with pytest.raises(PcoError) as e:
            sa.build_index(items[i][0], s.dt)
        ns = [c["n"] for c in f["chunks"]]
        m, p, r = _page_refs([([first], [s.fams[s.kept[0]]["chunks"][0]["n"]]), (items[i][1], ns),
                              ([first], [s.fams[s.kept[0]]["chunks"][0]["n"]])])
        o = _refused(_transcode(m, p, r, s.dt))
        assert o.err.kind == e.value.kind and o.st.page == 1 and ": page 1:" in str(o.err), (f["name"], o.err)


# ---- asynchronous index ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype_str", BY_DTYPE)
def test_async_index(oracle, crafted, scans, dtype_str):
    """AsyncIndexBuilder writes build_index's index for every family's file (record by record and entry by entry, as
    test_gpu_async_index.py compares them), or refuses it with build_index's kind and chunk; and likewise for one file of all the indexed
    families' chunks, whose many chunk sizes leave most of it to the serial walker."""
    from pcodec_b200 import PcoError
    from pcodec_b200 import standalone as sa

    s = scans[dtype_str]
    for f in s.fams:
        data = crafted[f["name"]][0]
        got, st = _build(data, s.dt)
        want = _blocking(data, s.dt)
        if isinstance(want, tuple):
            assert isinstance(got, PcoError), (f["name"], want)
            assert (got.kind, None if st.chunk == (1 << 64) - 1 else st.chunk) == want, (f["name"], got.message, want)
        else:
            assert _fields(got) == _fields(want), f["name"]
    chunks = [{k: v for k, v in c.items() if k != "route"} for i in s.kept for c in s.fams[i]["chunks"]]
    data, _ = oracle.write_explicit_file(s.dt, chunks)
    got, st = _build(data, s.dt)
    assert not isinstance(got, PcoError), got
    assert _fields(got) == _fields(sa.build_index(data, s.dt))
    assert st.n_chunks == len(chunks) and st.n_total == s.files_want.size
    runs = 1 + sum(a["n"] != b["n"] for a, b in zip(chunks, chunks[1:]))
    if runs > 2:  # the two rounds take two runs of equal sizes; the serial walker the rest
        assert st.serial_chunks > 0, (runs, st.serial_chunks)
