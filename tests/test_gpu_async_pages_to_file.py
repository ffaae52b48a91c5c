"""Transcode of wrapped pages into one indexed standalone file on the GPU (pco_b200_pages_to_file_async, wrapped.AsyncPagesToFile).  The
file and index are compared byte for byte with pco_b200_compress_ex's for the same chunks, with the oracle's standalone decoder and with
pco_b200_build_index_async's index of the file; the files calls on the output are compared with the pages calls on the pages; every
refusal with the pages call's kind and page."""
import numpy as np
import pytest

from tests.golden_generators import bits_view
from tests.test_gpu_async_pages import _cold_batch, _dev, _refs_dev
from tests.test_gpu_async_pages import _run as _pages_run
from tests.test_gpu_encode import _cfgs, _walk
from tests.test_gpu_wrapped_batch import _container, _data, _mixed_chunks, _shuffled, _six_pages

pytestmark = pytest.mark.gpu

SENTINEL = 0x5A
NONE = (1 << 64) - 1
ALL = [np.uint8, np.int8, np.uint16, np.int16, np.float16, np.uint32, np.int32, np.float32, np.uint64, np.int64, np.float64]


def _entries_room(refs):
    r = np.asarray(refs)
    return 64 + 32 * len(r) + int(sum((2 * ((int(n) + 255) // 256) * 12 + 15) // 16 * 16 for n in r["page_n"])) if len(r) else 64


def _frames(refs):
    r = np.asarray(refs)
    return int(sum((4 + int(m) + int(p) + 15) // 16 * 16 for m, p in zip(r["meta_len"], r["page_len"]))) if len(r) else 0


def _chunk_bytes(refs):
    r = np.asarray(refs)
    return int(sum(4 + int(m) + int(p) for m, p in zip(r["meta_len"], r["page_len"]))) if len(r) else 0


class _Out:
    pass


def _transcode(metas, pages, refs, dtype, max_pages=None, dst_cap=None, index_cap=None, frame_cap=None, n=None, uniform=False):
    """The call over host bytes copied to the device, its outputs filled with SENTINEL first.  Returns an _Out with the transcoder t, the
    whole file and index buffers (bytes), the ref, the error (or None) and the status."""
    import torch

    from pcodec_b200 import PcoError, wrapped

    max_pages = max_pages or max(len(refs), 1)
    dst_cap = dst_cap if dst_cap is not None else 32 + _chunk_bytes(refs)
    index_cap = index_cap if index_cap is not None else _entries_room(refs)
    frame_cap = frame_cap if frame_cap is not None else 2 * _frames(refs) + 64
    t = wrapped.AsyncPagesToFile(dtype, len(metas), len(pages), max_pages, dst_cap, index_cap, frame_cap, uniform_type_header=uniform)
    t.file.fill_(SENTINEL)
    t.index.fill_(SENTINEL)
    t.file_ref.fill_(-1)
    nt = torch.tensor([len(refs) if n is None else n], dtype=torch.int64, device="cuda")
    t(_dev(metas), _dev(pages), _refs_dev(refs, max_pages), nt)
    o = _Out()
    o.t, o.st = t, t.status_record()
    try:
        (o.file_len, o.index_len), o.err = t.result(), None
    except PcoError as e:
        o.file_len, o.index_len, o.err = 0, 0, e
    o.file_buf, o.index_buf = t.file.cpu().numpy().tobytes(), t.index.cpu().numpy().tobytes()
    o.file, o.index = o.file_buf[: o.file_len], o.index_buf[: o.index_len]
    o.ref = t.file_ref.cpu().numpy().reshape(-1).tolist()
    return o


def _ok(o):
    assert o.err is None, o.err
    assert o.ref == [0, o.file_len, 0, o.index_len] and o.st.page == NONE
    assert o.file_buf[o.file_len:] == bytes([SENTINEL]) * (len(o.file_buf) - o.file_len), "written past the file"
    assert o.index_buf[o.index_len:] == bytes([SENTINEL]) * (len(o.index_buf) - o.index_len), "written past the index"
    return o


def _refused(o):
    assert o.err is not None and o.st.kind != 0
    assert o.ref == [0, 0, 0, 0], "the ref must be zeroed on a failure"
    assert set(o.file_buf) == {SENTINEL} and set(o.index_buf) == {SENTINEL}, "a refused call wrote its outputs"
    return o


def _files_decode(o, dtype, dst_cap):
    """AsyncFilesDecompressor over the call's own output tensors and ref: (numbers, error)."""
    import torch

    from pcodec_b200 import PcoError, standalone
    from pcodec_b200.wrapped import _torch_dtypes

    d = standalone.AsyncFilesDecompressor(**o.t.files_args(), dst_cap=max(dst_cap, 1))
    dst = torch.zeros(max(dst_cap, 1), dtype=_torch_dtypes()[np.dtype(dtype)], device="cuda")
    ns = torch.zeros(1, dtype=torch.int64, device="cuda")
    d(o.t.file, o.t.index, o.t.file_ref, o.t.n_files, dst, ns)
    try:
        nw, err = d.result(), None
    except PcoError as e:
        nw, err = 0, e
    return dst.cpu().numpy()[:nw], err, d.status_record()


def _built_index(file, dtype, max_chunks, index_cap):
    import torch

    from pcodec_b200 import standalone

    b = standalone.AsyncIndexBuilder(file[:32], dtype, len(file) + 16, index_cap, max_chunks)
    idx = torch.full((index_cap + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
    b(_dev(file, len(file) + 16), torch.tensor([len(file)], dtype=torch.int64, device="cuda"), idx)
    il = b.result()
    return idx.cpu().numpy().tobytes()[:il]


# ---- byte identity with compress_ex

def _configs(dtype):
    kind = np.dtype(dtype).kind
    out = [("classic", o, 8) for o in range(8)] + [("classic", 1, 12), ("classic", 0, 10)]
    if kind == "f":
        out += [("float_quant", 1, 8)] + ([] if np.dtype(dtype).itemsize == 2 else [("float_mult", 0, 8), ("float_mult", 2, 12)])
    else:
        out += [("int_mult", 0, 8), ("int_mult", 3, 12)]
    return out


@pytest.mark.parametrize("dtype", ALL)
def test_file_and_index_equal_compress_ex(oracle, dtype):
    from pcodec_b200 import standalone, wrapped

    for k, (mode, order, level) in enumerate(_configs(dtype)):
        n = 5000 + 777 * k
        x = _data(dtype, mode, n, seed=300 + k)
        cfg, _ = _cfgs(oracle, mode=mode, order=order, level=level, max_page_n=2048, k=13 if np.dtype(dtype).itemsize > 2 else 5)
        uniform = k % 2 == 1
        want_file, want_index = standalone.simple_compress_with_index(x, cfg, uniform_type=uniform)
        metas, pages, refs = wrapped.compress_chunks(x, cfg)
        o = _ok(_transcode(metas, pages, refs, dtype, uniform=uniform))
        assert o.file == want_file, (mode, order, level, uniform)
        assert o.index == want_index, (mode, order, level, uniform)
        assert o.st.n_pages == len(refs) and o.st.n_total == n


def test_level_12_tables_take_the_wide_walk(oracle):
    """A chunk with 2^11- or 2^12-state tables is declined by the 2^10-state walker and taken by the wide one."""
    from pcodec_b200 import standalone, wrapped

    O = oracle
    rng = np.random.default_rng(3)
    centers = np.sort(rng.integers(0, 1 << 30, size=600))
    p = rng.lognormal(0.0, 1.0, size=centers.size)
    wide = (centers[rng.choice(centers.size, size=1 << 17, p=p / p.sum())] + rng.integers(0, 16, size=1 << 17)).astype(np.int32)
    metas, pages, refs, pieces = _container([(wide, O.make_config(level=12, mode=O.MODE_CLASSIC, delta=O.DELTA_NOOP))])
    o = _ok(_transcode(metas, pages, refs, np.int32))
    np.testing.assert_array_equal(O.simple_decompress(o.file, np.int32), wide)
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec

    cfg = ChunkConfig(compression_level=12, mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.no_op())
    want_file, want_index = standalone.simple_compress_with_index(wide, cfg)
    m2, p2, r2 = wrapped.compress_chunks(wide, cfg)
    o2 = _ok(_transcode(m2, p2, r2, np.int32))
    assert o2.file == want_file and o2.index == want_index


# ---- containers the oracle wrote

def _oracle_batches(oracle):
    O = oracle
    out = []
    for dtype in (np.uint64, np.float32, np.int16, np.float16, np.uint8):
        metas, pages, refs, pieces = _container(_mixed_chunks(oracle, dtype))
        refs, pieces = _shuffled(refs, pieces, seed=int(np.dtype(dtype).num))  # out of order, one page twice
        out.append((f"mixed-{np.dtype(dtype).name}", dtype, metas, pages, refs, pieces))
    metas, pages, refs, pieces = _six_pages(oracle)
    out.append(("six", np.uint64, metas, pages, refs[::-1].copy(), pieces[::-1]))
    fm = (np.round(np.random.default_rng(4).normal(size=4000) * 40) * 0.25).astype(np.float16)
    plain = _walk(np.float16, 3000, seed=9)
    chunks = [(plain, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=1)),
              (fm, O.make_config(mode=O.MODE_FLOAT_MULT, float_mult_base=0.25, delta=O.DELTA_CONSECUTIVE, delta_order=1, max_page_n=1500)),
              (plain[:999], O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_NOOP))]
    metas, pages, refs, pieces = _container(chunks)
    out.append(("f16-float-mult", np.float16, metas, pages, refs, pieces))
    metas, pages, refs, pieces = _cold_batch(oracle)
    keep = [i for i in range(len(refs)) if _transcode(metas, pages, refs[i:i + 1], np.int32).err is None]
    out.append(("wide-and-fast", np.int32, metas, pages, refs[keep], [pieces[i] for i in keep]))
    return out


def test_oracle_containers(oracle):
    for name, dtype, metas, pages, refs, pieces in _oracle_batches(oracle):
        total = sum(len(p) for p in pieces)
        got_pages, nw, err, _ = _pages_run(metas, pages, refs, dtype, frame_cap=_frames(refs))
        assert err is None and nw == total, (name, err)
        want = got_pages[:total]
        o = _ok(_transcode(metas, pages, refs, dtype))
        assert o.st.n_total == total, name
        # the oracle's standalone decoder reads the file
        np.testing.assert_array_equal(bits_view(oracle.simple_decompress(o.file, dtype)), bits_view(want), err_msg=name)
        # the index is the one the device index builder finds for the file
        assert o.index == _built_index(o.file, dtype, len(refs), o.index_len + 64), name
        # and the files call serves it
        got, ferr, _ = _files_decode(o, dtype, total)
        assert ferr is None, (name, ferr)
        np.testing.assert_array_equal(bits_view(got), bits_view(want), err_msg=name)
        np.testing.assert_array_equal(bits_view(got), bits_view(np.concatenate(pieces)), err_msg=name)


# ---- scans: files calls on the output against pages calls on the pages

def test_filter_aggregate_and_take_match_the_pages_calls(oracle):
    import torch

    from pcodec_b200 import standalone, wrapped
    from pcodec_b200.wrapped import _torch_dtypes

    for dtype in (np.uint64, np.int32, np.float32):
        metas, pages, refs, pieces = _container(_mixed_chunks(oracle, dtype))
        refs, pieces = _shuffled(refs, pieces, seed=2)
        x = np.concatenate(pieces)
        total, mp, fc = x.size, len(refs), _frames(refs) + 64
        o = _ok(_transcode(metas, pages, refs, dtype))
        dm, dp, dr = _dev(metas), _dev(pages), _refs_dev(refs, mp)
        nt = torch.tensor([mp], dtype=torch.int64, device="cuda")
        tdt = _torch_dtypes()[np.dtype(dtype)]
        fa = o.t.files_args()
        s = np.sort(x)
        lo, hi = s[total // 3], s[total // 3 + total // 100]
        iv = torch.from_numpy(wrapped.pack_interval(lo, hi, dtype)).cuda()
        # filter, 1 %
        pf = wrapped.AsyncPagesFilter(dtype, len(metas), len(pages), mp, total, total, fc)
        ff = standalone.AsyncFilesFilter(**fa, rows_cap=total, out_cap=total)
        outs = []
        for call, src in ((pf, (dm, dp, dr, nt)), (ff, (o.t.file, o.t.index, o.t.file_ref, o.t.n_files))):
            vals = torch.zeros(total, dtype=tdt, device="cuda")
            pos = torch.zeros(total, dtype=torch.int64, device="cuda")
            nm = torch.zeros(1, dtype=torch.int64, device="cuda")
            call(*src, iv, vals, pos, nm)
            k = call.result()
            outs.append((k, bits_view(vals.cpu().numpy()[:k]), pos.cpu().numpy()[:k]))
        assert outs[0][0] == outs[1][0] > 0
        np.testing.assert_array_equal(outs[0][1], outs[1][1])
        np.testing.assert_array_equal(outs[0][2], outs[1][2])
        # aggregate: the pages' per-page records summed against the file's one record (exact for integers; counts, min and max for floats)
        pa = wrapped.AsyncPagesAggregate(dtype, len(metas), len(pages), mp, total, fc)
        fa_ = standalone.AsyncFilesAggregate(**fa, rows_cap=total)
        recs = []
        for call, src, groups in ((pa, (dm, dp, dr, nt), mp), (fa_, (o.t.file, o.t.index, o.t.file_ref, o.t.n_files), 1)):
            aggs = torch.zeros((groups, 6), dtype=torch.int64, device="cuda")
            tot = torch.zeros(6, dtype=torch.int64, device="cuda")
            call(*src, iv, aggs, tot)
            call.result()
            recs.append(wrapped.unpack_aggregates(tot.cpu().numpy(), dtype)[0])
        (n0, c0, mn0, mx0, s0), (n1, c1, mn1, mx1, s1) = recs
        assert (n0, c0) == (n1, c1) and bits_view(np.array([mn0, mx0])).tolist() == bits_view(np.array([mn1, mx1])).tolist()
        if np.dtype(dtype).kind != "f":
            assert s0 == s1
        # take, a contiguous 1 % and a uniform 1 %
        rng = np.random.default_rng(5)
        for positions in (np.arange(total // 2, total // 2 + total // 100), np.sort(rng.choice(total, total // 100, replace=False))):
            pos = torch.zeros(total, dtype=torch.int64, device="cuda")
            pos[: positions.size] = torch.from_numpy(positions.astype(np.int64)).cuda()
            npos = torch.tensor([positions.size], dtype=torch.int64, device="cuda")
            pt = wrapped.AsyncPagesTake(dtype, len(metas), len(pages), mp, total, total, fc)
            ft = standalone.AsyncFilesTake(**fa, rows_cap=total, max_positions=total)
            got = []
            for call, src in ((pt, (dm, dp, dr, nt)), (ft, (o.t.file, o.t.index, o.t.file_ref, o.t.n_files))):
                vals = torch.zeros(total, dtype=tdt, device="cuda")
                call(*src, pos, npos, vals)
                assert call.result() == positions.size
                got.append(bits_view(vals.cpu().numpy()[: positions.size]))
            np.testing.assert_array_equal(got[0], got[1])
            np.testing.assert_array_equal(got[1], bits_view(x[positions]))


# ---- refusals

def _same_failure(metas, pages, refs, dtype=np.uint64, **kw):
    _, _, perr, pst = _pages_run(metas, pages, refs, dtype, **{k: v for k, v in kw.items() if k in ("max_pages", "n", "frame_cap")})
    o = _refused(_transcode(metas, pages, refs, dtype, **kw))
    assert perr is not None, "the pages call accepted what the transcode refused"
    assert (o.st.kind, o.st.device_status, o.st.page) == (pst.kind, pst.device_status, pst.page)
    assert o.err.kind == perr.kind and str(o.err) == str(perr)
    return o


def test_front_end_refusals_match_the_pages_call(oracle):
    metas, pages, refs, pieces = _six_pages(oracle)
    _same_failure(metas, pages, refs, max_pages=len(refs), n=len(refs) + 1)
    for field, value, at in (("meta_offset", len(metas), 3), ("page_offset", len(pages), 2), ("page_n", 0, 4), ("page_n", (1 << 24) + 1, 1)):
        bad = refs.copy()
        bad[field][at] = value
        bad[field][at + 1] = value
        o = _same_failure(metas, pages, bad)
        assert o.st.page == at
    o = _same_failure(metas, pages, refs, frame_cap=_frames(refs) - 1)
    assert o.st.frames_needed == _frames(refs)


def test_meta_and_walk_failures_match_the_pages_call(oracle):
    metas, pages, refs, pieces = _six_pages(oracle)
    bad = refs.copy()
    bad["meta_len"][2] -= 1  # the meta parses to another length
    _same_failure(metas, pages, bad)
    bad = refs.copy()
    bad["page_len"][3] //= 2  # the walk runs out of the page
    bad["page_len"][5] //= 2
    o = _same_failure(metas, pages, bad)
    assert o.st.page == 3


def test_pages_no_walker_takes_are_unsupported(oracle):
    metas, pages, refs, pieces = _cold_batch(oracle)
    single = [_transcode(metas, pages, refs[i:i + 1], np.int32) for i in range(len(refs))]
    declined = [i for i, o in enumerate(single) if o.err is not None]
    for i in declined:
        assert single[i].err.kind == "Unsupported" and single[i].st.device_status == 7 and single[i].st.page == 0
    # Lookback (two pages), Conv1 (two pages) and Dict (two refs); the level-12 and the plain pages are taken
    assert len(declined) == 6 and declined[-2:] == [len(refs) - 2, len(refs) - 1], declined
    for seed in range(3):
        order = np.random.default_rng(seed).permutation(len(refs))
        o = _refused(_transcode(metas, pages, refs[order], np.int32))
        lowest = min(k for k, i in enumerate(order) if i in declined)
        assert o.err.kind == "Unsupported" and o.st.page == lowest and f": page {lowest}: neither walker" in str(o.err), o.err
    # a walk failure behind the lowest declined page comes first
    bad = refs.copy()
    fast = [i for i in range(len(refs)) if i not in declined]
    bad["page_len"][fast[-1]] //= 2
    o = _refused(_transcode(metas, pages, bad, np.int32))
    assert o.st.page == fast[-1] and o.err.kind != "Unsupported", o.err


def test_capacities_one_byte_short_and_exact(oracle):
    metas, pages, refs, pieces = _six_pages(oracle)
    o = _ok(_transcode(metas, pages, refs, np.uint64))
    fl, il = o.file_len, o.index_len
    assert (o.st.file_needed, o.st.index_needed) == (fl, il)
    short = _refused(_transcode(metas, pages, refs, np.uint64, dst_cap=fl - 1))
    assert short.err.kind == "Io" and (short.st.file_needed, short.st.index_needed) == (fl, il) and short.st.device_status == 0x118
    assert str(fl) in str(short.err)
    short = _refused(_transcode(metas, pages, refs, np.uint64, index_cap=il - 1))
    assert short.err.kind == "Io" and (short.st.file_needed, short.st.index_needed) == (fl, il) and short.st.device_status == 0x119
    assert str(il) in str(short.err)
    # both short: the file is named first
    assert _refused(_transcode(metas, pages, refs, np.uint64, dst_cap=fl - 1, index_cap=il - 1)).st.device_status == 0x118
    exact = _ok(_transcode(metas, pages, refs, np.uint64, dst_cap=fl, index_cap=il))
    assert exact.file == o.file and exact.index == o.index
    # an index far below the walks' room: still Io, without a size
    tiny = _refused(_transcode(metas, pages, refs, np.uint64, index_cap=64))
    assert tiny.err.kind == "Io" and tiny.st.device_status == 0x119


# ---- sizes

def test_page_sizes_from_1_to_2_24(oracle):
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec, standalone, wrapped

    sizes = [1, 2, 255, 256, 257, 4097, 1 << 18, (1 << 24)]
    x = np.cumsum(np.random.default_rng(8).geometric(0.01, size=sum(sizes))).astype(np.uint64)
    cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(1), paging_spec=PagingSpec.exact_page_sizes(sizes))
    want_file, want_index = standalone.simple_compress_with_index(x, cfg)
    metas, pages, refs = wrapped.compress_chunks(x, cfg)
    assert list(refs["page_n"]) == sizes
    o = _ok(_transcode(metas, pages, refs, np.uint64, dst_cap=len(want_file) + 100, index_cap=len(want_index) + 100))
    assert o.file == want_file and o.index == want_index
    got, err, _ = _files_decode(o, np.uint64, x.size)
    assert err is None
    np.testing.assert_array_equal(got, x)


def test_more_than_1000_small_pages(oracle):
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec, standalone, wrapped

    x = _walk(np.int32, 1100 * 97 + 5, seed=12)
    cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(2), paging_spec=PagingSpec.equal_pages_up_to(97))
    want_file, want_index = standalone.simple_compress_with_index(x, cfg, uniform_type=True)
    metas, pages, refs = wrapped.compress_chunks(x, cfg)
    assert len(refs) > 1000
    o = _ok(_transcode(metas, pages, refs, np.int32, uniform=True))
    assert o.file == want_file and o.index == want_index


@pytest.mark.parametrize("uniform", [False, True])
def test_empty_batch_is_compress_ex_of_nothing(oracle, uniform):
    from pcodec_b200 import standalone

    metas, pages, refs, _ = _six_pages(oracle)
    want_file, want_index = standalone.simple_compress_with_index(np.zeros(0, np.float64), None, uniform_type=uniform)
    o = _ok(_transcode(metas, pages, refs[:0], np.float64, max_pages=4, n=0, uniform=uniform))
    assert o.file == want_file and o.index == want_index and o.st.n_pages == 0 and o.st.n_total == 0
    got, err, _ = _files_decode(o, np.float64, 1)
    assert err is None and got.size == 0


# ---- bit flips

def test_bit_flips_match_the_pages_call(oracle):
    metas, pages, refs, pieces = _six_pages(oracle)
    rng = np.random.default_rng(21)
    total = sum(len(p) for p in pieces)
    seen = set()
    for trial in range(40):
        m, p = bytearray(metas), bytearray(pages)
        if trial % 4 == 0:
            at = int(rng.integers(0, len(m)))
            m[at] ^= 1 << int(rng.integers(0, 8))
        else:
            at = int(rng.integers(0, len(p)))
            p[at] ^= 1 << int(rng.integers(0, 8))
        m, p = bytes(m), bytes(p)
        got_pages, _, perr, pst = _pages_run(m, p, refs, np.uint64)
        o = _transcode(m, p, refs, np.uint64)
        if o.err is not None and o.st.device_status == 7:  # a flipped meta no walker takes: declined, as that page alone is
            _refused(o)
            page = int(o.st.page)
            assert _transcode(m, p, refs[page:page + 1], np.uint64).st.device_status == 7
            seen.add("declined")
            continue
        if o.err is not None:  # the walk's verdict: the pages call names the same page with the same kind
            _refused(o)
            assert perr is not None and (o.st.kind, o.st.device_status, o.st.page) == (pst.kind, pst.device_status, pst.page), (o.err, perr)
            seen.add("walk")
            continue
        _ok(o)
        got, ferr, fst = _files_decode(o, np.uint64, total)
        if perr is None:
            assert ferr is None, ferr
            np.testing.assert_array_equal(got, got_pages[:total])
            seen.add("ok")
        else:  # the walk passed; the files call's decode names chunk i for page i with the pages call's kind
            assert ferr is not None and ferr.kind == perr.kind and (fst.chunk, fst.device_status) == (pst.page, pst.device_status), (ferr, perr)
            seen.add("decode")
    assert "walk" in seen and ("ok" in seen or "decode" in seen), seen


# ---- graphs

def test_graph_transcode_then_filter_replays_new_refs_counts_and_bounds(oracle):
    import torch

    from pcodec_b200 import standalone, wrapped

    batches = [_six_pages(oracle)]
    xs = [_walk(np.uint64, 2500 + 300 * k, seed=90 + k) for k in range(5)]
    batches.append(_container([(x, _cfgs(oracle, mode="classic", order=k % 3, max_page_n=1024)[1]) for k, x in enumerate(xs)]))
    metas_cap = max(len(b[0]) for b in batches) + 64
    pages_cap = max(len(b[1]) for b in batches) + 64
    mp = max(len(b[2]) for b in batches) + 3
    rows = 2 * sum(sum(len(p) for p in b[3]) for b in batches)
    frame_cap = 4 * (metas_cap * mp + pages_cap)
    t = wrapped.AsyncPagesToFile(np.uint64, metas_cap, pages_cap, mp, 4 * (pages_cap + metas_cap * mp) + 4096, 64 + 32 * mp + 24 * rows // 256 + 32 * mp,
                                 frame_cap)
    f = standalone.AsyncFilesFilter(**t.files_args(), rows_cap=rows, out_cap=rows)
    dm = torch.zeros(metas_cap, dtype=torch.uint8, device="cuda")
    dp = torch.zeros(pages_cap, dtype=torch.uint8, device="cuda")
    dr = torch.zeros((mp, 5), dtype=torch.int64, device="cuda")
    nt = torch.zeros(1, dtype=torch.int64, device="cuda")
    iv = torch.zeros(2, dtype=torch.int64, device="cuda")
    vals = torch.zeros(rows, dtype=torch.uint64, device="cuda")
    pos = torch.zeros(rows, dtype=torch.int64, device="cuda")
    nm = torch.zeros(1, dtype=torch.int64, device="cuda")

    def load(k, order, lo, hi):
        metas, pages, refs, pieces = batches[k]
        dm[: len(metas)].copy_(torch.frombuffer(bytearray(metas), dtype=torch.uint8))
        dp[: len(pages)].copy_(torch.frombuffer(bytearray(pages), dtype=torch.uint8))
        dr.copy_(_refs_dev(refs[order], mp))
        nt.fill_(len(order))
        iv.copy_(torch.from_numpy(wrapped.pack_interval(lo, hi, np.uint64)))
        return np.concatenate([pieces[i] for i in order]) if order else np.zeros(0, np.uint64)

    def step():
        t(dm, dp, dr, nt)
        f(t.file, t.index, t.file_ref, t.n_files, iv, vals, pos, nm)

    load(0, [0, 1], 0, 1)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    n0, n1 = len(batches[0][2]), len(batches[1][2])
    for k, order, qlo, qhi in [(0, list(range(n0)), 0.1, 0.9), (1, list(range(n1))[::-1], 0.0, 0.5), (0, [], 0.0, 1.0), (1, [3, 3, 0], 0.5, 0.5),
                               (0, [2, 0, 4], 0.9, 1.0)]:
        probe = load(k, order, 0, 0)
        srt = np.sort(probe)
        lo, hi = (srt[int(qlo * (srt.size - 1))], srt[int(qhi * (srt.size - 1))]) if order else (np.uint64(0), np.uint64(5))
        x = load(k, order, lo, hi)
        g.replay()
        torch.cuda.synchronize()
        fl, il = t.result()
        assert t.file_ref.cpu().numpy().reshape(-1).tolist() == [0, fl, 0, il]
        got = f.result()
        want = np.nonzero((x >= lo) & (x <= hi))[0]
        assert got == want.size
        np.testing.assert_array_equal(pos.cpu().numpy()[:got], want)
        np.testing.assert_array_equal(vals.cpu().numpy()[:got], x[want])


def test_graph_compress_then_transcode_then_decode(oracle):
    import torch

    from pcodec_b200 import standalone, wrapped

    cfg, _ = _cfgs(oracle, mode="classic", order=1, max_page_n=3000)
    max_n = 20000
    comp = wrapped.AsyncChunksCompressor(np.int64, cfg, 1, max_n, max_n)
    t = wrapped.AsyncPagesToFile(np.int64, comp.metas_cap, comp.pages_cap, comp.max_chunks, comp.metas_cap + comp.pages_cap + 64,
                                 64 + 64 * comp.max_chunks + 24 * max_n // 256 + 64)
    d = standalone.AsyncFilesDecompressor(**t.files_args(), dst_cap=max_n)
    nums = torch.zeros(max_n, dtype=torch.int64, device="cuda")
    ns = torch.zeros(1, dtype=torch.int64, device="cuda")
    one = torch.ones(1, dtype=torch.int64, device="cuda")
    metas = torch.zeros(comp.metas_cap, dtype=torch.uint8, device="cuda")
    pages = torch.zeros(comp.pages_cap, dtype=torch.uint8, device="cuda")
    refs = torch.zeros((comp.max_chunks, 5), dtype=torch.int64, device="cuda")
    first = torch.zeros(2, dtype=torch.int64, device="cuda")
    dst = torch.zeros(max_n, dtype=torch.int64, device="cuda")
    file_ns = torch.zeros(1, dtype=torch.int64, device="cuda")

    def step():
        comp(nums, ns, one, metas, pages, refs, first)
        t(metas, pages, refs, first[1:2])
        d(t.file, t.index, t.file_ref, t.n_files, dst, file_ns)

    ns.fill_(100)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    for n, seed in ((max_n, 1), (1, 2), (7777, 3), (0, 4), (3001, 5)):
        x = _walk(np.int64, n, seed=seed) if n else np.zeros(0, np.int64)
        nums[:n].copy_(torch.from_numpy(x))
        ns.fill_(n)
        g.replay()
        torch.cuda.synchronize()
        comp.result()
        fl, il = t.result()
        assert d.result() == n
        np.testing.assert_array_equal(dst.cpu().numpy()[:n], x)
        want_file, want_index = standalone.simple_compress_with_index(x, cfg)
        assert t.file.cpu().numpy().tobytes()[:fl] == want_file and t.index.cpu().numpy().tobytes()[:il] == want_index
