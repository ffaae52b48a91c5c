"""Asynchronous batches of wrapped pages on the GPU (pco_b200_decompress_pages_async, wrapped.AsyncPagesDecompressor): every batch is
compared with the blocking pco_b200_decompress_pages and with the input, and every refusal with the blocking call's kind and page."""
import ctypes as C

import numpy as np
import pytest

from tests.golden_generators import bits_view
from tests.test_gpu_encode import _cfgs, _walk
from tests.test_gpu_wrapped_batch import _container, _data, _mixed_chunks, _shuffled, _six_pages, _standalone_dict_chunk

pytestmark = pytest.mark.gpu

SENTINEL = 0x5A
KERNELS = ["ap_pages_kernel", "ap_scan_kernel", "ap_place_kernel", "frame_pages_kernel", "walk_kernel", "ap_route_kernel", "ap_rewalk_kernel",
           "fused_narrow_kernel", "symwalk_kernel", "decode_kernel", "ap_cold_kernel", "ap_finish_kernel"]


def _dev(b, cap=None):
    import torch

    buf = bytearray(b) + bytearray(max((cap or 0) - len(b), 0))
    return torch.frombuffer(buf + bytearray(1), dtype=torch.uint8).cuda()  # one spare byte: an empty buffer is still a pointer


def _refs_dev(refs, max_pages):
    import torch

    t = torch.zeros((max_pages, 5), dtype=torch.int64)
    r = np.asarray(refs)
    for i, name in enumerate(("meta_offset", "meta_len", "page_offset", "page_len", "page_n")):
        t[: len(r), i] = torch.from_numpy(r[name].astype(np.int64))
    return t.cuda()


def _sync(metas, pages, refs, dtype):
    """(numbers, None) or (None, PcoError) of the blocking call."""
    from pcodec_b200 import PcoError, wrapped

    try:
        return wrapped.decompress_pages(metas, pages, refs, dtype), None
    except PcoError as e:
        return None, e


def _run(metas, pages, refs, dtype, max_pages=None, dst_cap=None, frame_cap=-1, n=None, same_buffer=False):
    """The asynchronous call over host bytes copied to the device; returns (dst as numpy, its total, PcoError or None, status).
    frame_cap -1 is room for every frame twice over; None is the decompressor's default."""
    import torch

    from pcodec_b200 import PcoError, wrapped
    from pcodec_b200.wrapped import _torch_dtypes

    total = int(np.asarray(refs)["page_n"].sum()) if len(refs) else 0
    max_pages = max_pages or max(len(refs), 1)
    dst_cap = total if dst_cap is None else dst_cap
    if frame_cap == -1:
        frame_cap = 2 * (len(metas) + len(pages)) + 32 * max_pages
    if same_buffer:
        dm = dp = _dev(metas)
    else:
        dm, dp = _dev(metas), _dev(pages)
    dec = wrapped.AsyncPagesDecompressor(dtype, len(metas), len(pages), max_pages, dst_cap, frame_cap)
    dst = torch.full(((max(dst_cap, 1) + 64) * np.dtype(dtype).itemsize,), SENTINEL, dtype=torch.uint8).cuda()
    dst = dst.view(_torch_dtypes()[np.dtype(dtype)])
    nt = torch.tensor([len(refs) if n is None else n], dtype=torch.int64).cuda()
    dec(dm, dp, _refs_dev(refs, max_pages), nt, dst)
    st = dec.status_record()
    try:
        nw, err = dec.result(), None
    except PcoError as e:
        nw, err = 0, e
    return dst.cpu().numpy(), nw, err, st


def _check(metas, pages, refs, pieces, dtype, **kw):
    got, nw, err, st = _run(metas, pages, refs, dtype, **kw)
    want, serr = _sync(metas, pages, refs, dtype)
    assert serr is None and err is None, (serr, err)
    total = sum(len(p) for p in pieces)
    assert nw == total == st.n_written and st.page == (1 << 64) - 1
    np.testing.assert_array_equal(bits_view(got[:total]), bits_view(want))
    if pieces:
        np.testing.assert_array_equal(bits_view(got[:total]), bits_view(np.concatenate(pieces)))
    assert (got.view(np.uint8)[total * got.itemsize:] == SENTINEL).all(), "written past the pages' numbers"
    return got[:total]


@pytest.mark.parametrize("dtype", [np.uint8, np.int8, np.uint16, np.int16, np.float16, np.uint32, np.int32, np.float32, np.uint64, np.int64, np.float64])
def test_mixed_batch(oracle, dtype):
    metas, pages, refs, pieces = _container(_mixed_chunks(oracle, dtype))
    refs, pieces = _shuffled(refs, pieces, seed=int(np.dtype(dtype).num))
    # the shuffled batch repeats a page: the default frame_cap does not fit it, an exact one does
    frames = int(sum((4 + r["meta_len"] + r["page_len"] + 15) // 16 * 16 for r in refs))
    _check(metas, pages, refs, pieces, dtype, frame_cap=frames)
    # metas and pages in one buffer
    both = pages + metas
    refs2 = refs.copy()
    refs2["meta_offset"] += len(pages)
    _check(both, both, refs2, pieces, dtype, frame_cap=frames, same_buffer=True)


@pytest.mark.parametrize("dtype,order", [(np.uint32, 0), (np.int64, 1), (np.float32, 2), (np.uint16, 7), (np.float64, 7), (np.int8, 7)])
def test_delta_orders(oracle, dtype, order):
    chunks = []
    for k, mode in enumerate(["classic", "classic", "int_mult" if np.dtype(dtype).kind != "f" else "float_quant"]):
        x = _data(dtype, mode, 3000 + 1111 * k, seed=order * 10 + k)
        _, ocfg = _cfgs(oracle, mode=mode, order=order, k=13 if np.dtype(dtype).itemsize > 2 else 5, max_page_n=1500 if mode == "classic" else 0)
        chunks.append((x, ocfg))
    if np.dtype(dtype).kind == "f" and np.dtype(dtype).itemsize > 2:
        x = _data(dtype, "float_mult", 2500, seed=order)
        chunks.append((x, _cfgs(oracle, mode="float_mult", order=order)[1]))
    metas, pages, refs, pieces = _container(chunks)
    _check(metas, pages, refs, pieces, dtype)


def _cold_batch(oracle):
    O = oracle
    rng = np.random.default_rng(11)
    motif = rng.integers(0, 1 << 14, size=97)
    lookback = np.tile(motif, 60)[:5000].astype(np.int32)
    dict_nums = np.array([3, 77, 200, 5, 131], dtype=np.int32)[rng.integers(0, 5, size=7000)]
    i = np.arange(6000)
    conv1 = (2000 * np.sin(i / 30.0) + 300 * np.cos(i / 7.0)).astype(np.int32)
    centers = np.sort(rng.integers(0, 1 << 30, size=600))
    p = rng.lognormal(0.0, 1.0, size=centers.size)
    wide = (centers[rng.choice(centers.size, size=1 << 17, p=p / p.sum())] + rng.integers(0, 16, size=1 << 17)).astype(np.int32)
    fast = _walk(np.int32, 3000, seed=4)
    chunks = [
        (fast, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=1)),
        (lookback, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_LOOKBACK, max_page_n=1 << 12)),
        (fast[:700], O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_NOOP)),
        (fast[:2999], O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=2)),
        (conv1, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONV1, delta_order=2, max_page_n=1 << 12)),
        (wide, O.make_config(level=12, mode=O.MODE_CLASSIC, delta=O.DELTA_NOOP)),
        (fast[5:], O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_NOOP)),
    ]
    metas, pages, refs, pieces = _container(chunks)
    d_meta, d_page = _standalone_dict_chunk(oracle.simple_compress(dict_nums, O.make_config(mode=O.MODE_DICT, delta=O.DELTA_NOOP)))
    refs = np.concatenate([refs, np.array([(len(metas), len(d_meta), len(pages), len(d_page), dict_nums.size)] * 2, dtype=refs.dtype)])
    pieces += [dict_nums, dict_nums]
    return metas + d_meta, pages + d_page, refs, pieces


def test_cold_pages_interleaved_with_fast_ones(oracle):
    from pcodec_b200 import _lib

    metas, pages, refs, pieces = _cold_batch(oracle)
    refs, pieces = _shuffled(refs, pieces, seed=5)
    _check(metas, pages, refs, pieces, np.int32)
    L = _lib.lib()
    L.pco_b200_profile_enable(1)
    try:
        assert _run(metas, pages, refs, np.int32)[2] is None
        buf = C.create_string_buffer(8192)
        L.pco_b200_profile_last(buf, C.c_size_t(len(buf)))
    finally:
        L.pco_b200_profile_enable(0)
    prof = buf.value.decode()
    at = [prof.find(k) for k in KERNELS]
    assert all(a >= 0 for a in at) and at == sorted(at), prof


def test_f16_float_mult_pages_beside_fast_ones(oracle):
    O = oracle
    fm = (np.round(np.random.default_rng(4).normal(size=4000) * 40) * 0.25).astype(np.float16)
    plain = _walk(np.float16, 3000, seed=9)
    chunks = [(plain, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=1)),
              (fm, O.make_config(mode=O.MODE_FLOAT_MULT, float_mult_base=0.25, delta=O.DELTA_CONSECUTIVE, delta_order=1, max_page_n=1500)),
              (plain[:999], O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_NOOP))]
    metas, pages, refs, pieces = _container(chunks)
    _check(metas, pages, refs, pieces, np.float16)


def test_page_counts_zero_one_and_max(oracle):
    metas, pages, refs, pieces = _six_pages(oracle)
    for n in (0, 1, len(refs)):
        _check(metas, pages, refs[:n], pieces[:n], np.uint64, max_pages=len(refs) + 3)
    # the count read on the device, below the refs the tensor holds
    got, nw, err, st = _run(metas, pages, refs, np.uint64, max_pages=len(refs), n=2, dst_cap=sum(len(p) for p in pieces))
    assert err is None and nw == len(pieces[0]) + len(pieces[1]) and st.n_pages == 2
    np.testing.assert_array_equal(got[:nw], np.concatenate(pieces[:2]))


def test_full_size_pages(oracle):
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec, wrapped

    rng = np.random.default_rng(2)
    nums = np.cumsum(rng.geometric(0.001, size=64 << 18)).astype(np.uint64)
    cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(1), paging_spec=PagingSpec.equal_pages_up_to(1 << 18))
    metas, pages, refs = wrapped.compress_chunks(nums, cfg)
    assert len(refs) == 64
    got = _check(metas, pages, refs, [nums], np.uint64, frame_cap=None)  # the default frame_cap fits compress_chunks' layout
    np.testing.assert_array_equal(got, nums)


class _Batch:
    """Device buffers a captured call reads: metas, pages, refs and the count are refilled in place between replays."""

    def __init__(self, dtype, metas_cap, pages_cap, max_pages, dst_cap, frame_cap=None):
        import torch

        from pcodec_b200 import wrapped
        from pcodec_b200.wrapped import _torch_dtypes

        if frame_cap is None:  # room for shared metas and repeated pages
            frame_cap = 2 * (metas_cap + pages_cap) + 32 * max_pages
        self.dec = wrapped.AsyncPagesDecompressor(dtype, metas_cap, pages_cap, max_pages, dst_cap, frame_cap)
        self.metas = torch.zeros(metas_cap, dtype=torch.uint8, device="cuda")
        self.pages = torch.zeros(pages_cap, dtype=torch.uint8, device="cuda")
        self.refs = torch.zeros((max_pages, 5), dtype=torch.int64, device="cuda")
        self.n = torch.zeros(1, dtype=torch.int64, device="cuda")
        self.dst = torch.zeros(dst_cap, dtype=_torch_dtypes()[np.dtype(dtype)], device="cuda")
        self.max_pages = max_pages

    def load(self, metas, pages, refs):
        import torch

        self.metas[: len(metas)].copy_(torch.frombuffer(bytearray(metas) + bytearray(1), dtype=torch.uint8)[: len(metas)])
        self.pages[: len(pages)].copy_(torch.frombuffer(bytearray(pages) + bytearray(1), dtype=torch.uint8)[: len(pages)])
        self.refs.copy_(_refs_dev(refs, self.max_pages))
        self.n.fill_(len(refs))

    def call(self):
        self.dec(self.metas, self.pages, self.refs, self.n, self.dst)


def test_graph_replays_new_refs_count_and_bytes(oracle):
    import torch

    from pcodec_b200 import _lib

    batches = [_six_pages(oracle), _container(_mixed_chunks(oracle, np.uint64))]
    b = _Batch(np.uint64, 1 << 14, 1 << 22, 32, 1 << 20, frame_cap=1 << 23)
    b.load(*batches[0][:3])
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        b.call()
    plans = [(0, [0, 1, 2, 3, 4, 5, 6, 7]), (1, [5, 5, 0]), (0, []), (1, [3, 9, 1]), (0, [7, 0, 4, 1, 3, 5, 0, 0])]
    for step, (k, order) in enumerate(plans):
        metas, pages, refs, pieces = batches[k]
        sel = refs[order] if order else refs[:0]
        b.load(metas, pages, sel)
        if step == 2:
            _lib.lib().pco_b200_thread_release()  # the library's per-thread scratch is gone; the graph refers to none of it
        g.replay()
        torch.cuda.synchronize()
        nw = b.dec.result()
        want = [pieces[i] for i in order]
        assert nw == sum(len(p) for p in want)
        if want:
            got = b.dst[:nw].cpu().numpy()
            np.testing.assert_array_equal(got, np.concatenate(want))
            np.testing.assert_array_equal(got, _sync(metas, pages, sel, np.uint64)[0])


def test_subset_picked_on_the_device(oracle):
    """A pruned scan: a torch kernel keeps the pages whose first number passes a predicate and writes their refs and count."""
    import torch

    metas, pages, refs, pieces = _container(_mixed_chunks(oracle, np.uint64))
    b = _Batch(np.uint64, len(metas), len(pages), len(refs), sum(len(p) for p in pieces))
    b.load(metas, pages, refs)
    firsts = torch.tensor([int(p[0]) % 3 for p in pieces], device="cuda")
    all_refs = b.refs.clone()
    keep = firsts != 1
    kept = all_refs[keep]
    b.refs.zero_()
    b.refs[: kept.shape[0]].copy_(kept)
    b.n.copy_(keep.sum().reshape(1))
    b.call()
    nw = b.dec.result()
    idx = [i for i in range(len(pieces)) if int(pieces[i][0]) % 3 != 1]
    assert 0 < len(idx) < len(pieces)
    np.testing.assert_array_equal(b.dst[:nw].cpu().numpy(), np.concatenate([pieces[i] for i in idx]))
    np.testing.assert_array_equal(b.dst[:nw].cpu().numpy(), _sync(metas, pages, refs[idx], np.uint64)[0])


def test_two_streams_two_workspaces(oracle):
    import torch

    sets = [_six_pages(oracle), _container(_mixed_chunks(oracle, np.uint64))]
    bs = []
    for metas, pages, refs, pieces in sets:
        b = _Batch(np.uint64, len(metas), len(pages), len(refs), sum(len(p) for p in pieces))
        b.load(metas, pages, refs)
        bs.append(b)
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for _ in range(3):
        for b, s in zip(bs, streams):
            with torch.cuda.stream(s):
                b.call()
    torch.cuda.synchronize()
    for b, (metas, pages, refs, pieces) in zip(bs, sets):
        nw = b.dec.result()
        np.testing.assert_array_equal(b.dst[:nw].cpu().numpy(), np.concatenate(pieces))


def _same_failure(metas, pages, refs, dtype=np.uint64, **kw):
    """The asynchronous call fails as the blocking one does (kind and page), and writes nothing at or behind the failing page's slot."""
    got, nw, err, st = _run(metas, pages, refs, dtype, **kw)
    _, serr = _sync(metas, pages, refs, dtype)
    assert serr is not None and err is not None, (serr, err)
    assert err.kind == serr.kind, (err, serr)
    if serr.message.startswith("page "):
        assert err.message.split(":")[0] == serr.message.split(":")[0], (err, serr)
    if st.page != (1 << 64) - 1:
        at = int(np.asarray(refs)["page_n"][: st.page].sum()) * got.itemsize
        assert (got.view(np.uint8)[at:] == SENTINEL).all(), "written at or behind the failing page"
    return err, st


def test_refusals_before_the_device(oracle):
    metas, pages, refs, pieces = _six_pages(oracle)
    total = sum(len(p) for p in pieces)
    # more pages than max_pages
    _, _, err, st = _run(metas, pages, refs, np.uint64, max_pages=len(refs), n=len(refs) + 1, dst_cap=total)
    assert err.kind == "InvalidArgument" and "*n_pages is" in err.message and st.device_status == 0x11a and st.n_pages == len(refs) + 1
    for field, value, code in [("meta_offset", len(metas), 0x11b), ("page_len", len(pages) + 1, 0x11c), ("page_n", 0, 0x11d), ("page_n", (1 << 24) + 1, 0x11d)]:
        bad = refs.copy()
        bad[4][field] = value
        bad[6]["page_offset"] = len(pages)  # a later refusal does not win
        err, st = _same_failure(metas, pages, bad, dst_cap=total + (1 << 25))
        assert st.page == 4 and st.device_status == code, (field, err)
    # the running count passes dst_cap at page 3: the blocking call's kind (it names no page), and the page named
    got, _, err, st = _run(metas, pages, refs, np.uint64, dst_cap=int(refs["page_n"][:3].sum()) + 1)
    assert err.kind == "InvalidArgument" and st.page == 3 and st.device_status == 0x11e and "page 3: " in err.message, err
    assert (got.view(np.uint8) == SENTINEL).all()


def test_refusals_on_the_device(oracle):
    metas, pages, refs, pieces = _six_pages(oracle)
    # a page cut short, whose walk runs into the next frame: the re-walk over its own frame gives the kind
    for cut in (1, int(refs[3]["page_len"]) // 2):
        bad = refs.copy()
        bad[3]["page_len"] -= cut
        bad[5]["meta_len"] += 1
        err, st = _same_failure(metas, pages, bad)
        assert err.kind == "InsufficientData" and st.page == 3, (cut, err)
    # a wrong meta_len
    for delta in (1, -1):
        bad = refs.copy()
        bad[2]["meta_len"] = int(bad[2]["meta_len"]) + delta
        err, st = _same_failure(metas, pages, bad)
        assert err.kind == "InvalidArgument" and st.page == 2, err
    # an unknown mode: the meta's first 4 bits
    buf = bytearray(metas)
    buf[int(refs[1]["meta_offset"])] = (buf[int(refs[1]["meta_offset"])] & 0xF0) | 0xE
    err, st = _same_failure(bytes(buf), pages, refs)
    assert err.kind == "Corruption" and st.page == 1, err


def test_bit_flips_match_the_blocking_call(oracle):
    metas, pages, refs, pieces = _six_pages(oracle)
    rng = np.random.default_rng(1)
    for trial in range(24):
        k = int(rng.integers(0, len(refs)))
        if trial % 2:
            buf = bytearray(pages)
            buf[int(refs[k]["page_offset"] + rng.integers(0, refs[k]["page_len"]))] ^= 1 << int(rng.integers(0, 8))
            m, p = metas, bytes(buf)
        else:
            buf = bytearray(metas)
            buf[int(refs[k]["meta_offset"] + rng.integers(0, refs[k]["meta_len"]))] ^= 1 << int(rng.integers(0, 8))
            m, p = bytes(buf), pages
        want, serr = _sync(m, p, refs, np.uint64)
        got, nw, err, st = _run(m, p, refs, np.uint64)
        if serr is None:
            assert err is None, err
            np.testing.assert_array_equal(got[:nw], want)
        else:
            assert err is not None and err.kind == serr.kind and err.message.split(":")[0] == serr.message.split(":")[0], (trial, err, serr)


def test_frame_cap_refusal_reports_the_bytes_needed(oracle):
    metas, pages, refs, pieces = _six_pages(oracle)
    frames = int(sum((4 + r["meta_len"] + r["page_len"] + 15) // 16 * 16 for r in refs))
    _check(metas, pages, refs, pieces, np.uint64, frame_cap=frames)
    got, nw, err, st = _run(metas, pages, refs, np.uint64, frame_cap=frames - 1)
    assert err.kind == "Io" and st.device_status == 0x11f and st.frames_needed == frames and str(frames) in err.message
    assert (got.view(np.uint8) == SENTINEL).all()


def test_lookback_window_above_2_16_is_unsupported(oracle):
    O = oracle
    rng = np.random.default_rng(3)
    x = np.tile(rng.integers(0, 1 << 14, size=97), 60)[:5000].astype(np.int32)
    metas, pages, refs, pieces = _container([(x, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_LOOKBACK))])
    # Classic: mode (4 bits), delta variant 2 (4 bits), then window_n_log - 1 (5 bits): 2^17
    b = bytearray(metas)
    bits = int.from_bytes(b[:4], "little")
    assert (bits >> 4) & 15 == 2, "Lookback"
    bits = (bits & ~(31 << 8)) | (16 << 8)
    b[:4] = bits.to_bytes(4, "little")
    want, serr = _sync(bytes(b), pages, refs, np.int32)
    assert serr is None
    np.testing.assert_array_equal(want, x)
    got, nw, err, st = _run(bytes(b), pages, refs, np.int32)
    assert err is not None and err.kind == "Unsupported" and st.page == 0, err


def test_captured_call_records_no_spans(oracle):
    import torch

    from pcodec_b200 import _lib

    metas, pages, refs, pieces = _six_pages(oracle)
    b = _Batch(np.uint64, len(metas), len(pages), len(refs), sum(len(p) for p in pieces))
    b.load(metas, pages, refs)
    torch.cuda.synchronize()
    L = _lib.lib()
    L.pco_b200_profile_enable(1)
    try:
        _sync(metas, pages, refs, np.uint64)  # the last spans recorded are the blocking call's
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            b.call()
        buf = C.create_string_buffer(8192)
        L.pco_b200_profile_last(buf, C.c_size_t(len(buf)))
    finally:
        L.pco_b200_profile_enable(0)
    assert "ap_pages_kernel" not in buf.value.decode()
    g.replay()
    torch.cuda.synchronize()
    np.testing.assert_array_equal(b.dst[: b.dec.result()].cpu().numpy(), np.concatenate(pieces))
