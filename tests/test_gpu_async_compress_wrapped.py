"""Asynchronous batch compress into wrapped chunks (pco_b200_compress_wrapped_async, wrapped.AsyncChunksCompressor): metas and pages (with
guard zones behind them), refs and first_chunk equal a loop of pco_b200_compress_wrapped over the arrays one by one, bit for bit, and the
pages decode back to the input - for every number type, the explicit modes, delta orders, levels, array sizes on both sides of batch and
page boundaries, chunks on every unoptimized_bins_log in one pass, inside a CUDA graph replayed over sizes a kernel wrote, on concurrent
streams, and chained with AsyncPagesDecompressor in one graph.  Refusals write nothing where the contract forbids it."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DTYPES = [np.uint8, np.int8, np.uint16, np.int16, np.float16, np.uint32, np.int32, np.float32, np.uint64, np.int64, np.float64]
GUARD = 4096
SENT = 0xA5
# at level 8 these sizes give every unoptimized_bins_log from 4 to 8: 1..63 -> 4, 64..255 -> 5, 256..1023 -> 6, 1024..4095 -> 7, 4096.. -> 8
ALL_BINS = [1, 20, 64, 300, 1500, 4000, 5000, 100, 2048, 0, 4095, 4096]


@pytest.fixture(scope="module")
def wr():
    from pcodec_b200 import wrapped

    return wrapped


def _walk(dtype, n, seed, scale=0.05):
    rng = np.random.default_rng(seed)
    if np.dtype(dtype).kind == "f":
        x = np.cumsum(rng.normal(size=n)).astype(dtype)
        if n > 5:
            x[3], x[4], x[5] = np.nan, -np.inf, -0.0
        return x
    steps = rng.geometric(scale, size=n).astype(np.int64) - int(1 / scale) // 2
    return np.cumsum(steps).astype(np.uint64).astype(np.dtype(dtype).str.replace("i", "u")).view(dtype)


def _cfg(order=0, page=1 << 14, level=8, mode="classic", base=0.01, ibase=8, k=13):
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec

    ms = {"classic": ModeSpec.classic(), "float_mult": ModeSpec.try_float_mult(base), "int_mult": ModeSpec.try_int_mult(ibase),
          "float_quant": ModeSpec.try_float_quant(k)}[mode]
    ds = DeltaSpec.try_consecutive(order) if order else DeltaSpec.no_op()
    return ChunkConfig(compression_level=level, mode_spec=ms, delta_spec=ds, paging_spec=PagingSpec.equal_pages_up_to(page), enable_8_bit=True)


def _tdtype(dtype):
    from pcodec_b200.wrapped import _torch_dtypes

    return _torch_dtypes()[np.dtype(dtype)]


class Bufs:
    """Device buffers of one compressor, with sentinel guard zones behind metas and pages and sentinels in refs and first_chunk."""

    def __init__(self, comp, dtype):
        import torch

        self.comp = comp
        self.nums = torch.zeros(max(comp._plan.nums_cap, 1), dtype=_tdtype(dtype), device="cuda")
        self.array_ns = torch.full((comp.max_arrays,), 7777, dtype=torch.int64, device="cuda")  # slots past n_arrays are never read
        self.n_arrays = torch.zeros(1, dtype=torch.int64, device="cuda")
        self.metas_full = torch.full((comp.metas_cap + GUARD,), SENT, dtype=torch.uint8, device="cuda")
        self.metas = self.metas_full[:comp.metas_cap]
        self.pages_full = torch.full((comp.pages_cap + GUARD,), SENT, dtype=torch.uint8, device="cuda")
        self.pages = self.pages_full[:comp.pages_cap]
        self.refs_full = torch.full((comp.max_chunks + 8, 5), -1, dtype=torch.int64, device="cuda")
        self.refs = self.refs_full[:comp.max_chunks]
        self.first_full = torch.full((comp.max_arrays + 9,), -1, dtype=torch.int64, device="cuda")
        self.first = self.first_full[:comp.max_arrays + 1]

    def reset(self):
        self.metas_full.fill_(SENT)
        self.pages_full.fill_(SENT)
        self.refs_full.fill_(-1)
        self.first_full.fill_(-1)

    def load(self, xs):
        import torch

        n = sum(len(x) for x in xs)
        if n:
            self.nums[:n].copy_(torch.from_numpy(np.concatenate(xs)).cuda())
        if xs:
            self.array_ns[:len(xs)].copy_(torch.tensor([len(x) for x in xs], dtype=torch.int64))
        self.n_arrays.fill_(len(xs))

    def run(self):
        self.comp(self.nums, self.array_ns, self.n_arrays, self.metas, self.pages, self.refs, self.first)

    def untouched(self, refs=True):
        ok = (self.metas_full.cpu().numpy() == SENT).all() and (self.pages_full.cpu().numpy() == SENT).all()
        if refs:
            ok = ok and (self.refs_full.cpu().numpy() == -1).all() and (self.first_full.cpu().numpy() == -1).all()
        return ok


def _reference(wr, xs, cfg):
    """The per-array compress_wrapped loop on device buffers: metas, pages, refs (shifted by the arrays before) and first_chunk."""
    import torch

    metas, pages, refs, first = [], [], [], [0]
    mo = po = 0
    for x in xs:
        if len(x):
            m, p, r = wr.compress_chunks(torch.from_numpy(x).cuda(), cfg)
            r = r.copy()
            r["meta_offset"] += mo
            r["page_offset"] += po
            metas.append(m.cpu().numpy())
            pages.append(p.cpu().numpy())
            refs.append(r)
            mo += m.numel()
            po += p.numel()
        first.append(first[-1] + (len(refs[-1]) if len(x) else 0))
    cat = (lambda a: np.concatenate(a) if a else np.zeros(0, np.uint8))
    r = np.concatenate(refs) if refs else np.zeros(0, dtype=wr.PAGE_REF)
    return cat(metas), cat(pages), r, first


def _ref_rows(r):
    return np.stack([r[f] for f in ("meta_offset", "meta_len", "page_offset", "page_len", "page_n")], axis=1).astype(np.int64).reshape(-1, 5)


def _check(wr, b, xs, dtype, cfg, decode=True):
    """The call's output against the compress_wrapped loop, the guard zones, and the decode."""
    ml, pl, nc = b.comp.result()
    metas, pages, refs, first = _reference(wr, xs, cfg)
    assert (ml, pl, nc) == (metas.size, pages.size, len(refs))
    mf, pf = b.metas_full.cpu().numpy(), b.pages_full.cpu().numpy()
    assert np.array_equal(mf[:ml], metas) and np.array_equal(pf[:pl], pages)
    assert (mf[ml:] == SENT).all() and (pf[pl:] == SENT).all()  # nothing behind the batch's bytes
    rf = b.refs_full.cpu().numpy()
    assert np.array_equal(rf[:nc], _ref_rows(refs))
    assert (rf[nc:] == -1).all()  # pad chunk slots leave no trace
    ff = b.first_full.cpu().numpy()
    assert ff[:len(xs) + 1].tolist() == first
    assert (ff[len(xs) + 1:] == -1).all()
    if decode and nc:
        back = wr.decompress_pages(b.metas[:ml], b.pages[:pl], refs, dtype).cpu().numpy()
        assert np.array_equal(back.view(np.uint8), np.concatenate(xs).view(np.uint8))
    return ml, pl, nc


def _comp(wr, dtype, cfg, max_arrays=16, nums_cap=1 << 16, max_array_n=1 << 15, **kw):
    return wr.AsyncChunksCompressor(dtype, cfg, max_arrays, nums_cap, max_array_n, **kw)


def _one(wr, dtype, cfg, sizes, seed=0, data=None, **kw):
    xs = data if data is not None else [_walk(dtype, n, seed + i) for i, n in enumerate(sizes)]
    comp = _comp(wr, dtype, cfg, max_arrays=max(len(sizes), 1), nums_cap=max(sum(sizes), 1), max_array_n=max(max(sizes, default=1), 1), **kw)
    b = Bufs(comp, dtype)
    b.load(xs)
    b.run()
    return _check(wr, b, xs, dtype, cfg)


@pytest.mark.parametrize("dtype", DTYPES)
def test_every_type(wr, dtype):
    _one(wr, dtype, _cfg(order=1, page=4096), [3000, 0, 1, 9000, 257], seed=1)


@pytest.mark.parametrize("dtype,mode", [(np.int64, "int_mult"), (np.uint32, "int_mult"), (np.float32, "float_mult"), (np.float64, "float_mult"),
                                        (np.float32, "float_quant"), (np.float64, "float_quant"), (np.float16, "float_quant")])
def test_modes(wr, dtype, mode):
    sizes = [5000, 700, 64, 1]
    xs = [_walk(dtype, n, 2 + i) for i, n in enumerate(sizes)]
    if mode == "int_mult":
        xs = [(x.astype(np.uint64) // 8 * 8 + 3).astype(dtype) for x in xs]
    if mode == "float_mult":
        xs = [(np.round(np.cumsum(np.random.default_rng(9 + i).normal(size=n)) * 4) * 0.25).astype(dtype) for i, n in enumerate(sizes)]
    _one(wr, dtype, _cfg(mode=mode, k=5, base=0.25 if mode == "float_mult" else 0.01), sizes, data=xs)


@pytest.mark.parametrize("order", range(8))
@pytest.mark.parametrize("level", [0, 3, 8])
def test_orders_and_levels(wr, order, level):
    _one(wr, np.int64, _cfg(order=order, level=level, page=3000), ALL_BINS, seed=3)


@pytest.mark.parametrize("sizes", [[0], [1], [255], [256], [257], [(1 << 18) - 1], [1 << 18], [(1 << 18) + 1], [0, 0, 0],
                                   [(1 << 18) + 1, 1, 255, 0, 257, (1 << 18) - 1]])
def test_array_sizes(wr, sizes):
    _one(wr, np.uint64, _cfg(order=2, page=1 << 18), sizes, seed=5)


def test_arrays_above_max_page_n(wr):
    # 10007 numbers at pages of 1000: 11 chunks with rem != 0
    _one(wr, np.uint32, _cfg(order=1, page=1000), [10007, 999, 1001, 3, 2000], seed=6)


def test_bins_boundaries_in_one_pass(wr):
    # chunks of one batch on every unoptimized_bins_log, and arrays whose chunks straddle a boundary (4096 -> 8 bins_log, 4095 -> 7)
    _one(wr, np.int32, _cfg(order=1, page=4096), ALL_BINS + [8191, 8193, 12287, 63, 64, 255, 256, 1023, 1024], seed=7)


def test_n_arrays_zero_one_and_below_max_arrays(wr):
    cfg = _cfg(order=1, page=2048)
    comp = _comp(wr, np.int16, cfg, max_arrays=64, nums_cap=40000, max_array_n=9000)
    b = Bufs(comp, np.int16)
    b.load([])
    b.run()
    assert comp.result() == (0, 0, 0)
    assert b.untouched(refs=False) and (b.refs_full.cpu().numpy() == -1).all()
    ff = b.first_full.cpu().numpy()
    assert ff[0] == 0 and (ff[1:] == -1).all()  # first_chunk[0] = 0 and nothing else
    st = comp.status_record()
    assert (st.kind, st.n_arrays, st.n_chunks) == (0, 0, 0)
    for sizes in ([5000], [9000, 1, 0, 300]):
        xs = [_walk(np.int16, n, 10 + i) for i, n in enumerate(sizes)]
        b.reset()
        b.load(xs)
        b.run()
        _check(wr, b, xs, np.int16, cfg)


def test_oracle_bytes(wr):
    from oracle import pyoracle

    xs = [np.cumsum(np.random.default_rng(11 + i).geometric(0.01, size=n)).astype(np.uint64) for i, n in enumerate([3000, 1, 70000, 32769])]
    cfg = _cfg(order=1, page=1 << 15)
    comp = _comp(wr, np.uint64, cfg, max_arrays=4, nums_cap=110000, max_array_n=70000)
    b = Bufs(comp, np.uint64)
    b.load(xs)
    b.run()
    ml, pl, nc = _check(wr, b, xs, np.uint64, cfg)
    metas, pages = b.metas[:ml].cpu().numpy().tobytes(), b.pages[:pl].cpu().numpy().tobytes()
    refs = b.refs[:nc].cpu().numpy()
    first = b.first.cpu().numpy()
    for i, x in enumerate(xs):
        start = 0
        for r in refs[first[i]:first[i + 1]]:
            mo, mlen, po, plen, pn = (int(v) for v in r)
            occ = pyoracle.ChunkCompressor(x[start:start + pn], pyoracle.make_config(mode=pyoracle.MODE_CLASSIC, delta=pyoracle.DELTA_CONSECUTIVE,
                                                                                     delta_order=1, exact_pages=[pn]))
            assert metas[mo:mo + mlen] == occ.write_meta() and pages[po:po + plen] == occ.write_page(0)
            start += pn
        assert start == x.size


def test_graph_replay_with_sizes_from_a_kernel(wr):
    """One captured graph: a kernel writes the count and the sizes, the call compresses; replays with new counts, sizes and numbers."""
    import torch

    cfg = _cfg(order=1, page=4096)
    comp = _comp(wr, np.int32, cfg, max_arrays=8, nums_cap=30000, max_array_n=12000)
    b = Bufs(comp, np.int32)
    plan_ns = torch.zeros(9, dtype=torch.int64, device="cuda")  # [count, sizes...], set on the host between replays
    b.run()  # warm up outside the capture
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            b.n_arrays.copy_(plan_ns[:1])
            b.array_ns.copy_(plan_ns[1:] * 1)  # a kernel inside the graph writes the sizes
            b.run()
    rng = np.random.default_rng(12)
    for rep, sizes in enumerate([[100, 12000, 0, 5], [4096], [], [1] * 8, [12000, 12000, 5999]]):
        xs = [_walk(np.int32, n, 100 * rep + i) for i, n in enumerate(sizes)]
        b.reset()
        if xs and sum(sizes):
            b.nums[:sum(sizes)].copy_(torch.from_numpy(np.concatenate(xs)).cuda())
        row = [len(sizes)] + sizes + [int(rng.integers(0, 1 << 20))] * (8 - len(sizes))
        plan_ns.copy_(torch.tensor(row, dtype=torch.int64))
        g.replay()
        torch.cuda.synchronize()
        _check(wr, b, xs, np.int32, cfg)


def test_two_streams_with_their_own_workspaces(wr):
    import torch

    cfg = _cfg(order=2, page=2048)
    sets = [[_walk(np.float32, n, 20 + i) for i, n in enumerate(s)] for s in ([5000, 300, 0], [70, 6000, 6000, 1])]
    comps = [_comp(wr, np.float32, cfg, max_arrays=4, nums_cap=13000, max_array_n=6000) for _ in sets]
    bufs = [Bufs(c, np.float32) for c in comps]
    for b, xs in zip(bufs, sets):
        b.load(xs)
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in sets]
    for _ in range(3):
        for b, st in zip(bufs, streams):
            with torch.cuda.stream(st):
                b.run()
    torch.cuda.synchronize()
    for b, xs in zip(bufs, sets):
        _check(wr, b, xs, np.float32, cfg)


def test_compress_then_async_pages_decompress_in_one_graph(wr):
    import torch

    cfg = _cfg(order=1, page=4096)
    sizes = [3000, 0, 9000, 1, 4096]
    xs = [_walk(np.uint16, n, 30 + i) for i, n in enumerate(sizes)]
    comp = _comp(wr, np.uint16, cfg, max_arrays=6, nums_cap=20000, max_array_n=9000)
    b = Bufs(comp, np.uint16)
    b.load(xs)
    dec = wr.AsyncPagesDecompressor(np.uint16, comp.metas_cap, comp.pages_cap, comp.max_chunks, 20000)
    out = torch.zeros(20000, dtype=_tdtype(np.uint16), device="cuda")
    n_pages = torch.zeros(1, dtype=torch.int64, device="cuda")

    def step():
        b.run()
        n_pages.copy_(b.first.index_select(0, b.n_arrays))  # first_chunk[n_arrays]: the chunks of the batch
        dec(b.metas, b.pages, b.refs, n_pages, out)

    step()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            step()
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert dec.result() == sum(sizes)
    assert np.array_equal(out[:sum(sizes)].cpu().numpy().view(np.uint16), np.concatenate(xs))
    _check(wr, b, xs, np.uint16, cfg, decode=False)


def test_refusals_write_only_the_status(wr):
    import torch

    from pcodec_b200 import PcoError

    cfg = _cfg(order=1, page=4096)
    comp = _comp(wr, np.int64, cfg, max_arrays=4, nums_cap=10000, max_array_n=5000)
    cases = [
        ([100] * 5, 0x10E, None),              # more arrays than max_arrays
        ([100, 5001, 100], 0x116, 1),          # an array above max_array_n
        ([5000, 5000, 1], 0x117, 2),           # the running sum passes nums_cap at array 2
        ([5000, 5000, 1, 5001], 0x117, 2),     # the lowest failing array wins
        ([100, 5001, 5000, 5000], 0x116, 1),
    ]
    for sizes, code, array in cases:
        b = Bufs(comp, np.int64)
        b.array_ns[:min(len(sizes), 4)].copy_(torch.tensor(sizes[:4], dtype=torch.int64))
        b.n_arrays.fill_(len(sizes))
        b.run()
        with pytest.raises(PcoError) as e:
            comp.result()
        st = comp.status_record()
        assert e.value.kind == "InvalidArgument" and st.device_status == code, (sizes, st.device_status)
        assert st.n_arrays == len(sizes) and (st.n_chunks, st.metas_bytes, st.pages_bytes) == (0, 0, 0)
        if array is not None:
            assert st.array == array and e.value.message.startswith(f"array {array}: ")
        assert b.untouched(), sizes


@pytest.mark.parametrize("short", ["metas", "pages"])
def test_caps_one_byte_short(wr, short):
    from pcodec_b200 import PcoError

    cfg = _cfg(order=1, page=4096)
    sizes = [3000, 0, 7000, 2]
    xs = [_walk(np.uint32, n, 40 + i) for i, n in enumerate(sizes)]
    metas, pages, refs, first = _reference(wr, xs, cfg)
    comp = wr.AsyncChunksCompressor(np.uint32, cfg, 4, 10002, 7000, metas_cap=metas.size - (short == "metas"),
                                    pages_cap=pages.size - (short == "pages"))
    b = Bufs(comp, np.uint32)
    b.load(xs)
    b.run()
    with pytest.raises(PcoError) as e:
        comp.result()
    st = comp.status_record()
    assert e.value.kind == "Io" and st.device_status == 0x118
    assert (st.metas_bytes, st.pages_bytes, st.metas_written, st.pages_written, st.n_chunks) == (metas.size, pages.size, 0, 0, len(refs))
    assert f"need {metas.size} meta bytes and {pages.size} page bytes" in e.value.message
    # refs and first_chunk report the layout the batch needs; metas and pages are untouched
    assert np.array_equal(b.refs[:len(refs)].cpu().numpy(), _ref_rows(refs))
    assert b.first[:len(sizes) + 1].cpu().tolist() == first
    assert (b.metas_full.cpu().numpy() == SENT).all() and (b.pages_full.cpu().numpy() == SENT).all()


def test_profiler_spans_outside_a_capture_only(wr):
    import ctypes as C

    import torch

    from pcodec_b200 import _lib

    cfg = _cfg(order=1, page=4096)
    comp = _comp(wr, np.uint32, cfg, max_arrays=4, nums_cap=20000, max_array_n=9000)
    b = Bufs(comp, np.uint32)
    xs = [_walk(np.uint32, n, 50 + i) for i, n in enumerate([9000, 100, 5000])]
    b.load(xs)
    torch.cuda.synchronize()
    L = _lib.lib()

    def last():
        buf = C.create_string_buffer(1 << 16)
        L.pco_b200_profile_last(buf, C.c_size_t(len(buf)))
        return buf.value.decode()

    L.pco_b200_profile_enable(1)
    try:
        b.run()
        prof = last()
        kernels = ["acf_files_kernel", "pack_kernel", "acw_lens_kernel", "acw_scan_kernel", "acw_refs_kernel", "acw_split_kernel", "acw_finish_kernel"]
        at = [prof.find(k) for k in kernels]
        assert all(a >= 0 for a in at) and at == sorted(at), prof
        wr.compress_chunks(torch.from_numpy(xs[1]).cuda(), cfg)  # the last spans recorded are the blocking call's
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                b.run()
        prof = last()
    finally:
        L.pco_b200_profile_enable(0)
    assert "chunk_refs_kernel" in prof and "acw_" not in prof and "acf_" not in prof, prof
    b.reset()
    g.replay()
    torch.cuda.synchronize()
    _check(wr, b, xs, np.uint32, cfg)
