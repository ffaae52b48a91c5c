"""Asynchronous batch compress (pco_b200_compress_files_async, standalone.AsyncFilesCompressor): dst (with guard zones on both sides), the
side indexes and the refs equal pco_b200_compress_files on the same numbers, sizes and config, bit for bit, and decode back to the input -
for every number type, the explicit modes, delta orders, levels, both header flavours, with and without an index, file sizes on every
unoptimized_bins_log, inside a CUDA graph replayed over new counts, sizes and numbers, on concurrent streams, and chained with
AsyncFilesDecompressor in one graph.  Refusals write nothing where the contract forbids it."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DTYPES = [np.uint8, np.int8, np.uint16, np.int16, np.float16, np.uint32, np.int32, np.float32, np.uint64, np.int64, np.float64]
GUARD = 4096
SENT = 0xA5
# at level 8 these sizes give every unoptimized_bins_log from 4 to 8: 1..63 -> 4, 64..255 -> 5, 256..1023 -> 6, 1024..4095 -> 7, 4096.. -> 8
ALL_BINS = [1, 20, 64, 300, 1500, 4000, 5000, 100, 2048, 0, 4095, 4096]


@pytest.fixture(scope="module")
def sa():
    from pcodec_b200 import standalone

    return standalone


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
    """Device buffers of one compressor, with sentinel guard zones around dst, index and files."""

    def __init__(self, comp, dtype, index=True):
        import torch

        self.comp = comp
        self.nums = torch.zeros(comp._plan.nums_cap + 1, dtype=_tdtype(dtype), device="cuda")
        self.file_ns = torch.full((comp.max_files,), 7777, dtype=torch.int64, device="cuda")  # slots past n_files are never read
        self.n_files = torch.zeros(1, dtype=torch.int64, device="cuda")
        self.dst_full = torch.full((comp.dst_cap + 2 * GUARD,), SENT, dtype=torch.uint8, device="cuda")
        self.dst = self.dst_full[GUARD:GUARD + comp.dst_cap]
        self.idx_full = torch.full((comp.index_cap + 2 * GUARD,), SENT, dtype=torch.uint8, device="cuda") if index else None
        self.index = self.idx_full[GUARD:GUARD + comp.index_cap] if index else None
        self.files_full = torch.full((comp.max_files + 8, 4), -1, dtype=torch.int64, device="cuda")
        self.files = self.files_full[:comp.max_files]

    def load(self, xs):
        import torch

        n = sum(len(x) for x in xs)
        if n:
            self.nums[:n].copy_(torch.from_numpy(np.concatenate(xs)).cuda())
        if xs:
            self.file_ns[:len(xs)].copy_(torch.tensor([len(x) for x in xs], dtype=torch.int64))
        self.n_files.fill_(len(xs))

    def run(self):
        self.comp(self.nums, self.file_ns, self.n_files, self.dst, self.index, self.files)


def _reference(sa, xs, dtype, cfg, uniform, index):
    import torch

    nums = torch.from_numpy(np.concatenate(xs) if xs else np.zeros(0, dtype)).cuda()
    out = sa.compress_files(nums, [len(x) for x in xs], cfg, uniform_type=uniform, with_index=index)
    return out


def _check(sa, b, xs, dtype, cfg, uniform, index, decode=True):
    """The call's output against compress_files, and the guard zones."""
    import torch

    dl, il = b.comp.result()
    ref = _reference(sa, xs, dtype, cfg, uniform, index)
    data, files = ref[0], ref[1]
    assert dl == data.numel() and torch.equal(b.dst[:dl], data)
    dfull = b.dst_full.cpu().numpy()
    assert (dfull[:GUARD] == SENT).all() and (dfull[GUARD + dl:] == SENT).all()  # nothing in front of dst or behind the files
    got = b.files[:len(xs)].cpu().numpy().astype(np.uint64)
    want = np.stack([files["offset"], files["len"], files["index_offset"], files["index_len"]], axis=1).astype(np.uint64) if len(xs) else got
    assert np.array_equal(got, want)
    assert (b.files_full[len(xs):].cpu().numpy() == -1).all()
    if index:
        idx = ref[2]
        assert il == idx.numel() and torch.equal(b.index[:il], idx)
        ifull = b.idx_full.cpu().numpy()
        assert (ifull[:GUARD] == SENT).all() and (ifull[GUARD + il:] == SENT).all()
    else:
        assert il == 0
    if decode and xs and sum(len(x) for x in xs):
        back, _ = sa.decompress_files(data.cpu().numpy().tobytes(), files, dtype, ref[2].cpu().numpy().tobytes() if index else None)
        want_nums = np.concatenate(xs)
        assert np.array_equal(back.view(np.uint8), want_nums.view(np.uint8))
    return dl, il


def _comp(sa, dtype, cfg, max_files=16, nums_cap=1 << 16, max_file_n=1 << 15, index=True, uniform=False, dst_cap=None):
    return sa.AsyncFilesCompressor(dtype, cfg, max_files, nums_cap, max_file_n, dst_cap=dst_cap, index=index, uniform_type_header=uniform)


def _one(sa, dtype, cfg, sizes, seed=0, index=True, uniform=False, **kw):
    xs = [_walk(dtype, n, seed + i) for i, n in enumerate(sizes)]
    comp = _comp(sa, dtype, cfg, max_files=max(len(sizes), 1), nums_cap=max(sum(sizes), 1), max_file_n=max(max(sizes, default=1), 1), index=index,
                 uniform=uniform, **kw)
    b = Bufs(comp, dtype, index)
    b.load(xs)
    b.run()
    return _check(sa, b, xs, dtype, cfg, uniform, index)


@pytest.mark.parametrize("dtype", DTYPES)
def test_every_type(sa, dtype):
    _one(sa, dtype, _cfg(order=1, page=4096), [3000, 0, 1, 9000, 257], seed=1)


@pytest.mark.parametrize("dtype,mode", [(np.int64, "int_mult"), (np.uint32, "int_mult"), (np.float32, "float_mult"), (np.float64, "float_mult"),
                                        (np.float32, "float_quant"), (np.float64, "float_quant"), (np.float16, "float_quant")])
def test_modes(sa, dtype, mode):
    _one(sa, dtype, _cfg(mode=mode, k=5, base=0.25 if mode == "float_mult" else 0.01), [5000, 700, 64, 1], seed=2)


@pytest.mark.parametrize("order", [0, 1, 2, 7])
@pytest.mark.parametrize("level", [0, 4, 8])
def test_orders_and_levels(sa, order, level):
    _one(sa, np.int64, _cfg(order=order, level=level, page=3000), ALL_BINS, seed=3)


@pytest.mark.parametrize("uniform", [False, True])
@pytest.mark.parametrize("index", [False, True])
def test_header_flavours_and_index(sa, uniform, index):
    _one(sa, np.uint32, _cfg(order=1), [1000, 0, 20000], seed=4, index=index, uniform=uniform)


@pytest.mark.parametrize("sizes", [[0], [1], [255], [256], [257], [2047], [4095], [4096], [0, 0, 0], ALL_BINS, ALL_BINS[::-1]])
def test_file_sizes(sa, sizes):
    _one(sa, np.uint64, _cfg(order=2, page=1 << 18), sizes, seed=5)


def test_files_above_max_page_n_and_a_chunk_of_2_20(sa):
    # 10007 numbers at pages of 1000: 11 chunks, rem != 0; and a file of one chunk of 2^20
    _one(sa, np.uint32, _cfg(order=1, page=1000), [10007, 999, 1001, 3], seed=6)
    _one(sa, np.int32, _cfg(order=1, page=1 << 20), [1 << 20, 5], seed=7)


def test_two_var_two_kernel_path_and_wide_ranges(sa):
    rng = np.random.default_rng(8)
    xs = [rng.integers(0, 1 << 62, size=n, dtype=np.uint64) for n in (3000, 40000, 1)]
    cfg = _cfg(page=1 << 14)
    comp = _comp(sa, np.uint64, cfg, max_files=4, nums_cap=50000, max_file_n=40000)
    b = Bufs(comp, np.uint64)
    b.load(xs)
    b.run()
    _check(sa, b, xs, np.uint64, cfg, False, True)


def test_n_files_zero_one_and_below_max_files(sa):
    import torch

    cfg = _cfg(order=1, page=2048)
    comp = _comp(sa, np.int16, cfg, max_files=64, nums_cap=40000, max_file_n=9000)
    b = Bufs(comp, np.int16)
    b.load([])
    b.run()
    assert comp.result() == (0, 0)
    assert (b.dst_full.cpu().numpy() == SENT).all() and (b.idx_full.cpu().numpy() == SENT).all()
    assert (b.files_full.cpu().numpy() == -1).all()
    st = comp.status_record()
    assert (st.kind, st.n_files) == (0, 0)
    for sizes in ([5000], [9000, 1, 0, 300]):
        xs = [_walk(np.int16, n, 10 + i) for i, n in enumerate(sizes)]
        b = Bufs(comp, np.int16)
        b.load(xs)
        b.run()
        _check(sa, b, xs, np.int16, cfg, False, True)  # the pad chunk slots leave no trace behind the files


def test_oracle_bytes(sa):
    from oracle import pyoracle

    xs = [np.cumsum(np.random.default_rng(11 + i).geometric(0.01, size=n)).astype(np.uint64) for i, n in enumerate([3000, 1, 70000])]
    cfg = _cfg(order=1, page=1 << 15)
    comp = _comp(sa, np.uint64, cfg, max_files=3, nums_cap=80000, max_file_n=70000, index=False)
    b = Bufs(comp, np.uint64, index=False)
    b.load(xs)
    b.run()
    dl, _ = _check(sa, b, xs, np.uint64, cfg, False, False)
    data = b.dst[:dl].cpu().numpy().tobytes()
    files = b.files[:3].cpu().numpy()
    ocfg = pyoracle.make_config(mode=pyoracle.MODE_CLASSIC, delta=pyoracle.DELTA_CONSECUTIVE, delta_order=1, max_page_n=1 << 15)
    for (off, ln, _, _), x in zip(files, xs):
        assert data[off:off + ln] == pyoracle.simple_compress(x, ocfg)


def test_graph_replay_with_sizes_from_a_kernel(sa):
    """One captured graph: a kernel writes the count and the sizes, the call compresses; replays with new counts, sizes and numbers."""
    import torch

    cfg = _cfg(order=1, page=4096)
    comp = _comp(sa, np.int32, cfg, max_files=8, nums_cap=30000, max_file_n=12000)
    b = Bufs(comp, np.int32)
    plan_ns = torch.zeros(9, dtype=torch.int64, device="cuda")  # [count, sizes...], set on the host between replays
    comp(b.nums, b.file_ns, b.n_files, b.dst, b.index, b.files)  # warm up outside the capture
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            b.n_files.copy_(plan_ns[:1])
            b.file_ns.copy_(plan_ns[1:] * 1)  # a kernel inside the graph writes the sizes
            b.run()
    rng = np.random.default_rng(12)
    for rep, sizes in enumerate([[100, 12000, 0, 5], [4096], [], [1] * 8, [12000, 12000, 5999]]):
        xs = [_walk(np.int32, n, 100 * rep + i) for i, n in enumerate(sizes)]
        b.dst_full.fill_(SENT)
        b.idx_full.fill_(SENT)
        b.files_full.fill_(-1)
        if xs and sum(sizes):
            b.nums[:sum(sizes)].copy_(torch.from_numpy(np.concatenate(xs)).cuda())
        row = [len(sizes)] + sizes + [int(rng.integers(0, 1 << 20))] * (8 - len(sizes))
        plan_ns.copy_(torch.tensor(row, dtype=torch.int64))
        g.replay()
        torch.cuda.synchronize()
        _check(sa, b, xs, np.int32, cfg, False, True)


def test_two_streams_with_their_own_workspaces(sa):
    import torch

    cfg = _cfg(order=2, page=2048)
    sets = [[_walk(np.float32, n, 20 + i) for i, n in enumerate(s)] for s in ([5000, 300, 0], [70, 6000, 6000, 1])]
    comps = [_comp(sa, np.float32, cfg, max_files=4, nums_cap=13000, max_file_n=6000) for _ in sets]
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
        _check(sa, b, xs, np.float32, cfg, False, True)


def test_compress_then_async_decompress_in_one_graph(sa):
    import torch

    cfg = _cfg(order=1, page=4096)
    sizes = [3000, 0, 9000, 1, 4096]
    xs = [_walk(np.uint16, n, 30 + i) for i, n in enumerate(sizes)]
    comp = _comp(sa, np.uint16, cfg, max_files=6, nums_cap=20000, max_file_n=9000)
    b = Bufs(comp, np.uint16)
    b.load(xs)
    head = sa.compress_files(np.zeros(1, np.uint16), [1], cfg)[0][:32]
    dec = sa.AsyncFilesDecompressor(head, np.uint16, comp.dst_cap, comp.index_cap, 6, comp._plan.max_chunks, 20000)
    out = torch.zeros(20000, dtype=_tdtype(np.uint16), device="cuda")
    file_ns = torch.zeros(6, dtype=torch.int64, device="cuda")
    b.run()
    dec(b.dst, b.index, b.files, b.n_files, out, file_ns)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            b.run()
            dec(b.dst, b.index, b.files, b.n_files, out, file_ns)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert dec.result() == sum(sizes)
    assert np.array_equal(out[:sum(sizes)].cpu().numpy().view(np.uint16), np.concatenate(xs))
    assert file_ns[:len(sizes)].cpu().tolist() == sizes
    _check(sa, b, xs, np.uint16, cfg, False, True)


def _untouched(b):
    return (b.dst_full.cpu().numpy() == SENT).all() and (b.idx_full.cpu().numpy() == SENT).all() and (b.files_full.cpu().numpy() == -1).all()


def test_refusals_write_nothing(sa):
    import torch

    from pcodec_b200 import PcoError

    cfg = _cfg(order=1, page=4096)
    comp = _comp(sa, np.int64, cfg, max_files=4, nums_cap=10000, max_file_n=5000)
    cases = [
        ([100] * 5, 0x10E, None),              # more files than max_files
        ([100, 5001, 100], 0x116, 1),          # a file above max_file_n
        ([5000, 5000, 1], 0x117, 2),           # the running sum passes nums_cap at file 2
        ([5000, 5000, 1, 5001], 0x117, 2),     # the lowest failing file wins
        ([100, 5001, 5000, 5000], 0x116, 1),
    ]
    for sizes, code, file in cases:
        b = Bufs(comp, np.int64)
        b.file_ns[:min(len(sizes), 4)].copy_(torch.tensor(sizes[:4], dtype=torch.int64))
        b.n_files.fill_(len(sizes))
        b.run()
        with pytest.raises(PcoError) as e:
            comp.result()
        st = comp.status_record()
        assert e.value.kind == "InvalidArgument" and st.device_status == code, (sizes, st.device_status)
        assert st.n_files == len(sizes)
        if file is not None:
            assert st.file == file and e.value.message.startswith(f"file {file}: ")
        assert _untouched(b), sizes


@pytest.mark.parametrize("short", ["dst", "index"])
def test_caps_one_byte_short(sa, short):
    from pcodec_b200 import PcoError

    cfg = _cfg(order=1, page=4096)
    sizes = [3000, 0, 7000, 2]
    xs = [_walk(np.uint32, n, 40 + i) for i, n in enumerate(sizes)]
    ref = _reference(sa, xs, np.uint32, cfg, False, True)
    need_d, need_i = ref[0].numel(), ref[2].numel()
    comp = sa.AsyncFilesCompressor(np.uint32, cfg, 4, 10002, 7000, dst_cap=need_d - (short == "dst"), index=True)
    comp._plan.index_cap = need_i - (short == "index")  # the plan does not depend on index_cap beyond this field
    b = Bufs(comp, np.uint32)
    b.load(xs)
    b.run()
    with pytest.raises(PcoError) as e:
        comp.result()
    st = comp.status_record()
    assert e.value.kind == "Io" and st.device_status == (0x118 if short == "dst" else 0x119)
    assert (st.dst_bytes, st.index_bytes, st.dst_written, st.index_written) == (need_d, need_i, 0, 0)
    assert f"need {need_d} file bytes and {need_i} index bytes" in e.value.message
    files = ref[1]
    want = np.stack([files["offset"], files["len"], files["index_offset"], files["index_len"]], axis=1).astype(np.int64)
    assert np.array_equal(b.files[:4].cpu().numpy(), want)  # the refs report the sizes needed
    assert (b.dst_full.cpu().numpy() == SENT).all() and (b.idx_full.cpu().numpy() == SENT).all()  # nothing written, nothing past the caps
