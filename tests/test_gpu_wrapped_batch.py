"""Batched wrapped pages on the GPU (pco_b200_decompress_pages, pco_b200_compress_wrapped), against the oracle: pages written by the
oracle's ChunkCompressor decode to the input and to what the one-page decoder gives, and the batched writer's metas and pages are the
oracle's ChunkCompressor bytes chunk by chunk."""
import ctypes as C

import numpy as np
import pytest

from tests.golden_generators import bits_view
from tests.test_gpu_encode import _cfgs, _walk

pytestmark = pytest.mark.gpu

PAGE_SIZES = [1, 255, 256, 257, 4097, 1 << 18]


def _data(dtype, mode, n, seed):
    if mode == "float_mult":
        return (np.round(np.cumsum(np.random.default_rng(seed).normal(size=n)) * 100) * 0.01).astype(dtype)
    x = _walk(dtype, n, seed=seed)
    if mode == "int_mult":
        x = (x.astype(np.uint64) // 8 * 8 + 3).astype(dtype)
    return x


def _container(chunks):
    """chunks: [(nums, oracle config)] -> (metas, pages, refs, pieces): every chunk written by the oracle's ChunkCompressor, metas
    back to back, pages back to back; pieces[i] = the numbers of ref i."""
    from oracle import pyoracle
    from pcodec_b200 import wrapped

    metas, pages, refs, pieces = bytearray(), bytearray(), [], []
    for nums, cfg in chunks:
        occ = pyoracle.ChunkCompressor(nums, cfg)
        meta = occ.write_meta()
        m_off = len(metas)
        metas += meta
        start = 0
        for i, pn in enumerate(occ.n_per_page()):
            page = occ.write_page(i)
            refs.append((m_off, len(meta), len(pages), len(page), pn))
            pages += page
            pieces.append(nums[start:start + pn])
            start += pn
    return bytes(metas), bytes(pages), np.array(refs, dtype=wrapped.PAGE_REF), pieces


def _mixed_chunks(oracle, dtype):
    is_float = np.dtype(dtype).kind == "f"
    modes = ["classic"] + (["float_quant"] + ([] if np.dtype(dtype).itemsize == 2 else ["float_mult"]) if is_float else ["int_mult"])
    chunks = []
    for k, pn in enumerate(PAGE_SIZES):
        mode = modes[k % len(modes)]
        order = k % 4
        x = _data(dtype, mode, pn, seed=100 + k)
        _, ocfg = _cfgs(oracle, mode=mode, order=order, max_page_n=pn, k=13 if np.dtype(dtype).itemsize > 2 else 5)
        chunks.append((x, ocfg))
    # a multi-page chunk: four pages share one meta
    x = _data(dtype, "classic", 3 * 1000 + 7, seed=7)
    _, ocfg = _cfgs(oracle, mode="classic", order=1, exact=[1000, 1, 1006, 1000])
    chunks.append((x, ocfg))
    return chunks


def _shuffled(refs, pieces, seed):
    rng = np.random.default_rng(seed)
    order = list(rng.permutation(len(refs))) + [int(rng.integers(0, len(refs)))]  # shuffled, and one page twice
    return refs[order], [pieces[i] for i in order]


def _read_page_into(meta, page, pn, dtype):
    from pcodec_b200 import wrapped

    cd, _ = wrapped.FileDecompressor().chunk_decompressor(meta, dtype)
    dst = np.zeros(pn, dtype=dtype)
    prog, _ = cd.read_page_into(page, pn, dst)
    assert prog.finished
    return dst


@pytest.mark.parametrize("dtype", [np.uint8, np.int8, np.uint16, np.int16, np.float16, np.uint32, np.int32, np.float32, np.uint64, np.int64, np.float64])
def test_one_mixed_call(oracle, dtype):
    from pcodec_b200 import wrapped

    metas, pages, refs, pieces = _container(_mixed_chunks(oracle, dtype))
    refs, pieces = _shuffled(refs, pieces, seed=int(np.dtype(dtype).num))
    got = wrapped.decompress_pages(metas, pages, refs, dtype)
    np.testing.assert_array_equal(bits_view(got), bits_view(np.concatenate(pieces)))
    # page by page, the one-page decoder gives the same numbers
    start = 0
    for r, want in zip(refs, pieces):
        one = _read_page_into(metas[r["meta_offset"]:r["meta_offset"] + r["meta_len"]], pages[r["page_offset"]:r["page_offset"] + r["page_len"]], int(r["page_n"]), dtype)
        np.testing.assert_array_equal(bits_view(got[start:start + len(want)]), bits_view(one))
        start += len(want)
    # metas and pages in one buffer
    both = pages + metas
    refs2 = refs.copy()
    refs2["meta_offset"] += len(pages)
    np.testing.assert_array_equal(bits_view(wrapped.decompress_pages(both, both, refs2, dtype)), bits_view(got))


@pytest.mark.parametrize("dtype", [np.uint16, np.float32, np.int64])
def test_device_resident_on_a_side_stream(oracle, dtype):
    import torch

    from pcodec_b200 import wrapped

    metas, pages, refs, pieces = _container(_mixed_chunks(oracle, dtype))
    refs, pieces = _shuffled(refs, pieces, seed=3)
    dm = torch.frombuffer(bytearray(metas), dtype=torch.uint8).cuda()
    dp = torch.frombuffer(bytearray(pages), dtype=torch.uint8).cuda()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        out = wrapped.decompress_pages(dm, dp, refs, dtype)
    s.synchronize()
    assert out.is_cuda and out.numel() == sum(len(p) for p in pieces)
    np.testing.assert_array_equal(bits_view(out.cpu().numpy()), bits_view(np.concatenate(pieces)))


def _standalone_dict_chunk(data):
    """(meta, page) of the one int32 chunk of a standalone file in Dict mode without delta: header (magic, version, uniform type,
    size varint, format version), the chunk's type byte and n - 1, then the meta (mode 4 bits, dict length 25 bits, byte padding,
    the dict values, delta variant 4 bits, one latent var: ans_size_log 4 bits, bin count 15 bits, bins of ans_size_log + 32 + 6
    bits, byte padding), the page, and the terminator byte."""
    power = (data[6] & 63) + 1
    chunk = 6 + (6 + power + 7) // 8 + 2 + 4
    bits = int.from_bytes(data[chunk:chunk + 8], "little")
    assert bits & 15 == 4, "Dict mode"
    dict_len = (bits >> 4) & ((1 << 25) - 1)
    pos = 32 + dict_len * 32
    tail = int.from_bytes(data[chunk + pos // 8:chunk + pos // 8 + 8], "little")
    assert tail & 15 == 0, "no delta"
    size_log, n_bins = (tail >> 4) & 15, (tail >> 8) & 0x7FFF
    pos += 4 + 4 + 15 + n_bins * (size_log + 32 + 6)
    meta_len = (pos + 7) // 8
    return data[chunk:chunk + meta_len], data[chunk + meta_len:-1]


def _profile(L):
    buf = C.create_string_buffer(4096)
    L.pco_b200_profile_last(buf, 4096)
    return buf.value.decode()


def test_cold_pages_interleaved_with_fast_ones(oracle):
    from pcodec_b200 import _lib, wrapped

    rng = np.random.default_rng(11)
    motif = rng.integers(0, 1 << 14, size=97)
    lookback = np.tile(motif, 60)[:5000].astype(np.int32)
    lookback_im = (np.tile(rng.integers(0, 5000, size=50), 80) * 8 + rng.integers(0, 3, size=4000)).astype(np.int32)
    dict_nums = np.array([3, 77, 200, 5, 131], dtype=np.int32)[rng.integers(0, 5, size=7000)]
    i = np.arange(6000)
    conv1 = (2000 * np.sin(i / 30.0) + 300 * np.cos(i / 7.0)).astype(np.int32)
    centers = np.sort(rng.integers(0, 1 << 30, size=600))  # 600 narrow clusters, lognormal popularity: bins stay above 256 at level 12
    p = rng.lognormal(0.0, 1.0, size=centers.size)
    wide = (centers[rng.choice(centers.size, size=1 << 17, p=p / p.sum())] + rng.integers(0, 16, size=1 << 17)).astype(np.int32)
    fast = _walk(np.int32, 3000, seed=4)
    O = oracle
    chunks = [
        (fast, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=1)),
        (lookback, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_LOOKBACK, max_page_n=1 << 12)),
        (fast[:700], O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_NOOP)),
        (lookback_im, O.make_config(mode=O.MODE_INT_MULT, int_mult_base=8, delta=O.DELTA_LOOKBACK, max_page_n=1500)),
        (fast[:2999], O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=2)),
        (conv1, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONV1, delta_order=2, max_page_n=1 << 12)),
        (wide, O.make_config(level=12, mode=O.MODE_CLASSIC, delta=O.DELTA_NOOP)),
        (fast[5:], O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_NOOP)),
    ]
    metas, pages, refs, pieces = _container(chunks)
    # Dict mode: the oracle writes it through simple_compress only; its one chunk becomes two more pages of the container
    d_meta, d_page = _standalone_dict_chunk(oracle.simple_compress(dict_nums, O.make_config(mode=O.MODE_DICT, delta=O.DELTA_NOOP)))
    refs = np.concatenate([refs, np.array([(len(metas), len(d_meta), len(pages), len(d_page), dict_nums.size)] * 2, dtype=refs.dtype)])
    pieces += [dict_nums, dict_nums]
    dict_meta_at = len(metas)
    metas, pages = metas + d_meta, pages + d_page
    wide_meta = metas[refs[-4]["meta_offset"]:refs[-4]["meta_offset"] + refs[-4]["meta_len"]]
    # Classic, no delta: mode (4 bits), delta variant (4), then the var's ans_size_log (4) and bin count (15)
    assert (int.from_bytes(wide_meta[:4], "little") >> 12) & 0x7FFF > 256, "the level-12 chunk keeps more than 256 bins"
    refs, pieces = _shuffled(refs, pieces, seed=5)
    L = _lib.lib()
    L.pco_b200_profile_enable(1)
    try:
        got = wrapped.decompress_pages(metas, pages, refs, np.int32)
        prof = _profile(L)
    finally:
        L.pco_b200_profile_enable(0)
    assert "cold_decode_kernel" in prof and "fused_narrow_kernel" in prof, prof
    np.testing.assert_array_equal(got, np.concatenate(pieces))
    start = 0
    for r, want in zip(refs, pieces):
        meta, page = metas[r["meta_offset"]:r["meta_offset"] + r["meta_len"]], pages[r["page_offset"]:r["page_offset"] + r["page_len"]]
        if r["meta_offset"] != dict_meta_at:  # the Dict page: its numbers were checked above
            theirs, _, _ = oracle.wrapped_decompress_page(meta, page, np.int32, int(r["page_n"]))
            np.testing.assert_array_equal(got[start:start + len(want)], theirs)
        start += len(want)


def test_f16_float_mult_pages_beside_fast_ones(oracle):
    from pcodec_b200 import wrapped

    O = oracle
    fm = (np.round(np.random.default_rng(4).normal(size=4000) * 40) * 0.25).astype(np.float16)
    plain = _walk(np.float16, 3000, seed=9)
    chunks = [(plain, O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_CONSECUTIVE, delta_order=1)),
              (fm, O.make_config(mode=O.MODE_FLOAT_MULT, float_mult_base=0.25, delta=O.DELTA_CONSECUTIVE, delta_order=1, max_page_n=1500)),
              (plain[:999], O.make_config(mode=O.MODE_CLASSIC, delta=O.DELTA_NOOP))]
    metas, pages, refs, pieces = _container(chunks)
    refs, pieces = _shuffled(refs, pieces, seed=8)
    got = wrapped.decompress_pages(metas, pages, refs, np.float16)
    np.testing.assert_array_equal(bits_view(got), bits_view(np.concatenate(pieces)))


def _six_pages(oracle):
    chunks = []
    for k in range(6):
        x = _walk(np.uint64, 3000 + 500 * k, seed=40 + k)
        _, ocfg = _cfgs(oracle, mode="classic", order=k % 3)
        chunks.append((x, ocfg))
    x = _walk(np.uint64, 4000, seed=60)  # a chunk of two pages sharing a meta
    _, ocfg = _cfgs(oracle, mode="classic", order=1, exact=[1500, 2500])
    chunks.append((x, ocfg))
    return _container(chunks)


def _fails(metas, pages, refs):
    from pcodec_b200 import PcoError, wrapped

    with pytest.raises(PcoError) as e:
        wrapped.decompress_pages(metas, pages, refs, np.uint64)
    return e.value


def test_failures_name_the_lowest_failing_page(oracle):
    from pcodec_b200 import PcoError, wrapped

    metas, pages, refs, pieces = _six_pages(oracle)
    # a page cut short, as the lowest of two bad pages
    for cut in (1, refs[3]["page_len"] // 2):
        bad = refs.copy()
        bad[3]["page_len"] -= cut
        bad[5]["meta_len"] += 1
        e = _fails(metas, pages, bad)
        assert e.kind == "InsufficientData" and e.message.startswith("page 3: "), (cut, e)
    # a meta_len that disagrees with the meta's own length
    for delta in (1, -1):
        bad = refs.copy()
        bad[2]["meta_len"] = int(bad[2]["meta_len"]) + delta
        e = _fails(metas, pages, bad)
        assert e.kind == "InvalidArgument" and e.message.startswith("page 2: "), e
    # bit flips in pages: the call decodes or fails naming the flipped page; later pages do not matter
    rng = np.random.default_rng(1)
    for _ in range(40):
        k = int(rng.integers(0, len(refs)))
        buf = bytearray(pages)
        buf[int(refs[k]["page_offset"] + rng.integers(0, refs[k]["page_len"]))] ^= 1 << int(rng.integers(0, 8))
        try:
            out = wrapped.decompress_pages(metas, bytes(buf), refs, np.uint64)
            assert out.size == sum(len(p) for p in pieces)
        except PcoError as e:
            assert e.kind in ("Corruption", "InsufficientData"), e
            assert e.message.startswith(f"page {k}: "), (k, e)
    # bit flips in metas: the lowest page of the chunk fails first
    first_page_of_meta = {}
    for i, r in enumerate(refs):
        first_page_of_meta.setdefault(int(r["meta_offset"]), i)
    for _ in range(40):
        k = int(rng.integers(0, len(refs)))
        buf = bytearray(metas)
        buf[int(refs[k]["meta_offset"] + rng.integers(0, refs[k]["meta_len"]))] ^= 1 << int(rng.integers(0, 8))
        try:
            wrapped.decompress_pages(bytes(buf), pages, refs, np.uint64)
        except PcoError as e:
            assert e.kind in ("Corruption", "InsufficientData", "InvalidArgument", "Unsupported"), e
            assert e.message.startswith(f"page {first_page_of_meta[int(refs[k]['meta_offset'])]}: "), (k, e)
    # and the library is fine afterwards
    np.testing.assert_array_equal(wrapped.decompress_pages(metas, pages, refs, np.uint64), np.concatenate(pieces))


def _oracle_chunks_equal(oracle, nums, ocfg_kw, metas, pages, refs):
    start = 0
    assert len(refs) > 0
    for r in refs:
        pn = int(r["page_n"])
        occ = oracle.ChunkCompressor(nums[start:start + pn], oracle.make_config(exact_pages=[pn], **ocfg_kw))
        assert occ.n_per_page() == [pn]
        assert metas[r["meta_offset"]:r["meta_offset"] + r["meta_len"]] == occ.write_meta()
        assert pages[r["page_offset"]:r["page_offset"] + r["page_len"]] == occ.write_page(0)
        start += pn
    assert start == nums.size


MODE_KW = {"classic": {}, "int_mult": {"int_mult_base": 8}, "float_mult": {"float_mult_base": 0.01}, "float_quant": {"float_quant_k": 13}}


@pytest.mark.parametrize("dtype,mode,order", [(np.uint64, "classic", 1), (np.int32, "classic", 0), (np.uint16, "classic", 3), (np.int8, "classic", 2),
                                              (np.uint32, "int_mult", 1), (np.int64, "int_mult", 0), (np.float64, "float_mult", 2),
                                              (np.float32, "float_mult", 1), (np.float32, "float_quant", 0), (np.float64, "float_quant", 3),
                                              (np.float16, "classic", 1)])
def test_writer_bytes_equal_the_oracle(oracle, dtype, mode, order):
    from pcodec_b200 import wrapped

    x = _data(dtype, mode, 3 * 7000 + 11, seed=17)
    ours, _ = _cfgs(oracle, mode=mode, order=order, max_page_n=7000)
    metas, pages, refs = wrapped.compress_chunks(x, ours)
    assert list(refs["page_n"]) == [5253, 5253, 5253, 5252]  # EqualPagesUpTo(7000) over 21011 numbers
    om = {"classic": oracle.MODE_CLASSIC, "int_mult": oracle.MODE_INT_MULT, "float_mult": oracle.MODE_FLOAT_MULT, "float_quant": oracle.MODE_FLOAT_QUANT}[mode]
    kw = dict(mode=om, delta=oracle.DELTA_CONSECUTIVE, delta_order=order, **MODE_KW[mode])
    _oracle_chunks_equal(oracle, x, kw, metas, pages, refs)
    assert refs["meta_offset"][0] == 0 and refs["page_offset"][0] == 0
    assert int(refs["meta_offset"][-1] + refs["meta_len"][-1]) == len(metas) and int(refs["page_offset"][-1] + refs["page_len"][-1]) == len(pages)
    np.testing.assert_array_equal(bits_view(wrapped.decompress_pages(metas, pages, refs, dtype)), bits_view(x))


def test_writer_auto(oracle):
    from pcodec_b200 import ChunkConfig, PagingSpec, datagen, wrapped

    rng = np.random.default_rng(3)
    n = 30000
    a = (np.cumsum(rng.integers(-50, 50, size=n)) * 1000 + 10**9).astype(np.int64)
    b = np.cumsum(rng.geometric(0.01, size=n)).astype(np.int64)
    for x in (np.concatenate([a, b, a]), datagen.c2_u64_cumsum_geometric(seed=0)):
        info = oracle.inspect(oracle.simple_compress(x, oracle.make_config(mode=oracle.MODE_AUTO, delta=oracle.DELTA_AUTO, max_page_n=n)), x.dtype)
        assert all(c["delta"] in (0, 1) for c in info["chunks"]), "an input on which the oracle picks Lookback / Conv1"
        metas, pages, refs = wrapped.compress_chunks(x, ChunkConfig(paging_spec=PagingSpec.equal_pages_up_to(n)))
        _oracle_chunks_equal(oracle, x, dict(mode=oracle.MODE_AUTO, delta=oracle.DELTA_AUTO), metas, pages, refs)
        np.testing.assert_array_equal(wrapped.decompress_pages(metas, pages, refs, x.dtype), x)


@pytest.mark.parametrize("level", [8, 9, 12])
def test_writer_exact_paging_and_levels(oracle, level):
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec, wrapped

    sizes = [100, 5000, 70000, 300, 1]  # unoptimized_bins_log differs between them
    x = np.minimum(np.random.default_rng(level).lognormal(10, 2, size=sum(sizes)), 2**60).astype(np.uint64)
    cfg = ChunkConfig(compression_level=level, mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.no_op(), paging_spec=PagingSpec.exact_page_sizes(sizes))
    metas, pages, refs = wrapped.compress_chunks(x, cfg)
    assert list(refs["page_n"]) == sizes
    _oracle_chunks_equal(oracle, x, dict(level=level, mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_NOOP), metas, pages, refs)
    np.testing.assert_array_equal(wrapped.decompress_pages(metas, pages, refs, np.uint64), x)


def test_writer_device_buffers(oracle):
    import torch

    from pcodec_b200 import wrapped

    x = _walk(np.int64, 50000, seed=2)
    ours, _ = _cfgs(oracle, mode="classic", order=2, max_page_n=12000)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        dx = torch.from_numpy(x).cuda()
        dm, dp, refs = wrapped.compress_chunks(dx, ours)
        back = wrapped.decompress_pages(dm, dp, refs, np.int64)
    s.synchronize()
    assert dm.is_cuda and dp.is_cuda and back.is_cuda
    hm, hp, hrefs = wrapped.compress_chunks(x, ours)
    assert bytes(dm.cpu().numpy()) == hm and bytes(dp.cpu().numpy()) == hp and (hrefs == refs).all()
    _oracle_chunks_equal(oracle, x, dict(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_CONSECUTIVE, delta_order=2), hm, hp, hrefs)
    np.testing.assert_array_equal(back.cpu().numpy(), x)


def test_writer_errors(oracle):
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec, PcoError, _lib, wrapped

    x = _walk(np.uint32, 20000, seed=5)
    cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(1), paging_spec=PagingSpec.equal_pages_up_to(8000))
    metas, pages, refs = wrapped.compress_chunks(x, cfg)
    L = wrapped._lib_batch()
    c = cfg._to_c()
    for caps in [(0, 0, 0), (len(metas) - 1, len(pages), len(refs)), (len(metas), len(pages) - 1, len(refs)), (len(metas), len(pages), len(refs) - 1)]:
        mb, pb, rb = np.zeros(max(caps[0], 1), np.uint8), np.zeros(max(caps[1], 1), np.uint8), np.zeros(max(caps[2], 1), wrapped.PAGE_REF)
        ml, pl, nc = C.c_size_t(), C.c_size_t(), C.c_size_t()
        rc = L.pco_b200_compress_wrapped(x.ctypes.data_as(C.c_void_p), C.c_size_t(x.size), C.c_ubyte(1), C.byref(c), mb.ctypes.data_as(C.c_void_p),
                                         C.c_size_t(caps[0]), C.byref(ml), pb.ctypes.data_as(C.c_void_p), C.c_size_t(caps[1]), C.byref(pl),
                                         rb.ctypes.data_as(C.c_void_p), C.c_size_t(caps[2]), C.byref(nc), C.c_uint32(0), None)
        assert rc == 4, caps  # PCO_B200_IO
        assert (ml.value, pl.value, nc.value) == (len(metas), len(pages), len(refs))
    # refused with the kinds pco_b200_compress_ex gives
    for bad, kind in [(ChunkConfig(compression_level=13), "InvalidArgument"), (ChunkConfig(mode_spec=ModeSpec.try_dict()), "Unsupported"),
                      (ChunkConfig(delta_spec=DeltaSpec.try_lookback()), "Unsupported"), (ChunkConfig(paging_spec=PagingSpec.exact_page_sizes([5, 5])), "InvalidArgument")]:
        with pytest.raises(PcoError) as e:
            wrapped.compress_chunks(x, bad)
        assert e.value.kind == kind, (bad, e.value)
    motif = np.random.default_rng(1).integers(0, 1 << 30, size=97)
    lookback_wins = np.tile(motif, 700)[:60000].astype(np.uint32)
    with pytest.raises(PcoError) as e:  # Auto picks Lookback on this chunk
        wrapped.compress_chunks(lookback_wins, ChunkConfig())
    assert e.value.kind == "Unsupported"
    # empty input: no chunk
    m0, p0, r0 = wrapped.compress_chunks(np.zeros(0, np.uint32), cfg)
    assert m0 == b"" and p0 == b"" and len(r0) == 0


def test_full_size_round_trip(oracle):
    import torch

    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, datagen, wrapped

    n_chunks, chunk_n = 64, 1 << 18
    x = np.concatenate([datagen.c2_u64_cumsum_geometric(chunk_n, seed=c) for c in range(n_chunks)])
    cfg = ChunkConfig(mode_spec=ModeSpec.classic(), delta_spec=DeltaSpec.try_consecutive(1))
    x = x.view(np.int64)
    dx = torch.from_numpy(x).cuda()
    dm, dp, refs = wrapped.compress_chunks(dx, cfg)
    assert len(refs) == n_chunks and (refs["page_n"] == chunk_n).all()
    back = wrapped.decompress_pages(dm, dp, refs, np.int64)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(back.cpu().numpy(), x)
    hm, hp = bytes(dm.cpu().numpy()), bytes(dp.cpu().numpy())
    for c in (0, n_chunks - 1):
        occ = oracle.ChunkCompressor(x[c * chunk_n:(c + 1) * chunk_n], oracle.make_config(mode=oracle.MODE_CLASSIC, delta=oracle.DELTA_CONSECUTIVE, delta_order=1,
                                                                                       exact_pages=[chunk_n]))
        r = refs[c]
        assert hm[r["meta_offset"]:r["meta_offset"] + r["meta_len"]] == occ.write_meta()
        assert hp[r["page_offset"]:r["page_offset"] + r["page_len"]] == occ.write_page(0)
