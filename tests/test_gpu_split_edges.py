"""GPU compress at the edges of every mode split and of the size-guarantee fallback, on every compress entry point, against the oracle.

The families of tests/split_edges.py (special values of every float type, FloatMult at negative, subnormal and huge bases with ties,
overflows and multipliers either side of 2^MANTISSA_DIGITS, FloatQuant at every k, IntMult at the type's width, Classic on the
one-pass front end and the sort path) and its chunks one byte either side of the size guarantee go through:

* standalone.simple_compress, simple_compress_with_index (its index must equal build_index's), and pco_b200_compress_ex with every
  buffer on the device and guard bytes behind dst_cap;
* AsyncCompressor, compress_files and AsyncFilesCompressor (the family cut into files of different sizes, so per-chunk bins logs
  differ, and the whole family as one more file), wrapped.ChunkCompressor, compress_chunks and AsyncChunksCompressor;
* the boundary chunks of one config (margins -1, 0 and +1) as the files and arrays of one batch;
* a config with DeltaSpec.auto() beside the explicit mode, which runs the split in gather_primary_sample_kernel.

Every file must equal the oracle's byte for byte; the GPU and the oracle must decode it to the input, bit for bit; and the chunk must
keep the family's mode and delta exactly when the oracle's size guarantee does not fall back.  A mismatch prints both files' chunk
metas and keeps the case like test_gpu_properties.
"""
import ctypes as C

import numpy as np
import pytest

from tests import split_edges as se
from tests.test_gpu_properties import _dump_failure

pytestmark = pytest.mark.gpu

FAMILIES = se.families()
BOUNDARY = [se.boundary_family(combo, *v) | {"margin": m} for (combo, m), v in se.BOUNDARY.items()]
STANDALONE = FAMILIES + [f for f in BOUNDARY if not f.get("pages")]
SHARED_PAGES = [f for f in BOUNDARY if f.get("pages")]
GUARD, SENT = 1024, 0xA5
LOOKBACK = 2  # DeltaKind in the chunk meta


def _ids(fams):
    return [f["name"] for f in fams]


def _bits(x):
    return np.ascontiguousarray(x).view(se._u(x.dtype))


def _ours(fam, delta_auto=False, pages=None):
    from pcodec_b200 import ChunkConfig, DeltaSpec, ModeSpec, PagingSpec

    ms = {"classic": lambda: ModeSpec.classic(), "int_mult": lambda: ModeSpec.try_int_mult(fam["base"]),
          "float_mult": lambda: ModeSpec.try_float_mult(fam["base"]), "float_quant": lambda: ModeSpec.try_float_quant(fam["k"])}[fam["mode"]]()
    ds = DeltaSpec.auto() if delta_auto else DeltaSpec.try_consecutive(fam["order"]) if fam["order"] else DeltaSpec.no_op()
    ps = PagingSpec.exact_page_sizes(pages) if pages else PagingSpec.equal_pages_up_to(1 << 18)
    return ChunkConfig(compression_level=fam["level"], mode_spec=ms, delta_spec=ds, paging_spec=ps, enable_8_bit=True)


def _metas(oracle, data, dtype):
    try:
        return [{k: v for k, v in ch.items() if k not in ("chunk_start", "meta_start", "page_start", "chunk_end")}
                for ch in oracle.inspect(data, dtype)["chunks"]]
    except Exception as e:  # a file the oracle cannot read is its own finding
        return f"unreadable: {e}"


def _same(oracle, fam, where, got, want, nums=None):
    if got == want:
        return
    nums = fam["nums"] if nums is None else nums
    _dump_failure(nums, {"family": fam["name"], "where": where}, got, want)
    if where.startswith("wrapped") or where.startswith("chunks"):
        print("(wrapped meta/page bytes; no standalone chunk metas to print)")
    else:
        print("GPU chunk metas:   ", _metas(oracle, got, nums.dtype))
        print("oracle chunk metas:", _metas(oracle, want, nums.dtype))
    m = min(len(got), len(want))
    d = np.flatnonzero(np.frombuffer(got[:m], np.uint8) != np.frombuffer(want[:m], np.uint8))
    raise AssertionError(f"{fam['name']} via {where}: {len(got)} bytes vs the oracle's {len(want)}, first difference at byte "
                         f"{int(d[0]) if d.size else m}")


def _want(oracle, fam, nums=None, delta_auto=False):
    """The oracle's file."""
    nums = fam["nums"] if nums is None else nums
    return oracle.simple_compress(nums, se.oracle_configs(oracle, fam, delta_auto=delta_auto))


def _intent(oracle, fam, data):
    """Call right after _want: the chunk keeps the family's mode and delta exactly when the oracle's size guarantee holds."""
    (w, b), = oracle.last_fallback_margins()
    ch, = oracle.inspect(data, fam["dtype"])["chunks"]
    fell_back = w > b and not (fam["mode"] == "classic" and fam["order"] == 0)
    want = (0, 0, 0) if fell_back else (se.MODE_CODE[fam["mode"]], 1 if fam["order"] else 0, fam["order"])
    assert (ch["mode"], ch["delta"], ch["delta_order"]) == want, (fam["name"], w - b, ch)
    if "margin" in fam:
        assert w - b == fam["margin"], fam["name"]


def _device(x):
    import torch

    from pcodec_b200.wrapped import _torch_dtypes

    return torch.as_tensor(np.ascontiguousarray(x).view(np.uint8).copy(), device="cuda").view(_torch_dtypes()[x.dtype])


def _compress_ex_device(nums, cfg):
    """pco_b200_compress_ex with nums and dst on the device; dst_cap is followed by GUARD sentinel bytes that must stay untouched."""
    import torch

    from pcodec_b200 import _lib

    L = _lib.lib()
    c = cfg._to_c()
    cap = L.pco_standalone_guarantee_file_size(nums.size, _lib.dtype_byte(nums.dtype)) + 160
    d_x = _device(nums)
    dst = torch.full((cap + GUARD,), SENT, dtype=torch.uint8, device="cuda")
    written = C.c_size_t()
    _lib.check(L.pco_b200_compress_ex(C.c_void_p(d_x.data_ptr()), C.c_size_t(nums.size), C.c_ubyte(_lib.dtype_byte(nums.dtype)), C.byref(c), C.c_int(0),
                                      C.c_void_p(dst.data_ptr()), C.c_size_t(cap), C.byref(written), None, C.c_size_t(0), None, C.c_uint32(3),
                                      C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    host = dst.cpu().numpy()
    assert (host[cap:] == SENT).all(), "compress_ex wrote past dst_cap"
    return host[: written.value].tobytes()


def _index_fields(index):
    """What a side index says (IndexHeader, each IndexChunk and its BatchEntry array; pcodec_b200/csrc/codec_common.cuh), without
    where it puts the entry arrays: the compressor and build_index lay them out in different places."""
    import struct

    magic, version, n_chunks, n_total, file_len, chunks_offset, end_byte = struct.unpack_from("<IIQQQQQ", index, 0)
    chunks = []
    for c in range(n_chunks):
        chunk_offset, n, n_vars, entries_offset, out_offset = struct.unpack_from("<QIIQQ", index, chunks_offset + 32 * c)
        n_entries = n_vars * -(-n // 256)
        chunks.append((chunk_offset, n, n_vars, out_offset, index[entries_offset: entries_offset + 12 * n_entries]))
    return magic, version, n_chunks, n_total, file_len, end_byte, chunks


def _pieces(nums):
    """The family cut into files of different sizes (so their unoptimized bins logs differ), then the whole family as one more file,
    so the batch also holds the chunk at its own margin."""
    cuts = [c for c in (17, 17 + 300, 17 + 300 + 1030) if c < nums.size]
    return [p for p in np.split(nums, cuts) if p.size] + [nums]


def _files_batch(oracle, fam, parts, ours):
    """compress_files and AsyncFilesCompressor (sizes in device memory) over `parts` as files: each equals the oracle's file."""
    import torch

    from pcodec_b200 import PcoError, standalone

    dt = fam["dtype"]
    ns = [p.size for p in parts]
    nums = np.concatenate(parts)
    wants = [_want(oracle, fam, p) for p in parts]
    data, files, _ = standalone.compress_files(nums, ns, ours)
    for i, (p, w) in enumerate(zip(parts, wants)):
        _same(oracle, fam, f"compress_files file {i}", data[int(files[i]["offset"]): int(files[i]["offset"] + files[i]["len"])], w, p)
    if fam["level"] > 8:  # the asynchronous plans take unoptimized bins logs up to 8 only
        with pytest.raises(PcoError) as e:
            standalone.AsyncFilesCompressor(dt, ours, max_files=len(ns), nums_cap=nums.size, max_file_n=max(ns), index=False)
        assert e.value.kind == "Unsupported"
        return
    fc = standalone.AsyncFilesCompressor(dt, ours, max_files=len(ns), nums_cap=nums.size, max_file_n=max(ns), index=False)
    fdst = torch.empty(fc.dst_cap, dtype=torch.uint8, device="cuda")
    refs = torch.zeros((fc.max_files, 4), dtype=torch.int64, device="cuda")
    fc(_device(nums), torch.tensor(ns, dtype=torch.int64, device="cuda"), torch.tensor([len(ns)], dtype=torch.int64, device="cuda"), fdst, None, refs)
    dl, _ = fc.result()
    out, r = fdst[:dl].cpu().numpy().tobytes(), refs.cpu().numpy()
    for i, (p, w) in enumerate(zip(parts, wants)):
        _same(oracle, fam, f"AsyncFilesCompressor file {i}", out[int(r[i, 0]): int(r[i, 0] + r[i, 1])], w, p)


def _chunks_batch(oracle, fam, parts, ours):
    """AsyncChunksCompressor over `parts` as arrays: each array's one wrapped chunk equals the oracle's meta and page."""
    import torch

    from pcodec_b200 import PcoError, wrapped

    dt = fam["dtype"]
    nums = np.concatenate(parts)
    if fam["level"] > 8:
        with pytest.raises(PcoError) as e:
            wrapped.AsyncChunksCompressor(dt, ours, len(parts), nums.size, max(p.size for p in parts))
        assert e.value.kind == "Unsupported"
        return
    wants = [_oracle_wrapped(oracle, fam, p) for p in parts]
    comp = wrapped.AsyncChunksCompressor(dt, ours, len(parts), nums.size, max(p.size for p in parts))
    m_buf = torch.full((comp.metas_cap,), SENT, dtype=torch.uint8, device="cuda")
    p_buf = torch.full((comp.pages_cap,), SENT, dtype=torch.uint8, device="cuda")
    r_buf = torch.full((comp.max_chunks, 5), -1, dtype=torch.int64, device="cuda")
    first = torch.full((comp.max_arrays + 1,), -1, dtype=torch.int64, device="cuda")
    comp(_device(nums), torch.tensor([p.size for p in parts], dtype=torch.int64, device="cuda"), torch.tensor([len(parts)], dtype=torch.int64, device="cuda"),
         m_buf, p_buf, r_buf, first)
    ml, pl, nc = comp.result()
    assert nc == len(parts)
    assert first[: len(parts) + 1].cpu().tolist() == list(range(len(parts) + 1))
    mh, ph, rh = m_buf[:ml].cpu().numpy().tobytes(), p_buf[:pl].cpu().numpy().tobytes(), r_buf.cpu().numpy()
    for i, (p, (wm, wp, _)) in enumerate(zip(parts, wants)):
        _same(oracle, fam, f"chunks AsyncChunksCompressor meta {i}", mh[rh[i, 0]: rh[i, 0] + rh[i, 1]], wm, p)
        _same(oracle, fam, f"chunks AsyncChunksCompressor page {i}", ph[rh[i, 2]: rh[i, 2] + rh[i, 3]], wp[0], p)


def _oracle_wrapped(oracle, fam, nums, pages=None):
    occ = oracle.ChunkCompressor(nums, se.oracle_configs(oracle, dict(fam, pages=pages)))
    return occ.write_meta(), [occ.write_page(i) for i in range(len(occ.n_per_page()))], occ.n_per_page()


@pytest.mark.parametrize("fam", STANDALONE, ids=_ids(STANDALONE))
def test_standalone_entry_points(oracle, fam):
    from pcodec_b200 import PcoError, standalone

    nums, dt = fam["nums"], fam["dtype"]
    want = _want(oracle, fam)
    _intent(oracle, fam, want)
    ours = _ours(fam)
    _same(oracle, fam, "simple_compress", standalone.simple_compress(nums, ours), want)
    np.testing.assert_array_equal(_bits(standalone.simple_decompress(want, dt)), _bits(nums))
    np.testing.assert_array_equal(_bits(oracle.simple_decompress(want, dt)), _bits(nums))
    data, index = standalone.simple_compress_with_index(nums, ours)
    _same(oracle, fam, "simple_compress_with_index", data, want)
    assert _index_fields(index) == _index_fields(standalone.build_index(data, dt)), fam["name"]
    _same(oracle, fam, "compress_ex (device)", _compress_ex_device(nums, ours), want)
    # Auto delta with the explicit mode: the sample for the delta choice is split in gather_primary_sample_kernel.  Where the choice
    # is Lookback, which the GPU does not encode, the call refuses as Unsupported rather than write other bytes.
    want_auto = _want(oracle, fam, delta_auto=True)
    if oracle.inspect(want_auto, dt)["chunks"][0]["delta"] == LOOKBACK:
        with pytest.raises(PcoError) as e:
            standalone.simple_compress(nums, _ours(fam, delta_auto=True))
        assert e.value.kind == "Unsupported" and "Lookback" in e.value.message
    else:
        _same(oracle, fam, "simple_compress (Auto delta)", standalone.simple_compress(nums, _ours(fam, delta_auto=True)), want_auto)


@pytest.mark.parametrize("fam", STANDALONE, ids=_ids(STANDALONE))
def test_async_and_batch_entry_points(oracle, fam):
    import torch

    from pcodec_b200 import PcoError, standalone

    nums, dt = fam["nums"], fam["dtype"]
    ours = _ours(fam)
    want = _want(oracle, fam)
    _files_batch(oracle, fam, _pieces(nums), ours)
    if fam["level"] > 8:  # the asynchronous plans take unoptimized bins logs up to 8 only
        with pytest.raises(PcoError) as e:
            standalone.AsyncCompressor(nums.size, dt, ours, index=False)
        assert e.value.kind == "Unsupported"
        return
    comp = standalone.AsyncCompressor(nums.size, dt, ours, index=False)
    dst = torch.full((comp.dst_cap + GUARD,), SENT, dtype=torch.uint8, device="cuda")
    comp(_device(nums), dst[: comp.dst_cap])
    nw, _ = comp.result()
    host = dst.cpu().numpy()
    assert (host[comp.dst_cap:] == SENT).all()
    _same(oracle, fam, "AsyncCompressor", host[:nw].tobytes(), want)


@pytest.mark.parametrize("fam", STANDALONE, ids=_ids(STANDALONE))
def test_wrapped_entry_points(oracle, fam):
    from pcodec_b200 import wrapped

    nums, dt = fam["nums"], fam["dtype"]
    ours = _ours(fam)
    meta, pages, pns = _oracle_wrapped(oracle, fam, nums)
    assert len(pages) == 1
    cc = wrapped.FileCompressor().chunk_compressor(nums, ours)
    _same(oracle, fam, "wrapped.ChunkCompressor meta", cc.write_meta(), meta)
    _same(oracle, fam, "wrapped.ChunkCompressor page", cc.write_page(0), pages[0])
    back, _, _ = oracle.wrapped_decompress_page(meta, pages[0], dt, nums.size)
    np.testing.assert_array_equal(_bits(back), _bits(nums))
    metas, pgs, refs = wrapped.compress_chunks(nums, ours)
    assert len(refs) == 1
    _same(oracle, fam, "compress_chunks meta", metas[int(refs[0]["meta_offset"]): int(refs[0]["meta_offset"] + refs[0]["meta_len"])], meta)
    _same(oracle, fam, "compress_chunks page", pgs[int(refs[0]["page_offset"]): int(refs[0]["page_offset"] + refs[0]["page_len"])], pages[0])
    _chunks_batch(oracle, fam, _pieces(nums), ours)


BATCH_COMBOS = sorted({f["name"].split("-n")[0][len("boundary-"):] for f in BOUNDARY if not f.get("pages")})


@pytest.mark.parametrize("combo", BATCH_COMBOS)
def test_boundary_chunks_in_one_batch(oracle, combo):
    """The chunks of one config at margins -1, 0 and +1 as the files (and arrays) of one batch, each at its own margin."""
    fams = [f for f in BOUNDARY if f["name"].startswith(f"boundary-{combo}-n")]
    assert sorted(f["margin"] for f in fams) == [-1, 0, 1]
    for f in fams:
        _intent(oracle, f, _want(oracle, f))
    parts = [f["nums"] for f in fams]
    ours = _ours(fams[0])
    _files_batch(oracle, fams[0], parts, ours)
    _chunks_batch(oracle, fams[0], parts, ours)


@pytest.mark.parametrize("fam", SHARED_PAGES, ids=_ids(SHARED_PAGES))
def test_shared_page_fallback(oracle, fam):
    """A classic order-2 chunk of several pages: one fallback decision over all pages, counting P page metas."""
    from pcodec_b200 import wrapped

    nums, dt = fam["nums"], fam["dtype"]
    assert se.margin(oracle, fam) == fam["margin"]
    meta, pages, pns = _oracle_wrapped(oracle, fam, nums, fam["pages"])
    assert pns == fam["pages"]
    cc = wrapped.FileCompressor().chunk_compressor(nums, _ours(fam, pages=fam["pages"]))
    _same(oracle, fam, "wrapped shared pages meta", cc.write_meta(), meta)
    assert cc.n_per_page() == pns
    off = 0
    for i, pn in enumerate(pns):
        _same(oracle, fam, f"wrapped shared pages page {i}", cc.write_page(i), pages[i], nums[off: off + pn])
        back, _, _ = oracle.wrapped_decompress_page(meta, pages[i], dt, pn)
        np.testing.assert_array_equal(_bits(back), _bits(nums[off: off + pn]))
        dst = np.empty(pn, dtype=dt)
        wrapped.ChunkDecompressor(meta, dt).read_page_into(pages[i], pn, dst)
        np.testing.assert_array_equal(_bits(dst), _bits(nums[off: off + pn]))
        off += pn


REFUSALS = [
    ("f16 FloatMult", np.float16, "float_mult", 0.5, "Unsupported"),
    ("u8 IntMult 256", np.uint8, "int_mult", 256, "InvalidArgument"),
    ("u16 IntMult 2^17", np.uint16, "int_mult", 1 << 17, "InvalidArgument"),
    ("u32 IntMult 0", np.uint32, "int_mult", 0, "InvalidArgument"),
    ("f64 FloatMult 0", np.float64, "float_mult", 0.0, "InvalidArgument"),
    ("f32 FloatMult inf", np.float32, "float_mult", float("inf"), "InvalidArgument"),
    ("f64 FloatMult -inf", np.float64, "float_mult", float("-inf"), "InvalidArgument"),
    ("f64 FloatMult nan", np.float64, "float_mult", float("nan"), "InvalidArgument"),
    ("f32 FloatQuant 0", np.float32, "float_quant", 0, "InvalidArgument"),
    ("f32 FloatQuant 24", np.float32, "float_quant", 24, "InvalidArgument"),
    ("f16 FloatQuant 11", np.float16, "float_quant", 11, "InvalidArgument"),
    ("f64 FloatQuant 53", np.float64, "float_quant", 53, "InvalidArgument"),
]


@pytest.mark.parametrize("case", REFUSALS, ids=[c[0] for c in REFUSALS])
def test_refusals_on_every_entry_point(case):
    import torch

    from pcodec_b200 import PcoError, standalone, wrapped

    _, dt, mode, param, kind = case
    nums = (np.arange(1000) % 50).astype(dt)
    fam = se.family("refusal", dt, nums, mode, 1, base=param if mode != "float_quant" else None, k=param if mode == "float_quant" else None)
    ours = _ours(fam)
    calls = {
        "simple_compress": lambda: standalone.simple_compress(nums, ours),
        "simple_compress_with_index": lambda: standalone.simple_compress_with_index(nums, ours),
        "compress_ex (device)": lambda: _compress_ex_device(nums, ours),
        "compress_files": lambda: standalone.compress_files(nums, [400, 600], ours),
        "wrapped.ChunkCompressor": lambda: wrapped.FileCompressor().chunk_compressor(nums, ours),
        "compress_chunks": lambda: wrapped.compress_chunks(nums, ours),
        "compress_chunks (device)": lambda: wrapped.compress_chunks(_device(nums), ours),
        "AsyncCompressor plan": lambda: standalone.AsyncCompressor(nums.size, dt, ours, index=False),
        "AsyncFilesCompressor plan": lambda: standalone.AsyncFilesCompressor(dt, ours, max_files=2, nums_cap=nums.size, max_file_n=600, index=False),
        "AsyncChunksCompressor plan": lambda: wrapped.AsyncChunksCompressor(dt, ours, 2, nums.size, 600),
    }
    for where, call in calls.items():
        with pytest.raises(PcoError) as e:
            call()
        assert e.value.kind == kind, (case[0], where, e.value.kind, e.value.message)
    torch.cuda.synchronize()
