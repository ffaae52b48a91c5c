"""The asynchronous pipelines' one-CTA scans at more than one tile (cta_scan.cuh): batches of more than 1024 CTA sums (more than 262,144
ranges, pages or files), and a file of more than 16384 find counts (above 64 MB), so every scan carries its running sums, and the carry
flag, from one tile into the next.  Each result is compared with the input, or with the overflow or refusal numpy finds."""
import struct

import numpy as np
import pytest

from tests.golden_generators import bits_view

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from pcodec_b200 import PcoError, standalone as sa  # noqa: E402

TILE = 1024 * 256  # items whose CTA sums fill one tile of a one-CTA scan
N = 300_000        # items of every batch below: two tiles


def test_ranges_across_tiles():
    from tests.test_gpu_async_ranges import Bufs, _cfg, _walk

    n = 1 << 16
    x = _walk(np.uint32, n, seed=21)
    data, index = sa.simple_compress_with_index(x, _cfg(1))
    rng = np.random.default_rng(22)
    starts = rng.integers(0, n, N)
    counts = np.minimum(rng.integers(0, 20, N), n - starts)
    total = int(counts.sum())
    b = Bufs(sa, data[:32], np.uint32, len(data), len(index), 4, N, total, n)
    b.load(data, index, list(zip(starts.tolist(), counts.tolist())))
    b.call()
    got, err, st = b.outcome(total)
    assert err is None, err
    first = np.cumsum(counts) - counts
    want = x[np.repeat(starts - first, counts) + np.arange(total)]
    np.testing.assert_array_equal(bits_view(got), bits_view(want))
    assert st.n_written == total


def test_range_counts_passing_2_64_in_the_second_tile():
    """An index of 16384 chunks of 2^32 - 1 numbers (nothing is decoded: the call is refused first) and ranges inside it whose counts
    add up past 2^64 at a range of the second tile: RANGE_OVERFLOW names that range."""
    from tests.test_gpu_async_ranges import Bufs, _cfg, _walk

    data, index = sa.simple_compress_with_index(_walk(np.uint32, 1 << 14, seed=23), _cfg(1))
    k, cn = 16384, (1 << 32) - 1
    co = struct.unpack_from("<Q", index, 32)[0]
    chunk_offset, _, n_vars = struct.unpack_from("<QII", index, co)
    head = bytearray(index[:64])
    struct.pack_into("<QQ", head, 8, k, k * cn)
    struct.pack_into("<Q", head, 32, 64)
    recs = b"".join(struct.pack("<QIIQQ", chunk_offset, cn, n_vars, 0, c * cn) for c in range(k))
    crafted = bytes(head) + recs
    c = (1 << 64) // 270_000 + 1
    assert c <= k * cn
    over = -(-(1 << 64) // c) - 1  # the first range whose running sum reaches 2^64
    assert TILE < over < N and over * c < (1 << 64) <= (over + 1) * c
    pairs = [(i % 1000, c if i <= over else 0) for i in range(N)]
    b = Bufs(sa, data[:32], np.uint32, len(data), len(crafted), k, N, 1024, 1 << 16)
    b.load(data, crafted, pairs)
    b.call()
    got, err, st = b.outcome()
    assert got is None and err == ("InvalidArgument", over) and st.device_status == 0x10B, (err, st.device_status)


def test_pages_across_tiles():
    from pcodec_b200 import wrapped
    from tests.test_gpu_async_pages import SENTINEL, _run

    values = np.array([7, 0, 4_000_000_000, 12345, 1, 99, 65536], dtype=np.uint32)
    metas, pages, one = bytearray(), bytearray(), []
    for v in values:
        m, p, r = wrapped.compress_chunks(np.array([v], dtype=np.uint32))
        one.append((len(metas), len(m), len(pages), len(p), 1))
        metas += m
        pages += p
    pick = np.arange(N) % len(values)
    refs = np.array([one[j] for j in pick], dtype=wrapped.PAGE_REF)
    frames = int(sum((4 + r["meta_len"] + r["page_len"] + 15) // 16 * 16 for r in refs))
    got, nw, err, st = _run(bytes(metas), bytes(pages), refs, np.uint32, frame_cap=frames)
    assert err is None and nw == N == st.n_written, err
    np.testing.assert_array_equal(got[:N], values[pick])
    # the running count passes dst_cap at a page of the second tile
    got, _, err, st = _run(bytes(metas), bytes(pages), refs, np.uint32, frame_cap=frames, dst_cap=280_000)
    assert err.kind == "InvalidArgument" and st.page == 280_000 and st.device_status == 0x11E, err
    assert (got.view(np.uint8) == SENTINEL).all()


def test_compress_files_across_tiles():
    """300,000 files of 0-3 numbers compressed in one call and decoded back in one AsyncFilesDecompressor call (whose front end scans as
    many files); then file sizes whose running sum passes nums_cap at a file of the second tile."""
    from tests.test_gpu_async_compress_files import Bufs, _cfg, _comp, _untouched

    nums_cap = 2 * 280_000 + 1
    comp = _comp(sa, np.uint32, _cfg(order=1), max_files=N, nums_cap=nums_cap, max_file_n=3)
    rng = np.random.default_rng(24)
    sizes = rng.integers(0, 4, N)
    flat = rng.integers(0, 1 << 32, int(sizes.sum()), dtype=np.uint64).astype(np.uint32)
    assert flat.size <= nums_cap
    b = Bufs(comp, np.uint32)
    b.nums.view(torch.int32)[:flat.size].copy_(torch.from_numpy(flat.view(np.int32)))
    b.file_ns[:N].copy_(torch.from_numpy(sizes.astype(np.int64)))
    b.n_files.fill_(N)
    b.run()
    dl, il = comp.result()
    files = b.files.cpu().numpy()
    lens = files[:, 1]
    assert (files[:, 0] == np.cumsum(lens) - lens).all() and files[:, 0][-1] + lens[-1] == dl
    ilens = files[:, 3]
    assert (files[:, 2] == np.cumsum(ilens) - ilens).all() and files[:, 2][-1] + ilens[-1] == il

    dec = sa.AsyncFilesDecompressor(b.dst, np.uint32, dl, il, N, int((sizes > 0).sum()), flat.size)
    dst = torch.zeros(flat.size, dtype=torch.int32, device="cuda")
    file_ns = torch.zeros(N, dtype=torch.int64, device="cuda")
    dec(b.dst, b.index, b.files, torch.tensor([N], dtype=torch.int64, device="cuda"), dst.view(torch.uint32), file_ns)
    assert dec.result() == flat.size
    np.testing.assert_array_equal(dst.cpu().numpy().view(np.uint32), flat)
    np.testing.assert_array_equal(file_ns.cpu().numpy(), sizes)

    b = Bufs(comp, np.uint32)
    b.file_ns[:N].fill_(2)
    b.n_files.fill_(N)
    b.run()
    with pytest.raises(PcoError) as e:
        comp.result()
    st = comp.status_record()
    assert e.value.kind == "InvalidArgument" and st.device_status == 0x117 and st.file == 280_000, st.device_status
    assert _untouched(b)


def test_index_of_a_file_above_64_mb():
    """ai_scan_kernel scans one count per 4096 bytes of the file, 16384 per tile: a file above 64 MB spans two tiles."""
    from tests.test_gpu_async_index import _build, _cfg

    x = np.random.default_rng(25).integers(0, 1 << 64, 10_000_000, dtype=np.uint64)
    data, index = sa.simple_compress_with_index(x, _cfg(0, page=1 << 18))
    assert len(data) > 16384 * 4096
    got, st = _build(data, np.uint64)
    assert got == index
    assert st.n_total == x.size and st.serial_chunks == 0
