// Batches of standalone files (pco_b200_compress_files / pco_b200_decompress_files) on the device.
//
// Compress: the files' chunks go through the CHUNKS_ONLY pipeline as the chunks of one call; the kernels here turn that output into
// standalone files.  Decompress: the side indexes of many files become ONE chunk list for the ordinary decode kernels, and the
// index-free files are walked together, every file's candidate chunk starts found in one launch.
//   frame_files_kernel       one CTA per file: [header][its chunks][terminator] at the file's offset in dst, and its side index -
//                            IndexHeader, the chunk records rebased to the file, the batch entries - at its offset in `index`;
//   check_index_kernel       one CTA per indexed file: every record inside its own file, index and count, and the file's route;
//   merge_index_kernel       one CTA per indexed file: its IndexChunk records, rebased to the call's buffers, into the merged list;
//   find_file_starts_kernel  every position in each file's unread range whose 4 bytes equal THAT file's chunk pattern;
//   peek_bytes_kernel        a few bytes at many positions (file heads, index headers, chunk patterns) into one table for one readback.
// Byte copies go through cta_copy_bytes (gather_kernels.cuh): aligned 16-byte stores assembled from unaligned sources by funnel shifts.
#pragma once
#include "decode_kernels.cuh"
#include "gather_kernels.cuh"
#include "wrapped_kernels.cuh"  // wrapped_meta_len: a chunk meta's route

namespace pcob200 {

constexpr int FILES_THREADS = GATHER_THREADS;  // cta_copy_bytes strides by GATHER_THREADS
constexpr uint32_t FILE_HEADER_CAP = 24;       // a standalone header is at most 4 + 1 + 1 + 10 + 2 bytes

// One file of a compress_files call, as the host laid it out from the pipeline's chunk table.
struct FileFrame {
  uint64_t chunks_src;     // byte offset of the file's first chunk in the pipeline's output
  uint64_t chunks_len;     // bytes of its chunks
  uint64_t dst_off;        // offset of the file in dst
  uint64_t recs_src;       // byte offset of its first IndexChunk in the pipeline's index (0 when n_chunks == 0)
  uint64_t entries_src;    // byte offset of its first BatchEntry there
  uint64_t entries_len;    // bytes of its entries (16-byte aligned pieces, as compress_ex lays them out)
  uint64_t index_off;      // offset of its side index in `index` (a multiple of 16)
  uint64_t n;              // numbers in the file
  uint32_t n_chunks, hdr_len;
  uint8_t hdr[FILE_HEADER_CAP];
};
static_assert(sizeof(FileFrame) % 8 == 0, "frame table layout");

// One CTA per file.  `index` may be nullptr (no side indexes wanted).  Index layout per file, as compress_ex writes it: IndexHeader |
// IndexChunk[n_chunks] | entries, with chunk_offset counted from the file's first byte, out_offset from its first number and
// entries_offset from its index's first byte.
__global__ void __launch_bounds__(FILES_THREADS) frame_files_kernel(const uint8_t* __restrict__ chunks, const uint8_t* __restrict__ pidx,
                                                                    const FileFrame* __restrict__ tab, uint8_t* __restrict__ dst,
                                                                    uint8_t* __restrict__ index) {
  const FileFrame& f = tab[blockIdx.x];
  uint8_t* out = dst + f.dst_off;
  const uint64_t file_len = f.hdr_len + f.chunks_len + 1;
  if (threadIdx.x < f.hdr_len) out[threadIdx.x] = f.hdr[threadIdx.x];  // read in place: no local copy of the header bytes
  if (threadIdx.x == 0) out[file_len - 1] = 0;  // the terminator
  cta_copy_bytes(out + f.hdr_len, chunks + f.chunks_src, f.chunks_len);
  if (!index) return;
  uint8_t* ix = index + f.index_off;
  const uint64_t entries_begin = sizeof(IndexHeader) + uint64_t(f.n_chunks) * sizeof(IndexChunk);  // 64 + 32 k: 16-byte aligned
  if (threadIdx.x == 0) {
    IndexHeader h;
    h.magic = INDEX_MAGIC;
    h.version = 1;
    h.n_chunks = f.n_chunks;
    h.n_total = f.n;
    h.file_len = file_len;
    h.chunks_offset = sizeof(IndexHeader);
    h.end_byte = file_len;
    h.reserved[0] = 0;
    h.reserved[1] = 0;
    *reinterpret_cast<IndexHeader*>(ix) = h;
  }
  const IndexChunk* src_recs = reinterpret_cast<const IndexChunk*>(pidx + f.recs_src);
  IndexChunk* recs = reinterpret_cast<IndexChunk*>(ix + sizeof(IndexHeader));
  if (f.n_chunks) {
    const IndexChunk first = src_recs[0];
    for (uint32_t k = threadIdx.x; k < f.n_chunks; k += blockDim.x) {
      IndexChunk r = src_recs[k];
      r.chunk_offset = r.chunk_offset - first.chunk_offset + f.hdr_len;
      r.entries_offset = r.entries_offset - first.entries_offset + entries_begin;
      r.out_offset -= first.out_offset;
      recs[k] = r;
    }
  }
  cta_copy_bytes(ix + entries_begin, pidx + f.entries_src, f.entries_len);
}

// One indexed file of a decompress_files call: where its records are, where they go and what to add to their offsets.
struct FileMerge {
  uint64_t recs_src;      // byte offset of the file's IndexChunk[0] in the staged index
  uint64_t list_at;       // slot of its first record in the merged list
  uint64_t chunk_add;     // the file's byte offset in src
  uint64_t entries_add;   // its index's byte offset in the staged index
  uint64_t out_add;       // element offset of its first number in the output
  uint64_t n_chunks;
};

__global__ void __launch_bounds__(256) merge_index_kernel(const uint8_t* __restrict__ idx, const FileMerge* __restrict__ tab, IndexChunk* __restrict__ list) {
  const FileMerge m = tab[blockIdx.x];
  const IndexChunk* src = reinterpret_cast<const IndexChunk*>(idx + m.recs_src);
  for (uint64_t k = threadIdx.x; k < m.n_chunks; k += blockDim.x) {
    IndexChunk r = src[k];
    r.chunk_offset += m.chunk_add;
    r.entries_offset += m.entries_add;
    r.out_offset += m.out_add;
    list[m.list_at + k] = r;
  }
}

// One indexed file of a decompress_files call, for check_index_kernel.
struct FileCheck {
  uint64_t recs_src;      // byte offset of the file's IndexChunk[0] in the staged index
  uint64_t n_chunks;
  uint64_t file_begin;    // the file's bytes in src
  uint64_t file_len;
  uint64_t idx_base;      // its index's byte offset in the staged index, and length
  uint64_t idx_len;
  uint64_t n_total;       // the index header's count
  uint32_t format_major, pad;
};
constexpr uint32_t IDX_OK = 0, IDX_COLD = 1, IDX_OUTSIDE = 2, IDX_MISALIGNED = 3;

// One CTA per indexed file: is every record inside its own file - chunk start inside the file, entries inside the file's index, numbers
// inside the file's count - so that the merged decode, whose bounds are the whole src, index and dst, cannot touch another file's bytes,
// entries or output?  out[i]: IDX_OUTSIDE if not (the file then decodes on its own, with its own bounds, as decompress_ex would),
// IDX_MISALIGNED for entries the kernels cannot load, else IDX_COLD when a format 4.x chunk meta routes the file to the catch-all decoder.
__global__ void __launch_bounds__(256) check_index_kernel(const uint8_t* __restrict__ src, const uint8_t* __restrict__ idx, uint32_t dtype,
                                                          const FileCheck* __restrict__ tab, uint32_t* __restrict__ out) {
  __shared__ uint32_t verdict;
  const FileCheck f = tab[blockIdx.x];
  if (threadIdx.x == 0) verdict = IDX_OK;
  __syncthreads();
  const IndexChunk* recs = reinterpret_cast<const IndexChunk*>(idx + f.recs_src);
  for (uint64_t k = threadIdx.x; k < f.n_chunks; k += blockDim.x) {
    const IndexChunk r = recs[k];
    uint32_t v = IDX_OK;
    const uint64_t need = uint64_t(r.n_vars) * n_batches_of(r.n) * sizeof(BatchEntry);
    if (r.n == 0 || r.n > (1u << 24) || r.n_vars == 0 || r.n_vars > uint32_t(MAX_VARS) || r.chunk_offset >= f.file_len || r.entries_offset > f.idx_len ||
        need > f.idx_len - r.entries_offset || r.out_offset > f.n_total || r.n > f.n_total - r.out_offset)
      v = IDX_OUTSIDE;
    else if ((f.idx_base + r.entries_offset) % 4 != 0)
      v = IDX_MISALIGNED;
    else if (f.format_major == 4 && r.chunk_offset + 4 < f.file_len) {
      uint64_t len = 0;
      bool cold = false;
      if (wrapped_meta_len(src + f.file_begin + r.chunk_offset + 4, f.file_len - r.chunk_offset - 4, dtype, &len, &cold) == ST_OK && cold) v = IDX_COLD;
    }
    if (v != IDX_OK) atomicMax(&verdict, v);
  }
  __syncthreads();
  if (threadIdx.x == 0) out[blockIdx.x] = verdict;
}

// The unread range of one index-free file in a speculative round: positions [begin, end) are searched for `pattern`.  block0 is the
// first block of the launch that serves the file (an exclusive scan over the files' block counts).
struct FileScan {
  uint64_t begin, end;
  uint32_t pattern, block0;
};

// Every byte position in each file's [begin, end) whose 4 bytes equal its `pattern` (a chunk's type byte and its 24-bit count - 1,
// docs/format.md:186-192).  Chunk lengths are not in a standalone file, so the index-free decompressor cannot know where chunk k + 1
// starts before it has walked chunk k - but chunks of one file almost always share their first 4 bytes (same type, same count), so
// every position that LOOKS like such a chunk start is walked speculatively, all in parallel, and the host then follows the chain of
// (start, end) pairs from the first chunk: a candidate is a real chunk start exactly when a verified chunk ends on it (host_api.cu,
// speculative_walk_rounds).  A block finds its file by binary search over block0; a thread takes 8 positions.  (position, file) pairs
// are appended in no particular order; positions past `cap` are counted but not stored.
constexpr int FIND_THREADS = 256;
constexpr int FIND_PER_THREAD = 8;
__global__ void __launch_bounds__(FIND_THREADS) find_file_starts_kernel(const uint8_t* __restrict__ src, const FileScan* __restrict__ scans, uint32_t n_scans,
                                                                       uint64_t* __restrict__ out_pos, uint32_t* __restrict__ out_file, uint32_t cap,
                                                                       uint32_t* __restrict__ count) {
  uint32_t lo = 0, hi = n_scans;  // last scan whose block0 <= blockIdx.x
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) / 2;
    if (scans[mid].block0 <= blockIdx.x) lo = mid; else hi = mid;
  }
  const FileScan s = scans[lo];
  const uint64_t p0 = s.begin + (uint64_t(blockIdx.x - s.block0) * FIND_THREADS + threadIdx.x) * FIND_PER_THREAD;
  if (p0 >= s.end) return;
  uint32_t b[FIND_PER_THREAD + 3];
#pragma unroll
  for (int i = 0; i < FIND_PER_THREAD + 3; i++) b[i] = (p0 + i < s.end + 3) ? uint32_t(src[p0 + i]) : 0x100u;  // 0x100 never matches
#pragma unroll
  for (int i = 0; i < FIND_PER_THREAD; i++) {
    const uint32_t w = b[i] | (b[i + 1] << 8) | (b[i + 2] << 16) | (b[i + 3] << 24);
    if (w == s.pattern && (b[i] | b[i + 1] | b[i + 2] | b[i + 3]) < 0x100u && p0 + i < s.end) {
      const uint32_t k = atomicAdd(count, 1u);
      if (k < cap) { out_pos[k] = p0 + i; out_file[k] = lo; }
    }
  }
}

// out[i * width + j] = src[offs[i] + j] for j < min(width, lens[i]), 0 behind that.  One warp per position.
__global__ void __launch_bounds__(256) peek_bytes_kernel(const uint8_t* __restrict__ src, const uint64_t* __restrict__ offs, const uint64_t* __restrict__ lens,
                                                         uint32_t n, uint32_t width, uint8_t* __restrict__ out) {
  const uint32_t i = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (i >= n) return;
  const uint64_t o = offs[i], l = lens[i];
  for (uint32_t j = threadIdx.x & 31; j < width; j += 32) out[size_t(i) * width + j] = j < l ? src[o + j] : 0;
}

}  // namespace pcob200
