// Batched wrapped-format pages (pco/src/wrapped/: page_decompressor.rs, chunk_compressor.rs) on the device.
//
// A wrapped container stores a chunk's meta once, apart from its pages, and a page carries no preamble.  The decode kernels
// (walk_kernel, fused_narrow_kernel, symwalk_kernel + decode_kernel, cold_decode_kernel) address a chunk as ONE byte range that
// starts with the standalone preamble [type byte][n - 1, 24 bits] and continues with the chunk meta and the page: their bit offsets
// (BatchEntry::bit_pos) count from the type byte and the fused kernel copies the chunk head in one piece.  So the pages are framed
// on the device instead of teaching every kernel a second pointer:
//   frame_pages_kernel   one CTA per page: [dtype][page_n - 1][meta][page] at a 16-byte aligned offset of library scratch, and the
//                        page's meta parsed to its byte length (checked against the caller's meta_len) and its decode route;
//   chunk_refs_kernel    compress side: meta / page lengths of every CHUNKS_ONLY chunk, scanned into the caller's PcoB200PageRef;
//   split_chunks_kernel  compress side: every chunk's meta and page copied into the caller's two buffers.
// Byte copies go through cta_copy_bytes (gather_kernels.cuh): aligned 16-byte stores assembled from unaligned sources.
#pragma once
#include "../../include/pco_b200.h"
#include "cta_scan.cuh"
#include "decode_kernels.cuh"
#include "gather_kernels.cuh"

namespace pcob200 {

constexpr int WRAP_THREADS = GATHER_THREADS;  // cta_copy_bytes strides by GATHER_THREADS
constexpr uint32_t WP_COLD = 200;             // frame_pages_kernel: valid meta whose pages only the catch-all decoder takes

// One page of a pco_b200_decompress_pages call, as the host resolved it from the caller's PcoB200PageRef.
struct WrappedPage {
  uint64_t meta_off, meta_len;  // in `metas`
  uint64_t page_off, page_len;  // in `pages`
  uint64_t frame_off;           // of the framed standalone chunk in scratch (16-byte aligned)
  uint32_t page_n, pad;
};
static_assert(sizeof(WrappedPage) == 48, "page table layout");

// LSB-first bit reader over [p, p + avail) (docs/format.md: bits fill a byte from its low end); bytes past the end read as 0.
struct MetaBits {
  const uint8_t* p;
  uint64_t avail;
  uint64_t pos;
  __host__ __device__ uint64_t read(uint32_t nb) {
    uint64_t v = 0;
    for (uint32_t i = 0; i < nb; i++) {
      const uint64_t bit = pos + i;
      if ((bit >> 3) < avail) v |= uint64_t((p[bit >> 3] >> (bit & 7)) & 1) << i;
    }
    pos += nb;
    return v;
  }
};

// Byte length of the chunk meta at p (metadata/chunk.rs:127-174, mode.rs:102-167, delta_encoding.rs:118-202,
// chunk_latent_var.rs:102-143; format 4.x), for every mode and delta encoding: the same fields cold_decode_kernel reads, skipped
// by their sizes.  *cold: the fast kernels decline the chunk (Dict, Lookback, Conv1, secondary_uses_delta, tables above 2^10 states
// or 256 bins, FloatMult below 32 bits).  Only an unknown mode or delta variant makes the length undefined (ST_CORRUPTION); every
// other defect is reported by the kernels that decode the chunk.  *mode and *variant, when asked for, are set as soon as they are read.
// Bytes past avail read as 0, so a meta cut short parses to a length past avail.
__host__ __device__ inline uint32_t wrapped_meta_len(const uint8_t* p, uint64_t avail, uint32_t dtype, uint64_t* len, bool* cold,
                                                     uint32_t* mode = nullptr, uint32_t* variant = nullptr) {
  const uint32_t nb = nt_bits(dtype);
  MetaBits r{p, avail, 0};
  bool c = false;
  uint32_t n_vars = 1, prim_bits = nb;
  const uint32_t m = uint32_t(r.read(4));
  if (mode) *mode = m;
  switch (m) {
    case MODE_CLASSIC: break;
    case MODE_INT_MULT: r.pos += nb; n_vars = 2; break;
    case MODE_FLOAT_MULT: r.pos += nb; n_vars = 2; c |= nb < 32; break;
    case MODE_FLOAT_QUANT: r.pos += 8; n_vars = 2; break;
    case MODE_DICT: {
      const uint64_t dict_len = r.read(25);
      r.pos = (r.pos + 7) & ~uint64_t(7);
      r.pos += dict_len * nb;
      prim_bits = 32;  // the primary latents are dictionary indices
      c = true;
      break;
    }
    default: return ST_CORRUPTION;
  }
  const uint32_t dv = uint32_t(r.read(4));
  if (variant) *variant = dv;
  uint32_t lookback = 0;
  if (dv == 1) {
    r.pos += 3;                               // order
    c |= r.read(1) != 0 && n_vars > 1;        // secondary_uses_delta
  } else if (dv == 2) {
    r.pos += 5 + 4;                           // window_n_log - 1, state_n_log
    r.pos += 1;                               // secondary_uses_delta
    lookback = 1;
    c = true;
  } else if (dv == 3) {
    r.pos += 5 + 64;                          // quantization, bias
    const uint32_t order = 1 + uint32_t(r.read(5));
    r.pos += 32ull * order;                   // weights
    c = true;
  } else if (dv != 0) {
    return ST_CORRUPTION;
  }
  // latent vars: [lookback (32-bit latents)], primary, [secondary]
  for (uint32_t v = 0; v < n_vars + lookback; v++) {
    const uint32_t lb = (lookback && v == 0) ? 32u : v == lookback ? prim_bits : nb;
    const uint32_t size_log = uint32_t(r.read(4)), n_bins = uint32_t(r.read(15));
    c |= size_log > uint32_t(SMALL_MAX_SIZE_LOG) || n_bins > uint32_t(SMALL_MAX_BINS);
    r.pos += uint64_t(n_bins) * (size_log + lb + offset_bits_bits(lb));
  }
  *len = (r.pos + 7) >> 3;
  *cold = c;
  return ST_OK;
}

// One CTA per page: the framed standalone chunk, and the page's route in pstat[i] - ST_OK (fast kernels), WP_COLD (catch-all decoder),
// ST_INVALID_ARGUMENT (meta_len is not the length its meta parses to) or ST_CORRUPTION (meta of unknown layout).  The host has
// checked every range against metas_len / pages_len; the meta parse reads at most to the end of `metas`.
__global__ void __launch_bounds__(WRAP_THREADS) frame_pages_kernel(const uint8_t* __restrict__ metas, uint64_t metas_len, const uint8_t* __restrict__ pages,
                                                                   uint32_t dtype, const WrappedPage* __restrict__ tab, uint8_t* __restrict__ frames,
                                                                   uint32_t* __restrict__ pstat) {
  const WrappedPage pg = tab[blockIdx.x];
  uint8_t* f = frames + pg.frame_off;
  if (threadIdx.x == 0) {
    const uint32_t nm1 = pg.page_n - 1;
    f[0] = uint8_t(dtype);
    f[1] = uint8_t(nm1);
    f[2] = uint8_t(nm1 >> 8);
    f[3] = uint8_t(nm1 >> 16);
  } else if (threadIdx.x == 32) {  // a warp of its own: the byte copies below do not wait for the parse
    uint64_t len = 0;
    bool cold = false;
    uint32_t st = wrapped_meta_len(metas + pg.meta_off, metas_len - pg.meta_off, dtype, &len, &cold);
    if (st == ST_OK) st = len != pg.meta_len ? ST_INVALID_ARGUMENT : cold ? WP_COLD : ST_OK;
    pstat[blockIdx.x] = st;
  }
  cta_copy_bytes(f + 4, metas + pg.meta_off, pg.meta_len);
  cta_copy_bytes(f + 4 + pg.meta_len, pages + pg.page_off, pg.page_len);
}

// Compress side, one CTA: chunk i of a CHUNKS_ONLY compress is [type byte][n - 1][meta][page] at its IndexChunk's chunk_offset and
// sizes[i] bytes long (chunk_sizes_kernel).  Its meta length is parsed here; the exclusive scans of meta and page lengths give the
// refs, and tot[0], tot[1] the byte totals.  *err is set if a chunk does not parse (it cannot: the chunks are this library's own).
__global__ void __launch_bounds__(1024) chunk_refs_kernel(const uint8_t* __restrict__ file, const IndexChunk* __restrict__ chunks, const uint64_t* __restrict__ sizes,
                                                          uint32_t n_chunks, uint32_t dtype, PcoB200PageRef* __restrict__ refs, uint64_t* __restrict__ tot,
                                                          uint32_t* __restrict__ err) {
  for (uint32_t i = threadIdx.x; i < n_chunks; i += 1024) {
    const uint64_t sz = sizes[i];
    uint64_t ml = 0, pl = 0;
    bool cold = false;
    const uint32_t st = sz >= 4 ? wrapped_meta_len(file + chunks[i].chunk_offset + 4, sz - 4, dtype, &ml, &cold) : ST_CORRUPTION;
    if (st != ST_OK || ml > sz - 4) { *err = ST_CORRUPTION; ml = 0; }
    else pl = sz - 4 - ml;
    refs[i] = PcoB200PageRef{0, ml, 0, pl, chunks[i].n};
  }
  __syncthreads();
  uint64_t total[2] = {};
  cta_scan_inplace<1024, 1>(
      n_chunks, [&](uint64_t i, int k) { return k ? refs[i].page_len : refs[i].meta_len; },
      [&](uint64_t i, int k, uint64_t v) { (k ? refs[i].page_offset : refs[i].meta_offset) = v; }, total);
  if (threadIdx.x == 0) { tot[0] = total[0]; tot[1] = total[1]; }
}

// One CTA per chunk: its meta to metas + meta_offset, its page to pages + page_offset - unless the totals chunk_refs_kernel found do
// not fit the capacities (or the refs do not fit, refs_fit = 0, or a chunk did not parse): then nothing is written.
__global__ void __launch_bounds__(WRAP_THREADS) split_chunks_kernel(const uint8_t* __restrict__ file, const IndexChunk* __restrict__ chunks,
                                                                    const PcoB200PageRef* __restrict__ refs, const uint64_t* __restrict__ tot,
                                                                    const uint32_t* __restrict__ err, uint64_t metas_cap, uint64_t pages_cap, uint32_t refs_fit,
                                                                    uint8_t* __restrict__ metas, uint8_t* __restrict__ pages) {
  if (!refs_fit || *err != 0 || tot[0] > metas_cap || tot[1] > pages_cap) return;
  const PcoB200PageRef r = refs[blockIdx.x];
  const uint8_t* c = file + chunks[blockIdx.x].chunk_offset + 4;
  cta_copy_bytes(metas + r.meta_offset, c, r.meta_len);
  cta_copy_bytes(pages + r.page_offset, c + r.meta_len, r.page_len);
}

}  // namespace pcob200
