// The one cross-rank step of the sharded path (SURVEY.md 8e): chunks are compressed where they live - chunk c of the logical file on
// rank c mod G - and every rank ends up holding the whole standalone file
//     header | chunk_0 | chunk_1 | ... | 0x00          (pco/src/standalone/simple.rs:62-91, compressor.rs:85-105,157)
// byte-identical to what one GPU (or the reference) writes for the same numbers.  The exchange is done by the compressing GPUs
// themselves: after a device-side scan of all ranks' chunk sizes (no size ever visits the host) each rank STORES its chunks
// straight into every rank's file buffer at their final offsets - peer memory mapped over NVLink / NVSwitch (cudaIpc handles
// exchanged once at set-up), 16-byte stores, no staging copy and no second pass to put chunks in order.
#pragma once
#include "codec_common.cuh"

namespace pcob200 {

constexpr int GATHER_THREADS = 256;
constexpr int GATHER_MAX_WORLD = 16;

struct GatherPeers {
  uint8_t* file[GATHER_MAX_WORLD];  // every rank's file buffer as mapped in THIS process (file[rank] is local memory)
};

// sizes[i] of this rank's chunks from the side index of its compress (chunk offsets are in the IndexChunk records)
__global__ void chunk_sizes_kernel(const uint8_t* __restrict__ index, uint64_t index_len, uint64_t* __restrict__ sizes, uint32_t n_chunks, uint32_t* __restrict__ err) {
  const IndexHeader* ih = reinterpret_cast<const IndexHeader*>(index);
  if (index_len < sizeof(IndexHeader) || ih->magic != INDEX_MAGIC || ih->n_chunks != n_chunks || ih->chunks_offset > index_len ||
      uint64_t(n_chunks) > (index_len - ih->chunks_offset) / sizeof(IndexChunk)) {
    // an index that is not this compress's: sizes no file buffer can hold, so that the gather refuses (PCO_B200_IO) instead of copying garbage
    if (blockIdx.x == 0 && threadIdx.x == 0) *err = ST_INVALID_ARGUMENT;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_chunks; i += gridDim.x * blockDim.x) sizes[i] = uint64_t(1) << 56;
    return;
  }
  const IndexChunk* ic = reinterpret_cast<const IndexChunk*>(index + ih->chunks_offset);
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_chunks; i += gridDim.x * blockDim.x) {
    const uint64_t end = ih->end_byte ? ih->end_byte - 1 : ih->file_len;  // a whole standalone file ends with its terminator byte, bare chunks do not
    const uint64_t a = ic[i].chunk_offset, b = i + 1 < n_chunks ? ic[i + 1].chunk_offset : end;
    sizes[i] = b - a;
  }
}

// One CTA: file offset of each of this rank's chunks and the file length.
//   all_sizes[r * n_local + i] = bytes of rank r's i-th chunk = chunk i * G + r of the file (ranks with fewer chunks report 0).
//   src_off[i] = offset in this rank's own chunk bytes; dst_off[i] = offset in the file.
__global__ void __launch_bounds__(1024) gather_offsets_kernel(const uint64_t* __restrict__ all_sizes, uint32_t world, uint32_t rank, uint32_t n_local, uint64_t header_len,
                                                              uint64_t* __restrict__ src_off, uint64_t* __restrict__ dst_off, uint64_t* __restrict__ file_len) {
  __shared__ uint64_t warp_tot[2][32];
  __shared__ uint64_t carry[2];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) { carry[0] = header_len; carry[1] = 0; }
  __syncthreads();
  for (uint32_t base = 0; base < n_local; base += 1024) {
    const uint32_t i = base + tid;
    uint64_t row = 0, before_me = 0, mine = 0;
    if (i < n_local) {
      for (uint32_t r = 0; r < world; r++) {
        const uint64_t sz = all_sizes[size_t(r) * n_local + i];
        if (r < rank) before_me += sz;
        if (r == rank) mine = sz;
        row += sz;
      }
    }
    // inclusive scans of `row` (file) and `mine` (local) over the tile
    uint64_t a = row, b = mine;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint64_t oa = __shfl_up_sync(0xffffffffu, a, d), ob = __shfl_up_sync(0xffffffffu, b, d);
      if (lane >= d) { a += oa; b += ob; }
    }
    if (lane == 31) { warp_tot[0][warp] = a; warp_tot[1][warp] = b; }
    __syncthreads();
    if (warp == 0) {
      uint64_t ta = warp_tot[0][lane], tb = warp_tot[1][lane];
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint64_t oa = __shfl_up_sync(0xffffffffu, ta, d), ob = __shfl_up_sync(0xffffffffu, tb, d);
        if (lane >= d) { ta += oa; tb += ob; }
      }
      warp_tot[0][lane] = ta;
      warp_tot[1][lane] = tb;
    }
    __syncthreads();
    const uint64_t pa = (warp ? warp_tot[0][warp - 1] : 0) + carry[0], pb = (warp ? warp_tot[1][warp - 1] : 0) + carry[1];
    if (i < n_local) {
      dst_off[i] = pa + (a - row) + before_me;
      src_off[i] = pb + (b - mine);
    }
    __syncthreads();
    if (tid == 0) { carry[0] += warp_tot[0][31]; carry[1] += warp_tot[1][31]; }
    __syncthreads();
  }
  if (tid == 0) *file_len = carry[0] + 1;  // + the terminator byte (compressor.rs:157)
}

// `n` bytes from src to dst by one CTA, any alignment on either side.  dst is written in aligned 16-byte stores (the unit NVLink moves
// well); each is assembled from two ALIGNED 16-byte loads of the source (the second one is the next thread's first: an L1 hit) with a
// word select and a funnel shift.  A thread keeps GATHER_UNROLL units in flight - the loop is bound by the latency of its loads, the
// stores are posted - which is what lets a few CTAs fill the links (four units per thread and iteration nearly doubled a CTA's rate over one).
#ifndef PCOB_GATHER_UNROLL
#define PCOB_GATHER_UNROLL 8
#endif
constexpr int GATHER_UNROLL = PCOB_GATHER_UNROLL;

__device__ __forceinline__ uint4 ld16(const uint4* p) {
  uint32_t x, y, z, w;
  asm volatile("ld.global.nc.L1::evict_last.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(x), "=r"(y), "=r"(z), "=r"(w) : "l"(p));
  return make_uint4(x, y, z, w);
}
__device__ __forceinline__ uint4 splice16(uint4 a, uint4 b, uint32_t ws, uint32_t bs) {
  // bytes [4 ws + bs / 8, + 16) of the 32 bytes a | b
  uint32_t w0 = a.x, w1 = a.y, w2 = a.z, w3 = a.w, w4 = b.x, w5 = b.y, w6 = b.z, w7 = b.w;
  if (ws & 2) { w0 = w2; w1 = w3; w2 = w4; w3 = w5; w4 = w6; w5 = w7; }
  if (ws & 1) { w0 = w1; w1 = w2; w2 = w3; w3 = w4; w4 = w5; }
  return make_uint4(__funnelshift_r(w0, w1, bs), __funnelshift_r(w1, w2, bs), __funnelshift_r(w2, w3, bs), __funnelshift_r(w3, w4, bs));
}

__device__ __forceinline__ void cta_copy_bytes(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, uint64_t n) {
  const int tid = threadIdx.x;
  const uint64_t head = min(n, uint64_t((16 - (reinterpret_cast<uintptr_t>(dst) & 15)) & 15));
  if (uint64_t(tid) < head) dst[tid] = src[tid];
  const uint8_t* s = src + head;
  const uint32_t mis = uint32_t(reinterpret_cast<uintptr_t>(s) & 15);
  // units whose two loads stay inside [src, src + n) rounded out to 16-byte blocks; the rest (< 32 bytes) goes byte by byte
  uint64_t body = (n - head) / 16;
  if (mis != 0 && body > 0) body -= 1;
  uint4* __restrict__ d16 = reinterpret_cast<uint4*>(dst + head);
  const uint4* __restrict__ s16 = reinterpret_cast<const uint4*>(s - mis);
  const uint32_t ws = mis >> 2, bs = (mis & 3) * 8;
  uint64_t j = tid;
  for (; j + uint64_t(GATHER_UNROLL - 1) * GATHER_THREADS < body; j += uint64_t(GATHER_UNROLL) * GATHER_THREADS) {
    uint4 a[GATHER_UNROLL], b[GATHER_UNROLL];
#pragma unroll
    for (int u = 0; u < GATHER_UNROLL; u++) {
      a[u] = ld16(s16 + j + uint64_t(u) * GATHER_THREADS);
      b[u] = mis ? ld16(s16 + j + uint64_t(u) * GATHER_THREADS + 1) : a[u];
    }
#pragma unroll
    for (int u = 0; u < GATHER_UNROLL; u++) {
      const uint4 v = mis ? splice16(a[u], b[u], ws, bs) : a[u];
      asm volatile("st.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(d16 + j + uint64_t(u) * GATHER_THREADS), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
    }
  }
  for (; j < body; j += GATHER_THREADS) {
    const uint4 a = ld16(s16 + j);
    const uint4 v = mis ? splice16(a, ld16(s16 + j + 1), ws, bs) : a;
    asm volatile("st.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(d16 + j), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
  }
  const uint64_t done = head + body * 16;  // n - done < 32
  if (uint64_t(tid) < n - done) dst[done + tid] = src[done + tid];
}

// Persistent CTAs over the (chunk, peer) pairs: chunk i of this rank goes to file offset dst_off[i] of EVERY rank's buffer.
// Consecutive work items of a CTA target different peers, so the outgoing stores spread over all NVLink ports at any moment.
__global__ void __launch_bounds__(GATHER_THREADS) push_pages_kernel(const uint8_t* __restrict__ chunks, const uint64_t* __restrict__ all_sizes, const uint64_t* __restrict__ src_off,
                                                                    const uint64_t* __restrict__ dst_off, const uint64_t* __restrict__ file_len, GatherPeers peers, uint32_t world,
                                                                    uint32_t rank, uint32_t n_local, uint64_t file_cap, const uint8_t* __restrict__ header, uint32_t header_len,
                                                                    uint32_t* __restrict__ err) {
  const uint64_t total = *file_len;
  if (total > file_cap) {
    if (blockIdx.x == 0 && threadIdx.x == 0) *err = ST_INSUFFICIENT_DATA;  // reported as "file buffer too small" by the host
    return;
  }
  if (blockIdx.x == 0) {  // header and terminator of this rank's own copy of the file
    uint8_t* mine = peers.file[rank];
    for (uint32_t i = threadIdx.x; i < header_len; i += GATHER_THREADS) mine[i] = header[i];
    if (threadIdx.x == 0) mine[total - 1] = 0;
  }
  const uint64_t items = uint64_t(n_local) * world;
  for (uint64_t it = blockIdx.x; it < items; it += gridDim.x) {
    const uint32_t i = uint32_t(it / world);
    const uint32_t p = uint32_t((it + i + rank) % world);
    const uint64_t sz = all_sizes[size_t(rank) * n_local + i];
    if (sz == 0) continue;
    cta_copy_bytes(peers.file[p] + dst_off[i], chunks + src_off[i], sz);
  }
}

}  // namespace pcob200
