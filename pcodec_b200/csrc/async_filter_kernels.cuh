// Kernels of pco_b200_filter_pages_async: the pages pco_b200_decompress_pages_async decodes, with only the numbers inside a closed
// interval written out, in row order, with their positions in the pages' concatenation.  The front end (ap_pages_kernel .. ap_rewalk_kernel,
// async_pages_kernels.cuh) runs unchanged with rows_cap in the role of dst_cap; what changes is the store side of the decode:
//   fused_narrow_kernel<L, false, true>, symwalk_kernel<false>, decode_kernel<L, 1 / 2, false, true>  the FILT instantiations: each batch's
//                        matches and their in-batch offsets staged compactly in its own slot, and the batch's count (filt_store8,
//                        decode_kernels.cuh);
//   ap_cold_kernel<L>    unchanged, decoding the cold pages into the value staging (each page's numbers at its rows);
//   fl_cold_kernel<L>    one CTA per cold-list entry: the cold page's batches filtered in place into the same slots;
//   ap_finish_kernel     unchanged, into the workspace: the pages call's outcome, whose refusals this call keeps;
//   fl_count_kernel      per CTA of FL_THREADS slots, the sum of their counts;
//   fl_finish_kernel     (one CTA) the CTA sums scanned into CTA offsets (cta_scan_inplace), the total against out_cap, the
//                        PcoB200AsyncFilterStatus and *n_matches;
//   fl_gather_kernel     per CTA of FL_THREADS slots, each slot's output offset; its warps copy the slots' matches to out_values and
//                        build out_positions (row + offset), the first out_cap matches only.
// The value staging is rows_cap numbers and the offset staging rows_cap bytes; the counts are cleared by a memset before the decode.
#pragma once
#include "async_pages_kernels.cuh"

namespace pcob200 {

constexpr int FL_THREADS = 256;        // slots per CTA of fl_count_kernel and fl_gather_kernel
constexpr int FL_SCAN_THREADS = 1024;  // fl_finish_kernel

// decided by fl_finish_kernel
struct FlState {
  uint32_t ok, reserved;  // 1: the pages decoded, fl_gather_kernel writes the matches
  uint64_t n_matches;     // the total, in row order
};

// Batch slots of a plan: the slot of batch b of page p, whose numbers start at row O, is O / 256 + p + b; over any batch within rows_cap
// and max_pages the largest is below floor(rows_cap / 256) + max_pages.
__host__ __device__ inline uint64_t fl_slots(uint64_t max_pages, uint64_t rows_cap) { return rows_cap / BATCH_N + max_pages; }

// Workspace of one in-flight call: the pages call's (ap_layout with dst_cap = rows_cap) | the pages status | FlState | per slot: count,
// row | CTA sums of the counts | value staging (rows_cap numbers of elem bytes) | offset staging (rows_cap bytes).  Each region 256-byte
// aligned.
struct FlLayout : ApLayout {
  uint64_t pstatus, fstate, counts, rows, cparts, stage, soffs, fl_total;
};
__host__ __device__ inline FlLayout fl_layout(uint64_t max_pages, uint64_t rows_cap, uint64_t frame_cap, uint32_t elem) {
  FlLayout l;
  static_cast<ApLayout&>(l) = ap_layout(max_pages, rows_cap, frame_cap);
  const uint64_t slots = fl_slots(max_pages, rows_cap);
  l.pstatus = l.total;
  l.fstate = l.pstatus + async_align(sizeof(PcoB200AsyncPagesStatus));
  l.counts = l.fstate + async_align(sizeof(FlState));
  l.rows = l.counts + async_align(slots * sizeof(uint32_t));
  l.cparts = l.rows + async_align(slots * sizeof(uint64_t));
  l.stage = l.cparts + async_align(ctas_of<FL_THREADS>(slots) * sizeof(uint64_t));
  l.soffs = l.stage + async_align(rows_cap * elem);
  l.fl_total = l.soffs + async_align(rows_cap);
  return l;
}

// The batches of record `p` (its numbers at rows rec.out_offset .., decoded into the value staging by a catch-all decoder) filtered in
// place by the CTA's warps: a warp reads its batch into registers before filt_store8 writes the matches back at the batch's start, into
// slot rec.out_offset / 256 + p + b.  AGG: agg_store8 reduces the batch into the slot instead (the aggregate calls).
template <typename L, bool AGG = false>
__device__ __forceinline__ void fl_filter_in_place(const FiltStage& f, const FiltKey& key, const IndexChunk& rec, uint64_t p, L* __restrict__ stage) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t nb = n_batches_of(rec.n);
  for (uint32_t b = warp; b < nb; b += FL_THREADS / 32) {
    const uint64_t row = rec.out_offset + uint64_t(b) * BATCH_N;
    const uint32_t cnt = min(uint32_t(BATCH_N), rec.n - b * BATCH_N);
    L r[8];
#pragma unroll
    for (int e = 0; e < 8; e++) r[e] = uint32_t(lane * 8 + e) < cnt ? stage[row + lane * 8 + e] : L(0);
    if constexpr (AGG) {
      agg_store8<L>(f, key, rec.out_offset / BATCH_N + p + b, cnt, lane, r);
    } else {
      __syncwarp();
      filt_store8<L>(f, key, stage, row, rec.out_offset / BATCH_N + p + b, cnt, lane, r);
    }
  }
}

// One CTA per cold-list entry k: the cold page, decoded into the value staging by ap_cold_kernel, filtered in place.  Cold pages at or
// behind a failure were not decoded; their staging is left alone (a failed call gathers nothing).  AGG: reduced into the slots instead.
template <typename L, bool AGG = false>
__global__ void __launch_bounds__(FL_THREADS) fl_cold_kernel(const ApState* __restrict__ state, const IndexChunk* __restrict__ recs,
                                                             const uint32_t* __restrict__ cold_list, FiltStage f, uint32_t dtype, L* __restrict__ stage) {
  const uint64_t k = blockIdx.x;
  if (k >= state->n_cold) return;
  const uint32_t p = cold_list[k];
  if (p >= state->fail_page || p >= (state->decode_fail >> 32)) return;
  const IndexChunk rec = recs[p];
  const FiltKey key = filt_bounds<L>(f.interval, dtype);
  fl_filter_in_place<L, AGG>(f, key, rec, p, stage);
}

// ceil(slots / FL_THREADS) CTAs: the sum of each CTA's counts.
__global__ void __launch_bounds__(FL_THREADS) fl_count_kernel(const uint32_t* __restrict__ counts, uint64_t slots, uint64_t* __restrict__ parts) {
  const uint64_t i = uint64_t(blockIdx.x) * FL_THREADS + threadIdx.x;
  uint64_t tot;
  block_exscan<FL_THREADS>(uint64_t(i < slots ? counts[i] : 0u), &tot);
  if (threadIdx.x == 0) parts[blockIdx.x] = tot;
}

// The step both finish kernels share, on one CTA of FL_SCAN_THREADS: the CTA sums scanned into CTA offsets (in place); returns the total.
__device__ __forceinline__ uint64_t fl_scan_parts(uint64_t* __restrict__ parts, uint64_t n_parts) {
  uint64_t total[1] = {0};
  cta_scan_inplace<FL_SCAN_THREADS, 1>(
      n_parts, [&](uint64_t c, int) { return parts[c]; }, [&](uint64_t c, int, uint64_t v) { parts[c] = v; }, total);
  return total[0];
}

// Thread 0 of a finish kernel, with the upstream call's outcome already in r (kind and device_status): no matches when that call failed
// (ok false), else `total` matches of which out_cap at most are written, PCO_B200_IO (PCO_B200_FILTER_OUT_FULL) when there are more.
// Writes the FlState fl_gather_kernel reads and *n_matches.
template <typename S>
__device__ __forceinline__ void fl_decide(bool ok, uint64_t total, uint64_t out_cap, S& r, FlState* __restrict__ fs, uint64_t* __restrict__ n_matches) {
  r.n_matches = 0;
  r.matches_needed = 0;
  if (ok) {
    r.matches_needed = total;
    r.n_matches = min(total, out_cap);
    if (total > out_cap) {
      r.kind = PCO_B200_IO;
      r.device_status = PCO_B200_FILTER_OUT_FULL;
    }
  }
  *fs = FlState{ok ? 1u : 0u, 0u, r.n_matches};
  *n_matches = r.n_matches;
}

// One CTA: the CTA sums scanned into CTA offsets (in place) and the total; then, from the pages call's outcome, the status: a refusal or
// failure as that call reports it (no matches), else success, or PCO_B200_IO when the matches outnumber out_cap (out_cap of them written).
__global__ void __launch_bounds__(FL_SCAN_THREADS) fl_finish_kernel(const PcoB200AsyncPagesStatus* __restrict__ ps, uint64_t* __restrict__ parts,
                                                                    uint64_t n_parts, uint64_t out_cap, FlState* __restrict__ fs,
                                                                    uint64_t* __restrict__ n_matches, PcoB200AsyncFilterStatus* __restrict__ out) {
  const uint64_t total = fl_scan_parts(parts, n_parts);
  if (threadIdx.x != 0) return;
  const PcoB200AsyncPagesStatus p = *ps;
  PcoB200AsyncFilterStatus r;
  r.kind = p.kind;
  r.device_status = p.device_status;
  r.page = p.page;
  r.n_written = p.n_written;
  r.n_pages = p.n_pages;
  r.frames_needed = p.frames_needed;
  fl_decide(p.kind == PCO_B200_OK, total, out_cap, r, fs, n_matches);
  *out = r;
}

// ceil(slots / FL_THREADS) CTAs: each slot's output offset (its CTA's offset and the CTA's exclusive scan of the counts); then warp w
// copies the matches of the CTA's slots 32 w .. 32 w + 31, one slot after another, a lane per match: the staged value, and the row plus
// the staged offset as the position.  Offsets at or past out_cap are not written.
template <typename L>
__global__ void __launch_bounds__(FL_THREADS) fl_gather_kernel(const FlState* __restrict__ fs, const uint32_t* __restrict__ counts,
                                                               const uint64_t* __restrict__ rows, const uint64_t* __restrict__ parts, uint64_t slots,
                                                               const L* __restrict__ stage, const uint8_t* __restrict__ soffs, uint64_t out_cap,
                                                               L* __restrict__ out_values, uint64_t* __restrict__ out_positions) {
  __shared__ uint64_t s_off[FL_THREADS];
  __shared__ uint32_t s_cnt[FL_THREADS];
  if (!fs->ok) return;  // uniform: every thread leaves
  const uint32_t tid = threadIdx.x;
  const uint64_t i = uint64_t(blockIdx.x) * FL_THREADS + tid;
  const uint32_t c = i < slots ? counts[i] : 0u;
  uint64_t tot;
  s_off[tid] = parts[blockIdx.x] + block_exscan<FL_THREADS>(uint64_t(c), &tot);
  s_cnt[tid] = c;
  __syncthreads();
  const uint32_t lane = tid & 31, warp = tid >> 5;
  for (uint32_t s = warp * 32; s < warp * 32 + 32; s++) {
    const uint32_t cnt = s_cnt[s];
    const uint64_t off = s_off[s];
    if (cnt == 0 || off >= out_cap) continue;
    const uint64_t row = rows[uint64_t(blockIdx.x) * FL_THREADS + s];
    for (uint32_t j = lane; j < cnt && off + j < out_cap; j += 32) {
      out_values[off + j] = stage[row + j];
      out_positions[off + j] = row + soffs[row + j];
    }
  }
}

}  // namespace pcob200
