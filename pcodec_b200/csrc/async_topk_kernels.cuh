// Kernels of pco_b200_topk_pages_async and pco_b200_topk_files_async: the k smallest or largest numbers inside a closed interval of the
// concatenation the matching decompress call writes, with their positions.  The decompress call's launches run unchanged with rows_cap in
// the role of dst_cap (and, for files, ff_map_kernel and ff_cold_list_kernel around them, as the take runs them).  Before them:
//   topk_table_kernel    (one thread) the top-k table the decode kernels read (decode_kernels.cuh, TOPK_* words): the caller's interval,
//                        k, the direction, the global threshold (all ones) and the match count (0);
// between the front end and the decode stage the histogram's gate: hg_front_*_kernel, hg_mark_*_kernel (every record flagged when the
// front end passed) and, for pages, tk_cold_list_kernel.  Then the decode stage in top-k mode: fused_narrow_kernel<L, false, true, false,
// false, false, false, true> lets an unflagged record go at once, and the TOPK instantiations keep each CTA's best matches in a candidate
// buffer in shared memory (topk_store8) whose k best, sorted, go to the record's slot when the record is done.  Cold records, decoded into
// the value staging, go through the same store by topk_cold_pages_kernel / topk_cold_files_kernel.  Then:
//   topk_merge_kernel    ceil(log2(slots)) launches, each merging pairs of sorted slot lists into the first of the pair, keeping the k best
//                        (slot 0 ends with the k best of all);
//   topk_finish_pages_kernel / topk_finish_files_kernel  (one CTA) the decision, the outputs and *n_out (0 on a failure), the status.
// Entries are ranked by (key, row), rows are distinct, so every list and the output are unique functions of the numbers, whatever the
// grids or the order the CTAs and warps ran in.
#pragma once
#include "async_histogram_kernels.cuh"

namespace pcob200 {

constexpr int TOPK_THREADS = 256;      // every topk_* kernel but the table one
constexpr uint64_t TOPK_MAX_K = 1024;  // the plans' bound on k: a CTA's buffer stays within 32 KB of shared memory

// Workspace of one in-flight pages call: the pages call's (ap_layout with dst_cap = rows_cap) | the pages status | HgState | a flag per
// page | the top-k table | value staging (rows_cap numbers of elem bytes) | the slots' entry counts (a uint32 per page) | the slots (k
// entries of 16 bytes per page).  Each region 256-byte aligned.
struct TopkLayout : ApLayout {
  uint64_t pstatus, hstate, flags, topk_table, stage, counts, lists, topk_total;
};
__host__ __device__ inline TopkLayout topk_layout(uint64_t max_pages, uint64_t rows_cap, uint64_t frame_cap, uint64_t k, uint32_t elem) {
  TopkLayout l;
  static_cast<ApLayout&>(l) = ap_layout(max_pages, rows_cap, frame_cap);
  l.pstatus = l.total;
  l.hstate = l.pstatus + async_align(sizeof(PcoB200AsyncPagesStatus));
  l.flags = l.hstate + async_align(sizeof(HgState));
  l.topk_table = l.flags + async_align(max_pages * sizeof(uint32_t));
  l.stage = l.topk_table + async_align(TOPK_WORDS * sizeof(uint64_t));
  l.counts = l.stage + async_align(rows_cap * elem);
  l.lists = l.counts + async_align(max_pages * sizeof(uint32_t));
  l.topk_total = l.lists + async_align(max_pages * k * sizeof(ulonglong2));
  return l;
}

// Workspace of one in-flight files call: the files call's (af_layout with dst_cap = rows_cap) | the files status | HgState | a flag per
// chunk | the top-k table | value staging | the slot map (max_chunks words) | the cold list (its length, then up to max_chunks records) |
// the slots' entry counts (a uint32 per chunk) | the slots (k entries of 16 bytes per chunk).
struct TopkfLayout : AfLayout {
  uint64_t fstatus, hstate, flags, topk_table, stage, slot_map, cold_list, counts, lists, topkf_total;
};
__host__ __device__ inline TopkfLayout topkf_layout(uint64_t max_files, uint64_t max_chunks, uint64_t rows_cap, uint64_t k, uint32_t elem) {
  TopkfLayout l;
  static_cast<AfLayout&>(l) = af_layout(max_files, max_chunks, rows_cap);
  l.fstatus = l.total;
  l.hstate = l.fstatus + async_align(sizeof(PcoB200AsyncFilesStatus));
  l.flags = l.hstate + async_align(sizeof(HgState));
  l.topk_table = l.flags + async_align(max_chunks * sizeof(uint32_t));
  l.stage = l.topk_table + async_align(TOPK_WORDS * sizeof(uint64_t));
  l.slot_map = l.stage + async_align(rows_cap * elem);
  l.cold_list = l.slot_map + async_align(max_chunks * sizeof(uint32_t));
  l.counts = l.cold_list + async_align((max_chunks + 1) * sizeof(uint32_t));
  l.lists = l.counts + async_align(max_chunks * sizeof(uint32_t));
  l.topkf_total = l.lists + async_align(max_chunks * k * sizeof(ulonglong2));
  return l;
}

// One thread: the top-k table from the caller's interval and the plan's k and direction.
__global__ void __launch_bounds__(32) topk_table_kernel(const uint64_t* __restrict__ interval, uint32_t k, uint32_t largest, uint64_t* __restrict__ table) {
  if (threadIdx.x != 0) return;
  table[TOPK_LO] = interval[0];
  table[TOPK_HI] = interval[1];
  table[TOPK_K] = k;
  table[TOPK_LARGEST] = largest;
  table[TOPK_GLOBAL] = ~uint64_t(0);
  table[TOPK_MATCHES] = 0;
}

// The batches of record `rec` (its numbers at rows rec.out_offset .., decoded into the value staging by a catch-all decoder) stored by the
// CTA's warps through topk_store8, then flushed to `slot`.  Every thread calls it.
template <typename L>
__device__ __forceinline__ void topk_select_in_place(const FiltStage& f, const FiltKey& key, const IndexChunk& rec, uint32_t slot,
                                                     const L* __restrict__ stage, void* buf) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  topk_clear(buf, threadIdx.x);
  __syncthreads();
  const uint32_t nb = n_batches_of(rec.n);
  for (uint32_t b = warp; b < nb; b += TOPK_THREADS / 32) {
    const uint64_t row = rec.out_offset + uint64_t(b) * BATCH_N;
    const uint32_t cnt = min(uint32_t(BATCH_N), rec.n - b * BATCH_N);
    L v[8];
#pragma unroll
    for (int e = 0; e < 8; e++) v[e] = uint32_t(lane * 8 + e) < cnt ? stage[row + lane * 8 + e] : L(0);
    topk_store8<L>(f, key, buf, row, cnt, lane, v);
  }
  __syncthreads();
  topk_flush(f, buf, slot, threadIdx.x, TOPK_THREADS);
  __syncthreads();
}

// One CTA per cold-list entry k (pages, the list kept to flagged pages), with topk_smem_bytes(k) of dynamic shared memory: the cold page,
// decoded into the value staging by ap_cold_kernel, selected in place.  Cold pages at or behind a failure were not decoded; they are left
// alone.
template <typename L>
__global__ void __launch_bounds__(TOPK_THREADS) topk_cold_pages_kernel(const ApState* __restrict__ state, const IndexChunk* __restrict__ recs,
                                                                       const uint32_t* __restrict__ cold_list, FiltStage f, uint32_t dtype,
                                                                       const L* __restrict__ stage) {
  extern __shared__ __align__(16) unsigned char topk_buf[];
  const uint64_t k = blockIdx.x;
  if (k >= state->n_cold) return;
  const uint32_t p = cold_list[k];
  if (p >= state->fail_page || p >= (state->decode_fail >> 32)) return;
  topk_select_in_place<L>(f, filt_bounds<L>(f.interval, dtype), recs[p], p, stage, topk_buf);
}

// min(max_chunks, FF_COLD_CTAS) CTAs striding over the cold list (files), with topk_smem_bytes(k) of dynamic shared memory: each record
// cold_chunks_kernel decoded into the value staging without failure, selected in place (unflagged records never reach the list: the
// fused kernel reported them done).
template <typename L>
__global__ void __launch_bounds__(TOPK_THREADS) topk_cold_files_kernel(const uint32_t* __restrict__ cold_list, const IndexChunk* __restrict__ table,
                                                                       const uint32_t* __restrict__ statuses, FiltStage f, uint32_t dtype,
                                                                       const L* __restrict__ stage) {
  extern __shared__ __align__(16) unsigned char topk_buf[];
  const uint32_t n_cold = cold_list[0];
  const FiltKey key = filt_bounds<L>(f.interval, dtype);
  for (uint32_t k = blockIdx.x; k < n_cold; k += gridDim.x) {  // uniform: every thread runs the same records
    const uint32_t r = cold_list[1 + k];
    if (statuses[r] != ST_OK) continue;
    topk_select_in_place<L>(f, key, table[r], r, stage, topk_buf);
  }
}

// The entries of the sorted list s[0 : n) that rank before x.
__device__ __forceinline__ uint32_t topk_rank_in(const ulonglong2* s, uint32_t n, ulonglong2 x) {
  uint32_t lo = 0;
  for (uint32_t len = n; len > 0;) {
    const uint32_t half = len >> 1;
    if (topk_before(s[lo + half].x, s[lo + half].y, x.x, x.y)) {
      lo += half + 1;
      len -= half + 1;
    } else {
      len = half;
    }
  }
  return lo;
}

// ceil(slots / (2 stride)) CTAs, with 2 k entries of dynamic shared memory: the sorted lists of slots a = 2 stride j and b = a + stride
// merged into slot a, keeping its k best.  Both lists are read into shared memory before slot a is written; an entry's place in the merge
// is its index plus the entries of the other list that rank before it (no two entries rank equal).
__global__ void __launch_bounds__(TOPK_THREADS) topk_merge_kernel(ulonglong2* __restrict__ lists, uint32_t* __restrict__ counts, uint64_t slots,
                                                                  uint32_t k, uint64_t stride) {
  extern __shared__ ulonglong2 topk_pair[];
  const uint64_t a = uint64_t(blockIdx.x) * 2 * stride, b = a + stride;
  if (b >= slots) return;
  const uint32_t nb = counts[b];
  if (nb == 0) return;  // uniform: every thread leaves
  const uint32_t na = counts[a];
  ulonglong2* la = lists + a * k;
  const ulonglong2* lb = lists + b * k;
  ulonglong2* sa = topk_pair;
  ulonglong2* sb = topk_pair + k;
  for (uint32_t i = threadIdx.x; i < na; i += TOPK_THREADS) sa[i] = la[i];
  for (uint32_t i = threadIdx.x; i < nb; i += TOPK_THREADS) sb[i] = lb[i];
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < na; i += TOPK_THREADS) {
    const uint32_t at = i + topk_rank_in(sb, nb, sa[i]);
    if (at < k) la[at] = sa[i];
  }
  for (uint32_t i = threadIdx.x; i < nb; i += TOPK_THREADS) {
    const uint32_t at = i + topk_rank_in(sa, na, sb[i]);
    if (at < k) la[at] = sb[i];
  }
  if (threadIdx.x == 0) counts[a] = min(k, na + nb);
}

// The outputs from slot 0 when `ok`: values (their own bits) and rows, and *n_out; only *n_out (0) otherwise.  Every thread calls it.
template <typename L>
__device__ __forceinline__ void topk_write(bool ok, const uint64_t* __restrict__ table, uint32_t dtype, const ulonglong2* __restrict__ lists,
                                           const uint32_t* __restrict__ counts, L* __restrict__ out_values, uint64_t* __restrict__ out_positions,
                                           uint64_t* __restrict__ n_out) {
  const uint32_t kind = nt_is_float(dtype) ? 2u : nt_is_signed(dtype) ? 1u : 0u;
  const bool largest = table[TOPK_LARGEST] != 0;
  const uint32_t n = ok ? counts[0] : 0u;
  for (uint32_t i = threadIdx.x; i < n; i += TOPK_THREADS) {
    const ulonglong2 e = lists[i];
    out_values[i] = topk_value<L>(e, kind, largest);
    out_positions[i] = e.y & TOPK_ROW_MASK;
  }
  if (threadIdx.x == 0) *n_out = n;
}

// One CTA: the pages top-k's outputs and status from the pages call's and slot 0.
template <typename L>
__global__ void __launch_bounds__(TOPK_THREADS) topk_finish_pages_kernel(const PcoB200AsyncPagesStatus* __restrict__ ps, const uint64_t* __restrict__ table,
                                                                         uint32_t dtype, const ulonglong2* __restrict__ lists,
                                                                         const uint32_t* __restrict__ counts, L* __restrict__ out_values,
                                                                         uint64_t* __restrict__ out_positions, uint64_t* __restrict__ n_out,
                                                                         PcoB200AsyncTopkStatus* __restrict__ out) {
  const PcoB200AsyncPagesStatus p = *ps;
  const bool ok = p.kind == PCO_B200_OK;
  topk_write<L>(ok, table, dtype, lists, counts, out_values, out_positions, n_out);
  if (threadIdx.x == 0) *out = PcoB200AsyncTopkStatus{p.kind, p.device_status, p.page, p.n_written, p.n_pages, p.frames_needed, ok ? table[TOPK_MATCHES] : 0};
}

// One CTA: the files top-k's outputs and status from the files call's and slot 0.
template <typename L>
__global__ void __launch_bounds__(TOPK_THREADS) topk_finish_files_kernel(const PcoB200AsyncFilesStatus* __restrict__ fs, const uint64_t* __restrict__ table,
                                                                         uint32_t dtype, const ulonglong2* __restrict__ lists,
                                                                         const uint32_t* __restrict__ counts, L* __restrict__ out_values,
                                                                         uint64_t* __restrict__ out_positions, uint64_t* __restrict__ n_out,
                                                                         PcoB200AsyncFilesTopkStatus* __restrict__ out) {
  const PcoB200AsyncFilesStatus f = *fs;
  const bool ok = f.kind == PCO_B200_OK;
  topk_write<L>(ok, table, dtype, lists, counts, out_values, out_positions, n_out);
  if (threadIdx.x == 0) *out = PcoB200AsyncFilesTopkStatus{f.kind, f.device_status, f.file, f.chunk, f.n_written, f.n_files, ok ? table[TOPK_MATCHES] : 0};
}

}  // namespace pcob200
