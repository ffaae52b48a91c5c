// Kernels of pco_b200_histogram_pages_async and pco_b200_histogram_files_async: how many numbers of the concatenation the matching
// decompress call writes fall in each bucket of B caller-given edges, per page / file and in all.  The decompress call's launches run
// unchanged with rows_cap in the role of dst_cap (and, for files, ff_map_kernel and ff_cold_list_kernel around them, as the take runs
// them).  Between its front end and its decode stage runs the plan:
//   hg_front_pages_kernel / hg_front_files_kernel  (one thread) the HgState: whether the front end passed;
//   hg_check_kernel<L>   the edges' keys staged in the workspace behind B (the edge table the decode kernels read), and the lowest index
//                        of an edge that is a NaN or not above the one before it;
//   hg_mark_pages_kernel / hg_mark_files_kernel  when the gate passes, each record's group + 1 (page p: p + 1; a chunk: its file + 1),
//                        read by the decode kernels as a touched flag and as the row to flush into; on a refusal every record stays 0;
//   tk_cold_list_kernel  (pages, the take's) the cold list kept to the flagged pages.
// Then the decode stage in histogram mode: fused_narrow_kernel<L, false, true, false, false, false, true> lets an unflagged record go at
// once, and the HIST instantiations count each batch's numbers into CTA-private counters (hist_store8, decode_kernels.cuh) that the CTA
// adds to its group's row when the record is done.  Cold records, decoded into the value staging, are counted by hg_cold_pages_kernel /
// hg_cold_files_kernel through the same hist_store8 and flush.  Then:
//   hg_rows_kernel       a (column tile, group share) grid: on success the group rows copied to hists and each share's column sums
//                        added to the workspace's sum row by atomics;
//   hg_finish_pages_kernel / hg_finish_files_kernel  (one CTA) the decision, *total from the sum row (zeros on a failure), the status.
// Counts are exact integers met by atomics, so nothing here depends on order or grids.
#pragma once
#include "async_take_kernels.cuh"

namespace pcob200 {

constexpr int HG_THREADS = 256;            // every hg_* kernel but the front ones
constexpr uint64_t HG_MAX_BUCKETS = 4096;  // the plans' bound on B: a CTA's counters stay within 4 (4096 + 3) bytes of shared memory
constexpr uint64_t HG_MAX_CTAS = 4096;     // the largest grid of hg_mark_*_kernel; their CTAs stride
constexpr uint32_t HG_ROW_SHARES = 512;    // hg_rows_kernel's most group shares (gridDim.y)

// decided by the plan kernels, in launch order
struct HgState {
  uint32_t front_ok, reserved;    // 1: the decompress call's front end refused nothing (pages: nor did the walk)
  unsigned long long nbad_edge;   // ~j of the lowest j whose edge is a NaN or not above edge j - 1 (0: none)
};
static_assert(sizeof(HgState) == 16, "workspace layout");

__device__ __forceinline__ bool hg_gate(const HgState& t) { return t.front_ok && t.nbad_edge == 0; }

// Group shares of hg_rows_kernel (gridDim.y) for up to max_groups groups: about 32 groups each.
__host__ __device__ inline uint32_t hg_row_shares(uint64_t max_groups) {
  const uint64_t k = (max_groups + 31) / 32;
  return uint32_t(k < 1 ? 1 : k > HG_ROW_SHARES ? HG_ROW_SHARES : k);
}

// Workspace of one in-flight pages call: the pages call's (ap_layout with dst_cap = rows_cap) | the pages status | HgState | group + 1 per
// page | the edge table (B + 2 words) | value staging (rows_cap numbers of elem bytes) | the pages' rows (W = B + 3 words each) | the sum
// row (W words).  Each region 256-byte aligned.
struct HgLayout : ApLayout {
  uint64_t pstatus, hstate, flags, edges, stage, rows, sums, hg_total;
};
__host__ __device__ inline HgLayout hg_layout(uint64_t max_pages, uint64_t rows_cap, uint64_t frame_cap, uint64_t n_buckets, uint32_t elem) {
  HgLayout l;
  static_cast<ApLayout&>(l) = ap_layout(max_pages, rows_cap, frame_cap);
  const uint64_t w = n_buckets + 3;
  l.pstatus = l.total;
  l.hstate = l.pstatus + async_align(sizeof(PcoB200AsyncPagesStatus));
  l.flags = l.hstate + async_align(sizeof(HgState));
  l.edges = l.flags + async_align(max_pages * sizeof(uint32_t));
  l.stage = l.edges + async_align((n_buckets + 2) * sizeof(uint64_t));
  l.rows = l.stage + async_align(rows_cap * elem);
  l.sums = l.rows + async_align(max_pages * w * sizeof(uint64_t));
  l.hg_total = l.sums + async_align(w * sizeof(uint64_t));
  return l;
}

// Workspace of one in-flight files call: the files call's (af_layout with dst_cap = rows_cap) | the files status | HgState | group + 1
// per chunk | the edge table | value staging | the slot map (max_chunks words) | the cold list (its length, then up to max_chunks records)
// | the files' rows | the sum row.
struct HgfLayout : AfLayout {
  uint64_t fstatus, hstate, flags, edges, stage, slot_map, cold_list, rows, sums, hgf_total;
};
__host__ __device__ inline HgfLayout hgf_layout(uint64_t max_files, uint64_t max_chunks, uint64_t rows_cap, uint64_t n_buckets, uint32_t elem) {
  HgfLayout l;
  static_cast<AfLayout&>(l) = af_layout(max_files, max_chunks, rows_cap);
  const uint64_t w = n_buckets + 3;
  l.fstatus = l.total;
  l.hstate = l.fstatus + async_align(sizeof(PcoB200AsyncFilesStatus));
  l.flags = l.hstate + async_align(sizeof(HgState));
  l.edges = l.flags + async_align(max_chunks * sizeof(uint32_t));
  l.stage = l.edges + async_align((n_buckets + 2) * sizeof(uint64_t));
  l.slot_map = l.stage + async_align(rows_cap * elem);
  l.cold_list = l.slot_map + async_align(max_chunks * sizeof(uint32_t));
  l.rows = l.cold_list + async_align((max_chunks + 1) * sizeof(uint32_t));
  l.sums = l.rows + async_align(max_files * w * sizeof(uint64_t));
  l.hgf_total = l.sums + async_align(w * sizeof(uint64_t));
  return l;
}

// One thread: the HgState of a pages call, behind ap_route_kernel.
__global__ void __launch_bounds__(32) hg_front_pages_kernel(const ApState* __restrict__ s, HgState* __restrict__ hs) {
  if (threadIdx.x != 0) return;
  *hs = HgState{s->status == ST_OK && s->fail_page == NONE64 ? 1u : 0u, 0u, 0};
}

// One thread: the HgState of a files call, behind merge_index_kernel.
__global__ void __launch_bounds__(32) hg_front_files_kernel(const AsyncCheck* __restrict__ chk, HgState* __restrict__ hs) {
  if (threadIdx.x != 0) return;
  *hs = HgState{chk->status == ST_OK ? 1u : 0u, 0u, 0};
}

// ceil((B + 1) / HG_THREADS) CTAs over edges[0 : B + 1): edge j's key (hist_edge_key) to table[1 + j] behind table[0] = B, and the lowest
// j whose edge is a NaN or whose key is not above edge j - 1's, met by atomicMax of ~j.
template <typename L>
__global__ void __launch_bounds__(HG_THREADS) hg_check_kernel(const uint64_t* __restrict__ edges, uint32_t n_buckets, uint32_t dtype,
                                                              HgState* __restrict__ hs, uint64_t* __restrict__ table) {
  const uint32_t kind = nt_is_float(dtype) ? 2u : nt_is_signed(dtype) ? 1u : 0u;
  const uint64_t j = uint64_t(blockIdx.x) * HG_THREADS + threadIdx.x;
  if (j == 0) table[0] = n_buckets;
  if (j > n_buckets) return;
  const L x = L(edges[j]);
  const L k = hist_key<L>(x, kind);
  table[1 + j] = uint64_t(k);
  bool bad = hist_is_nan<L>(x, kind);
  if (j > 0 && !bad) {
    const L p = L(edges[j - 1]);
    bad = !hist_is_nan<L>(p, kind) && k <= hist_key<L>(p, kind);
  }
  if (bad) atomicMax(&hs->nbad_edge, ~(unsigned long long)j);
}

// min(max_pages, HG_MAX_CTAS * HG_THREADS) threads over the pages: flags[p] = p + 1 when the gate passes, else 0.
__global__ void __launch_bounds__(HG_THREADS) hg_mark_pages_kernel(const HgState* __restrict__ hs, uint64_t max_pages, uint32_t* __restrict__ flags) {
  const bool ok = hg_gate(*hs);
  for (uint64_t p = uint64_t(blockIdx.x) * HG_THREADS + threadIdx.x; p < max_pages; p += uint64_t(gridDim.x) * HG_THREADS)
    flags[p] = ok ? uint32_t(p + 1) : 0u;
}

// min(max_files, HG_MAX_CTAS) CTAs, a file at a time (striding), behind a memset of the flags: when the gate passes, every chunk record of
// file g (merges[g].list_at .. + n_chunks of the merged table) gets g + 1.
__global__ void __launch_bounds__(HG_THREADS) hg_mark_files_kernel(const HgState* __restrict__ hs, const uint64_t* __restrict__ n_files,
                                                                   uint64_t max_files, const FileMerge* __restrict__ merges,
                                                                   uint32_t* __restrict__ flags) {
  if (!hg_gate(*hs)) return;  // uniform: every thread leaves
  const uint64_t nf = min(*n_files, max_files);
  for (uint64_t g = blockIdx.x; g < nf; g += gridDim.x) {
    const FileMerge m = merges[g];
    for (uint64_t k = threadIdx.x; k < m.n_chunks; k += HG_THREADS) flags[m.list_at + k] = uint32_t(g + 1);
  }
}

// The batches of record `rec` (its numbers at rows rec.out_offset .., decoded into the value staging by a catch-all decoder) counted by
// the CTA's warps into the counters hc through hist_store8, then added to the row of group `g1 - 1`.  Every thread calls it.
template <typename L>
__device__ __forceinline__ void hg_count_in_place(const FiltStage& f, const FiltKey& key, const IndexChunk& rec, uint32_t g1, const L* __restrict__ stage,
                                                  uint32_t* hc) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  hist_clear(f, hc, threadIdx.x, HG_THREADS);
  __syncthreads();
  const uint32_t nb = n_batches_of(rec.n);
  for (uint32_t b = warp; b < nb; b += HG_THREADS / 32) {
    const uint64_t row = rec.out_offset + uint64_t(b) * BATCH_N;
    const uint32_t cnt = min(uint32_t(BATCH_N), rec.n - b * BATCH_N);
    L v[8];
#pragma unroll
    for (int e = 0; e < 8; e++) v[e] = uint32_t(lane * 8 + e) < cnt ? stage[row + lane * 8 + e] : L(0);
    hist_store8<L>(f, key, hc, cnt, lane, v);
  }
  __syncthreads();
  hist_flush(f, hc, g1, threadIdx.x, HG_THREADS);
  __syncthreads();
}

// One CTA per cold-list entry k (pages, the list kept to flagged pages), with 4 W bytes of dynamic shared memory: the cold page, decoded
// into the value staging by ap_cold_kernel, counted in place.  Cold pages at or behind a failure were not decoded; they are left alone.
template <typename L>
__global__ void __launch_bounds__(HG_THREADS) hg_cold_pages_kernel(const ApState* __restrict__ state, const IndexChunk* __restrict__ recs,
                                                                   const uint32_t* __restrict__ cold_list, FiltStage f, uint32_t dtype,
                                                                   const L* __restrict__ stage) {
  extern __shared__ uint32_t hg_counters[];
  const uint64_t k = blockIdx.x;
  if (k >= state->n_cold) return;
  const uint32_t p = cold_list[k];
  if (p >= state->fail_page || p >= (state->decode_fail >> 32)) return;
  hg_count_in_place<L>(f, hist_fkey(dtype), recs[p], f.counts[p], stage, hg_counters);
}

// min(max_chunks, FF_COLD_CTAS) CTAs striding over the cold list (files), with 4 W bytes of dynamic shared memory: each record
// cold_chunks_kernel decoded into the value staging without failure, counted in place (unflagged records never reach the list: the fused
// kernel reported them done).
template <typename L>
__global__ void __launch_bounds__(HG_THREADS) hg_cold_files_kernel(const uint32_t* __restrict__ cold_list, const IndexChunk* __restrict__ table,
                                                                   const uint32_t* __restrict__ statuses, FiltStage f, uint32_t dtype,
                                                                   const L* __restrict__ stage) {
  extern __shared__ uint32_t hg_counters[];
  const uint32_t n_cold = cold_list[0];
  for (uint32_t k = blockIdx.x; k < n_cold; k += gridDim.x) {  // uniform: every thread runs the same records
    const uint32_t r = cold_list[1 + k];
    if (statuses[r] != ST_OK) continue;
    hg_count_in_place<L>(f, hist_fkey(dtype), table[r], f.counts[r], stage, hg_counters);
  }
}

// (ceil(W / HG_THREADS), hg_row_shares(max_groups)) CTAs, when the decompress call succeeded and the gate passed: column c of the rows of
// this CTA's share of the *n_groups groups copied to hists, and their sum added to sums[c].
__global__ void __launch_bounds__(HG_THREADS) hg_rows_kernel(const uint32_t* __restrict__ pkind, const uint64_t* __restrict__ n_groups,
                                                             const HgState* __restrict__ hs, uint32_t w, const uint64_t* __restrict__ rows,
                                                             uint64_t* __restrict__ hists, unsigned long long* __restrict__ sums) {
  if (*pkind != PCO_B200_OK || !hg_gate(*hs)) return;  // uniform: every thread leaves
  const uint32_t c = blockIdx.x * HG_THREADS + threadIdx.x;
  if (c >= w) return;
  const uint64_t n = *n_groups, per = (n + gridDim.y - 1) / gridDim.y;
  const uint64_t g0 = min(n, per * blockIdx.y), g1 = min(n, per * (blockIdx.y + 1));
  uint64_t s = 0;
  for (uint64_t g = g0; g < g1; g++) {
    const uint64_t v = rows[g * w + c];
    hists[g * w + c] = v;
    s += v;
  }
  if (s) atomicAdd(&sums[c], (unsigned long long)s);
}

// Thread 0 of a finish kernel, with the decompress call's outcome already in r: that outcome when it failed, else the edge refusal, else
// success.
template <typename S>
__device__ __forceinline__ void hg_decide(const HgState& t, S& r) {
  r.edge = NONE64;
  if (r.kind != PCO_B200_OK || t.nbad_edge == 0) return;
  r.kind = PCO_B200_INVALID_ARGUMENT;
  r.device_status = PCO_B200_HIST_EDGES_ORDER;
  r.edge = ~t.nbad_edge;
}

// One CTA: the pages histogram's total and status from the pages call's and the HgState.
__global__ void __launch_bounds__(HG_THREADS) hg_finish_pages_kernel(const PcoB200AsyncPagesStatus* __restrict__ ps, const HgState* __restrict__ hs,
                                                                     uint32_t w, const uint64_t* __restrict__ sums, uint64_t* __restrict__ total,
                                                                     PcoB200AsyncHistogramStatus* __restrict__ out) {
  const PcoB200AsyncPagesStatus p = *ps;
  PcoB200AsyncHistogramStatus r{p.kind, p.device_status, p.page, p.n_written, p.n_pages, p.frames_needed, NONE64};
  hg_decide(*hs, r);
  const bool ok = r.kind == PCO_B200_OK;
  for (uint32_t c = threadIdx.x; c < w; c += HG_THREADS) total[c] = ok ? sums[c] : 0;
  if (threadIdx.x == 0) *out = r;
}

// One CTA: the files histogram's total and status from the files call's and the HgState.
__global__ void __launch_bounds__(HG_THREADS) hg_finish_files_kernel(const PcoB200AsyncFilesStatus* __restrict__ fs, const HgState* __restrict__ hs,
                                                                     uint32_t w, const uint64_t* __restrict__ sums, uint64_t* __restrict__ total,
                                                                     PcoB200AsyncFilesHistogramStatus* __restrict__ out) {
  const PcoB200AsyncFilesStatus f = *fs;
  PcoB200AsyncFilesHistogramStatus r{f.kind, f.device_status, f.file, f.chunk, f.n_written, f.n_files, NONE64};
  hg_decide(*hs, r);
  const bool ok = r.kind == PCO_B200_OK;
  for (uint32_t c = threadIdx.x; c < w; c += HG_THREADS) total[c] = ok ? sums[c] : 0;
  if (threadIdx.x == 0) *out = r;
}

}  // namespace pcob200
