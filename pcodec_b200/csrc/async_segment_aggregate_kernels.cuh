// Kernels of pco_b200_segment_aggregate_pages_async and pco_b200_segment_aggregate_files_async: count, min, max and sum of the numbers
// inside a closed interval per caller-given row segment [bounds[g], bounds[g + 1]) of the concatenation the matching decompress call
// writes, decoding only the pages or chunks the segments cover.  The decompress call's launches run unchanged with rows_cap in the role of
// dst_cap (and, for files, ff_map_kernel and ff_cold_list_kernel around them, as the take runs them).  Between its front end and its
// decode stage runs the plan:
//   sg_front_pages_kernel / sg_front_files_kernel  (one thread) the SgState: whether the front end passed, the rows placed, the records
//                        and *n_segments as read;
//   sg_check_kernel      the bounds copied behind the interval into the workspace (what the decode kernels read), and the lowest
//                        index of each refusal: a bound below the one before it, a bound past the rows;
//   sg_mark_kernel       a CTA per record (striding): when the gate passes, its touched flag (its rows meet [bounds[0], bounds[M])) and
//                        for a touched record every batch's SegRun; on a refusal every record untouched;
//   tk_cold_list_kernel  (pages, the take's) the cold list kept to the touched pages.
// Then the decode stage in segment mode: fused_narrow_kernel<L, false, true, false, false, true> lets an untouched record go at once, and
// the SEG instantiations reduce each batch per segment into the SegRec records (seg_store8, decode_kernels.cuh).  Cold records, decoded
// into the value staging, are reduced in place by sg_cold_pages_kernel / sg_cold_files_kernel through the same seg_store8.  Then:
//   sg_group_kernel      a warp per segment (striding): the segment's records walked record by record in row order, the order-free parts
//                        (short segments only) reduced and the float sum's lane chains run, into the segment's AgGroup; long segments
//                        (more than 2^18 rows) listed;
//   sg_long_kernel       the long segments' order-free parts, each record range split over every CTA and met by atomics (as ag_share);
//   sg_finish_pages_kernel / sg_finish_files_kernel  (one CTA) aggs and *total by the aggregate's ag_total, and the status.
// Records: batch slot s (the filters' slots, fl_slots) keeps its partial of segment g in record s + g, so a plan holds S + max_segments
// records.  They are cleared before the decode, so the record range of a long segment (from its first batch's slot + g to its last's)
// holds its records and the empty records of the slot gaps between pages / chunks.
//
// Sum order (floats, in f64): a batch's partial of a segment is agg_store8's with the batch's rows outside the segment as non-matches; a
// segment's sum puts its batch j (the batches holding rows of the segment, in row order, running on across pages and chunks) on lane
// j mod 32, each lane adding in order from +0.0, then the pairwise tree; the total does the same with segment g in place of batch j.
#pragma once
#include "async_aggregate_kernels.cuh"
#include "async_take_kernels.cuh"

namespace pcob200 {

constexpr int SG_THREADS = 256;        // sg_check_kernel, sg_mark_kernel, sg_group_kernel, the cold kernels
constexpr uint64_t SG_MAX_CTAS = 4096;  // the largest grid of sg_check_kernel, sg_mark_kernel and sg_group_kernel; their CTAs stride
constexpr uint64_t SG_LONG_ROWS = uint64_t(1) << 18;  // a segment of more rows is long: its order-free parts go to sg_long_kernel
constexpr uint32_t SG_LONG_CTAS = 512;                 // sg_long_kernel's grid: every CTA takes a part of every long segment

// A long segment on sg_group_kernel's list: its index and its record range [s0, s1).  Entry 0's g is the list's length.
struct SgLong {
  uint64_t g, s0, s1;
};
static_assert(sizeof(SgLong) == 24, "workspace layout");
// Entries of the long list (its length, then one per long segment): at most rows_cap / 2^18 segments have more than 2^18 rows.
__host__ __device__ inline uint64_t sg_long_entries(uint64_t rows_cap) { return rows_cap / SG_LONG_ROWS + 2; }

// decided by the plan kernels, in launch order
struct SgState {
  uint32_t front_ok, reserved;    // 1: the decompress call's front end refused nothing (pages: nor did the walk)
  uint64_t n_read;                // *n_segments as read
  uint64_t rows;                  // the rows of the concatenation (valid when front_ok)
  uint64_t n_records;             // pages of the batch / chunks of the merged table
  unsigned long long nbad_order;  // ~j of the lowest j with bounds[j] < bounds[j - 1] (0: none)
  unsigned long long nbad_past;   // ~j of the lowest j with bounds[j] > rows (0: none)
  unsigned long long n_touched;   // records the segments touch (once the gate passed)
};
static_assert(sizeof(SgState) == 56, "workspace layout");

__device__ __forceinline__ bool sg_gate(const SgState& t, uint64_t max_segments) {
  return t.front_ok && t.n_read <= max_segments && t.nbad_order == 0 && t.nbad_past == 0;
}

// Records of a plan: S batch slots, each with max_segments segments in reach.
__host__ __device__ inline uint64_t sg_records(uint64_t slots, uint64_t max_segments) { return slots + max_segments; }

// Workspace of one in-flight pages call: the pages call's (ap_layout with dst_cap = rows_cap) | the pages status | SgState | SegRun per
// slot | touched flag per page | the interval and bounds (max_segments + 3 words) | SegRec per record | value staging (rows_cap numbers
// of elem bytes) | AgGroup per segment | the long list.  Each region 256-byte aligned.
struct SgLayout : ApLayout {
  uint64_t pstatus, sstate, runs, touched, bounds, recs, stage, groups, longs, sg_total;
};
__host__ __device__ inline SgLayout sg_layout(uint64_t max_pages, uint64_t rows_cap, uint64_t frame_cap, uint64_t max_segments, uint32_t elem) {
  SgLayout l;
  static_cast<ApLayout&>(l) = ap_layout(max_pages, rows_cap, frame_cap);
  const uint64_t slots = fl_slots(max_pages, rows_cap);
  l.pstatus = l.total;
  l.sstate = l.pstatus + async_align(sizeof(PcoB200AsyncPagesStatus));
  l.runs = l.sstate + async_align(sizeof(SgState));
  l.touched = l.runs + async_align(slots * sizeof(SegRun));
  l.bounds = l.touched + async_align(max_pages * sizeof(uint32_t));
  l.recs = l.bounds + async_align((max_segments + 3) * sizeof(uint64_t));
  l.stage = l.recs + async_align(sg_records(slots, max_segments) * sizeof(SegRec));
  l.groups = l.stage + async_align(rows_cap * elem);
  l.longs = l.groups + async_align(max_segments * sizeof(AgGroup));
  l.sg_total = l.longs + async_align(sg_long_entries(rows_cap) * sizeof(SgLong));
  return l;
}

// Workspace of one in-flight files call: the files call's (af_layout with dst_cap = rows_cap) | the files status | SgState | SegRun per
// slot | touched flag per chunk | the interval and bounds | SegRec per record | value staging | the slot map (max_chunks words) | the cold
// list (its length, then up to max_chunks records) | AgGroup per segment | the long list.
struct SgfLayout : AfLayout {
  uint64_t fstatus, sstate, runs, touched, bounds, recs, stage, slot_map, cold_list, groups, longs, sgf_total;
};
__host__ __device__ inline SgfLayout sgf_layout(uint64_t max_files, uint64_t max_chunks, uint64_t rows_cap, uint64_t max_segments, uint32_t elem) {
  SgfLayout l;
  static_cast<AfLayout&>(l) = af_layout(max_files, max_chunks, rows_cap);
  const uint64_t slots = fl_slots(max_chunks, rows_cap);
  l.fstatus = l.total;
  l.sstate = l.fstatus + async_align(sizeof(PcoB200AsyncFilesStatus));
  l.runs = l.sstate + async_align(sizeof(SgState));
  l.touched = l.runs + async_align(slots * sizeof(SegRun));
  l.bounds = l.touched + async_align(max_chunks * sizeof(uint32_t));
  l.recs = l.bounds + async_align((max_segments + 3) * sizeof(uint64_t));
  l.stage = l.recs + async_align(sg_records(slots, max_segments) * sizeof(SegRec));
  l.slot_map = l.stage + async_align(rows_cap * elem);
  l.cold_list = l.slot_map + async_align(max_chunks * sizeof(uint32_t));
  l.groups = l.cold_list + async_align((max_chunks + 1) * sizeof(uint32_t));
  l.longs = l.groups + async_align(max_segments * sizeof(AgGroup));
  l.sgf_total = l.longs + async_align(sg_long_entries(rows_cap) * sizeof(SgLong));
  return l;
}

// One thread: the SgState of a pages call, behind ap_route_kernel (as tk_front_pages_kernel).
__global__ void __launch_bounds__(32) sg_front_pages_kernel(const ApState* __restrict__ s, const uint64_t* __restrict__ n_segments,
                                                            SgState* __restrict__ ss) {
  if (threadIdx.x != 0) return;
  *ss = SgState{s->status == ST_OK && s->fail_page == NONE64 ? 1u : 0u, 0u, *n_segments, s->nums.s, s->n_pages, 0, 0, 0};
}

// One thread: the SgState of a files call, behind af_table_kernel (as tk_front_files_kernel).
__global__ void __launch_bounds__(32) sg_front_files_kernel(const AfState* __restrict__ s, const AsyncCheck* __restrict__ chk,
                                                            const uint64_t* __restrict__ n_segments, SgState* __restrict__ ss) {
  if (threadIdx.x != 0) return;
  *ss = SgState{chk->status == ST_OK ? 1u : 0u, 0u, *n_segments, s->total.s, chk->n_chunks, 0, 0, 0};
}

// min(ceil((max_segments + 1) / SG_THREADS), SG_MAX_CTAS) CTAs striding over bounds[0 : M + 1) (M = *n_segments; none when M is 0 or
// above max_segments): each bound copied to copy[2 + j] behind the interval (copy[0 .. 1], by thread 0 of CTA 0), the lowest j with
// bounds[j] < bounds[j - 1] and the lowest j with bounds[j] past the rows, each met by atomicMax of ~j.
__global__ void __launch_bounds__(SG_THREADS) sg_check_kernel(const uint64_t* __restrict__ bounds, const uint64_t* __restrict__ interval,
                                                              uint64_t max_segments, SgState* __restrict__ ss, uint64_t* __restrict__ copy) {
  __shared__ unsigned long long s_order, s_past;
  if (threadIdx.x == 0) s_order = s_past = 0;
  if (blockIdx.x == 0 && threadIdx.x < 2) copy[threadIdx.x] = interval[threadIdx.x];
  __syncthreads();
  const uint64_t m = ss->n_read, rows = ss->rows;
  const uint64_t n = m >= 1 && m <= max_segments ? m + 1 : 0;
  uint64_t order = NONE64, past = NONE64;  // a thread's first of each is its lowest
  for (uint64_t j = uint64_t(blockIdx.x) * SG_THREADS + threadIdx.x; j < n; j += uint64_t(gridDim.x) * SG_THREADS) {
    const uint64_t b = bounds[j];
    copy[2 + j] = b;
    if (order == NONE64 && j > 0 && b < bounds[j - 1]) order = j;
    if (past == NONE64 && b > rows) past = j;
  }
  if (order != NONE64) atomicMax(&s_order, ~order);
  if (past != NONE64) atomicMax(&s_past, ~past);
  __syncthreads();
  if (threadIdx.x != 0) return;
  if (s_order) atomicMax(&ss->nbad_order, s_order);
  if (s_past) atomicMax(&ss->nbad_past, s_past);
}

// The segment that holds row x, for bounds[0] <= x < bounds[m]: the last g < m with bounds[g] <= x.
__device__ __forceinline__ uint32_t sg_segment_of(const uint64_t* __restrict__ bounds, uint64_t m, uint64_t x) {
  uint64_t lo = 0, hi = m;  // bounds[lo] <= x < bounds[hi]
  while (hi - lo > 1) {
    const uint64_t mid = lo + (hi - lo) / 2;
    if (bounds[mid] <= x) lo = mid;
    else hi = mid;
  }
  return uint32_t(lo);
}

// min(max_records, SG_MAX_CTAS) CTAs, a record at a time (records[0 : n_records): the pages' placed records or the merged chunk table;
// record r's slots start at out_offset / 256 + r).  When the gate refuses, every record is left untouched.  Otherwise a record is touched
// when its rows meet [bounds[0], bounds[M]), and then every batch of it gets its run of segments (none for a batch outside the range).
__global__ void __launch_bounds__(SG_THREADS) sg_mark_kernel(const uint64_t* __restrict__ copy, uint64_t max_segments, const IndexChunk* __restrict__ recs,
                                                             SgState* __restrict__ ss, uint32_t* __restrict__ touched, SegRun* __restrict__ runs) {
  const SgState t = *ss;
  const bool ok = sg_gate(t, max_segments) && t.n_read > 0;
  const uint64_t m = t.n_read;
  const uint64_t* __restrict__ bounds = copy + 2;
  const uint64_t w0 = ok ? bounds[0] : 0, w1 = ok ? bounds[m] : 0;
  for (uint64_t r = blockIdx.x; r < t.n_records; r += gridDim.x) {  // uniform: every thread runs the same records
    const IndexChunk rec = recs[r];
    const uint64_t o = rec.out_offset, e = o + rec.n;
    const bool hit = ok && o < w1 && e > w0;
    if (threadIdx.x == 0) {
      touched[r] = hit ? 1u : 0u;
      if (hit) atomicAdd(&ss->n_touched, 1ull);
    }
    if (!hit) continue;
    const uint32_t nb = n_batches_of(rec.n);
    const uint64_t slot0 = o / BATCH_N + r;
    for (uint32_t b = threadIdx.x; b < nb; b += SG_THREADS) {
      const uint64_t a = max(o + uint64_t(b) * BATCH_N, w0), z = min(min(o + uint64_t(b + 1) * BATCH_N, e), w1);
      runs[slot0 + b] = a < z ? SegRun{sg_segment_of(bounds, m, a), sg_segment_of(bounds, m, z - 1)} : SegRun{1u, 0u};
    }
  }
}

// The batches of record r (its numbers at rows rec.out_offset .., decoded into the value staging by a catch-all decoder) reduced by the
// CTA's warps through seg_store8.
template <typename L>
__device__ __forceinline__ void sg_reduce_in_place(const FiltStage& f, const FiltKey& key, const IndexChunk& rec, uint64_t r, const L* __restrict__ stage) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t nb = n_batches_of(rec.n);
  for (uint32_t b = warp; b < nb; b += SG_THREADS / 32) {
    const uint64_t row = rec.out_offset + uint64_t(b) * BATCH_N;
    const uint32_t cnt = min(uint32_t(BATCH_N), rec.n - b * BATCH_N);
    L v[8];
#pragma unroll
    for (int e = 0; e < 8; e++) v[e] = uint32_t(lane * 8 + e) < cnt ? stage[row + lane * 8 + e] : L(0);
    seg_store8<L>(f, key, row, rec.out_offset / BATCH_N + r + b, cnt, lane, v);
  }
}

// One CTA per cold-list entry k (pages, the list kept to touched pages): the cold page, decoded into the value staging by ap_cold_kernel,
// reduced in place.  Cold pages at or behind a failure were not decoded; they are left alone.
template <typename L>
__global__ void __launch_bounds__(SG_THREADS) sg_cold_pages_kernel(const ApState* __restrict__ state, const IndexChunk* __restrict__ recs,
                                                                   const uint32_t* __restrict__ cold_list, FiltStage f, uint32_t dtype,
                                                                   const L* __restrict__ stage) {
  const uint64_t k = blockIdx.x;
  if (k >= state->n_cold) return;
  const uint32_t p = cold_list[k];
  if (p >= state->fail_page || p >= (state->decode_fail >> 32)) return;
  sg_reduce_in_place<L>(f, filt_bounds<L>(f.interval, dtype), recs[p], p, stage);
}

// min(max_chunks, FF_COLD_CTAS) CTAs striding over the cold list (files): each record cold_chunks_kernel decoded into the value staging
// without failure, reduced in place (untouched records never reach the list: the fused kernel reported them done).
template <typename L>
__global__ void __launch_bounds__(SG_THREADS) sg_cold_files_kernel(const uint32_t* __restrict__ cold_list, const IndexChunk* __restrict__ table,
                                                                   const uint32_t* __restrict__ statuses, FiltStage f, uint32_t dtype,
                                                                   const L* __restrict__ stage) {
  const uint32_t n_cold = cold_list[0];
  if (blockIdx.x >= n_cold) return;
  const FiltKey key = filt_bounds<L>(f.interval, dtype);
  for (uint32_t k = blockIdx.x; k < n_cold; k += gridDim.x) {
    const uint32_t r = cold_list[1 + k];
    if (statuses[r] != ST_OK) continue;
    sg_reduce_in_place<L>(f, key, table[r], r, stage);
  }
}

// The first record whose rows end after row a (records[0 : n) in row order; n when none).
__device__ __forceinline__ uint64_t sg_first_record(const IndexChunk* __restrict__ recs, uint64_t n, uint64_t a) {
  uint64_t r0 = 0, r1 = n;
  while (r0 < r1) {
    const uint64_t mid = r0 + (r1 - r0) / 2;
    const IndexChunk rm = recs[mid];
    if (rm.out_offset + rm.n <= a) r0 = mid + 1;
    else r1 = mid;
  }
  return r0;
}

// The record range [s0, s1) of a long segment g with rows [a, b): from its first batch's slot + g to its last batch's slot + g.  The
// range holds only segment g's records and the cleared records of the slot gaps between pages / chunks.
__device__ __forceinline__ SgLong sg_long_range(const IndexChunk* __restrict__ recs, uint64_t n, uint64_t g, uint64_t a, uint64_t b) {
  const uint64_t r0 = sg_first_record(recs, n, a);
  uint64_t r1 = sg_first_record(recs, n, b - 1);  // the record that holds row b - 1
  const IndexChunk f = recs[r0], l = recs[r1];
  const uint64_t s0 = f.out_offset / BATCH_N + r0 + (a - f.out_offset) / BATCH_N;
  const uint64_t s1 = l.out_offset / BATCH_N + r1 + (b - 1 - l.out_offset) / BATCH_N + 1;
  return SgLong{g, s0 + g, s1 + g};
}

// min(ceil(max_segments / 8), SG_MAX_CTAS) CTAs of 8 warps, a warp per segment (striding), when the gate passed and the decompress call
// succeeded: segment g's rows [a, b) (none: an all-zero group), the records that hold them found by binary search, then walked in row order;
// in record r its batches bf .. bl meet the segment, and their partials sit in records slot + g.  Lane l takes the segment's batches
// j = l (mod 32) in order.  A short segment (at most SG_LONG_ROWS rows): count, least and greatest key and the 128-bit sum in any order,
// the f64 sum from +0.0 in that order, then the warp's reductions (agg_warp: the pairwise tree for the f64 sum) into groups[g].  A long
// segment: only the f64 chain (from each record's count and sum word), groups[g] written with it and zero order-free parts, and the segment
// appended to the long list, whose order-free parts sg_long_kernel then spreads over every CTA.
__global__ void __launch_bounds__(SG_THREADS) sg_group_kernel(const uint32_t* __restrict__ pkind, const SgState* __restrict__ ss, uint64_t max_segments,
                                                              const uint64_t* __restrict__ copy, const IndexChunk* __restrict__ recs,
                                                              const SegRec* __restrict__ srecs, uint32_t dtype, AgGroup* __restrict__ groups,
                                                              SgLong* __restrict__ longs) {
  const SgState t = *ss;
  if (*pkind != PCO_B200_OK || !sg_gate(t, max_segments)) return;  // uniform: every thread leaves
  const uint64_t* __restrict__ bounds = copy + 2;
  const bool is_float = ag_kind(dtype) == 2;
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = uint64_t(gridDim.x) * (SG_THREADS / 32);
  for (uint64_t g = uint64_t(blockIdx.x) * (SG_THREADS / 32) + (threadIdx.x >> 5); g < t.n_read; g += warps) {
    const uint64_t a = bounds[g], b = bounds[g + 1];
    const bool is_long = b - a > SG_LONG_ROWS;  // uniform over the warp
    uint64_t cnt = 0, kmin = ~uint64_t(0), kmax = 0, lo = 0, hi = 0;
    double fs = 0.0;
    if (a < b && (!is_long || is_float)) {
      uint64_t j0 = 0;
      for (uint64_t r = sg_first_record(recs, t.n_records, a); r < t.n_records; r++) {
        const IndexChunk rec = recs[r];
        if (rec.out_offset >= b) break;
        if (rec.n == 0) continue;
        const uint64_t bf = (max(a, rec.out_offset) - rec.out_offset) / BATCH_N, bl = (min(b, rec.out_offset + rec.n) - 1 - rec.out_offset) / BATCH_N;
        const uint64_t nb = bl - bf + 1;
        const SegRec* __restrict__ base = srecs + rec.out_offset / BATCH_N + r + bf + g;
        if (is_long) {  // the float chain alone, as ag_chain runs it
#pragma unroll 4
          for (uint64_t k = (uint64_t(lane) - j0) & 31u; k < nb; k += 32) {
            const uint64_t c = base[k].count;
            const double v = __longlong_as_double((long long)base[k].lo);
            fs = fs + (c ? v : 0.0);
          }
        } else {
#pragma unroll 4
          for (uint64_t k = (uint64_t(lane) - j0) & 31u; k < nb; k += 32) {
            const SegRec s = base[k];
            if (s.count) {
              cnt += s.count;
              kmin = min(kmin, s.kmin);
              kmax = max(kmax, s.kmax);
              if (!is_float) agg_add128(lo, hi, s.lo, s.hi);
            }
            fs = fs + (s.count ? __longlong_as_double((long long)s.lo) : 0.0);
          }
        }
        j0 += nb;
      }
    }
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, d);
    agg_warp(kmin, kmax, lo, hi, fs, is_float);
    if (lane == 0) {
      groups[g] = AgGroup{cnt, ~kmin, kmax, lo, hi, fs};  // a long segment: the identity of every order-free part, and its f64 sum
      if (is_long) {
        const unsigned long long at = atomicAdd(reinterpret_cast<unsigned long long*>(longs), 1ull);
        longs[1 + at] = sg_long_range(recs, t.n_records, g, a, b);
      }
    }
  }
}

// SG_LONG_CTAS CTAs, after sg_group_kernel: CTA c takes part c of every long segment's record range (gridDim.x equal parts), as ag_share
// takes its share of a group's slots: the order-free parts of the records with a match, reduced in each warp and met in groups[g] by
// atomics.  Gap records inside a range were cleared before the decode and count nothing.
__global__ void __launch_bounds__(AG_THREADS) sg_long_kernel(const uint32_t* __restrict__ pkind, const SgState* __restrict__ ss, uint64_t max_segments,
                                                             const SgLong* __restrict__ longs, const SegRec* __restrict__ srecs, uint32_t dtype,
                                                             AgGroup* __restrict__ groups) {
  if (*pkind != PCO_B200_OK || !sg_gate(*ss, max_segments)) return;  // uniform: every thread leaves
  const bool is_float = ag_kind(dtype) == 2;
  const uint64_t n_long = longs[0].g;
  for (uint64_t i = 0; i < n_long; i++) {
    const SgLong e = longs[1 + i];
    const uint64_t n = e.s1 - e.s0, per = (n + gridDim.x - 1) / gridDim.x;
    const uint64_t s0 = e.s0 + min(n, per * blockIdx.x), s1 = e.s0 + min(n, per * (blockIdx.x + 1));
    uint64_t cnt = 0, kmin = ~uint64_t(0), kmax = 0, lo = 0, hi = 0;
    for (uint64_t s = s0 + threadIdx.x; s < s1; s += AG_THREADS) {
      const SegRec r = srecs[s];
      if (r.count) {
        cnt += r.count;
        kmin = min(kmin, r.kmin);
        kmax = max(kmax, r.kmax);
        if (!is_float) agg_add128(lo, hi, r.lo, r.hi);
      }
    }
    double unused = 0.0;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, d);
    agg_warp(kmin, kmax, lo, hi, unused, false);
    if ((threadIdx.x & 31) != 0 || cnt == 0) continue;
    AgGroup* acc = &groups[e.g];
    atomicAdd(&acc->count, cnt);
    atomicMax(&acc->nkmin, ~kmin);
    atomicMax(&acc->kmax, kmax);
    if (!is_float) {  // the 128-bit sum: the low word's carry out of each addition goes to the high word
      const unsigned long long old = atomicAdd(&acc->lo, lo);
      atomicAdd(&acc->hi, hi + (old + lo < old ? 1u : 0u));
    }
  }
}

// Thread 0 of a finish kernel, with the decompress call's outcome already in r: that outcome when it failed, else the segment call's own
// refusal in its order (the count, then the lowest j out of order, then the lowest j past the rows), else success with the records decoded.
template <typename S>
__device__ __forceinline__ void sg_decide(const SgState& t, uint64_t max_segments, S& r) {
  r.n_segments = t.n_read;
  r.segment = NONE64;
  r.records_decoded = 0;
  if (r.kind != PCO_B200_OK) return;
  uint32_t code = ST_OK;
  if (t.n_read > max_segments) code = PCO_B200_SEGMENTS_TOO_MANY;
  else if (t.nbad_order) code = PCO_B200_SEGMENTS_ORDER, r.segment = ~t.nbad_order;
  else if (t.nbad_past) code = PCO_B200_SEGMENTS_PAST, r.segment = ~t.nbad_past;
  if (code != ST_OK) {
    r.kind = PCO_B200_INVALID_ARGUMENT;
    r.device_status = code;
  } else {
    r.records_decoded = t.n_touched;
  }
}

// The step both finish kernels share, on one CTA of AG_THREADS: the decision, then aggs and *total by ag_total (n_rows of segment g is
// bounds[g + 1] - bounds[g]; of the total, bounds[M] - bounds[0]) and the match count.
template <typename L, typename S>
__device__ __forceinline__ void sg_finish(const SgState& t, uint64_t max_segments, const uint64_t* __restrict__ copy, const AgGroup* __restrict__ groups,
                                          uint32_t dtype, PcoB200Aggregate* __restrict__ aggs, PcoB200Aggregate* __restrict__ total, S& r) {
  sg_decide(t, max_segments, r);
  const bool ok = r.kind == PCO_B200_OK;
  const uint64_t m = ok ? t.n_read : 0;
  const uint64_t* __restrict__ bounds = copy + 2;
  r.n_matches = ag_total<L>(ok, m, m ? bounds[m] - bounds[0] : 0, groups, [&](uint64_t g) { return bounds[g + 1] - bounds[g]; }, dtype, aggs, total);
}

// One CTA: the pages segment aggregate's records and status from the pages call's and the SgState.
template <typename L>
__global__ void __launch_bounds__(AG_THREADS) sg_finish_pages_kernel(const PcoB200AsyncPagesStatus* __restrict__ ps, const SgState* __restrict__ ss,
                                                                     uint64_t max_segments, const uint64_t* __restrict__ copy,
                                                                     const AgGroup* __restrict__ groups, uint32_t dtype, PcoB200Aggregate* __restrict__ aggs,
                                                                     PcoB200Aggregate* __restrict__ total, PcoB200AsyncSegmentAggregateStatus* __restrict__ out) {
  const PcoB200AsyncPagesStatus p = *ps;
  PcoB200AsyncSegmentAggregateStatus r;
  r.kind = p.kind;
  r.device_status = p.device_status;
  r.page = p.page;
  r.n_written = p.n_written;
  r.n_pages = p.n_pages;
  r.frames_needed = p.frames_needed;
  sg_finish<L>(*ss, max_segments, copy, groups, dtype, aggs, total, r);
  if (threadIdx.x == 0) *out = r;
}

// One CTA: the files segment aggregate's records and status from the files call's and the SgState.
template <typename L>
__global__ void __launch_bounds__(AG_THREADS) sg_finish_files_kernel(const PcoB200AsyncFilesStatus* __restrict__ fs, const SgState* __restrict__ ss,
                                                                     uint64_t max_segments, const uint64_t* __restrict__ copy,
                                                                     const AgGroup* __restrict__ groups, uint32_t dtype, PcoB200Aggregate* __restrict__ aggs,
                                                                     PcoB200Aggregate* __restrict__ total,
                                                                     PcoB200AsyncFilesSegmentAggregateStatus* __restrict__ out) {
  const PcoB200AsyncFilesStatus f = *fs;
  PcoB200AsyncFilesSegmentAggregateStatus r;
  r.kind = f.kind;
  r.device_status = f.device_status;
  r.file = f.file;
  r.chunk = f.chunk;
  r.n_written = f.n_written;
  r.n_files = f.n_files;
  sg_finish<L>(*ss, max_segments, copy, groups, dtype, aggs, total, r);
  if (threadIdx.x == 0) *out = r;
}

}  // namespace pcob200
