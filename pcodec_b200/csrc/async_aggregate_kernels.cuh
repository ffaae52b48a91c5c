// Kernels of pco_b200_aggregate_pages_async and pco_b200_aggregate_files_async: the pages or files the matching decompress call decodes,
// reduced to count, min, max and sum of the numbers inside a closed interval, per page / file and in all.  The decompress call's launches
// run unchanged with rows_cap in the role of dst_cap (and, for files, ff_map_kernel and ff_cold_list_kernel around them, as the files
// filter runs them); what changes is the store side of the decode:
//   fused_narrow_kernel<L, false, true, true>, symwalk_kernel<false>, decode_kernel<L, 1 / 2, false, true, true>  the AGG instantiations:
//                        each batch's matches reduced in registers into its slot (agg_store8, decode_kernels.cuh); nothing is stored to dst;
//   ap_cold_kernel<L> / cold_chunks_kernel<L>  unchanged, decoding the cold pages / chunks into the value staging;
//   fl_cold_kernel<L, true> / ff_cold_kernel<L, true>  those batches reduced in place into their slots by the same agg_store8;
//   ag_pages_kernel / ag_files_kernel  a (group, share) grid: each page's / file's slots split across gridDim.y CTAs, whose
//                        order-free parts (count, min, max, integer sum) meet in the group's AgGroup by atomics; the float sum's lane
//                        chains run on warp 0 of the group's first CTA;
//   ag_finish_kernel<L> / agf_finish_kernel<L>  (one CTA) each group's record written to aggs[g], the groups reduced into *total, and the
//                        status from the decompress call's.
// The batch slots are the filters' (fl_slots, async_filter_kernels.cuh): batch b of record r, its numbers from row O, has slot O / 256 + r + b.
// Only the slot counts are cleared before the decode; a count of 0 marks a slot no batch with matches wrote.
//
// Sum order (floats, in f64; integers are exact, so any order gives them): a batch's sum is agg_store8's (each lane's 8 numbers left to
// right from +0.0, then the lanes as a pairwise tree); a group's sum puts its batch j (in row order, over all its pages' / chunks'
// batches) on lane j mod 32, each lane adds its batches in order from +0.0, then the same tree; the total does the same with group g in
// place of batch j.  Count, min, max and the integer sums do not depend on the order, so any number of CTAs may take shares of them.
#pragma once
#include "async_filter_files_kernels.cuh"

namespace pcob200 {

constexpr int AG_THREADS = 256;       // the group and finish CTAs
constexpr uint64_t AG_TILE = 2048;    // slots per group CTA, on average over a plan's capacity

// A group's accumulator in the workspace, cleared before the call: the order-free parts, met by atomics (exact, so in any order), and
// the f64 sum.  The least key is kept complemented, so that a cleared record is the identity of every field.
struct AgGroup {
  unsigned long long count, nkmin, kmax, lo, hi;
  double fs;
};
static_assert(sizeof(AgGroup) == 48, "workspace layout");

// CTAs per group (gridDim.y of the group kernels): about AG_TILE slots each when the slots are spread over max_groups groups.
__host__ __device__ inline uint32_t ag_split(uint64_t slots, uint64_t max_groups) {
  const uint64_t k = (slots + max_groups * AG_TILE - 1) / (max_groups * AG_TILE);
  return uint32_t(k < 1 ? 1 : k > 65535 ? 65535 : k);
}

// Workspace of one in-flight pages call: the pages call's (ap_layout with dst_cap = rows_cap) | the pages status | per slot: count,
// AggSlot | value staging (rows_cap numbers of elem bytes) | AgGroup[max_pages].  Each region 256-byte aligned.
struct AgLayout : ApLayout {
  uint64_t pstatus, counts, aslots, stage, groups, ag_total;
};
__host__ __device__ inline AgLayout ag_layout(uint64_t max_pages, uint64_t rows_cap, uint64_t frame_cap, uint32_t elem) {
  AgLayout l;
  static_cast<ApLayout&>(l) = ap_layout(max_pages, rows_cap, frame_cap);
  const uint64_t slots = fl_slots(max_pages, rows_cap);
  l.pstatus = l.total;
  l.counts = l.pstatus + async_align(sizeof(PcoB200AsyncPagesStatus));
  l.aslots = l.counts + async_align(slots * sizeof(uint32_t));
  l.stage = l.aslots + async_align(slots * sizeof(AggSlot));
  l.groups = l.stage + async_align(rows_cap * elem);
  l.ag_total = l.groups + async_align(max_pages * sizeof(AgGroup));
  return l;
}

// Workspace of one in-flight files call: the files call's (af_layout with dst_cap = rows_cap) | the files status | per slot: count,
// AggSlot | value staging | the slot map (max_chunks words) | the cold list (its length, then up to max_chunks records) | AgGroup[max_files].
struct AgfLayout : AfLayout {
  uint64_t fstatus, counts, aslots, stage, slot_map, cold_list, groups, agf_total;
};
__host__ __device__ inline AgfLayout agf_layout(uint64_t max_files, uint64_t max_chunks, uint64_t rows_cap, uint32_t elem) {
  AgfLayout l;
  static_cast<AfLayout&>(l) = af_layout(max_files, max_chunks, rows_cap);
  const uint64_t slots = fl_slots(max_chunks, rows_cap);
  l.fstatus = l.total;
  l.counts = l.fstatus + async_align(sizeof(PcoB200AsyncFilesStatus));
  l.aslots = l.counts + async_align(slots * sizeof(uint32_t));
  l.stage = l.aslots + async_align(slots * sizeof(AggSlot));
  l.slot_map = l.stage + async_align(rows_cap * elem);
  l.cold_list = l.slot_map + async_align(max_chunks * sizeof(uint32_t));
  l.groups = l.cold_list + async_align((max_chunks + 1) * sizeof(uint32_t));
  l.agf_total = l.groups + async_align(max_files * sizeof(AgGroup));
  return l;
}

// The inverse of filt_key: the bit pattern of the number whose key is k.
template <typename L>
__device__ __forceinline__ L filt_unkey(L k, uint32_t kind) {
  constexpr L TOP = L(L(1) << (LT<L>::BITS - 1));
  if (kind == 1) return L(k ^ TOP);
  if (kind == 2) return (k & TOP) ? L(k ^ TOP) : L(~k);
  return k;
}
__device__ __forceinline__ uint32_t ag_kind(uint32_t dtype) { return nt_is_float(dtype) ? 2u : nt_is_signed(dtype) ? 1u : 0u; }

// This CTA's share (blockIdx.y of gridDim.y equal parts) of the group's slot range [a, b): the order-free parts of its slots with a
// match, reduced in each warp, then met in *acc by atomics (lane 0 of each warp that saw a match).  Slots in the range that no batch
// wrote have a count of 0.  Every thread calls it.
__device__ __forceinline__ void ag_share(AgGroup* __restrict__ acc, const uint32_t* __restrict__ counts, const AggSlot* __restrict__ aslots,
                                         uint64_t a, uint64_t b, bool is_float) {
  const uint64_t n = b - a, per = (n + gridDim.y - 1) / gridDim.y;
  const uint64_t s0 = a + min(n, per * blockIdx.y), s1 = a + min(n, per * (blockIdx.y + 1));
  uint64_t cnt = 0, kmin = ~uint64_t(0), kmax = 0, lo = 0, hi = 0;
  for (uint64_t s = s0 + threadIdx.x; s < s1; s += AG_THREADS) {
    const uint32_t c = counts[s];
    if (c) {
      const AggSlot r = aslots[s];
      cnt += c;
      kmin = min(kmin, r.kmin);
      kmax = max(kmax, r.kmax);
      if (!is_float) agg_add128(lo, hi, r.lo, r.hi);
    }
  }
  double unused = 0.0;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, d);
  agg_warp(kmin, kmax, lo, hi, unused, false);
  if ((threadIdx.x & 31) != 0 || cnt == 0) return;
  atomicAdd(&acc->count, cnt);
  atomicMax(&acc->nkmin, ~kmin);
  atomicMax(&acc->kmax, kmax);
  if (!is_float) {  // the 128-bit sum: the low word's carry out of each addition goes to the high word
    const unsigned long long old = atomicAdd(&acc->lo, lo);
    atomicAdd(&acc->hi, hi + (old + lo < old ? 1u : 0u));
  }
}

// Lane `lane`'s chain of the f64 sum over slots slot0 .. slot0 + nb - 1 (a record's batches, the first of which is batch j0 of its
// group): batches j = lane (mod 32), in order.  A slot without a match adds +0.0, which leaves a sum that started from +0.0 as it was.
__device__ __forceinline__ double ag_chain(double fs, const uint32_t* __restrict__ counts, const AggSlot* __restrict__ aslots, uint64_t slot0,
                                           uint64_t nb, uint64_t j0, uint32_t lane) {
#pragma unroll 4
  for (uint64_t b = (uint64_t(lane) - j0) & 31u; b < nb; b += 32) {
    const uint32_t c = counts[slot0 + b];
    const double v = __longlong_as_double((long long)aslots[slot0 + b].lo);
    fs = fs + (c ? v : 0.0);
  }
  return fs;
}
__device__ __forceinline__ double ag_tree(double fs) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) fs = fs + __shfl_xor_sync(0xffffffffu, fs, d);
  return fs;
}

// (max_pages, ag_split) CTAs: when the pages call succeeded, page g's slots (from recs[g].out_offset / 256 + g, one per batch) into
// groups[g]; CTA (g, 0)'s warp 0 runs the float sum's chains.
__global__ void __launch_bounds__(AG_THREADS) ag_pages_kernel(const PcoB200AsyncPagesStatus* __restrict__ ps, const IndexChunk* __restrict__ recs,
                                                              const uint32_t* __restrict__ counts, const AggSlot* __restrict__ aslots, uint32_t dtype,
                                                              AgGroup* __restrict__ groups) {
  const uint64_t g = blockIdx.x;
  if (ps->kind != PCO_B200_OK || g >= ps->n_pages) return;  // uniform: every thread leaves
  const bool is_float = ag_kind(dtype) == 2;
  const IndexChunk rec = recs[g];
  const uint64_t a = rec.out_offset / BATCH_N + g, nb = n_batches_of(rec.n);
  ag_share(&groups[g], counts, aslots, a, a + nb, is_float);
  if (is_float && blockIdx.y == 0 && threadIdx.x < 32) {
    const double fs = ag_tree(ag_chain(0.0, counts, aslots, a, nb, 0, threadIdx.x));
    if (threadIdx.x == 0) groups[g].fs = fs;
  }
}

// (max_files, ag_split) CTAs: when the files call succeeded, file g's slots into groups[g].  Its chunks are the records merges[g].list_at
// .. + n_chunks of the merged table; their slots lie in one range (from the first record's first slot to the last's last), whose slots no
// other file's batch writes.  CTA (g, 0)'s warp 0 runs the float chains record by record, the batch number running on through the file.
__global__ void __launch_bounds__(AG_THREADS) ag_files_kernel(const PcoB200AsyncFilesStatus* __restrict__ fst, const FileMerge* __restrict__ merges,
                                                              const IndexChunk* __restrict__ table, const uint32_t* __restrict__ counts,
                                                              const AggSlot* __restrict__ aslots, uint32_t dtype, AgGroup* __restrict__ groups) {
  const uint64_t g = blockIdx.x;
  if (fst->kind != PCO_B200_OK || g >= fst->n_files) return;  // uniform: every thread leaves
  const FileMerge m = merges[g];
  if (m.n_chunks == 0) return;
  const bool is_float = ag_kind(dtype) == 2;
  const uint64_t r0 = m.list_at, r1 = m.list_at + m.n_chunks - 1;
  const IndexChunk last = table[r1];
  ag_share(&groups[g], counts, aslots, table[r0].out_offset / BATCH_N + r0, last.out_offset / BATCH_N + r1 + n_batches_of(last.n), is_float);
  if (is_float && blockIdx.y == 0 && threadIdx.x < 32) {
    double fs = 0.0;
    uint64_t j0 = 0;
    for (uint64_t r = r0; r <= r1; r++) {
      const IndexChunk rec = table[r];
      const uint64_t nb = n_batches_of(rec.n);
      fs = ag_chain(fs, counts, aslots, rec.out_offset / BATCH_N + r, nb, j0, threadIdx.x);
      j0 += nb;
    }
    fs = ag_tree(fs);
    if (threadIdx.x == 0) groups[g].fs = fs;
  }
}

// The step both finish kernels share, on one CTA of AG_THREADS: when ok, each of the n groups' accumulators written to aggs[g] as a
// record (n_rows from rows_of(g)), and the groups reduced into *total (group g on lane g mod 32 of the f64 sum); else *total all zeros
// and aggs untouched.  Returns the match count (0 when not ok) to thread 0.
template <typename L, typename RowsOf>
__device__ __forceinline__ uint64_t ag_total(bool ok, uint64_t n, uint64_t n_rows, const AgGroup* __restrict__ groups, RowsOf rows_of, uint32_t dtype,
                                             PcoB200Aggregate* __restrict__ aggs, PcoB200Aggregate* __restrict__ total) {
  __shared__ unsigned long long s_cnt[AG_THREADS / 32], s_min[AG_THREADS / 32], s_max[AG_THREADS / 32], s_lo[AG_THREADS / 32],
      s_hi[AG_THREADS / 32];
  const uint32_t kind = ag_kind(dtype), lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool is_float = kind == 2;
  auto record = [&](uint64_t rows, uint64_t cnt, uint64_t kmin, uint64_t kmax, uint64_t lo, uint64_t hi, double fs) {
    PcoB200Aggregate r{rows, cnt, 0, 0, is_float ? uint64_t(__double_as_longlong(fs)) : lo, is_float ? 0 : hi};
    if (cnt) {
      r.min_bits = uint64_t(filt_unkey<L>(L(kmin), kind));
      r.max_bits = uint64_t(filt_unkey<L>(L(kmax), kind));
    }
    return r;
  };
  uint64_t cnt = 0, kmin = ~uint64_t(0), kmax = 0, lo = 0, hi = 0;
  double fs = 0.0;
  if (ok) {
    for (uint64_t g = threadIdx.x; g < n; g += AG_THREADS) {
      const AgGroup a = groups[g];
      aggs[g] = record(rows_of(g), a.count, ~a.nkmin, a.kmax, a.lo, a.hi, a.fs);
      if (a.count) {
        cnt += a.count;
        kmin = min(kmin, uint64_t(~a.nkmin));
        kmax = max(kmax, uint64_t(a.kmax));
        if (!is_float) agg_add128(lo, hi, a.lo, a.hi);
      }
    }
    if (is_float && warp == 0) {
      for (uint64_t g = lane; g < n; g += 32) fs = fs + (groups[g].count ? groups[g].fs : 0.0);
      fs = ag_tree(fs);
    }
  }
  double unused = 0.0;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, d);
  agg_warp(kmin, kmax, lo, hi, unused, false);
  if (lane == 0) {
    s_cnt[warp] = cnt;
    s_min[warp] = kmin;
    s_max[warp] = kmax;
    s_lo[warp] = lo;
    s_hi[warp] = hi;
  }
  __syncthreads();
  if (threadIdx.x != 0) return 0;
  for (uint32_t w = 1; w < AG_THREADS / 32; w++) {
    cnt += s_cnt[w];
    kmin = min(kmin, uint64_t(s_min[w]));
    kmax = max(kmax, uint64_t(s_max[w]));
    agg_add128(lo, hi, s_lo[w], s_hi[w]);
  }
  *total = ok ? record(n_rows, cnt, kmin, kmax, lo, hi, fs) : PcoB200Aggregate{0, 0, 0, 0, 0, 0};
  return ok ? cnt : 0;
}

// One CTA: aggs and *total from the pages' accumulators (n_rows = page_n), then the status: the pages call's outcome (a refusal or failure
// as that call reports it, with *total zeroed), with the match count.
template <typename L>
__global__ void __launch_bounds__(AG_THREADS) ag_finish_kernel(const PcoB200AsyncPagesStatus* __restrict__ ps, const AgGroup* __restrict__ groups,
                                                               const IndexChunk* __restrict__ recs, uint32_t dtype, PcoB200Aggregate* __restrict__ aggs,
                                                               PcoB200Aggregate* __restrict__ total, PcoB200AsyncAggregateStatus* __restrict__ out) {
  const PcoB200AsyncPagesStatus p = *ps;
  const bool ok = p.kind == PCO_B200_OK;
  const uint64_t count = ag_total<L>(ok, ok ? p.n_pages : 0, p.n_written, groups, [&](uint64_t g) { return uint64_t(recs[g].n); }, dtype, aggs, total);
  if (threadIdx.x != 0) return;
  *out = PcoB200AsyncAggregateStatus{p.kind, p.device_status, p.page, p.n_written, p.n_pages, p.frames_needed, count};
}

// One CTA: ag_finish_kernel with the files call's outcome (n_rows = the file's count).
template <typename L>
__global__ void __launch_bounds__(AG_THREADS) agf_finish_kernel(const PcoB200AsyncFilesStatus* __restrict__ fst, const AgGroup* __restrict__ groups,
                                                                const FileCheck* __restrict__ fchk, uint32_t dtype, PcoB200Aggregate* __restrict__ aggs,
                                                                PcoB200Aggregate* __restrict__ total, PcoB200AsyncFilesAggregateStatus* __restrict__ out) {
  const PcoB200AsyncFilesStatus f = *fst;
  const bool ok = f.kind == PCO_B200_OK;
  const uint64_t count = ag_total<L>(ok, ok ? f.n_files : 0, f.n_written, groups, [&](uint64_t g) { return fchk[g].n_total; }, dtype, aggs, total);
  if (threadIdx.x != 0) return;
  *out = PcoB200AsyncFilesAggregateStatus{f.kind, f.device_status, f.file, f.chunk, f.n_written, f.n_files, count};
}

}  // namespace pcob200
