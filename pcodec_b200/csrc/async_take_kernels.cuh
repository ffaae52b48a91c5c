// Kernels of pco_b200_take_pages_async and pco_b200_take_files_async: the numbers at caller-given, strictly ascending positions of the
// concatenation the matching decompress call writes, decoding only the pages or chunks some position touches.  The decompress call's
// launches run unchanged with rows_cap in the role of dst_cap (and, for files, ff_map_kernel and ff_cold_list_kernel around them, as the
// files filter runs them).  Between its front end and its decode stage runs the take's plan:
//   tk_front_pages_kernel / tk_front_files_kernel  (one thread) the TkState: whether the front end passed, the rows placed, the records
//                        and *n_positions as read;
//   tk_check_kernel      the positions against max_positions, their order and the rows: the lowest offending index of each check;
//   tk_mark_kernel       a CTA per record (striding): when the gate passes, the record's positions found by binary search, its touched
//                        flag, and for a touched record every batch's run [first, end) of position indices in its slot; on a refusal
//                        every record untouched;
//   tk_cold_list_kernel  (pages, one CTA) the cold list kept to the touched pages, in page order, so ap_cold_kernel decodes only those.
// Then the decode stage in take mode: fused_narrow_kernel<L, false, true, false, true> lets an untouched record go at its first lines
// with ST_OK, and the TAKE instantiations store each batch's numbers at its run's positions (take_store8, decode_kernels.cuh).  Cold
// records (those routed to ap_cold_kernel / cold_chunks_kernel, decoded into the value staging at their rows) are taken in place by
// tk_cold_pages_kernel / tk_cold_files_kernel through the same take_store8.  tk_finish_pages_kernel / tk_finish_files_kernel write the
// status.
// The batch slots are the filters' (fl_slots, async_filter_kernels.cuh): batch b of record r, its numbers from row O, has slot
// O / 256 + map[r] + b, with map the pages' fast_page (record -> page, and the take's records are pages) or ff_map_kernel's identity.
#pragma once
#include "async_filter_files_kernels.cuh"

namespace pcob200 {

constexpr int TK_THREADS = 256;         // tk_check_kernel, tk_mark_kernel, the cold take kernels
constexpr int TK_SCAN_THREADS = 1024;   // tk_cold_list_kernel, tk_finish_files_kernel
constexpr uint64_t TK_MAX_CTAS = 4096;  // the largest grid of tk_check_kernel and tk_mark_kernel; their CTAs stride

// decided by the plan kernels, in launch order
struct TkState {
  uint32_t front_ok, reserved;   // 1: the decompress call's front end refused nothing (pages: nor did the walk)
  uint64_t n_read;               // *n_positions as read
  uint64_t rows;                 // the rows of the concatenation (valid when front_ok)
  uint64_t n_records;            // pages of the batch / chunks of the merged table
  unsigned long long nbad_order;  // ~j of the lowest j with positions[j] <= positions[j - 1] (0: none)
  unsigned long long nbad_past;   // ~j of the lowest j with positions[j] >= rows (0: none)
  unsigned long long n_touched;   // records some position touches (once the gate passed)
};
static_assert(sizeof(TkState) == 56, "workspace layout");

__device__ __forceinline__ bool tk_gate(const TkState& t, uint64_t max_positions) {
  return t.front_ok && t.n_read <= max_positions && t.nbad_order == 0 && t.nbad_past == 0;
}

// Workspace of one in-flight pages call: the pages call's (ap_layout with dst_cap = rows_cap) | the pages status | TkState | TakeRun per
// slot | touched flag per page | value staging (rows_cap numbers of elem bytes).  Each region 256-byte aligned.
struct TkLayout : ApLayout {
  uint64_t pstatus, tstate, runs, touched, stage, tk_total;
};
__host__ __device__ inline TkLayout tk_layout(uint64_t max_pages, uint64_t rows_cap, uint64_t frame_cap, uint32_t elem) {
  TkLayout l;
  static_cast<ApLayout&>(l) = ap_layout(max_pages, rows_cap, frame_cap);
  l.pstatus = l.total;
  l.tstate = l.pstatus + async_align(sizeof(PcoB200AsyncPagesStatus));
  l.runs = l.tstate + async_align(sizeof(TkState));
  l.touched = l.runs + async_align(fl_slots(max_pages, rows_cap) * sizeof(TakeRun));
  l.stage = l.touched + async_align(max_pages * sizeof(uint32_t));
  l.tk_total = l.stage + async_align(rows_cap * elem);
  return l;
}

// Workspace of one in-flight files call: the files call's (af_layout with dst_cap = rows_cap) | the files status | TkState | TakeRun per
// slot | touched flag per chunk | value staging | the slot map (max_chunks words) | the cold list (its length, then up to max_chunks
// records).
struct TkfLayout : AfLayout {
  uint64_t fstatus, tstate, runs, touched, stage, slot_map, cold_list, tkf_total;
};
__host__ __device__ inline TkfLayout tkf_layout(uint64_t max_files, uint64_t max_chunks, uint64_t rows_cap, uint32_t elem) {
  TkfLayout l;
  static_cast<AfLayout&>(l) = af_layout(max_files, max_chunks, rows_cap);
  l.fstatus = l.total;
  l.tstate = l.fstatus + async_align(sizeof(PcoB200AsyncFilesStatus));
  l.runs = l.tstate + async_align(sizeof(TkState));
  l.touched = l.runs + async_align(fl_slots(max_chunks, rows_cap) * sizeof(TakeRun));
  l.stage = l.touched + async_align(max_chunks * sizeof(uint32_t));
  l.slot_map = l.stage + async_align(rows_cap * elem);
  l.cold_list = l.slot_map + async_align(max_chunks * sizeof(uint32_t));
  l.tkf_total = l.cold_list + async_align((max_chunks + 1) * sizeof(uint32_t));
  return l;
}

// One thread: the TkState of a pages call, behind ap_route_kernel.  The front end passed when ap_scan_kernel refused nothing and no page
// failed its meta or walk.
__global__ void __launch_bounds__(32) tk_front_pages_kernel(const ApState* __restrict__ s, const uint64_t* __restrict__ n_positions,
                                                            TkState* __restrict__ ts) {
  if (threadIdx.x != 0) return;
  *ts = TkState{s->status == ST_OK && s->fail_page == NONE64 ? 1u : 0u, 0u, *n_positions, s->nums.s, s->n_pages, 0, 0, 0};
}

// One thread: the TkState of a files call, behind af_table_kernel (which left any refusal pending in chk->status and the merged table's
// chunk count in chk->n_chunks).
__global__ void __launch_bounds__(32) tk_front_files_kernel(const AfState* __restrict__ s, const AsyncCheck* __restrict__ chk,
                                                            const uint64_t* __restrict__ n_positions, TkState* __restrict__ ts) {
  if (threadIdx.x != 0) return;
  *ts = TkState{chk->status == ST_OK ? 1u : 0u, 0u, *n_positions, s->total.s, chk->n_chunks, 0, 0, 0};
}

// min(ceil(max_positions / TK_THREADS), TK_MAX_CTAS) CTAs striding over positions[0 : *n_positions) (none when the count is above
// max_positions): the lowest j that breaks the strict order and the lowest j at or past the rows, each met by atomicMax of ~j.
__global__ void __launch_bounds__(TK_THREADS) tk_check_kernel(const uint64_t* __restrict__ pos, uint64_t max_positions, TkState* __restrict__ ts) {
  __shared__ unsigned long long s_order, s_past;
  if (threadIdx.x == 0) s_order = s_past = 0;
  __syncthreads();
  const uint64_t n = ts->n_read <= max_positions ? ts->n_read : 0, rows = ts->rows;
  uint64_t order = NONE64, past = NONE64;  // a thread's first of each is its lowest
  for (uint64_t j = uint64_t(blockIdx.x) * TK_THREADS + threadIdx.x; j < n; j += uint64_t(gridDim.x) * TK_THREADS) {
    const uint64_t p = pos[j];
    if (order == NONE64 && j > 0 && p <= pos[j - 1]) order = j;
    if (past == NONE64 && p >= rows) past = j;
    if (order != NONE64 && past != NONE64) break;
  }
  if (order != NONE64) atomicMax(&s_order, ~order);
  if (past != NONE64) atomicMax(&s_past, ~past);
  __syncthreads();
  if (threadIdx.x != 0) return;
  if (s_order) atomicMax(&ts->nbad_order, s_order);
  if (s_past) atomicMax(&ts->nbad_past, s_past);
}

// The first index in [lo, hi] whose position is at least x, where positions[lo .. hi) are strictly ascending and lie in [o, e), and
// o <= x <= e.  At most e - x of them are at or above x and at most x - o below it, which narrows the search (to one index when every
// row is taken).
__device__ __forceinline__ uint64_t tk_search(const uint64_t* __restrict__ pos, uint64_t lo, uint64_t hi, uint64_t o, uint64_t e, uint64_t x) {
  uint64_t a = hi - min(hi - lo, e - x), b = min(hi, lo + (x - o));
  while (a < b) {
    const uint64_t m = a + (b - a) / 2;
    if (pos[m] < x) a = m + 1;
    else b = m;
  }
  return a;
}

// The first index in [lo, hi) whose position is at least x, else hi (any order: an unsorted array gives some index in range).
__device__ __forceinline__ uint64_t tk_lower_bound(const uint64_t* __restrict__ pos, uint64_t lo, uint64_t hi, uint64_t x) {
  while (lo < hi) {
    const uint64_t m = lo + (hi - lo) / 2;
    if (pos[m] < x) lo = m + 1;
    else hi = m;
  }
  return lo;
}

// min(max_records, TK_MAX_CTAS) CTAs, a record at a time (records[0 : n_records): the pages' placed records or the merged chunk table;
// record r's slots start at out_offset / 256 + r).  When the gate refuses, every record is left untouched.  Otherwise thread 0 finds the
// record's positions [lo, hi) and writes its touched flag; for a touched record the CTA writes every batch's run.
__global__ void __launch_bounds__(TK_THREADS) tk_mark_kernel(const uint64_t* __restrict__ pos, uint64_t max_positions, const IndexChunk* __restrict__ recs,
                                                             TkState* __restrict__ ts, uint32_t* __restrict__ touched, TakeRun* __restrict__ runs) {
  __shared__ uint64_t s_lo, s_hi, s_first[TK_THREADS];
  const TkState t = *ts;
  const bool ok = tk_gate(t, max_positions);
  for (uint64_t r = blockIdx.x; r < t.n_records; r += gridDim.x) {  // uniform: every thread runs the same records
    if (!ok) {
      if (threadIdx.x == 0) touched[r] = 0;
      continue;
    }
    const IndexChunk rec = recs[r];
    const uint64_t o = rec.out_offset, e = o + rec.n;
    if (threadIdx.x == 0) {
      const uint64_t lo = tk_lower_bound(pos, 0, t.n_read, o), hi = tk_lower_bound(pos, lo, t.n_read, e);
      s_lo = lo;
      s_hi = hi;
      touched[r] = hi > lo ? 1u : 0u;
      if (hi > lo) atomicAdd(&ts->n_touched, 1ull);
    }
    __syncthreads();
    const uint64_t lo = s_lo, hi = s_hi;
    __syncthreads();  // s_lo, s_hi are read before the next record writes them
    if (hi == lo) continue;
    const uint32_t nb = n_batches_of(rec.n);
    const uint64_t slot0 = o / BATCH_N + r;
    // a tile of batches at a time: each thread finds its batch's first position, and its end is the next batch's first
    for (uint32_t t0 = 0; t0 < nb; t0 += TK_THREADS) {
      const uint32_t b = t0 + threadIdx.x;
      const uint64_t first = b < nb ? tk_search(pos, lo, hi, o, e, o + uint64_t(b) * BATCH_N) : hi;
      s_first[threadIdx.x] = first;
      __syncthreads();
      if (b < nb) {
        const uint64_t end = b + 1 == nb ? hi : threadIdx.x + 1 < TK_THREADS ? s_first[threadIdx.x + 1]
                                                                            : tk_search(pos, lo, hi, o, e, o + uint64_t(b + 1) * BATCH_N);
        runs[slot0 + b] = TakeRun{first, end};
      }
      __syncthreads();
    }
  }
}

// One CTA (pages): the cold list ap_route_kernel made kept to its touched pages, in page order, and its length, so ap_cold_kernel decodes
// only those.  A tile's reads all happen before its barrier-ended scan, and an entry moves only down, so the compaction runs in place.
__global__ void __launch_bounds__(TK_SCAN_THREADS) tk_cold_list_kernel(ApState* __restrict__ state, uint32_t* __restrict__ cold_list,
                                                                       const uint32_t* __restrict__ touched) {
  const uint64_t n_cold = state->n_cold;
  uint64_t carry = 0;
  for (uint64_t base = 0; base < n_cold; base += TK_SCAN_THREADS) {
    const uint64_t k = base + threadIdx.x;
    uint32_t p = 0;
    uint64_t keep = 0;
    if (k < n_cold) {
      p = cold_list[k];
      keep = touched[p] ? 1 : 0;
    }
    uint64_t tot;
    const uint64_t at = carry + block_exscan<TK_SCAN_THREADS>(keep, &tot);
    if (keep) cold_list[at] = p;
    carry += tot;
  }
  if (threadIdx.x == 0) state->n_cold = carry;
}

// The batches of record r (its numbers at rows rec.out_offset .., decoded into the value staging by a catch-all decoder) taken by the
// CTA's warps: a warp whose batch has a run reads the batch into registers and take_store8 writes its positions' numbers.
template <typename L>
__device__ __forceinline__ void tk_take_in_place(const FiltStage& f, const IndexChunk& rec, uint64_t r, const L* __restrict__ stage) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t nb = n_batches_of(rec.n);
  for (uint32_t b = warp; b < nb; b += TK_THREADS / 32) {
    const uint64_t row = rec.out_offset + uint64_t(b) * BATCH_N, slot = rec.out_offset / BATCH_N + r + b;
    const TakeRun run = take_runs(f)[slot];
    if (run.end == run.first) continue;  // uniform over the warp
    const uint32_t cnt = min(uint32_t(BATCH_N), rec.n - b * BATCH_N);
    L v[8];
#pragma unroll
    for (int e = 0; e < 8; e++) v[e] = uint32_t(lane * 8 + e) < cnt ? stage[row + lane * 8 + e] : L(0);
    take_store8<L>(f, row, slot, cnt, lane, v);
  }
}

// One CTA per cold-list entry k (pages): the touched cold page, decoded into the value staging by ap_cold_kernel, taken in place.  Cold
// pages at or behind a failure were not decoded; they are left alone.
template <typename L>
__global__ void __launch_bounds__(TK_THREADS) tk_cold_pages_kernel(const ApState* __restrict__ state, const IndexChunk* __restrict__ recs,
                                                                   const uint32_t* __restrict__ cold_list, FiltStage f, const L* __restrict__ stage) {
  const uint64_t k = blockIdx.x;
  if (k >= state->n_cold) return;
  const uint32_t p = cold_list[k];
  if (p >= state->fail_page || p >= (state->decode_fail >> 32)) return;
  tk_take_in_place<L>(f, recs[p], p, stage);
}

// min(max_chunks, FF_COLD_CTAS) CTAs striding over the cold list (files): each touched cold record that cold_chunks_kernel decoded into
// the value staging without failure, taken in place.
template <typename L>
__global__ void __launch_bounds__(TK_THREADS) tk_cold_files_kernel(const uint32_t* __restrict__ cold_list, const IndexChunk* __restrict__ table,
                                                                   const uint32_t* __restrict__ statuses, FiltStage f, const L* __restrict__ stage) {
  const uint32_t n_cold = cold_list[0];
  for (uint32_t k = blockIdx.x; k < n_cold; k += gridDim.x) {
    const uint32_t r = cold_list[1 + k];
    if (statuses[r] != ST_OK) continue;
    tk_take_in_place<L>(f, table[r], r, stage);
  }
}

// Thread 0 of a finish kernel, with the decompress call's outcome already in r: that outcome when it failed (a refusal of its front end
// is decided before anything is decoded, and only touched records are decoded), else the take's own refusal in its order (the count,
// then the lowest j out of order, then the lowest j past the rows), else success with the records decoded.
template <typename S>
__device__ __forceinline__ void tk_decide(const TkState& t, uint64_t max_positions, S& r) {
  r.n_positions = t.n_read;
  r.position = NONE64;
  r.records_decoded = 0;
  if (r.kind != PCO_B200_OK) return;
  uint32_t code = ST_OK;
  if (t.n_read > max_positions) code = PCO_B200_TAKE_TOO_MANY;
  else if (t.nbad_order) code = PCO_B200_TAKE_ORDER, r.position = ~t.nbad_order;
  else if (t.nbad_past) code = PCO_B200_TAKE_PAST, r.position = ~t.nbad_past;
  if (code != ST_OK) {
    r.kind = PCO_B200_INVALID_ARGUMENT;
    r.device_status = code;
  } else {
    r.records_decoded = t.n_touched;
  }
}

// One thread: the pages take's status from the pages call's and the TkState.
__global__ void __launch_bounds__(32) tk_finish_pages_kernel(const PcoB200AsyncPagesStatus* __restrict__ ps, const TkState* __restrict__ ts,
                                                             uint64_t max_positions, PcoB200AsyncTakeStatus* __restrict__ out) {
  if (threadIdx.x != 0) return;
  const PcoB200AsyncPagesStatus p = *ps;
  PcoB200AsyncTakeStatus r;
  r.kind = p.kind;
  r.device_status = p.device_status;
  r.page = p.page;
  r.n_written = p.n_written;
  r.n_pages = p.n_pages;
  r.frames_needed = p.frames_needed;
  tk_decide(*ts, max_positions, r);
  *out = r;
}

// One CTA: the files take's status from the files call's and the TkState; on success, file_ns (the files call ran without it, so that a
// refused take writes none).
__global__ void __launch_bounds__(TK_SCAN_THREADS) tk_finish_files_kernel(const PcoB200AsyncFilesStatus* __restrict__ fs, const TkState* __restrict__ ts,
                                                                          const AfState* __restrict__ state, const FileCheck* __restrict__ fchk,
                                                                          uint64_t max_positions, uint64_t* __restrict__ file_ns,
                                                                          PcoB200AsyncFilesTakeStatus* __restrict__ out) {
  const PcoB200AsyncFilesStatus f = *fs;
  PcoB200AsyncFilesTakeStatus r;
  r.kind = f.kind;
  r.device_status = f.device_status;
  r.file = f.file;
  r.chunk = f.chunk;
  r.n_written = f.n_written;
  r.n_files = f.n_files;
  tk_decide(*ts, max_positions, r);
  if (r.kind == PCO_B200_OK && file_ns)
    for (uint64_t i = threadIdx.x; i < state->n_files; i += TK_SCAN_THREADS) file_ns[i] = fchk[i].n_total;
  if (threadIdx.x == 0) *out = r;
}

}  // namespace pcob200
