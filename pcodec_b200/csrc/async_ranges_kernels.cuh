// Kernels of pco_b200_decompress_ranges_async: ranges of an indexed standalone file decoded with the ranges in device memory and no host
// decision between launches, so random access can be queued behind the step that produced the positions or captured in a CUDA graph.
// What pco_b200_decompress_ranges plans on the host (plan_ranges and the loop of decompress_ranges_impl, host_api.cu) is planned here on
// the device, over grids fixed by the plan's capacities:
//   async_check_kernel (async_kernels.cuh)  the header / index check, the chunk table padded to max_chunks, the binomial table;
//   ar_chunks_kernel     checks that the chunk records tile [0, n_total) in order and clears the per-chunk marks;
//   ar_count_kernel      checks every range against n_total and sums the counts of each CTA's ranges;
//   ar_scan_kernel       (one CTA) the first refusals, and the CTA sums scanned into CTA offsets;
//   ar_mark_kernel       the destination offset of every range, the lowest range whose counts overflow 2^64, and the marks: for every
//                        chunk a range touches, its piece folded into the chunk's record by atomics (min lo, max hi, piece count,
//                        lowest range, destination of a lone piece), the lanes of a warp sharing the chunks of one range;
//   ar_window_kernel     per CTA of chunks: touched chunks and the sum of their windows;
//   ar_gate_kernel       (one CTA) scans those, and decides every refusal in the order pco_b200_decompress_ranges has them;
//   ar_tasks_kernel      the task table in chunk order: IndexChunk, WinTask (destination or slot, scratch rows), route; pads behind;
//   fused_narrow_kernel<L, true>, symwalk_kernel<true>, decode_kernel<L, 1 / 2, true>  (the window-mode decode, max_chunks CTAs);
//   ar_cold_kernel       the tasks the fast kernels reported ST_UNSUPPORTED for, one after another with the catch-all decoder;
//   ar_gather_kernel     the pieces of staged and catch-all tasks from their slots to the destination;
//   ar_finish_kernel     the lowest failing range, and the PcoB200AsyncRangesStatus.
// Window rule: a touched chunk's window is the chunk-relative end of the last number wanted of it (max hi) rounded up to 256, and
// window_needed is the sum over touched chunks.  A task's slot and its scratch rows are laid out by that scan: slot [W0, W0 + W) numbers
// (a staged window [lo, hi) needs hi - lo <= W, the catch-all decoder's [0, hi) needs hi <= W), rows [2 W0 / 256, 2 (W0 + W) / 256) (the
// general pair needs (vars) x (batches from the first decoded one to ceil(hi / 256)) <= 2 W / 256).
#pragma once
#include "async_kernels.cuh"
#include "cta_scan.cuh"
#include "decode_kernels.cuh"
#include "ranges_kernels.cuh"

namespace pcob200 {

constexpr int AR_THREADS = RANGES_THREADS;  // every multi-CTA launch; cta_copy_bytes strides by it
constexpr int AR_SCAN_THREADS = 1024;       // the one-CTA scans
constexpr uint32_t AR_GATHER_MAX_CTAS = 1u << 16;
constexpr uint32_t AR_NONE = 0xffffffffu;

enum : uint32_t { AR_DIRECT = 0, AR_STAGED = 1, AR_COLD = 2 };  // route of a task: straight into dst, into its slot, catch-all into its slot

// per chunk, the pieces of the ranges that touch it (ar_chunks_kernel clears, ar_mark_kernel folds, ar_tasks_kernel reads)
struct ArMark {
  uint32_t lo, hi;        // min lo, max hi of its pieces, chunk-relative
  uint32_t n_pieces;
  uint32_t first_range;   // lowest-index range with numbers in it
  uint32_t task, reserved;
  uint64_t lone_dst;      // min destination offset of its pieces: the place of a lone piece
};
struct ArChunkPart {      // per CTA of ar_chunks_kernel / ar_window_kernel (ar_gate_kernel turns the last two into offsets)
  uint32_t tile_bad;      // lowest chunk that breaks the tiling (n_chunks: the sum differs from n_total; AR_NONE: none)
  uint32_t reserved;
  uint64_t n_touched, window;
};
struct ArRangePart {      // per CTA of ar_count_kernel (ar_scan_kernel turns sum into an offset)
  CarrySum sum;
  uint64_t bad;           // lowest range past the file, as 2 i (NONE64: none)
  uint64_t reserved;
};
struct ArTask {
  uint32_t chunk, first_range;
  uint32_t route, reserved;
  uint64_t slot;          // first number of its slot in the staging area
};

// decided by ar_scan_kernel, ar_mark_kernel and ar_gate_kernel
struct ArState {
  uint32_t status;        // ST_OK or a PCO_B200_ASYNC_* refusal
  uint32_t n_ranges;      // ranges the call runs over (0 once refused before the ranges)
  uint32_t n_tasks;       // touched chunks (0 when refused)
  uint32_t reserved;
  uint64_t bad;           // lowest failing range as 2 i (past the file) or 2 i + 1 (the counts overflow there); NONE64: none
  uint64_t bad_chunk;     // the chunk a tiling refusal names
  uint64_t total;         // the sum of the counts
  uint64_t window_needed;
};

// everything the launches take by value; fp.src_len is src_cap
struct ArArgs {
  AsyncArgs a;            // what async_check_kernel takes (a.dst_cap is the plan's dst_cap)
  const PcoB200Range* ranges;
  const uint64_t* n_ranges;
  uint64_t window_cap;
  uint32_t max_ranges;
  uint32_t elem;          // bytes per number
};

// Workspace of one in-flight call, byte offsets, each region 256-byte aligned; the decode tail stages the window between the offset rows
// and the catch-all decoder's scratch.
struct ArLayout : AsyncDecodeTail {
  uint64_t state, table, marks, cparts, rparts, roff, rspan, tasks, wins, tinfo;
};
__host__ __device__ inline uint64_t ar_rows(uint64_t window_cap) { return 2 * (window_cap / BATCH_N); }
__host__ __device__ inline ArLayout ar_layout(uint64_t max_chunks, uint64_t max_ranges, uint64_t window_cap, uint32_t elem) {
  ArLayout l;
  l.state = async_align(sizeof(AsyncCheck));
  l.table = l.state + async_align(sizeof(ArState));
  l.marks = l.table + async_align(max_chunks * sizeof(IndexChunk));
  l.cparts = l.marks + async_align(max_chunks * sizeof(ArMark));
  l.rparts = l.cparts + async_align(ctas_of<AR_THREADS>(max_chunks) * sizeof(ArChunkPart));
  l.roff = l.rparts + async_align(ctas_of<AR_THREADS>(max_ranges) * sizeof(ArRangePart));
  l.rspan = l.roff + async_align(max_ranges * sizeof(uint64_t));
  l.tasks = l.rspan + async_align(max_ranges * sizeof(uint2));
  l.wins = l.tasks + async_align(max_chunks * sizeof(IndexChunk));
  l.tinfo = l.wins + async_align(max_chunks * sizeof(WinTask));
  static_cast<AsyncDecodeTail&>(l) =
      async_decode_tail(l.tinfo + async_align(max_chunks * sizeof(ArTask)), max_chunks, ar_rows(window_cap), window_cap * elem);
  return l;
}

// ceil(max_chunks / AR_THREADS) CTAs.  Chunk k breaks the tiling when n[k] = 0 or out_offset[k] differs from out_offset[k - 1] + n[k - 1]
// (out_offset[0] from 0); with every record in place, the last one must end at n_total.  This is plan_ranges' check (host_api.cu), in the
// same order: the lowest breaking chunk first, the sum after.
__global__ void __launch_bounds__(AR_THREADS) ar_chunks_kernel(const AsyncCheck* __restrict__ chk, const IndexChunk* __restrict__ table,
                                                              ArMark* __restrict__ marks, ArChunkPart* __restrict__ cparts) {
  __shared__ uint32_t s_bad;
  const uint32_t tid = threadIdx.x;
  if (tid == 0) s_bad = AR_NONE;
  __syncthreads();
  const uint32_t n_chunks = chk->status == ST_OK ? chk->n_chunks : 0u;
  const uint64_t k = uint64_t(blockIdx.x) * AR_THREADS + tid;
  if (k < n_chunks) {
    const IndexChunk r = table[k];
    const uint64_t expect = k == 0 ? 0 : table[k - 1].out_offset + table[k - 1].n;
    if (r.n == 0 || r.out_offset != expect) atomicMin(&s_bad, uint32_t(k));
    else if (k + 1 == n_chunks && r.out_offset + r.n != chk->n_total) atomicMin(&s_bad, n_chunks);
    marks[k] = ArMark{AR_NONE, 0u, 0u, AR_NONE, 0u, 0u, NONE64};
  }
  if (k == 0 && n_chunks == 0 && chk->status == ST_OK && chk->n_total != 0) s_bad = 0;  // no chunks: n_total must be 0
  __syncthreads();
  if (tid == 0) cparts[blockIdx.x] = ArChunkPart{s_bad, 0u, 0, 0};
}

// the ranges this call runs over: 0 when the file was refused or *n_ranges exceeds max_ranges
__device__ __forceinline__ uint64_t ar_n_ranges(const ArArgs& g, const AsyncCheck* chk) {
  const uint64_t n = *g.n_ranges;
  return chk->status == ST_OK && n <= g.max_ranges ? n : 0;
}

// ceil(max_ranges / AR_THREADS) CTAs, one range per thread: the CTA's sum of counts and its lowest range past the file.
__global__ void __launch_bounds__(AR_THREADS) ar_count_kernel(ArArgs g, const AsyncCheck* __restrict__ chk, ArRangePart* __restrict__ rparts) {
  __shared__ unsigned long long s_bad;
  const uint32_t tid = threadIdx.x;
  if (tid == 0) s_bad = NONE64;
  __syncthreads();
  const uint64_t n = ar_n_ranges(g, chk), n_total = chk->n_total;
  const uint64_t i = uint64_t(blockIdx.x) * AR_THREADS + tid;
  uint64_t cnt = 0;
  if (i < n) {
    const PcoB200Range r = g.ranges[i];
    cnt = r.count;
    if (r.count > n_total || r.start > n_total - r.count) atomicMin(&s_bad, 2ull * i);
  }
  CarrySum tot;
  block_exscan<AR_THREADS>(carry_sum(cnt), &tot);
  if (tid == 0) rparts[blockIdx.x] = ArRangePart{tot, s_bad, 0};
}

// One CTA: the refusals known so far (too many ranges, the header / index check, the tiling), and the CTA sums of the counts scanned into
// CTA offsets (in place).  Writes the ArState the next kernels read.
__global__ void __launch_bounds__(AR_SCAN_THREADS) ar_scan_kernel(ArArgs g, const AsyncCheck* __restrict__ chk, const ArChunkPart* __restrict__ cparts,
                                                                  ArRangePart* __restrict__ rparts, ArState* __restrict__ state) {
  __shared__ uint32_t s_tile;
  __shared__ unsigned long long s_bad;
  const uint32_t tid = threadIdx.x;
  if (tid == 0) {
    s_tile = AR_NONE;
    s_bad = NONE64;
  }
  __syncthreads();
  const uint64_t n_cparts = ctas_of<AR_THREADS>(g.a.max_chunks), n_rparts = ctas_of<AR_THREADS>(g.max_ranges);
  for (uint64_t c = tid; c < n_cparts; c += AR_SCAN_THREADS)
    if (cparts[c].tile_bad != AR_NONE) atomicMin(&s_tile, cparts[c].tile_bad);
  for (uint64_t c = tid; c < n_rparts; c += AR_SCAN_THREADS)
    if (rparts[c].bad != NONE64) atomicMin(&s_bad, rparts[c].bad);
  CarrySum total[1] = {};
  cta_scan_inplace<AR_SCAN_THREADS, 1>(
      n_rparts, [&](uint64_t c, int) { return rparts[c].sum; }, [&](uint64_t c, int, CarrySum v) { rparts[c].sum = v; }, total);
  __syncthreads();
  if (tid != 0) return;
  ArState s;
  s.status = ST_OK;
  s.bad = NONE64;
  s.bad_chunk = NONE64;
  s.n_tasks = 0;
  s.reserved = 0;
  s.window_needed = 0;
  s.total = total[0].s;
  if (*g.n_ranges > g.max_ranges) s.status = PCO_B200_ASYNC_TOO_MANY_RANGES;
  else if (chk->status != ST_OK) s.status = chk->status;
  else if (s_tile != AR_NONE) {
    s.status = s_tile < chk->n_chunks ? PCO_B200_ASYNC_INDEX_TILING : PCO_B200_ASYNC_INDEX_TOTAL;
    s.bad_chunk = s_tile;
  } else {
    s.bad = s_bad;  // ar_mark_kernel may lower it (a range where the counts overflow)
  }
  s.n_ranges = s.status == ST_OK ? uint32_t(ar_n_ranges(g, chk)) : 0u;
  *state = s;
}

// the last chunk whose out_offset <= x, over a table that tiles [0, n_total)
__device__ __forceinline__ uint32_t ar_find_chunk(const IndexChunk* __restrict__ table, uint32_t n_chunks, uint64_t x) {
  uint32_t a = 0, b = n_chunks;
  while (b - a > 1) {
    const uint32_t m = a + (b - a) / 2;
    if (table[m].out_offset <= x) a = m;
    else b = m;
  }
  return a;
}

// ceil(max_ranges / AR_THREADS) CTAs, one range per thread; then the warp's 32 ranges one at a time, the lanes over its chunks.
__global__ void __launch_bounds__(AR_THREADS) ar_mark_kernel(ArArgs g, const AsyncCheck* __restrict__ chk, const IndexChunk* __restrict__ table,
                                                             const ArRangePart* __restrict__ rparts, ArState* __restrict__ state, ArMark* __restrict__ marks,
                                                             uint64_t* __restrict__ roff, uint2* __restrict__ rspan) {
  if (state->status != ST_OK) return;  // uniform: every thread leaves
  const uint32_t tid = threadIdx.x, lane = tid & 31;
  const uint64_t n = state->n_ranges, n_total = chk->n_total;
  const uint32_t n_chunks = chk->n_chunks;
  const uint64_t i = uint64_t(blockIdx.x) * AR_THREADS + tid;
  PcoB200Range r{0, 0};
  if (i < n) r = g.ranges[i];
  CarrySum tot;
  const CarrySum ex = carry_add(rparts[blockIdx.x].sum, block_exscan<AR_THREADS>(carry_sum(r.count), &tot));
  const CarrySum inc = carry_add(ex, carry_sum(r.count));
  const bool valid = i < n && r.count <= n_total && r.start <= n_total - r.count;
  if (i < n && !ex.ovf && inc.ovf) atomicMin(reinterpret_cast<unsigned long long*>(&state->bad), 2ull * i + 1);
  uint32_t c0 = 0, c1 = 0;
  if (valid && r.count > 0) {
    c0 = ar_find_chunk(table, n_chunks, r.start);
    c1 = ar_find_chunk(table, n_chunks, r.start + r.count - 1);
  }
  if (i < n) {
    roff[i] = ex.s;
    rspan[i] = make_uint2(c0, c1);
  }
  const bool mine = valid && r.count > 0;
  uint32_t todo = __ballot_sync(0xffffffffu, mine);
  while (todo) {
    const int j = __ffs(todo) - 1;
    todo &= todo - 1;
    const uint64_t start = __shfl_sync(0xffffffffu, r.start, j), end = start + __shfl_sync(0xffffffffu, r.count, j);
    const uint64_t off = __shfl_sync(0xffffffffu, ex.s, j);
    const uint32_t a = __shfl_sync(0xffffffffu, c0, j), b = __shfl_sync(0xffffffffu, c1, j);
    const uint32_t range = uint32_t(__shfl_sync(0xffffffffu, i, j));
    for (uint32_t k = a + lane; k <= b; k += 32) {
      const IndexChunk rec = table[k];
      const uint64_t from = max(start, rec.out_offset), to = min(end, rec.out_offset + rec.n);
      ArMark* m = marks + k;
      atomicMin(&m->lo, uint32_t(from - rec.out_offset));
      atomicMax(&m->hi, uint32_t(to - rec.out_offset));
      atomicAdd(&m->n_pieces, 1u);
      atomicMin(&m->first_range, range);
      atomicMin(reinterpret_cast<unsigned long long*>(&m->lone_dst), off + (from - start));
    }
  }
}

// ceil(max_chunks / AR_THREADS) CTAs: the CTA's touched chunks and the sum of their windows.
__global__ void __launch_bounds__(AR_THREADS) ar_window_kernel(const AsyncCheck* __restrict__ chk, const ArState* __restrict__ state,
                                                               const ArMark* __restrict__ marks, ArChunkPart* __restrict__ cparts) {
  if (state->status != ST_OK) return;
  const uint64_t k = uint64_t(blockIdx.x) * AR_THREADS + threadIdx.x;
  uint64_t touched = 0, w = 0;
  if (k < chk->n_chunks && marks[k].n_pieces > 0) {
    touched = 1;
    w = (uint64_t(marks[k].hi) + BATCH_N - 1) / BATCH_N * BATCH_N;
  }
  uint64_t t_tot, w_tot;
  block_exscan<AR_THREADS>(touched, &t_tot);
  block_exscan<AR_THREADS>(w, &w_tot);
  if (threadIdx.x == 0) {
    cparts[blockIdx.x].n_touched = t_tot;
    cparts[blockIdx.x].window = w_tot;
  }
}

// One CTA: the touched chunks and windows of the CTAs scanned into offsets (in place), and every remaining refusal in the order of
// pco_b200_decompress_ranges: a range past the file or where the counts overflow, then a total above dst_cap; then the window.
__global__ void __launch_bounds__(AR_SCAN_THREADS) ar_gate_kernel(ArArgs g, ArChunkPart* __restrict__ cparts, ArState* __restrict__ state) {
  if (state->status != ST_OK) return;
  auto sum = [&](uint64_t c, int k) -> uint64_t& { return k ? cparts[c].window : cparts[c].n_touched; };
  uint64_t total[2] = {};
  cta_scan_inplace<AR_SCAN_THREADS, 1>(
      ctas_of<AR_THREADS>(g.a.max_chunks), [&](uint64_t c, int k) { return sum(c, k); }, [&](uint64_t c, int k, uint64_t v) { sum(c, k) = v; }, total);
  if (threadIdx.x != 0) return;
  ArState s = *state;
  if (s.bad != NONE64) s.status = (s.bad & 1) ? PCO_B200_ASYNC_RANGE_OVERFLOW : PCO_B200_ASYNC_RANGE_PAST;
  else if (s.total > g.a.dst_cap) s.status = PCO_B200_ASYNC_DST_SHORT;
  if (s.status == ST_OK || s.status == PCO_B200_ASYNC_DST_SHORT) s.window_needed = total[1];  // the windows are known once the ranges are
  if (s.status == ST_OK && s.window_needed > g.window_cap) s.status = PCO_B200_ASYNC_WINDOW;
  s.n_tasks = s.status == ST_OK ? uint32_t(total[0]) : 0u;
  *state = s;
}

// ceil(max_chunks / AR_THREADS) CTAs: touched chunk k becomes task t (its rank among the touched chunks) with the window scan's slot and
// rows; task entries from n_tasks to max_chunks are pads, which the decode kernels refuse without reading the file.  A refused call
// leaves pads only, so nothing reaches dst.
__global__ void __launch_bounds__(AR_THREADS) ar_tasks_kernel(ArArgs g, const AsyncCheck* __restrict__ chk, const ArState* __restrict__ state,
                                                              const IndexChunk* __restrict__ table, ArMark* __restrict__ marks,
                                                              const ArChunkPart* __restrict__ cparts, IndexChunk* __restrict__ tasks,
                                                              WinTask* __restrict__ wins, ArTask* __restrict__ tinfo, uint8_t* __restrict__ dst,
                                                              uint8_t* __restrict__ stage) {
  const uint64_t k = uint64_t(blockIdx.x) * AR_THREADS + threadIdx.x;
  const uint32_t n_tasks = state->n_tasks;
  ArMark m{AR_NONE, 0u, 0u, AR_NONE, 0u, 0u, NONE64};
  if (n_tasks && k < chk->n_chunks) m = marks[k];
  const uint64_t touched = m.n_pieces > 0 ? 1 : 0;
  const uint64_t w = touched ? (uint64_t(m.hi) + BATCH_N - 1) / BATCH_N * BATCH_N : 0;
  uint64_t tot;
  const uint64_t t = cparts[blockIdx.x].n_touched + block_exscan<AR_THREADS>(touched, &tot);
  const uint64_t w0 = cparts[blockIdx.x].window + block_exscan<AR_THREADS>(w, &tot);
  if (touched) {
    const bool lone = m.n_pieces == 1;
    const uint8_t* at = lone ? dst + m.lone_dst * g.elem : stage + w0 * g.elem;
    tasks[t] = table[k];
    wins[t] = WinTask{m.lo, m.hi, uint64_t(reinterpret_cast<uintptr_t>(at)), 2 * (w0 / BATCH_N)};
    tinfo[t] = ArTask{uint32_t(k), m.first_range, lone ? AR_DIRECT : AR_STAGED, 0u, w0};
    marks[k].task = uint32_t(t);
  }
  if (k < g.a.max_chunks && k >= n_tasks) tasks[k] = IndexChunk{g.a.fp.src_len, 0u, 0u, 0, 0};
}

// One CTA.  Its threads list the tasks in [0, n_tasks) whose status is ST_UNSUPPORTED, AR_THREADS at a time; thread 0 decodes each with
// the catch-all decoder from the chunk's start to max hi into the task's slot.  It stops there (ST_DST_FULL) or, when the window reaches
// the chunk's end, behind the chunk: the chunk is decoded once the decoder has counted it (decompress_ranges_impl's rule).
template <typename L>
__global__ void __launch_bounds__(AR_THREADS) ar_cold_kernel(FileParams fp, const ArState* __restrict__ state, const IndexChunk* __restrict__ tasks,
                                                             const WinTask* __restrict__ wins, ArTask* __restrict__ tinfo, uint32_t* __restrict__ statuses,
                                                             L* __restrict__ stage, uint8_t* __restrict__ scratch) {
  __shared__ uint32_t s_list[AR_THREADS];
  __shared__ uint32_t s_count;
  const int tid = threadIdx.x;
  const uint32_t n_tasks = state->n_tasks;
  for (uint32_t base = 0; base < n_tasks; base += AR_THREADS) {
    if (tid == 0) s_count = 0;
    __syncthreads();
    const uint32_t t = base + tid;
    if (t < n_tasks && statuses[t] == ST_UNSUPPORTED) s_list[atomicAdd(&s_count, 1u)] = t;
    __syncthreads();
    if (tid == 0) {
      for (uint32_t i = 0; i < s_count; i++) {
        const uint32_t c = s_list[i];
        ColdResult res;
        cold_decode_run<L>(fp, tasks[c].chunk_offset, stage + tinfo[c].slot, wins[c].hi, scratch, ASYNC_COLD_WINDOW_LOG, &res);
        statuses[c] = cold_status(res);
        tinfo[c].route = AR_COLD;
      }
    }
    __syncthreads();
  }
}

// min(max_ranges, AR_GATHER_MAX_CTAS) CTAs over the ranges.  A CTA lists, AR_THREADS chunks at a time, the chunks of its range whose task
// decoded into a slot and succeeded, and copies each piece from the slot to its place in dst.
__global__ void __launch_bounds__(AR_THREADS) ar_gather_kernel(ArArgs g, const ArState* __restrict__ state, const IndexChunk* __restrict__ table,
                                                               const ArMark* __restrict__ marks, const WinTask* __restrict__ wins,
                                                               const ArTask* __restrict__ tinfo, const uint32_t* __restrict__ statuses,
                                                               const uint64_t* __restrict__ roff, const uint2* __restrict__ rspan, uint8_t* __restrict__ dst,
                                                               const uint8_t* __restrict__ stage) {
  __shared__ uint32_t s_list[AR_THREADS];
  __shared__ uint32_t s_count;
  if (state->n_tasks == 0) return;  // refused, or nothing decoded
  const uint32_t tid = threadIdx.x, elem = g.elem;
  const uint64_t n = state->n_ranges;
  for (uint64_t i = blockIdx.x; i < n; i += gridDim.x) {
    const PcoB200Range r = g.ranges[i];
    if (r.count == 0) continue;
    const uint2 span = rspan[i];
    const uint64_t off = roff[i], end = r.start + r.count;
    for (uint64_t base = span.x; base <= span.y; base += AR_THREADS) {
      if (tid == 0) s_count = 0;
      __syncthreads();
      const uint64_t k = base + tid;
      if (k <= span.y) {
        const uint32_t t = marks[k].task;
        if (tinfo[t].route != AR_DIRECT && statuses[t] == ST_OK) s_list[atomicAdd(&s_count, 1u)] = uint32_t(k);
      }
      __syncthreads();
      const uint32_t cnt = s_count;
      for (uint32_t q = 0; q < cnt; q++) {
        const uint32_t kk = s_list[q];
        const IndexChunk rec = table[kk];
        const uint32_t t = marks[kk].task;
        const uint64_t from = max(r.start, rec.out_offset), to = min(end, rec.out_offset + rec.n);
        const uint64_t wlo = tinfo[t].route == AR_COLD ? 0 : wins[t].lo;
        cta_copy_bytes(dst + (off + (from - r.start)) * elem, stage + (tinfo[t].slot + (from - rec.out_offset) - wlo) * elem, (to - from) * elem);
      }
      __syncthreads();
    }
  }
}

// One CTA: the refusal, or the lowest failing range (ties: the lower task, i.e. chunk), or success.
__global__ void __launch_bounds__(AR_SCAN_THREADS) ar_finish_kernel(const ArState* __restrict__ state, const ArTask* __restrict__ tinfo,
                                                                    const uint32_t* __restrict__ statuses, PcoB200AsyncRangesStatus* __restrict__ out) {
  __shared__ unsigned long long s_min;
  const uint32_t tid = threadIdx.x;
  if (tid == 0) s_min = NONE64;
  __syncthreads();
  const ArState s = *state;
  for (uint32_t t = tid; t < s.n_tasks; t += AR_SCAN_THREADS)
    if (statuses[t] != ST_OK) atomicMin(&s_min, (uint64_t(tinfo[t].first_range) << 32) | t);
  __syncthreads();
  if (tid != 0) return;
  PcoB200AsyncRangesStatus r;
  r.kind = PCO_B200_OK;
  r.device_status = ST_OK;
  r.range = NONE64;
  r.chunk = NONE64;
  r.window_needed = s.window_needed;
  r.n_written = 0;
  const bool known = s.status == ST_OK || s.status == PCO_B200_ASYNC_DST_SHORT || s.status == PCO_B200_ASYNC_WINDOW;
  if (known) r.n_written = s.total;
  if (s.status != ST_OK) {
    r.kind = async_kind_of(s.status);
    r.device_status = s.status;
    if (s.status == PCO_B200_ASYNC_RANGE_PAST || s.status == PCO_B200_ASYNC_RANGE_OVERFLOW) r.range = s.bad >> 1;
    if (s.status == PCO_B200_ASYNC_INDEX_TILING) r.chunk = s.bad_chunk;
  } else if (s_min != NONE64) {
    const uint32_t t = uint32_t(s_min);
    const uint32_t st = statuses[t];
    r.kind = async_kind_of(st);
    r.device_status = st;
    r.range = s_min >> 32;
    r.chunk = tinfo[t].chunk;
  }
  *out = r;
}

}  // namespace pcob200
