// Kernels of pco_b200_decompress_pages_async: a batch of wrapped-format pages decoded with the page refs in device memory and no host
// decision between launches, so a list of pages a kernel picked (a filter on page statistics, a row-group selection) can be decoded behind
// that kernel or captured in a CUDA graph.  What decompress_pages_impl (host_api.cu) does on the host - the page table, the walk's
// placeholder records, the route of every page, the compaction of the fast pages' records, the re-walk of a failing page and one catch-all
// launch per cold page - is done here on the device, over grids fixed by the plan's max_pages:
//   ap_pages_kernel      one thread per page slot: its ref against metas_cap / pages_cap and page_n, its frame size and entries room, CTA
//                        sums of frame bytes, entry bytes and numbers, and (CTA 0) the binomial table decode_kernel reads;
//   ap_scan_kernel       (one CTA) *n_pages against max_pages, the lowest ref refusal, the CTA sums scanned into CTA offsets, and the totals
//                        against dst_cap and frame_cap;
//   ap_place_kernel      every page's WrappedPage row and IndexChunk placeholder (as lay_out_entries); pads for every other slot;
//   frame_pages_kernel, walk_kernel<SMALL_MAX_SIZE_LOG>  (wrapped_kernels.cuh, decode_kernels.cuh) unchanged, over max_pages CTAs;
//   ap_route_kernel      (one CTA) the lowest failing page from the meta statuses, walk statuses and walk ends; the walked records of the
//                        fast pages in front of it compacted into the decode table, and the cold pages in front of it listed;
//   ap_rewalk_kernel     (one CTA) the failing page walked once more over its own frame, for the kind pco_b200_page_decompress gives;
//   fused_narrow_kernel<L>, symwalk_kernel<false>, decode_kernel<L, 1 / 2>  over the decode table, as pco_b200_decompress_async;
//   ap_cold_kernel<L>    (one CTA) the cold pages in front of the lowest failure, in page order, with the catch-all decoder;
//   ap_finish_kernel     the lowest failing page, else the pending refusal, into the PcoB200AsyncPagesStatus.
// A refused batch, or one whose lowest failing page is j, decodes nothing at or behind j's slot of dst.
#pragma once
#include "async_kernels.cuh"
#include "cta_scan.cuh"
#include "wrapped_kernels.cuh"

namespace pcob200 {

constexpr int AP_THREADS = 256;        // the per-slot launches
constexpr int AP_SCAN_THREADS = 1024;  // the one-CTA launches

// per CTA of ap_pages_kernel (ap_scan_kernel turns the sums into CTA offsets, in place)
struct ApPart {
  CarrySum frames, entries, nums;
  uint64_t bad_ref;  // lowest ref refusal of the CTA as (page << 32) | status (NONE64: none)
};

// decided by the kernels, in launch order
struct ApState {
  uint32_t status;          // ST_OK, or a PCO_B200_ASYNC_* refusal decided before the device touches a page (ap_scan_kernel)
  uint32_t rewalk;          // 1: ap_rewalk_kernel walks the failing page again
  uint64_t n_read;          // *n_pages as read
  uint64_t n_pages;         // the pages the call runs over (0 when *n_pages is above max_pages)
  uint64_t bad;             // (page << 32) | status of a ref refusal, or the page that takes the numbers past dst_cap
  CarrySum frames, nums;    // the totals
  uint64_t fail_page;       // ap_route_kernel: the lowest page failing its meta or walk (NONE64: none)
  uint32_t fail_st, rewalk_st;
  uint64_t n_fast, n_cold;  // the decode table's records and the cold list's pages, all in front of fail_page
  uint64_t decode_fail;     // ap_cold_kernel: (page << 32) | status of the lowest failing decode (NONE64: none)
  WalkResult walk;          // walk_kernel's serial result, not written in per-chunk mode
};
static_assert(sizeof(ApPart) == 56 && sizeof(ApState) == 136 && sizeof(WalkSmem<SMALL_MAX_SIZE_LOG>) <= 48 * 1024, "workspace layout");

// everything the launches take by value
struct ApArgs {
  const uint8_t* metas;
  const uint8_t* pages;
  const PcoB200PageRef* refs;
  const uint64_t* n_pages;
  uint64_t metas_cap, pages_cap, dst_cap, frame_cap;
  uint32_t dtype, max_pages;
};

// Workspace of one in-flight call, byte offsets, each region 256-byte aligned:
// AsyncCheck (binomials) | ApState | WrappedPage[max_pages] | IndexChunk[max_pages + 1] and the batch entries | frames and a pad frame |
// per page: meta status, walk status, walk end | CTA sums | decode table | its pages | cold list | the decode tail.
struct ApLayout : AsyncDecodeTail {
  uint64_t state, tab, index, index_len, frames, pad_frame, pstat, wst, ends, parts, table, fast_page, cold_list;
};
// Batch entries of an accepted batch: each page's entries_bytes(MAX_VARS, n) (16-byte aligned room for MAX_VARS x ceil(n / 256) entries of 12 bytes)
// is at most 24 floor(n / 256) + 32 bytes, and the pages hold at most dst_cap numbers.
__host__ __device__ inline uint64_t ap_entries_bound(uint64_t max_pages, uint64_t dst_cap) { return 24 * (dst_cap / BATCH_N) + 32 * max_pages; }
__host__ __device__ inline ApLayout ap_layout(uint64_t max_pages, uint64_t dst_cap, uint64_t frame_cap) {
  ApLayout l;
  l.state = async_align(sizeof(AsyncCheck));
  l.tab = l.state + async_align(sizeof(ApState));
  l.index = l.tab + async_align(max_pages * sizeof(WrappedPage));
  l.index_len = (max_pages + 1) * sizeof(IndexChunk) + ap_entries_bound(max_pages, dst_cap);
  l.frames = l.index + async_align(l.index_len);
  l.pad_frame = (frame_cap + 15) & ~uint64_t(15);  // from l.frames
  l.pstat = l.frames + async_align(l.pad_frame + 64);
  l.wst = l.pstat + async_align(max_pages * sizeof(uint32_t));
  l.ends = l.wst + async_align(max_pages * sizeof(uint32_t));
  l.parts = l.ends + async_align(max_pages * sizeof(uint64_t));
  l.table = l.parts + async_align(ctas_of<AP_THREADS>(max_pages) * sizeof(ApPart));
  l.fast_page = l.table + async_align(max_pages * sizeof(IndexChunk));
  l.cold_list = l.fast_page + async_align(max_pages * sizeof(uint32_t));
  static_cast<AsyncDecodeTail&>(l) =
      async_decode_tail(l.cold_list + async_align(max_pages * sizeof(uint32_t)), max_pages, scratch_rows_total(dst_cap, uint32_t(max_pages)), 0);
  return l;
}

__device__ __forceinline__ uint64_t ap_n_pages(const ApArgs& g) {
  const uint64_t n = *g.n_pages;
  return n <= g.max_pages ? n : 0;
}
// a page's framed chunk: [dtype][page_n - 1, 24 bits][meta][page], 16-byte aligned (decompress_pages_impl)
__device__ __forceinline__ uint64_t ap_frame_bytes(const PcoB200PageRef& r) { return (4 + r.meta_len + r.page_len + 15) & ~uint64_t(15); }

// ceil(max_pages / AP_THREADS) CTAs, one page slot per thread: the argument checks decompress_pages_impl makes for each page, in its order
// (meta range, page range, page_n), and the sizes the placement scans.
__global__ void __launch_bounds__(AP_THREADS) ap_pages_kernel(ApArgs g, AsyncCheck* __restrict__ chk, ApPart* __restrict__ parts) {
  __shared__ unsigned long long s_bad;
  const uint32_t tid = threadIdx.x;
  if (tid == 0) s_bad = NONE64;
  if (blockIdx.x == 0 && tid == 32) PCOB_ASYNC_FILL_BINOMS(chk->binoms);
  __syncthreads();
  const uint64_t i = uint64_t(blockIdx.x) * AP_THREADS + tid;
  uint64_t frame = 0, room = 0, nums = 0;
  if (i < ap_n_pages(g)) {
    const PcoB200PageRef r = g.refs[i];
    uint32_t ref = ST_OK;
    if (r.meta_len > g.metas_cap || r.meta_offset > g.metas_cap - r.meta_len) ref = PCO_B200_ASYNC_META_OUTSIDE;
    else if (r.page_len > g.pages_cap || r.page_offset > g.pages_cap - r.page_len) ref = PCO_B200_ASYNC_PAGE_OUTSIDE;
    else if (r.page_n == 0 || r.page_n > (uint64_t(1) << 24)) ref = PCO_B200_ASYNC_PAGE_N;
    if (ref != ST_OK) {
      atomicMin(&s_bad, (i << 32) | ref);
    } else {
      frame = ap_frame_bytes(r);
      room = entries_bytes(MAX_VARS, r.page_n);
      nums = r.page_n;
    }
  }
  CarrySum f_tot, e_tot, n_tot;
  block_exscan<AP_THREADS>(carry_sum(frame), &f_tot);
  block_exscan<AP_THREADS>(carry_sum(room), &e_tot);
  block_exscan<AP_THREADS>(carry_sum(nums), &n_tot);
  if (tid == 0) parts[blockIdx.x] = ApPart{f_tot, e_tot, n_tot, s_bad};
}

// One CTA: *n_pages against max_pages, the lowest ref refusal over all pages, the CTA sums scanned into CTA offsets (in place), and the
// totals: more numbers than dst_cap (the page that passes it is found by ap_place_kernel), then more frame bytes than frame_cap.
__global__ void __launch_bounds__(AP_SCAN_THREADS) ap_scan_kernel(ApArgs g, ApPart* __restrict__ parts, ApState* __restrict__ state) {
  __shared__ unsigned long long s_bad;
  const uint32_t tid = threadIdx.x;
  if (tid == 0) s_bad = NONE64;
  __syncthreads();
  const uint64_t n_parts = ctas_of<AP_THREADS>(g.max_pages);
  for (uint64_t c = tid; c < n_parts; c += AP_SCAN_THREADS)
    if (parts[c].bad_ref != NONE64) atomicMin(&s_bad, parts[c].bad_ref);
  auto sum = [&](uint64_t c, int k) -> CarrySum& { return k == 0 ? parts[c].frames : k == 1 ? parts[c].entries : parts[c].nums; };
  CarrySum total[3] = {};
  cta_scan_inplace<AP_SCAN_THREADS, 1>(
      n_parts, [&](uint64_t c, int k) { return sum(c, k); }, [&](uint64_t c, int k, CarrySum v) { sum(c, k) = v; }, total);
  __syncthreads();
  if (tid != 0) return;
  ApState s;
  s.status = ST_OK;
  s.rewalk = 0;
  s.n_read = *g.n_pages;
  s.n_pages = ap_n_pages(g);
  s.bad = NONE64;
  s.frames = total[0];
  s.nums = total[2];
  s.fail_page = NONE64;
  s.fail_st = ST_OK;
  s.rewalk_st = ST_OK;
  s.n_fast = 0;
  s.n_cold = 0;
  s.decode_fail = NONE64;
  s.walk = WalkResult{0, 0, 0, 0, 0};
  if (s.n_read > g.max_pages) s.status = PCO_B200_ASYNC_TOO_MANY_PAGES;
  else if (s_bad != NONE64) {
    s.status = uint32_t(s_bad);
    s.bad = s_bad;
  } else if (s.nums.s > g.dst_cap) s.status = PCO_B200_ASYNC_PAGES_DST;  // the page: ap_place_kernel
  else if (s.frames.ovf || s.frames.s > g.frame_cap) s.status = PCO_B200_ASYNC_FRAMES;
  *state = s;
}

// ceil(max_pages / AP_THREADS) CTAs, one page slot per thread: the page's WrappedPage row and its IndexChunk placeholder (frame offset, n,
// entries offset, out offset), as decompress_pages_impl lays them out.  Every slot past *n_pages, and every slot of a refused batch, gets a
// pad: a page of one number whose frame is the pad frame (its type byte and count, then zeros), which frame_pages_kernel copies nothing
// into and walk_kernel refuses at its header.  Under PCO_B200_ASYNC_PAGES_DST the one page whose running count passes dst_cap is named.
__global__ void __launch_bounds__(AP_THREADS) ap_place_kernel(ApArgs g, const ApPart* __restrict__ parts, ApState* __restrict__ state,
                                                              WrappedPage* __restrict__ tab, IndexChunk* __restrict__ recs, uint8_t* __restrict__ frames,
                                                              uint64_t pad_frame, uint64_t entries_begin) {
  const uint32_t tid = threadIdx.x;
  const uint32_t pre = state->status;
  const uint64_t n = state->n_pages;
  const uint64_t i = uint64_t(blockIdx.x) * AP_THREADS + tid;
  if (blockIdx.x == 0 && tid < 16) reinterpret_cast<uint32_t*>(frames + pad_frame)[tid] = 0;
  const bool in = (pre == ST_OK || pre == PCO_B200_ASYNC_PAGES_DST || pre == PCO_B200_ASYNC_FRAMES) && i < n;
  PcoB200PageRef r{0, 0, 0, 0, 0};
  if (in) r = g.refs[i];
  const uint64_t frame = in ? ap_frame_bytes(r) : 0, room = in ? entries_bytes(MAX_VARS, r.page_n) : 0, nums = in ? r.page_n : 0;
  CarrySum tot;
  const CarrySum f_ex = carry_add(parts[blockIdx.x].frames, block_exscan<AP_THREADS>(carry_sum(frame), &tot));
  const CarrySum e_ex = carry_add(parts[blockIdx.x].entries, block_exscan<AP_THREADS>(carry_sum(room), &tot));
  const CarrySum n_ex = carry_add(parts[blockIdx.x].nums, block_exscan<AP_THREADS>(carry_sum(nums), &tot));
  if (i >= g.max_pages) return;
  if (in && pre == PCO_B200_ASYNC_PAGES_DST && n_ex.s <= g.dst_cap && n_ex.s + nums > g.dst_cap) state->bad = (i << 32) | pre;
  if (in && pre == ST_OK) {
    tab[i] = WrappedPage{r.meta_offset, r.meta_len, r.page_offset, r.page_len, f_ex.s, uint32_t(r.page_n), 0};
    recs[i] = IndexChunk{f_ex.s, uint32_t(r.page_n), 0u, entries_begin + e_ex.s, n_ex.s};
  } else {
    tab[i] = WrappedPage{0, 0, 0, 0, pad_frame, 1, 0};
    recs[i] = IndexChunk{pad_frame, 1u, 0u, entries_begin, 0};
  }
}

// One CTA.  The route of page i, as decompress_pages_impl decides it: its meta status (frame_pages_kernel) first - WP_COLD for the catch-all
// decoder, an error fails the page - then its walk: ST_UNSUPPORTED for the catch-all decoder, ST_OK and an end inside its frame for the fast
// kernels, ST_OK and an end past its frame fails it as ST_INSUFFICIENT_DATA, any other status fails it and asks for the re-walk.  The
// lowest failing page is found first; then the walked records of the fast pages in front of it go to the decode table in page order (pads
// behind them, up to max_pages: chunk_offset = src_len, which the decode kernels refuse without reading), and the cold pages in front of
// it to the cold list.  The spare record behind the page table gets the failing page's placeholder for ap_rewalk_kernel.
__global__ void __launch_bounds__(AP_SCAN_THREADS) ap_route_kernel(ApArgs g, ApState* __restrict__ state, const WrappedPage* __restrict__ tab,
                                                                   IndexChunk* __restrict__ recs, const uint32_t* __restrict__ pstat,
                                                                   const uint32_t* __restrict__ wst, const uint64_t* __restrict__ ends,
                                                                   IndexChunk* __restrict__ table, uint32_t* __restrict__ fast_page,
                                                                   uint32_t* __restrict__ cold_list, uint64_t src_len) {
  constexpr uint32_t R_FAST = 0, R_COLD = 1, R_FAIL = 2, R_FAIL_REWALK = 3;
  __shared__ unsigned long long s_fail;
  __shared__ uint64_t s_carry[2];
  const uint32_t tid = threadIdx.x;
  if (tid == 0) {
    s_fail = NONE64;
    s_carry[0] = s_carry[1] = 0;
  }
  __syncthreads();
  const uint64_t n = state->status == ST_OK ? state->n_pages : 0;
  auto route = [&](uint64_t i, uint32_t* st) -> uint32_t {
    *st = pstat[i];
    if (*st == WP_COLD) return R_COLD;
    if (*st != ST_OK) return R_FAIL;
    *st = wst[i];
    if (*st == ST_UNSUPPORTED) return R_COLD;
    if (*st == ST_OK) {
      const WrappedPage w = tab[i];
      if (ends[i] <= w.frame_off + 4 + w.meta_len + w.page_len) return R_FAST;
      *st = ST_INSUFFICIENT_DATA;  // the walk ran past the page into the next frame
      return R_FAIL;
    }
    return R_FAIL_REWALK;
  };
  for (uint64_t i = tid; i < n; i += AP_SCAN_THREADS) {
    uint32_t st;
    const uint32_t r = route(i, &st);
    if (r >= R_FAIL) {
      atomicMin(&s_fail, (i << 32) | (uint64_t(r == R_FAIL_REWALK) << 31) | st);  // a thread's first failure is its lowest
      break;
    }
  }
  __syncthreads();
  const unsigned long long fail = s_fail;
  const uint64_t limit = fail != NONE64 ? (fail >> 32) : n;
  const uint32_t lane = tid & 31, warp = tid >> 5;
  __shared__ uint32_t s_warp[2][AP_SCAN_THREADS / 32];
  for (uint64_t base = 0; base < limit; base += AP_SCAN_THREADS) {
    const uint64_t i = base + tid;
    uint32_t st = ST_OK;
    const uint32_t r = i < limit ? route(i, &st) : R_FAIL;
    const uint32_t f = r == R_FAST, c = r == R_COLD;
    const uint32_t fb = __ballot_sync(0xffffffffu, f), cb = __ballot_sync(0xffffffffu, c);
    if (lane == 0) {
      s_warp[0][warp] = __popc(fb);
      s_warp[1][warp] = __popc(cb);
    }
    __syncthreads();
    if (tid == 0) {
      uint32_t a = 0, b = 0;
      for (uint32_t w = 0; w < AP_SCAN_THREADS / 32; w++) {
        const uint32_t x = s_warp[0][w], y = s_warp[1][w];
        s_warp[0][w] = a;
        s_warp[1][w] = b;
        a += x;
        b += y;
      }
    }
    __syncthreads();
    const uint32_t below = (1u << lane) - 1;
    if (f) {
      const uint64_t k = s_carry[0] + s_warp[0][warp] + __popc(fb & below);
      table[k] = recs[i];
      fast_page[k] = uint32_t(i);
    }
    if (c) cold_list[s_carry[1] + s_warp[1][warp] + __popc(cb & below)] = uint32_t(i);
    __syncthreads();
    if (tid == AP_SCAN_THREADS - 1) {  // the last warp's offset and count: the tile's totals
      s_carry[0] += s_warp[0][warp] + __popc(fb);
      s_carry[1] += s_warp[1][warp] + __popc(cb);
    }
    __syncthreads();
  }
  const uint64_t n_fast = s_carry[0];
  for (uint64_t k = n_fast + tid; k < g.max_pages; k += AP_SCAN_THREADS) table[k] = IndexChunk{src_len, 0u, 0u, 0, 0};
  if (tid != 0) return;
  state->n_fast = n_fast;
  state->n_cold = s_carry[1];
  if (fail != NONE64) {
    const uint64_t p = fail >> 32;
    state->fail_page = p;
    state->fail_st = uint32_t(fail) & 0x7fffffffu;
    state->rewalk = uint32_t(fail >> 31) & 1u;
    state->rewalk_st = ST_OK;
    IndexChunk one = recs[p];
    one.chunk_offset = 0;
    recs[g.max_pages] = one;
  }
}

// One CTA of WALK_THREADS: when ap_route_kernel asked for it, the failing page walked once more over its own frame alone.  A walk that
// leaves its page reads the next frame, not the zeros pco_b200_page_decompress would see there; this walk gives that call's kind.
__global__ void __launch_bounds__(WALK_THREADS) ap_rewalk_kernel(ApArgs g, ApState* __restrict__ state, const WrappedPage* __restrict__ tab,
                                                                 const uint8_t* __restrict__ frames, uint8_t* __restrict__ index, uint64_t index_len) {
  if (!state->rewalk) return;  // uniform: every thread leaves
  const WrappedPage w = tab[state->fail_page];
  const FileParams fp{frames + w.frame_off, 4 + w.meta_len + w.page_len, g.dtype, 0, 4};
  walk_run<SMALL_MAX_SIZE_LOG>(fp, index, uint64_t(g.max_pages) * sizeof(IndexChunk), 1, 0, index_len, 0, 0, ~uint64_t(0), &state->rewalk_st,
                               &state->walk, 0, nullptr);
}

// One CTA.  Its threads find the lowest failing record of the decode table; thread 0 then decodes the cold pages in front of both that
// record's page and ap_route_kernel's failing page, in page order, each with the catch-all decoder over its own frame (bytes past the
// page read as zeros) straight into its slot of dst, and stops at the first that fails.  The lowest decode failure goes to the state.
template <typename L>
__global__ void __launch_bounds__(ASYNC_THREADS) ap_cold_kernel(ApArgs g, ApState* __restrict__ state, const WrappedPage* __restrict__ tab,
                                                                const IndexChunk* __restrict__ recs, const uint32_t* __restrict__ statuses,
                                                                const uint32_t* __restrict__ fast_page, const uint32_t* __restrict__ cold_list,
                                                                const uint8_t* __restrict__ frames, L* __restrict__ out, uint8_t* __restrict__ scratch) {
  __shared__ uint32_t s_min;
  const uint32_t tid = threadIdx.x;
  if (tid == 0) s_min = 0xffffffffu;
  __syncthreads();
  const uint64_t n_fast = state->n_fast;
  for (uint64_t k = tid; k < n_fast; k += ASYNC_THREADS)
    if (statuses[k] != ST_OK) {
      atomicMin(&s_min, uint32_t(k));  // a thread's first failure is its lowest
      break;
    }
  __syncthreads();
  if (tid != 0) return;
  uint64_t fail = NONE64;
  if (s_min != 0xffffffffu) fail = (uint64_t(fast_page[s_min]) << 32) | statuses[s_min];
  const uint64_t limit = min(state->fail_page, fail >> 32);
  const uint64_t n_cold = state->n_cold;
  for (uint64_t k = 0; k < n_cold; k++) {
    const uint32_t p = cold_list[k];
    if (p >= limit) break;
    const WrappedPage w = tab[p];
    const FileParams fp{frames + w.frame_off, 4 + w.meta_len + w.page_len, g.dtype, 0, 4};
    ColdResult res;
    cold_decode_run<L>(fp, 0, out + recs[p].out_offset, w.page_n, scratch, ASYNC_COLD_WINDOW_LOG, &res);
    if (res.n_chunks == 0) {  // the page is decoded once its chunk is (what the decoder reads behind it is not the page's)
      fail = (uint64_t(p) << 32) | cold_status(res);
      break;
    }
  }
  state->decode_fail = fail;
}

// One CTA, one thread: the lowest of ap_route_kernel's failing page (with the re-walk's status when it ran and failed) and ap_cold_kernel's
// decode failure, else the pending refusal, else success.
__global__ void __launch_bounds__(32) ap_finish_kernel(const ApState* __restrict__ state, PcoB200AsyncPagesStatus* __restrict__ out) {
  if (threadIdx.x != 0) return;
  const ApState s = *state;
  PcoB200AsyncPagesStatus r;
  r.kind = PCO_B200_OK;
  r.device_status = ST_OK;
  r.page = NONE64;
  const bool refs_ok = s.status == ST_OK || s.status == PCO_B200_ASYNC_FRAMES;
  r.n_written = refs_ok ? s.nums.s : 0;
  r.n_pages = s.n_read;
  r.frames_needed = refs_ok || s.status == PCO_B200_ASYNC_PAGES_DST ? (s.frames.ovf ? NONE64 : s.frames.s) : 0;
  if (s.status != ST_OK) {
    r.kind = async_kind_of(s.status);
    r.device_status = s.status;
    r.n_written = 0;
    if (s.status != PCO_B200_ASYNC_TOO_MANY_PAGES && s.status != PCO_B200_ASYNC_FRAMES) r.page = s.bad >> 32;
  } else if (s.fail_page != NONE64 || s.decode_fail != NONE64) {
    uint32_t st;
    if (s.fail_page <= (s.decode_fail >> 32)) {
      r.page = s.fail_page;
      st = s.rewalk && s.rewalk_st != ST_OK ? s.rewalk_st : s.fail_st;
    } else {
      r.page = s.decode_fail >> 32;
      st = uint32_t(s.decode_fail);
    }
    r.kind = async_kind_of(st);
    r.device_status = st;
    r.n_written = 0;
  }
  *out = r;
}

}  // namespace pcob200
