// Kernels and host steps of pco_b200_compress_wrapped_async: a batch of arrays compressed into wrapped chunks of one page each, with the
// array sizes and their count in device memory and no host decision between launches, so a GPU writer of a container that embeds pco (a
// columnar file, a page store) can queue its column chunks behind the step that sized them or capture the whole write in a CUDA graph.
//
// The encode is pco_b200_compress_files_async's one pass (async_compress_files.cuh, acf_launch_encode) with AcfArgs::framed = 0: an array
// has no header, no terminator and no index, so its chunks land back to back in a staging region of the workspace, each as the standalone
// chunk [type byte][n - 1][meta][page] that pco_b200_compress_wrapped also stages.  Then the tail splits them:
//   acw_lens_kernel         per chunk slot: the meta length of each live chunk, parsed with wrapped_meta_len (as chunk_refs_kernel parses
//                           it), and the CTA sums of the meta and page lengths;
//   acw_scan_kernel         (one CTA) the CTA sums scanned into CTA offsets (in place), the totals, and whether they fit metas_cap and
//                           pages_cap;
//   acw_refs_kernel         per chunk slot and per array slot: each live chunk's PcoB200PageRef, and first_chunk;
//   acw_split_kernel        one CTA per chunk slot: a live chunk's meta and page copied to their places (cta_copy_bytes);
//   acw_finish_kernel       the PcoB200AsyncCompressWrappedStatus.
// A refused batch (too many arrays, an array above max_array_n, the counts past nums_cap) runs every launch over chunks of 0 numbers and
// writes nothing but the status; a batch that does not fit writes refs, first_chunk and the status only.
#pragma once
#include "async_compress_files.cuh"
#include "cta_scan.cuh"
#include "wrapped_kernels.cuh"  // wrapped_meta_len, WRAP_THREADS, cta_copy_bytes

namespace pcob200 {

enum { ACW_META = 0, ACW_PAGE, ACW_BAD, ACW_SUMS };
struct AcwPart {  // per CTA of acw_lens_kernel: the sums of its chunks' meta lengths, page lengths and meta parse failures (the chunks are
                  // this library's own: none fails), then (acw_scan_kernel) the sums of the CTAs before it
  CarrySum s[ACW_SUMS];
};
struct AcwState {  // written by acw_scan_kernel
  uint32_t fits;       // the metas fit metas_cap and the pages pages_cap
  uint32_t split_err;  // some chunk's meta did not parse
  uint64_t metas_bytes, pages_bytes;
  uint64_t reserved;
};
static_assert(sizeof(AcwState) == 32 && sizeof(AcwPart) == 48, "the workspace formula in pco_b200.h");

// Workspace: pco_b200_compress_files_async's layout for the same capacities, then this call's regions, each 256-byte aligned.
struct AcwLayout {
  AcfLayout f;
  uint64_t stage, state, lens, parts, total;
};
inline AcwLayout acw_layout(const AcfLayout& f, uint64_t stage_bytes, uint64_t max_chunks) {
  AcwLayout l;
  l.f = f;
  uint64_t at = f.total;
  auto take = [&](uint64_t bytes) { const uint64_t o = at; at += acomp_align(bytes); return o; };
  l.stage = take(stage_bytes);
  l.state = take(sizeof(AcwState));
  l.lens = take(max_chunks * 4);
  l.parts = take(ctas_of<ACF_THREADS>(max_chunks + 1) * sizeof(AcwPart));
  l.total = at;
  return l;
}

struct AcwArgs {
  AcfArgs f;  // f.a.dst is the staging region, f.a.dst_cap its size
  AcwLayout l;
  uint8_t* metas;
  uint8_t* pages;
  PcoB200PageRef* refs;
  uint64_t* first_chunk;
  uint64_t metas_cap, pages_cap;
  uint32_t dtype, reserved;
};
__device__ __forceinline__ AcwState* acw_state(const AcwArgs& w) { return reinterpret_cast<AcwState*>(w.f.a.ws + w.l.state); }
__device__ __forceinline__ AcwPart* acw_parts(const AcwArgs& w) { return reinterpret_cast<AcwPart*>(w.f.a.ws + w.l.parts); }
__device__ __forceinline__ bool acw_placed(const AcfState* st) { return st->status == ST_OK && st->bad == NONE64; }
// The chunks staged: those of a placed batch (the staging region holds any batch within the capacities, so acf_bytes_scan_kernel finds
// that it fits; a staging that did not fit would have placed no chunk, and acw_scan_kernel reports it as chunks that do not split)
__device__ __forceinline__ uint64_t acw_live(const AcfState* st) { return acw_placed(st) && st->fits ? st->live_chunks : 0; }

// Chunk c's meta and page lengths (0, 0 for a slot that holds no live chunk).  ml comes from the lens table acw_lens_kernel wrote.
__device__ __forceinline__ void acw_chunk_lens(const AcwArgs& w, uint64_t c, uint64_t live, uint64_t* ml, uint64_t* pl) {
  *ml = *pl = 0;
  if (c >= live) return;
  const ChunkEnc* chunks = reinterpret_cast<const ChunkEnc*>(w.f.a.ws + w.f.a.lay.chunks);
  *ml = reinterpret_cast<const uint32_t*>(w.f.a.ws + w.l.lens)[c];  // 0 for a chunk that did not parse
  *pl = chunks[c].chunk_bytes - 4 - *ml;
}

// ceil((max_chunks + 1) / ACF_THREADS) CTAs: each live chunk's meta length, parsed from its staged bytes, and the CTA sums of the meta and
// page lengths.
__global__ void __launch_bounds__(ACF_THREADS) acw_lens_kernel(AcwArgs w) {
  const AcfState* st = acf_state(w.f);
  const uint64_t live = acw_live(st);
  const ChunkEnc* chunks = reinterpret_cast<const ChunkEnc*>(w.f.a.ws + w.f.a.lay.chunks);
  const uint64_t c = uint64_t(blockIdx.x) * ACF_THREADS + threadIdx.x;
  uint64_t v[ACW_SUMS] = {0, 0, 0};
  if (c < live) {
    const uint64_t sz = chunks[c].chunk_bytes;
    uint64_t ml = 0;
    bool cold = false;
    const uint32_t rc = sz >= 4 ? wrapped_meta_len(w.f.a.dst + chunks[c].out_offset + 4, sz - 4, w.dtype, &ml, &cold) : ST_CORRUPTION;
    if (rc != ST_OK || ml > sz - 4) {
      v[ACW_BAD] = 1;
      ml = 0;
    } else {
      v[ACW_META] = ml;
      v[ACW_PAGE] = sz - 4 - ml;
    }
    reinterpret_cast<uint32_t*>(w.f.a.ws + w.l.lens)[c] = uint32_t(ml);
  }
  CarrySum tot[ACW_SUMS];
  for (int k = 0; k < ACW_SUMS; k++) block_exscan<ACF_THREADS>(carry_sum(v[k]), &tot[k]);
  if (threadIdx.x == 0)
    for (int k = 0; k < ACW_SUMS; k++) acw_parts(w)[blockIdx.x].s[k] = tot[k];
}

// One CTA: the CTA sums scanned into CTA offsets (in place), the totals, and whether they fit the caps.
__global__ void __launch_bounds__(ACF_SCAN_THREADS) acw_scan_kernel(AcwArgs w) {
  AcwPart* parts = acw_parts(w);
  CarrySum total[ACW_SUMS] = {};
  cta_scan_inplace<ACF_SCAN_THREADS, 1>(
      ctas_of<ACF_THREADS>(w.f.a.n_chunks + 1), [&](uint64_t c, int k) { return parts[c].s[k]; },
      [&](uint64_t c, int k, CarrySum v) { parts[c].s[k] = v; }, total);
  if (threadIdx.x != 0) return;
  AcwState s;
  s.metas_bytes = total[ACW_META].s;
  s.pages_bytes = total[ACW_PAGE].s;
  s.split_err = total[ACW_BAD].s != 0 || !acf_state(w.f)->fits ? 1u : 0u;
  s.fits = s.split_err == 0 && s.metas_bytes <= w.metas_cap && s.pages_bytes <= w.pages_cap ? 1u : 0u;
  s.reserved = 0;
  *acw_state(w) = s;
}

// max(ceil((max_chunks + 1) / ACF_THREADS), ceil((max_arrays + 1) / ACF_THREADS)) CTAs, one chunk slot and one array slot per thread: a
// placed batch writes each live chunk's ref (offsets from the scans) and first_chunk[0 : n_arrays].
__global__ void __launch_bounds__(ACF_THREADS) acw_refs_kernel(AcwArgs w) {
  const AcfState* st = acf_state(w.f);
  if (!acw_placed(st)) return;
  const uint64_t live = acw_live(st), nf = st->n_files;
  const uint64_t c = uint64_t(blockIdx.x) * ACF_THREADS + threadIdx.x;
  uint64_t ml, pl;
  acw_chunk_lens(w, c, live, &ml, &pl);
  CarrySum tot;
  const CarrySum mex = block_exscan<ACF_THREADS>(carry_sum(ml), &tot);
  const CarrySum pex = block_exscan<ACF_THREADS>(carry_sum(pl), &tot);
  if (c < live) {
    const AcwPart& part = acw_parts(w)[blockIdx.x];
    const uint64_t* starts = acomp_starts(w.f.a);
    PcoB200PageRef r;
    r.meta_offset = part.s[0].s + mex.s;
    r.meta_len = ml;
    r.page_offset = part.s[1].s + pex.s;
    r.page_len = pl;
    r.page_n = starts[c + 1] - starts[c];
    w.refs[c] = r;
  }
  if (c < nf) w.first_chunk[c] = acf_files(w.f)[c].first[ACF_CHUNKS];
  else if (c == nf) w.first_chunk[c] = live;
}

// max_chunks CTAs, one per chunk slot: a live chunk of a batch that fits copies its meta and its page from the staging region to the
// places its ref names.
__global__ void __launch_bounds__(WRAP_THREADS) acw_split_kernel(AcwArgs w) {
  const AcfState* st = acf_state(w.f);
  const uint64_t c = blockIdx.x;
  if (c >= acw_live(st) || !acw_state(w)->fits) return;
  const ChunkEnc* chunks = reinterpret_cast<const ChunkEnc*>(w.f.a.ws + w.f.a.lay.chunks);
  const PcoB200PageRef r = w.refs[c];
  const uint8_t* src = w.f.a.dst + chunks[c].out_offset + 4;
  cta_copy_bytes(w.metas + r.meta_offset, src, r.meta_len);
  cta_copy_bytes(w.pages + r.page_offset, src + r.meta_len, r.page_len);
}

// One thread: the outcome.
__global__ void acw_finish_kernel(AcwArgs w, PcoB200AsyncCompressWrappedStatus* __restrict__ out) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  const AcfState* st = acf_state(w.f);
  const AcwState* ws = acw_state(w);
  PcoB200AsyncCompressWrappedStatus s;
  memset(&s, 0, sizeof(s));
  s.array = ~uint64_t(0);
  s.n_arrays = st->n_read;
  if (st->status != ST_OK) {
    s.device_status = st->status;
  } else if (st->bad != NONE64) {
    s.device_status = uint32_t(st->bad & 0xffffffffu);
    s.array = st->bad >> 32;
  } else {
    s.n_chunks = st->live_chunks;
    s.metas_bytes = ws->metas_bytes;
    s.pages_bytes = ws->pages_bytes;
    if (ws->split_err) {
      s.device_status = ST_CORRUPTION;  // the staged chunks did not split (it does not happen: the staging region holds any batch)
    } else if (ws->fits) {
      s.metas_written = ws->metas_bytes;
      s.pages_written = ws->pages_bytes;
    } else {
      s.device_status = PCO_B200_ASYNC_FILES_DST_FULL;
    }
  }
  s.kind = async_kind_of(s.device_status);
  *out = s;
}

// ---- host steps

// The bytes that hold the staged chunks of any batch within the capacities: max_chunks * (5 + B) + ceil(nums_cap * L / 8)
inline uint64_t acw_stage_bytes(uint32_t dtype, uint64_t max_chunks, uint64_t nums_cap) {
  const uint64_t lbits = nt_bits(dtype);
  return max_chunks * (5 + baseline_chunk_meta_size(uint32_t(lbits))) + (nums_cap * lbits + 7) / 8;
}

// The plan as pco_b200_compress_files_async's launches read it: files of no header flavour, the staging region as dst, no index.
inline PcoB200AsyncCompressFilesPlan acw_files_plan(const PcoB200AsyncCompressWrappedPlan& p) {
  PcoB200AsyncCompressFilesPlan f;
  std::memset(&f, 0, sizeof(f));
  f.dtype = p.dtype;
  f.mode = p.mode;
  f.order = p.order;
  f.n_vars = p.n_vars;
  f.level = p.level;
  f.mode_k = p.mode_k;
  f.max_files = p.max_arrays;
  f.nums_cap = p.nums_cap;
  f.max_file_n = p.max_array_n;
  f.max_page_n = p.max_page_n;
  f.max_chunks = p.max_chunks;
  f.dst_cap = acw_stage_bytes(p.dtype, p.max_chunks, p.nums_cap);
  f.mode_base = p.mode_base;
  f.base_bits = p.base_bits;
  f.inv_base_bits = p.inv_base_bits;
  return f;
}

struct AcwPlanGeom {
  AcfPlanGeom f;
  AcwLayout l;
};
inline AcwPlanGeom acw_plan_geom(const PcoB200AsyncCompressWrappedPlan& p) {
  AcwPlanGeom pg;
  const PcoB200AsyncCompressFilesPlan f = acw_files_plan(p);
  pg.f = acf_plan_geom(f);
  pg.l = acw_layout(pg.f.l, f.dst_cap, p.max_chunks);
  return pg;
}

inline PcoB200Error acw_check_plan(const PcoB200AsyncCompressWrappedPlan* p, AcwPlanGeom* pg) {
  const char* what = "the plan was not made by pco_b200_compress_wrapped_async_plan";
  if (!acomp_spec_ok(p) || p->level > 12 || p->max_arrays == 0 || p->max_arrays > 0x7fffffffu || p->max_array_n == 0 || p->nums_cap > (uint64_t(1) << 56) ||
      p->max_chunks != p->nums_cap / acf_chunk_n(p->max_page_n, p->max_array_n, p->nums_cap) + p->max_arrays || p->max_chunks > 0x7fffffffu)
    return fail(PCO_B200_INVALID_ARGUMENT, what);
  *pg = acw_plan_geom(*p);
  if (p->workspace_bytes != pg->l.total) return fail(PCO_B200_INVALID_ARGUMENT, what);
  return PCO_B200_OK;
}

template <typename L>
void acw_launch(const PcoB200AsyncCompressWrappedPlan& p, const AcwPlanGeom& pg, const AcwArgs& w, const void* nums,
                PcoB200AsyncCompressWrappedStatus* status, const AsyncLaunch& ln) {
  const cudaStream_t stream = ln.stream;
  acf_launch_encode<L>(acw_files_plan(p), pg.f.g, w.f, nums, ln);
  const uint64_t nc = pg.f.g.n_chunks;
  const uint32_t chunk_ctas = uint32_t(ctas_of<ACF_THREADS>(nc + 1)), ref_ctas = uint32_t(std::max(ctas_of<ACF_THREADS>(nc + 1), ctas_of<ACF_THREADS>(p.max_arrays + 1)));
  ln.begin("acw_lens_kernel");
  acw_lens_kernel<<<chunk_ctas, ACF_THREADS, 0, stream>>>(w);
  ln.end();
  ln.begin("acw_scan_kernel");
  acw_scan_kernel<<<1, ACF_SCAN_THREADS, 0, stream>>>(w);
  ln.end();
  ln.begin("acw_refs_kernel");
  acw_refs_kernel<<<ref_ctas, ACF_THREADS, 0, stream>>>(w);
  ln.end();
  ln.begin("acw_split_kernel");
  acw_split_kernel<<<uint32_t(nc), WRAP_THREADS, 0, stream>>>(w);
  ln.end();
  ln.begin("acw_finish_kernel");
  acw_finish_kernel<<<1, 32, 0, stream>>>(w, status);
  ln.end();
}

}  // namespace pcob200
