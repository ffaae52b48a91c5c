// Kernels of pco_b200_pages_to_file_async: a batch of wrapped-format pages written out as one indexed standalone file - page i as chunk i,
// its bytes pco's own - on the caller's stream, so later scans of the pages read the side index instead of walking every page again.
// The pages call's front end (async_pages_kernels.cuh: ap_pages, ap_scan, ap_place, frame_pages, walk<10>, ap_route, ap_rewalk) runs
// unchanged and leaves every page framed as a standalone chunk, [dtype][page_n - 1][meta][page], with its walked record and batch entries
// (bit positions counted from the frame's type byte, which is the side index's own layout).  Then, over grids fixed by the plan:
//   pf_walk_kernel      the pages walk<10> declined, walked again with the 2^12-state walker (as ai_walk_kernel<12>);
//   pf_gate_kernel      (one CTA) each page's verdict - its meta status, its walk (the wide walk's where walk<10> declined), its walk end
//                       inside its frame - the lowest failing page, then the lowest declined page; on success the chunk sizes (frame bytes up
//                       to the walk's end) and entry sizes (compacted to the chunk's n_vars) scanned into file and index offsets, and the
//                       file against dst_cap, the index against index_cap;
//   pf_file_kernel      the file: header, every chunk copied from its frame, terminator; each CTA owns spans of PF_SPAN output bytes and
//                       finds the chunks that cover them by binary search over the chunk offsets;
//   pf_index_kernel     one CTA per page: its record and its entries into the index (index_copy_chunk, as ai_copy_kernel);
//   pf_finish_kernel    the index header, the PcoB200FileRef and the PcoB200AsyncPagesToFileStatus.
// The file and the index are written only on success; the ref is zeroed on any failure.
#pragma once
#include "async_index_kernels.cuh"
#include "async_pages_kernels.cuh"
#include "compress_host.cuh"
#include "gather_kernels.cuh"

namespace pcob200 {

constexpr uint64_t PF_SPAN = 64 * 1024;  // output bytes per CTA step of pf_file_kernel
constexpr uint32_t PF_MAX_CTAS = 2048;   // pf_file_kernel's grid: one CTA per span of dst_cap, at most this many
constexpr int PF_SCAN_PER_THREAD = 4;

// decided by pf_gate_kernel
struct PfState {
  uint32_t status;     // ST_OK, the front end's refusal, the failing page's status, ST_UNSUPPORTED or a capacity refusal
  uint32_t hdr_len;    // bytes of the standalone header
  uint64_t page;       // the page a page failure names (NONE64: none)
  uint64_t file_len;   // bytes of the file, once every page passed (0 before)
  uint64_t index_len;  // bytes of the side index, likewise
};

// everything the launches take by value
struct PfArgs {
  uint8_t* ws;
  uint8_t* file;
  uint8_t* index;
  PcoB200FileRef* ref;
  uint64_t max_pages, frame_cap, dst_cap, index_cap;
  uint32_t dtype, uniform_type;
};

// The numbers whose walk entries the front end makes room for: rows_cap of ap_layout.  A page of n numbers has at least 12 ceil(n / 256)
// bytes of entries in any index, so the pages of an index that fits index_cap hold at most 256 floor(index_cap / 12) numbers' batches,
// and their entries at MAX_VARS fit ap_entries_bound of that.
__host__ __device__ inline uint64_t pf_rows(uint64_t index_cap) { return uint64_t(BATCH_N) * (index_cap / sizeof(BatchEntry)); }

// Workspace of one in-flight call, byte offsets, each region 256-byte aligned: the pages front end's regions of ap_layout (up to, not
// including, the decode tail) | PfState | per page: wide walk status, wide walk end, chunk offset, entries offset.
struct PfLayout {
  ApLayout ap;
  uint64_t state, wst, ends, coff, eoff, total;
};
__host__ __device__ inline PfLayout pf_layout(uint64_t max_pages, uint64_t frame_cap, uint64_t index_cap) {
  PfLayout l;
  l.ap = ap_layout(max_pages, pf_rows(index_cap), frame_cap);
  l.state = l.ap.cold_list + async_align(max_pages * sizeof(uint32_t));
  l.wst = l.state + async_align(sizeof(PfState));
  l.ends = l.wst + async_align(max_pages * sizeof(uint32_t));
  l.coff = l.ends + async_align(max_pages * sizeof(uint64_t));
  l.eoff = l.coff + async_align(max_pages * sizeof(uint64_t));
  l.total = l.eoff + async_align(max_pages * sizeof(uint64_t));
  return l;
}
__host__ __device__ inline uint32_t pf_file_ctas(uint64_t dst_cap) {
  const uint64_t n = (dst_cap + PF_SPAN - 1) / PF_SPAN;
  return uint32_t(n < 1 ? 1 : n > PF_MAX_CTAS ? PF_MAX_CTAS : n);
}

// the frames as one file, as the front end's walk reads them
__device__ __forceinline__ FileParams pf_frames(const PfArgs& g, const PfLayout& l) {
  return FileParams{g.ws + l.ap.frames, l.ap.pad_frame + 64, g.dtype, 0, 4};
}

// max_pages CTAs launched as walk_kernel<12> is: page blockIdx.x walked again, over the frames as the front end's walk saw them, when
// walk<10> declined it; the others leave at once.
__global__ void __launch_bounds__(WALK_THREADS, PCOB_WALK_MIN_BLOCKS) pf_walk_kernel(PfArgs g) {
  const PfLayout l = pf_layout(g.max_pages, g.frame_cap, g.index_cap);
  const ApState& a = *reinterpret_cast<const ApState*>(g.ws + l.ap.state);
  const uint32_t* wst = reinterpret_cast<const uint32_t*>(g.ws + l.ap.wst);
  if (a.status != ST_OK || blockIdx.x >= a.n_pages || wst[blockIdx.x] != ST_UNSUPPORTED) return;
  walk_run<12>(pf_frames(g, l), g.ws + l.ap.index, 0, uint32_t(g.max_pages), 0, l.ap.index_len, 0, 0, ~uint64_t(0),
               reinterpret_cast<uint32_t*>(g.ws + l.wst), nullptr, 0, reinterpret_cast<uint64_t*>(g.ws + l.ends));
}

// Page i's verdict: ST_OK with *len, the bytes of its chunk (its frame up to the walk's end); ST_UNSUPPORTED when both walkers decline it;
// ST_INDEX_FULL when its entries did not fit the room index_cap gives the walks; else the status it fails with - its meta status
// (frame_pages_kernel), its walk's, or ST_INSUFFICIENT_DATA for a walk that ran past its page into the next frame (as ap_route_kernel).
__device__ __forceinline__ uint32_t pf_verdict(const PfArgs& g, const PfLayout& l, uint64_t i, uint64_t* len) {
  const uint32_t p = reinterpret_cast<const uint32_t*>(g.ws + l.ap.pstat)[i];
  if (p != ST_OK && p != WP_COLD) return p;
  uint32_t w = reinterpret_cast<const uint32_t*>(g.ws + l.ap.wst)[i];
  uint64_t e = reinterpret_cast<const uint64_t*>(g.ws + l.ap.ends)[i];
  if (w == ST_UNSUPPORTED) {
    w = reinterpret_cast<const uint32_t*>(g.ws + l.wst)[i];
    e = reinterpret_cast<const uint64_t*>(g.ws + l.ends)[i];
  }
  if (w != ST_OK) return w;
  const WrappedPage t = reinterpret_cast<const WrappedPage*>(g.ws + l.ap.tab)[i];
  if (e > t.frame_off + 4 + t.meta_len + t.page_len) return ST_INSUFFICIENT_DATA;
  *len = e - t.frame_off;
  return ST_OK;
}

// One CTA.  The front end's refusal, else the verdicts: the lowest failing page (with the status of its walk over its own frame alone when
// ap_route_kernel found the same page and re-walked it), else the lowest declined page, else a batch whose walks ran out of room (the
// index is larger than index_cap).  Then each chunk's offset in the file (header, then the chunks back to back) and its entries' offset in
// the index (header, n_pages records, then each chunk's entries at entries_bytes(n_vars, n)), and the file and index against their caps.
__global__ void __launch_bounds__(AP_SCAN_THREADS) pf_gate_kernel(PfArgs g) {
  __shared__ unsigned long long s_fail, s_decl, s_full;
  const uint32_t tid = threadIdx.x;
  const PfLayout l = pf_layout(g.max_pages, g.frame_cap, g.index_cap);
  const ApState& a = *reinterpret_cast<const ApState*>(g.ws + l.ap.state);
  PfState& s = *reinterpret_cast<PfState*>(g.ws + l.state);
  if (tid == 0) {
    s_fail = s_decl = s_full = NONE64;
    s.status = a.status;
    s.hdr_len = standalone_header_len(a.nums.s);
    s.page = NONE64;
    s.file_len = s.index_len = 0;
  }
  __syncthreads();
  if (a.status != ST_OK) return;
  const uint64_t n = a.n_pages;
  const IndexChunk* recs = reinterpret_cast<const IndexChunk*>(g.ws + l.ap.index);
  uint64_t* coff = reinterpret_cast<uint64_t*>(g.ws + l.coff);
  uint64_t* eoff = reinterpret_cast<uint64_t*>(g.ws + l.eoff);
  for (uint64_t i = tid; i < n; i += AP_SCAN_THREADS) {
    uint64_t len = 0;
    const uint32_t st = pf_verdict(g, l, i, &len);
    if (st == ST_OK) {
      coff[i] = len;
      eoff[i] = entries_bytes(recs[i].n_vars, recs[i].n);
    } else if (st == ST_UNSUPPORTED) {
      atomicMin(&s_decl, (unsigned long long)i);
    } else if (st == ST_INDEX_FULL) {
      atomicMin(&s_full, (unsigned long long)i);
    } else {
      atomicMin(&s_fail, (unsigned long long)((i << 32) | st));
    }
  }
  __syncthreads();
  if (s_fail != NONE64 || s_decl != NONE64 || s_full != NONE64) {
    if (tid != 0) return;
    if (s_fail != NONE64) {
      const uint64_t p = s_fail >> 32;
      s.page = p;
      s.status = p == a.fail_page && a.rewalk && a.rewalk_st != ST_OK ? a.rewalk_st : uint32_t(s_fail);
    } else if (s_decl != NONE64) {
      s.page = s_decl;
      s.status = ST_UNSUPPORTED;
    } else {
      s.status = PCO_B200_ASYNC_FILES_INDEX_FULL;  // index_needed stays 0: the pages behind s_full were not walked
    }
    return;
  }
  uint64_t end[2] = {s.hdr_len, sizeof(IndexHeader) + n * sizeof(IndexChunk)};
  cta_scan_inplace<AP_SCAN_THREADS, PF_SCAN_PER_THREAD>(
      n, [&](uint64_t i, int k) { return k ? eoff[i] : coff[i]; }, [&](uint64_t i, int k, uint64_t v) { (k ? eoff[i] : coff[i]) = v; }, end);
  if (tid != 0) return;
  s.file_len = end[0] + 1;  // the terminator
  s.index_len = end[1];
  if (s.file_len > g.dst_cap) s.status = PCO_B200_ASYNC_FILES_DST_FULL;
  else if (s.index_len > g.index_cap) s.status = PCO_B200_ASYNC_FILES_INDEX_FULL;
}

// pf_file_ctas(dst_cap) CTAs of GATHER_THREADS, on success only.  CTA 0 writes the header and the terminator; every CTA copies the chunk
// bytes of its spans [k PF_SPAN, (k + 1) PF_SPAN) of the file, k = blockIdx.x, blockIdx.x + gridDim.x, ..., chunk after chunk from the
// one its span starts in.  Spans and chunks end at any byte: cta_copy_bytes stores whole aligned words inside a piece and single bytes at
// its edges, so no two CTAs write the same byte.
__global__ void __launch_bounds__(GATHER_THREADS) pf_file_kernel(PfArgs g) {
  __shared__ uint64_t s_first;
  const PfLayout l = pf_layout(g.max_pages, g.frame_cap, g.index_cap);
  const PfState s = *reinterpret_cast<const PfState*>(g.ws + l.state);
  if (s.status != ST_OK) return;
  const ApState& a = *reinterpret_cast<const ApState*>(g.ws + l.ap.state);
  const uint64_t n = a.n_pages, body_end = s.file_len - 1;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    uint8_t h[STANDALONE_HEADER_MAX];
    const uint32_t len = standalone_header_into(a.nums.s, uint8_t(g.uniform_type), h);
    for (uint32_t i = 0; i < len; i++) g.file[i] = h[i];
    g.file[body_end] = 0;
  }
  const uint64_t* coff = reinterpret_cast<const uint64_t*>(g.ws + l.coff);
  const WrappedPage* tab = reinterpret_cast<const WrappedPage*>(g.ws + l.ap.tab);
  const uint8_t* frames = g.ws + l.ap.frames;
  for (uint64_t lo = uint64_t(blockIdx.x) * PF_SPAN; lo < body_end; lo += uint64_t(gridDim.x) * PF_SPAN) {
    const uint64_t a0 = max(lo, uint64_t(s.hdr_len)), a1 = min(lo + PF_SPAN, body_end);
    if (a0 >= a1) continue;  // uniform across the CTA
    if (threadIdx.x == 0) {  // the last chunk that starts at or before a0
      uint64_t k0 = 0, k1 = n;
      while (k1 - k0 > 1) {
        const uint64_t m = (k0 + k1) / 2;
        if (coff[m] <= a0) k0 = m;
        else k1 = m;
      }
      s_first = k0;
    }
    __syncthreads();
    for (uint64_t k = s_first; k < n && coff[k] < a1; k++) {
      const uint64_t c0 = coff[k], c1 = k + 1 < n ? coff[k + 1] : body_end;
      const uint64_t x0 = max(a0, c0), x1 = min(a1, c1);
      if (x0 < x1) cta_copy_bytes(g.file + x0, frames + tab[k].frame_off + (x0 - c0), x1 - x0);
    }
    __syncthreads();  // s_first is rewritten for the next span
  }
}

// max_pages CTAs of AI_THREADS, on success only: page blockIdx.x's record (its chunk's offset in the file, its entries' offset in the
// index) and its walked entries, padding zeroed, into the index.
__global__ void __launch_bounds__(AI_THREADS) pf_index_kernel(PfArgs g) {
  const PfLayout l = pf_layout(g.max_pages, g.frame_cap, g.index_cap);
  const PfState& s = *reinterpret_cast<const PfState*>(g.ws + l.state);
  const uint64_t c = blockIdx.x;
  if (s.status != ST_OK || c >= reinterpret_cast<const ApState*>(g.ws + l.ap.state)->n_pages) return;
  const uint8_t* walked = g.ws + l.ap.index;
  IndexChunk r = reinterpret_cast<const IndexChunk*>(walked)[c];
  r.chunk_offset = reinterpret_cast<const uint64_t*>(g.ws + l.coff)[c];
  index_copy_chunk(r, reinterpret_cast<const uint32_t*>(walked + r.entries_offset), g.index, reinterpret_cast<const uint64_t*>(g.ws + l.eoff)[c], c);
}

// One thread: the index header and the ref (zeroed on a failure), and the status.  A front-end refusal is reported as
// ap_finish_kernel reports it.
__global__ void pf_finish_kernel(PfArgs g, PcoB200AsyncPagesToFileStatus* __restrict__ out) {
  const PfLayout l = pf_layout(g.max_pages, g.frame_cap, g.index_cap);
  const ApState a = *reinterpret_cast<const ApState*>(g.ws + l.ap.state);
  const PfState s = *reinterpret_cast<const PfState*>(g.ws + l.state);
  const bool refs_ok = a.status == ST_OK || a.status == PCO_B200_ASYNC_FRAMES;
  PcoB200AsyncPagesToFileStatus r;
  r.kind = async_kind_of(s.status);
  r.device_status = s.status;
  r.page = s.page;
  if (a.status != ST_OK && a.status != PCO_B200_ASYNC_TOO_MANY_PAGES && a.status != PCO_B200_ASYNC_FRAMES) r.page = a.bad >> 32;
  r.n_pages = a.n_read;
  r.n_total = refs_ok ? a.nums.s : 0;
  r.frames_needed = refs_ok ? (a.frames.ovf ? NONE64 : a.frames.s) : 0;
  r.file_needed = s.file_len;
  r.index_needed = s.index_len;
  const bool ok = s.status == ST_OK;
  r.file_len = ok ? s.file_len : 0;
  r.index_len = ok ? s.index_len : 0;
  if (ok) write_index_header(g.index, a.n_pages, a.nums.s, s.file_len, s.file_len);
  *g.ref = ok ? PcoB200FileRef{0, s.file_len, 0, s.index_len} : PcoB200FileRef{0, 0, 0, 0};
  *out = r;
}

}  // namespace pcob200
