// Kernels and host steps of pco_b200_compress_files_async: a batch of standalone files compressed with the file sizes and their count in
// device memory and no host decision between launches, so the write side of a batch (a checkpoint writer, an offload of evicted blocks,
// a columnar writer) can be queued behind the step that produced the numbers or captured in a CUDA graph.
//
// pco_b200_compress_files makes one pipeline pass per unoptimized_bins_log and frames the files on the host.  Here the whole batch is ONE
// pass over grids fixed by the plan's capacities (max_chunks chunk slots, each of up to the largest chunk's numbers):
//   acf_files_kernel        one thread per file slot: the CTA sums of the files' numbers, chunks, rows, frame bytes and index bytes;
//   acf_scan_kernel         (one CTA) *n_files against max_files, the CTA sums scanned into CTA offsets (in place);
//   acf_place_kernel        one thread per file slot: its first number, chunk, row, frame byte and index byte, and its refusal (above
//                           max_file_n, or the running sum of the counts past nums_cap, with exact 64-bit overflow detection);
//   acf_init_kernel         per chunk slot: its start and row base (EqualPagesUpTo per file in closed form; the chunks of a refused batch
//                           and the pad slots up to max_chunks hold 0 numbers), its file, its ChunkEnc reset; the zeroed offset-bit sums;
//   the encode kernels      enqueue_encode_kernels (async_compress.cuh), as pco_b200_compress_async runs them behind the same gates
//                           (which read the starts table this init kernel wrote); split_count_kernel, plan_probe_kernel and
//                           plan_solve_kernel in their CHUNK_BINS instantiations, which compute each chunk's unoptimized_bins_log from its n;
//   acf_bytes_kernel, acf_bytes_scan_kernel, acf_offsets_kernel
//                           a multi-CTA exclusive scan of the chunk sizes layout_kernel wrote: each chunk's place in dst behind its file's
//                           header, every file's place and length, and whether the batch fits dst_cap and index_cap.  A chunk that is not
//                           written (a pad slot, or a batch that does not fit) is placed past any dst_cap, as acomp_pack_gate_kernel does;
//   pack_kernel             per choice of keys (acomp_pack_gate_kernel), each chunk straight into its final place;
//   acf_frame_kernel        one thread per file slot: its header and terminator, its PcoB200FileRef and its side index header;
//   acf_index_kernel        one CTA per chunk slot: its record (offsets counted from its file) and its batch entries, padding zeroed;
//   acf_finish_kernel       the PcoB200AsyncCompressFilesStatus.
// A refused batch (too many files, a file above max_file_n, the counts past nums_cap) runs every launch over chunks of 0 numbers and
// writes nothing but the status; a batch that does not fit writes `files` and the status only, as pco_b200_compress_files does.
#pragma once
#include "async_compress.cuh"
#include "async_kernels.cuh"  // async_kind_of
#include "cta_scan.cuh"

namespace pcob200 {

constexpr int ACF_THREADS = 256;        // the per-file and per-chunk launches
constexpr int ACF_SCAN_THREADS = 1024;  // the one-CTA launches
constexpr int ACF_INDEX_THREADS = 128;
enum { ACF_NUMS = 0, ACF_CHUNKS, ACF_ROWS, ACF_FRAME, ACF_IDX, ACF_SUMS };

struct AcfPart {  // per CTA of acf_files_kernel: the CTA's sums, then (acf_scan_kernel) the sums of the CTAs before it
  CarrySum s[ACF_SUMS];
};
struct AcfFile {  // per file, by acf_place_kernel: where its numbers, chunks, rows, frame bytes and index start
  uint64_t n, first[ACF_SUMS], hdr_len;
};
struct AcfState {
  uint32_t status;      // ST_OK or PCO_B200_ASYNC_TOO_MANY_FILES
  uint32_t fits;        // acf_bytes_scan_kernel: the batch fits dst_cap and index_cap
  uint64_t n_read;      // *n_files as read
  uint64_t n_files;     // the files the call runs over (0 when *n_files is above max_files)
  unsigned long long bad;  // (file << 32) | status: the lowest file refusal (NONE64: none)
  uint64_t live_chunks; // chunks of the batch, 0 when refused
  uint64_t dst_bytes, index_bytes;  // what the batch needs (index_bytes 0 without an index)
  CarrySum total[ACF_SUMS];
};

static_assert(sizeof(AcfState) == 136 && sizeof(AcfFile) == 56 && sizeof(AcfPart) == 80, "the workspace formula in pco_b200.h");

// Workspace: the regions of pco_b200_compress_async's layout for max_chunks chunks of up to chunk_n numbers and nums_cap + 255 max_chunks
// rows (acomp_layout), then this call's, each 256-byte aligned.
struct AcfLayout {
  AcompLayout enc;
  uint64_t state, files, parts, cfile, cparts, pre, total;
};
inline AcompGeom acf_enc_geom(uint64_t max_chunks, uint64_t chunk_n, uint64_t nums_cap) {
  AcompGeom g = {};
  g.n_chunks = max_chunks;
  g.max_n = chunk_n;
  g.slots = nums_cap + 255 * max_chunks;
  g.bpc = n_batches_of(uint32_t(chunk_n));
  g.tiles = uint32_t((chunk_n + SPLIT_TILE - 1) / SPLIT_TILE);
  return g;
}
inline AcfLayout acf_layout(const AcompGeom& g, uint32_t lbytes, uint32_t n_vars, uint64_t max_files) {
  AcfLayout l;
  l.enc = acomp_layout(g, lbytes, n_vars);
  uint64_t at = l.enc.total;
  auto take = [&](uint64_t bytes) { const uint64_t o = at; at += acomp_align(bytes); return o; };
  l.state = take(sizeof(AcfState));
  l.files = take(max_files * sizeof(AcfFile));
  l.parts = take(ctas_of<ACF_THREADS>(max_files) * sizeof(AcfPart));
  l.cfile = take(g.n_chunks * 4);
  l.cparts = take(ctas_of<ACF_THREADS>(g.n_chunks + 1) * 8);
  l.pre = take((g.n_chunks + 1) * 8);
  l.total = at;
  return l;
}

// What the launches take by value.  `a` is what the shared gates and acomp_pack_gate_kernel read (ws, lay, n_chunks = max_chunks, n_vars).
struct AcfArgs {
  AcompArgs a;
  AcfLayout l;
  const uint64_t* file_ns;
  const uint64_t* n_files;
  PcoB200FileRef* files;
  uint64_t max_files, max_file_n, nums_cap, max_page_n, index_cap;
  uint32_t uniform_type, bpc;
  uint32_t framed;  // 1: standalone files (a header and a terminator around each file's chunks); 0: bare chunks (async_compress_wrapped.cuh)
  uint32_t reserved;
};
__device__ __forceinline__ AcfState* acf_state(const AcfArgs& g) { return reinterpret_cast<AcfState*>(g.a.ws + g.l.state); }
__device__ __forceinline__ AcfFile* acf_files(const AcfArgs& g) { return reinterpret_cast<AcfFile*>(g.a.ws + g.l.files); }
__device__ __forceinline__ AcfPart* acf_parts(const AcfArgs& g) { return reinterpret_cast<AcfPart*>(g.a.ws + g.l.parts); }

// The sizes of file slot f (zeros past the batch): its count for the nums_cap check, and the rest from its count clamped to max_file_n
// (a file above it refuses the batch, so its other sums only have to stay finite).
__device__ __forceinline__ void acf_file_sums(const AcfArgs& g, uint64_t f, uint64_t nf, CarrySum* s, uint64_t* n_out) {
  const uint64_t n = f < nf ? g.file_ns[f] : 0;
  const uint64_t nn = min(n, g.max_file_n);
  const EqualPages fp = equal_pages(nn, g.max_page_n);
  s[ACF_NUMS] = carry_sum(n);
  s[ACF_CHUNKS] = carry_sum(fp.n_chunks);
  s[ACF_ROWS] = carry_sum(fp.row_start(fp.n_chunks));
  s[ACF_FRAME] = carry_sum(f < nf && g.framed ? standalone_header_len(nn) + 1 : 0);
  s[ACF_IDX] = carry_sum(f < nf ? fp.index_bytes(g.a.n_vars) : 0);
  *n_out = n;
}
__device__ __forceinline__ uint64_t acf_n_files(const AcfArgs& g) {
  const uint64_t n = *g.n_files;
  return n <= g.max_files ? n : 0;
}

// ceil(max_files / ACF_THREADS) CTAs, one file slot per thread: the CTA's sums.
__global__ void __launch_bounds__(ACF_THREADS) acf_files_kernel(AcfArgs g) {
  const uint64_t nf = acf_n_files(g);
  CarrySum s[ACF_SUMS], tot[ACF_SUMS];
  uint64_t n;
  acf_file_sums(g, uint64_t(blockIdx.x) * ACF_THREADS + threadIdx.x, nf, s, &n);
  for (int k = 0; k < ACF_SUMS; k++) block_exscan<ACF_THREADS>(s[k], &tot[k]);
  if (threadIdx.x == 0)
    for (int k = 0; k < ACF_SUMS; k++) acf_parts(g)[blockIdx.x].s[k] = tot[k];
}

// One CTA: *n_files against max_files, and the CTA sums scanned into CTA offsets (in place).  Writes the AcfState the next kernels read.
__global__ void __launch_bounds__(ACF_SCAN_THREADS) acf_scan_kernel(AcfArgs g) {
  AcfPart* parts = acf_parts(g);
  CarrySum total[ACF_SUMS] = {};
  cta_scan_inplace<ACF_SCAN_THREADS, 1>(
      ctas_of<ACF_THREADS>(g.max_files), [&](uint64_t c, int k) { return parts[c].s[k]; }, [&](uint64_t c, int k, CarrySum v) { parts[c].s[k] = v; },
      total);
  if (threadIdx.x != 0) return;
  AcfState s;
  memset(&s, 0, sizeof(s));
  s.n_read = *g.n_files;
  s.n_files = acf_n_files(g);
  s.status = s.n_read > g.max_files ? uint32_t(PCO_B200_ASYNC_TOO_MANY_FILES) : uint32_t(ST_OK);
  s.bad = NONE64;
  for (int k = 0; k < ACF_SUMS; k++) s.total[k] = total[k];
  *acf_state(g) = s;
}

// ceil(max_files / ACF_THREADS) CTAs, one file slot per thread: the file's firsts (exclusive scans) and its refusal; the lowest failing
// file wins (atomicMin of (file << 32) | status).
__global__ void __launch_bounds__(ACF_THREADS) acf_place_kernel(AcfArgs g) {
  AcfState* st = acf_state(g);
  const uint64_t nf = st->n_files;
  const uint64_t f = uint64_t(blockIdx.x) * ACF_THREADS + threadIdx.x;
  CarrySum s[ACF_SUMS], ex[ACF_SUMS];
  uint64_t n;
  acf_file_sums(g, f, nf, s, &n);
  for (int k = 0; k < ACF_SUMS; k++) {
    CarrySum tot;
    ex[k] = carry_add(acf_parts(g)[blockIdx.x].s[k], block_exscan<ACF_THREADS>(s[k], &tot));
  }
  if (f >= nf) return;
  AcfFile r;
  r.n = n;
  for (int k = 0; k < ACF_SUMS; k++) r.first[k] = ex[k].s;
  r.hdr_len = g.framed ? standalone_header_len(n) : 0;
  acf_files(g)[f] = r;
  const CarrySum end = carry_add(ex[ACF_NUMS], s[ACF_NUMS]);
  uint32_t code = ST_OK;
  if (n > g.max_file_n) code = PCO_B200_ASYNC_FILE_TOO_LARGE;
  else if (end.ovf || end.s > g.nums_cap) code = PCO_B200_ASYNC_NUMS_CAP;
  if (code != ST_OK) atomicMin(&st->bad, (unsigned long long)((f << 32) | code));
}

// Grid-stride over the chunk slots [0, max_chunks] and the offset-bit sums: each chunk's start, row base and file (the pad slots and
// every slot of a refused batch: 0 numbers at the end of the batch's numbers), its ChunkEnc record reset, the sums zeroed.
__global__ void __launch_bounds__(ACF_THREADS) acf_init_kernel(AcfArgs g) {
  AcfState* st = acf_state(g);
  const bool ok = st->status == ST_OK && st->bad == NONE64;
  const uint64_t nf = ok ? st->n_files : 0, live = ok ? st->total[ACF_CHUNKS].s : 0;
  const uint64_t end_num = ok ? st->total[ACF_NUMS].s : 0, end_row = ok ? st->total[ACF_ROWS].s : 0;
  const uint64_t nc = g.a.n_chunks;
  const AcfFile* fl = acf_files(g);
  ChunkEnc* chunks = reinterpret_cast<ChunkEnc*>(g.a.ws + g.a.lay.chunks);
  uint64_t* starts = reinterpret_cast<uint64_t*>(g.a.ws + g.a.lay.starts);
  uint64_t* rows = reinterpret_cast<uint64_t*>(g.a.ws + g.a.lay.rows);
  uint32_t* cfile = reinterpret_cast<uint32_t*>(g.a.ws + g.l.cfile);
  uint32_t* ob_sum = reinterpret_cast<uint32_t*>(g.a.ws + g.a.lay.ob_sum);
  const uint64_t n_sums = nc * MAX_VARS * g.bpc;
  const uint64_t jobs = max(nc + 1, n_sums);
  for (uint64_t t = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; t < jobs; t += uint64_t(gridDim.x) * blockDim.x) {
    if (t <= nc) {
      uint64_t s = end_num, r = end_row;
      uint32_t file = ~0u;
      if (t < live) {
        // the file holding chunk t: the last one whose first chunk is at or before t (files of 0 chunks share their successor's)
        uint64_t lo = 0, hi = nf;  // invariant: fl[lo].first <= t < fl[hi].first (hi == nf: past the end)
        while (hi - lo > 1) {
          const uint64_t m = (lo + hi) >> 1;
          if (fl[m].first[ACF_CHUNKS] <= t) lo = m;
          else hi = m;
        }
        const AcfFile& f = fl[lo];
        const EqualPages fp = equal_pages(f.n, g.max_page_n);
        const uint64_t j = t - f.first[ACF_CHUNKS];
        s = f.first[ACF_NUMS] + fp.start(j);
        r = f.first[ACF_ROWS] + fp.row_start(j);
        file = uint32_t(lo);
      }
      starts[t] = s;
      rows[t] = r;
      if (t < nc) {
        cfile[t] = file;
        reset_chunk_enc(&chunks[t]);
      }
    }
    if (t < n_sums) ob_sum[t] = 0;
  }
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  AcompHead* h = reinterpret_cast<AcompHead*>(g.a.ws);
  h->flags[0] = h->flags[1] = 0;
  h->range_bits[0] = h->range_bits[1] = 0;
  h->total = 0;
  st->live_chunks = live;
}

// ceil((max_chunks + 1) / ACF_THREADS) CTAs: the CTA sums of the live chunks' sizes.
__global__ void __launch_bounds__(ACF_THREADS) acf_bytes_kernel(AcfArgs g) {
  const uint64_t live = acf_state(g)->live_chunks;
  const ChunkEnc* chunks = reinterpret_cast<const ChunkEnc*>(g.a.ws + g.a.lay.chunks);
  const uint64_t c = uint64_t(blockIdx.x) * ACF_THREADS + threadIdx.x;
  uint64_t tot;
  block_exscan<ACF_THREADS>(c < live ? chunks[c].chunk_bytes : 0, &tot);
  if (threadIdx.x == 0) reinterpret_cast<uint64_t*>(g.a.ws + g.l.cparts)[blockIdx.x] = tot;
}

// One CTA: the chunk CTA sums scanned into CTA offsets (in place), the bytes the batch needs, and whether it fits.
__global__ void __launch_bounds__(ACF_SCAN_THREADS) acf_bytes_scan_kernel(AcfArgs g) {
  uint64_t* parts = reinterpret_cast<uint64_t*>(g.a.ws + g.l.cparts);
  uint64_t total[1] = {};
  cta_scan_inplace<ACF_SCAN_THREADS, 1>(
      ctas_of<ACF_THREADS>(g.a.n_chunks + 1), [&](uint64_t c, int) { return parts[c]; }, [&](uint64_t c, int, uint64_t v) { parts[c] = v; }, total);
  if (threadIdx.x != 0) return;
  AcfState* st = acf_state(g);
  st->dst_bytes = total[0] + st->total[ACF_FRAME].s;
  st->index_bytes = g.a.index ? st->total[ACF_IDX].s : 0;
  st->fits = st->dst_bytes <= g.a.dst_cap && st->index_bytes <= g.index_cap ? 1u : 0u;
}

// ceil((max_chunks + 1) / ACF_THREADS) CTAs: pre[c] = the bytes of the live chunks before chunk c, for every slot up to max_chunks, and
// each chunk's place in dst (behind the frames of its file and the files before it), or past any dst_cap when it is not written.
__global__ void __launch_bounds__(ACF_THREADS) acf_offsets_kernel(AcfArgs g) {
  const AcfState* st = acf_state(g);
  const uint64_t live = st->live_chunks;
  const bool fits = st->fits != 0;
  ChunkEnc* chunks = reinterpret_cast<ChunkEnc*>(g.a.ws + g.a.lay.chunks);
  const uint64_t c = uint64_t(blockIdx.x) * ACF_THREADS + threadIdx.x;
  const uint64_t bytes = c < live ? chunks[c].chunk_bytes : 0;
  uint64_t tot;
  const uint64_t pre = reinterpret_cast<const uint64_t*>(g.a.ws + g.l.cparts)[blockIdx.x] + block_exscan<ACF_THREADS>(bytes, &tot);
  if (c > g.a.n_chunks) return;
  reinterpret_cast<uint64_t*>(g.a.ws + g.l.pre)[c] = pre;
  if (c == g.a.n_chunks) return;
  uint64_t off = ~uint64_t(0) - chunks[c].chunk_bytes;  // out_offset + chunk_bytes exceeds any out_cap below 2^64 - 1
  if (c < live && fits) {
    const AcfFile& f = acf_files(g)[reinterpret_cast<const uint32_t*>(g.a.ws + g.l.cfile)[c]];
    off = pre + f.first[ACF_FRAME] + f.hdr_len;
  }
  chunks[c].out_offset = off;
}

// ceil(max_files / ACF_THREADS) CTAs, one file slot per thread: a placed batch writes every file's PcoB200FileRef; one that fits also its
// header, its terminator and its side index header (as frame_files_kernel writes them).
__global__ void __launch_bounds__(ACF_THREADS) acf_frame_kernel(AcfArgs g) {
  const AcfState* st = acf_state(g);
  if (st->status != ST_OK || st->bad != NONE64) return;
  const uint64_t f = uint64_t(blockIdx.x) * ACF_THREADS + threadIdx.x;
  if (f >= st->n_files) return;
  const AcfFile r = acf_files(g)[f];
  const uint64_t* pre = reinterpret_cast<const uint64_t*>(g.a.ws + g.l.pre);
  const EqualPages fp = equal_pages(r.n, g.max_page_n);
  const uint64_t c0 = r.first[ACF_CHUNKS], k = fp.n_chunks;
  const uint64_t off = pre[c0] + r.first[ACF_FRAME];
  const uint64_t len = r.hdr_len + (pre[c0 + k] - pre[c0]) + 1;
  const uint64_t ilen = fp.index_bytes(g.a.n_vars);
  PcoB200FileRef ref;
  ref.offset = off;
  ref.len = len;
  ref.index_offset = g.a.index ? r.first[ACF_IDX] : 0;
  ref.index_len = g.a.index ? ilen : 0;
  g.files[f] = ref;
  if (!st->fits) return;
  uint8_t hdr[STANDALONE_HEADER_MAX];
  const uint32_t hl = standalone_header_into(r.n, uint8_t(g.uniform_type), hdr);
  for (uint32_t i = 0; i < hl; i++) g.a.dst[off + i] = hdr[i];
  g.a.dst[off + len - 1] = 0;
  if (!g.a.index) return;
  IndexHeader h;
  h.magic = INDEX_MAGIC;
  h.version = 1;
  h.n_chunks = k;
  h.n_total = r.n;
  h.file_len = len;
  h.chunks_offset = sizeof(IndexHeader);
  h.end_byte = len;
  h.reserved[0] = 0;
  h.reserved[1] = 0;
  *reinterpret_cast<IndexHeader*>(g.a.index + r.first[ACF_IDX]) = h;
}

// max_chunks CTAs, one per chunk slot: a live chunk of a batch that fits writes its record (chunk_offset counted from its file's first
// byte, out_offset from its first number, entries_offset from its index's first byte) and its region of batch entries: n_vars x batches
// records of the plan's n_vars (emit_index_kernel's, for the vars the chunk has) rounded up to 16 bytes, the rest zero, as the sync call's
// zeroed index holds it.
__global__ void __launch_bounds__(ACF_INDEX_THREADS) acf_index_kernel(AcfArgs g) {
  const AcfState* st = acf_state(g);
  const uint64_t c = blockIdx.x;
  if (c >= st->live_chunks || !st->fits) return;
  const ChunkEnc* chunks = reinterpret_cast<const ChunkEnc*>(g.a.ws + g.a.lay.chunks);
  const AcfFile& f = acf_files(g)[reinterpret_cast<const uint32_t*>(g.a.ws + g.l.cfile)[c]];
  const uint64_t j = c - f.first[ACF_CHUNKS];
  const uint64_t cs = acomp_starts(g.a)[c], n = acomp_starts(g.a)[c + 1] - cs;
  const uint32_t nb = n_batches_of(uint32_t(n));
  const uint32_t n_vars = chunks[c].fallback ? 1 : g.a.n_vars;
  const uint64_t eoff = equal_pages(f.n, g.max_page_n).entries_offset(g.a.n_vars, j);
  uint8_t* ix = g.a.index + f.first[ACF_IDX];
  if (threadIdx.x == 0) {
    IndexChunk ic;
    ic.chunk_offset = chunks[c].out_offset - (reinterpret_cast<const uint64_t*>(g.a.ws + g.l.pre)[f.first[ACF_CHUNKS]] + f.first[ACF_FRAME]);
    ic.n = uint32_t(n);
    ic.n_vars = n_vars;
    ic.entries_offset = eoff;
    ic.out_offset = cs - f.first[ACF_NUMS];
    reinterpret_cast<IndexChunk*>(ix + sizeof(IndexHeader))[j] = ic;
  }
  const BatchEntry* entries = reinterpret_cast<const BatchEntry*>(g.a.ws + g.a.lay.entries);
  const uint64_t words = entries_bytes(g.a.n_vars, n) / 4, used = uint64_t(n_vars) * nb * 3;
  uint32_t* dst = reinterpret_cast<uint32_t*>(ix + eoff);
  for (uint64_t w = threadIdx.x; w < words; w += ACF_INDEX_THREADS) {
    uint32_t x = 0;
    if (w < used) {
      const uint64_t i = w / 3, v = i / nb, b = i % nb;
      x = reinterpret_cast<const uint32_t*>(&entries[(c * MAX_VARS + v) * g.bpc + b])[w % 3];
    }
    dst[w] = x;
  }
}

// One thread: the outcome.
__global__ void acf_finish_kernel(AcfArgs g, PcoB200AsyncCompressFilesStatus* __restrict__ out) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  const AcfState* st = acf_state(g);
  PcoB200AsyncCompressFilesStatus s;
  memset(&s, 0, sizeof(s));
  s.file = ~uint64_t(0);
  s.n_files = st->n_read;
  if (st->status != ST_OK) {
    s.device_status = st->status;
  } else if (st->bad != NONE64) {
    s.device_status = uint32_t(st->bad & 0xffffffffu);
    s.file = st->bad >> 32;
  } else {
    s.dst_bytes = st->dst_bytes;
    s.index_bytes = st->index_bytes;
    if (st->fits) {
      s.dst_written = st->dst_bytes;
      s.index_written = st->index_bytes;
    } else {
      s.device_status = st->dst_bytes > g.a.dst_cap ? uint32_t(PCO_B200_ASYNC_FILES_DST_FULL) : uint32_t(PCO_B200_ASYNC_FILES_INDEX_FULL);
    }
  }
  s.kind = async_kind_of(s.device_status);
  *out = s;
}

// ---- host steps

// The plan's geometry: the encode regions' AcompGeom and the whole workspace
struct AcfPlanGeom {
  AcompGeom g;
  AcfLayout l;
};
inline uint64_t acf_chunk_n(uint64_t max_page_n, uint64_t max_file_n, uint64_t nums_cap) {
  return std::max<uint64_t>(1, std::min({page_cap(max_page_n), max_file_n, nums_cap}));
}
inline AcfPlanGeom acf_plan_geom(const PcoB200AsyncCompressFilesPlan& p) {
  AcfPlanGeom pg;
  pg.g = acf_enc_geom(p.max_chunks, acf_chunk_n(p.max_page_n, p.max_file_n, p.nums_cap), p.nums_cap);
  pg.l = acf_layout(pg.g, nt_bits(p.dtype) / 8, p.n_vars, p.max_files);
  return pg;
}

inline PcoB200Error acf_check_plan(const PcoB200AsyncCompressFilesPlan* p, AcfPlanGeom* pg) {
  if (!acomp_spec_ok(p) || p->level > 12 || p->max_files == 0 || p->max_files > 0x7fffffffu || p->max_file_n == 0 || p->nums_cap > (uint64_t(1) << 56) ||
      p->max_chunks != p->nums_cap / acf_chunk_n(p->max_page_n, p->max_file_n, p->nums_cap) + p->max_files || p->max_chunks > 0x7fffffffu)
    return fail(PCO_B200_INVALID_ARGUMENT, "the plan was not made by pco_b200_compress_files_async_plan");
  *pg = acf_plan_geom(*p);
  if (p->workspace_bytes != pg->l.total) return fail(PCO_B200_INVALID_ARGUMENT, "the plan was not made by pco_b200_compress_files_async_plan");
  return PCO_B200_OK;
}

// The launches up to and including pack_kernel, which every call of this layout shares: each chunk lands at its place in a.dst.
template <typename L>
void acf_launch_encode(const PcoB200AsyncCompressFilesPlan& p, const AcompGeom& g, const AcfArgs& fa, const void* nums, const AsyncLaunch& ln) {
  const cudaStream_t stream = ln.stream;
  const uint32_t file_ctas = uint32_t(ctas_of<ACF_THREADS>(p.max_files)), chunk_ctas = uint32_t(ctas_of<ACF_THREADS>(g.n_chunks + 1));
  ln.begin("acf_files_kernel");
  acf_files_kernel<<<file_ctas, ACF_THREADS, 0, stream>>>(fa);
  ln.end();
  ln.begin("acf_scan_kernel");
  acf_scan_kernel<<<1, ACF_SCAN_THREADS, 0, stream>>>(fa);
  ln.end();
  ln.begin("acf_place_kernel");
  acf_place_kernel<<<file_ctas, ACF_THREADS, 0, stream>>>(fa);
  ln.end();
  const uint32_t init_ctas = uint32_t(std::min<uint64_t>(1024, std::max<uint64_t>(g.n_chunks + 1, g.n_chunks * MAX_VARS * g.bpc) / ACF_THREADS + 1));
  ln.begin("acf_init_kernel");
  acf_init_kernel<<<init_ctas, ACF_THREADS, 0, stream>>>(fa);
  ln.end();
  // the CHUNK_BINS kernels compute each chunk's unoptimized_bins_log from the level and its n
  const EncParams ep = acomp_enc_params(p, g, fa.a, nums, p.nums_cap, p.level);
  enqueue_encode_kernels<L, true>(g, fa.a, ep, ln);
  // ---- placement: every chunk's final place in dst, behind its file's header
  ln.begin("acf_bytes_kernel");
  acf_bytes_kernel<<<chunk_ctas, ACF_THREADS, 0, stream>>>(fa);
  ln.end();
  ln.begin("acf_bytes_scan_kernel");
  acf_bytes_scan_kernel<<<1, ACF_SCAN_THREADS, 0, stream>>>(fa);
  ln.end();
  ln.begin("acf_offsets_kernel");
  acf_offsets_kernel<<<chunk_ctas, ACF_THREADS, 0, stream>>>(fa);
  ln.end();
  enqueue_pack<L>(g, fa.a, ep, ln);
}

template <typename L>
void acf_launch(const PcoB200AsyncCompressFilesPlan& p, const AcompGeom& g, const AcfArgs& fa, const void* nums, PcoB200AsyncCompressFilesStatus* status,
                const AsyncLaunch& ln) {
  acf_launch_encode<L>(p, g, fa, nums, ln);
  const cudaStream_t stream = ln.stream;
  const uint32_t nc = uint32_t(g.n_chunks), file_ctas = uint32_t(ctas_of<ACF_THREADS>(p.max_files));
  // ---- framing
  ln.begin("acf_frame_kernel");
  acf_frame_kernel<<<file_ctas, ACF_THREADS, 0, stream>>>(fa);
  ln.end();
  if (fa.a.index) {
    ln.begin("acf_index_kernel");
    acf_index_kernel<<<nc, ACF_INDEX_THREADS, 0, stream>>>(fa);
    ln.end();
  }
  ln.begin("acf_finish_kernel");
  acf_finish_kernel<<<1, 32, 0, stream>>>(fa, status);
  ln.end();
}

}  // namespace pcob200
