// Kernels of pco_b200_decompress_files_async: a batch of indexed standalone files decoded with the file list in device memory and no host
// decision between launches, so a batch a kernel picked (a sampler, a cache lookup) can be queued behind it or captured in a CUDA graph.
// What pco_b200_decompress_files does on the host (decompress_files_impl, host_api.cu: the reads of heads and index headers, the check
// verdicts, the placement, the merged chunk list) is done here on the device, over grids fixed by the plan's capacities:
//   af_files_kernel      one thread per file: its ref against src_cap / index_cap, its header (async_parse_header), its index header
//                        (index_header_ok), the FileCheck and FileMerge rows of the existing kernels, CTA sums of counts and chunks, and
//                        (CTA 0) the binomial table decode_kernel reads;
//   check_index_kernel   (files_kernels.cuh, one CTA per file slot) every record inside its own file, index and count;
//   af_scan_kernel       (one CTA) *n_files against max_files, the lowest ref refusal, and the CTA sums scanned into CTA offsets;
//   af_place_kernel      every file's dst base and table base, with exact 64-bit overflow detection, and the lowest failing file;
//   af_table_kernel      the gate: which files are decoded (all, those before the lowest refused file, or none); the other files'
//                        FileMerge rows emptied, pads behind the merged records;
//   merge_index_kernel   (files_kernels.cuh, one CTA per file slot) each file's records rebased into the one table;
//   fused_narrow_kernel<L>, symwalk_kernel<false>, decode_kernel<L, 1 / 2>, cold_chunks_kernel<L>  (as pco_b200_decompress_async);
//   af_finish_kernel     the lowest failing chunk and its file, else the refusal, the PcoB200AsyncFilesStatus and, on success, file_ns.
// Every refusal before the decode is decided before merge_index_kernel runs.  A call refused at file j decodes only the files before j
// (as pco_b200_decompress_files does, so that a decode failure in one of them is the one reported) and writes nothing at or behind file
// j's place in dst; a call refused before the files (too many, a ref outside the buffers) leaves a table of pads only.
#pragma once
#include "async_kernels.cuh"
#include "cta_scan.cuh"
#include "files_kernels.cuh"

namespace pcob200 {

constexpr int AF_THREADS = 256;        // the per-file and per-slot launches
constexpr int AF_SCAN_THREADS = 1024;  // the one-CTA launches

// per CTA of af_files_kernel (af_scan_kernel turns the sums into CTA offsets, in place)
struct AfPart {
  CarrySum count, chunks;
  uint64_t bad_ref;     // lowest ref refusal of the CTA as (file << 32) | status (NONE64: none)
  uint64_t reserved;
};

// decided by af_scan_kernel and af_place_kernel
struct AfState {
  uint32_t status;      // ST_OK, PCO_B200_ASYNC_TOO_MANY_FILES or a ref refusal
  uint32_t reserved;
  uint64_t n_read;      // *n_files as read
  uint64_t n_files;     // the files the call runs over (0 when *n_files is above max_files)
  uint64_t bad;         // (file << 32) | status: the lowest refusal (a ref refusal here, or af_place_kernel's by atomicMin)
  CarrySum total, chunks;  // the sums of the counts and of the chunk counts over the files
};

// everything the launches take by value; fp.src_len is src_cap
struct AfArgs {
  FileParams fp;
  const uint8_t* index;
  uint64_t index_cap;
  uint64_t dst_cap;
  const PcoB200FileRef* files;
  const uint64_t* n_files;
  uint32_t max_files, max_chunks;
};

// Workspace of one in-flight call, byte offsets, each region 256-byte aligned:
// AsyncCheck (binomials, chunk count) | AfState | per file: status, FileCheck, verdict, FileMerge | CTA sums | IndexChunk[max_chunks] |
// the decode tail.
struct AfLayout : AsyncDecodeTail {
  uint64_t state, fst, fchk, verdict, merges, parts, table;
};
__host__ __device__ inline AfLayout af_layout(uint64_t max_files, uint64_t max_chunks, uint64_t dst_cap) {
  AfLayout l;
  l.state = async_align(sizeof(AsyncCheck));
  l.fst = l.state + async_align(sizeof(AfState));
  l.fchk = l.fst + async_align(max_files * sizeof(uint32_t));
  l.verdict = l.fchk + async_align(max_files * sizeof(FileCheck));
  l.merges = l.verdict + async_align(max_files * sizeof(uint32_t));
  l.parts = l.merges + async_align(max_files * sizeof(FileMerge));
  l.table = l.parts + async_align(ctas_of<AF_THREADS>(max_files) * sizeof(AfPart));
  static_cast<AsyncDecodeTail&>(l) =
      async_decode_tail(l.table + async_align(max_chunks * sizeof(IndexChunk)), max_chunks, scratch_rows_total(dst_cap, uint32_t(max_chunks)), 0);
  return l;
}

__device__ __forceinline__ uint64_t af_n_files(const AfArgs& g) {
  const uint64_t n = *g.n_files;
  return n <= g.max_files ? n : 0;
}

// ceil(max_files / AF_THREADS) CTAs, one file per thread.  The ref checks are decompress_files_impl's argument checks (file inside
// src_cap, then for a ref with an index its offset a multiple of 16 and its bytes inside index_cap); a file that passes them gets its
// header parsed and checked against the plan's flavour, and its index header checked as decompress_files_impl checks it (chunk table
// 8-byte aligned).  Every slot up to max_files gets a FileCheck and a FileMerge row: files past *n_files or refused get zero chunks, which
// check_index_kernel and merge_index_kernel pass over.
__global__ void __launch_bounds__(AF_THREADS) af_files_kernel(AfArgs g, AsyncCheck* __restrict__ chk, uint32_t* __restrict__ fst,
                                                              FileCheck* __restrict__ fchk, FileMerge* __restrict__ merges, AfPart* __restrict__ parts) {
  __shared__ unsigned long long s_bad;
  const uint32_t tid = threadIdx.x;
  if (tid == 0) s_bad = NONE64;
  if (blockIdx.x == 0 && tid == 32) PCOB_ASYNC_FILL_BINOMS(chk->binoms);
  __syncthreads();
  const uint64_t n = af_n_files(g);
  const uint64_t i = uint64_t(blockIdx.x) * AF_THREADS + tid;
  uint32_t st = ST_OK;
  uint64_t count = 0, n_chunks = 0;
  FileCheck fc{0, 0, 0, 0, 0, 0, 0, 0, 0};
  FileMerge fm{0, 0, 0, 0, 0, 0};
  if (i < n) {
    const PcoB200FileRef r = g.files[i];
    const uint64_t src_cap = g.fp.src_len;
    uint32_t ref = ST_OK;
    if (r.len > src_cap || r.offset > src_cap - r.len) ref = PCO_B200_ASYNC_FILE_OUTSIDE;
    else if (r.index_len && r.index_offset % 16) ref = PCO_B200_ASYNC_INDEX_OFFSET;
    else if (r.index_len && (r.index_len > g.index_cap || r.index_offset > g.index_cap - r.index_len)) ref = PCO_B200_ASYNC_INDEX_OUTSIDE;
    if (ref != ST_OK) {
      atomicMin(&s_bad, (i << 32) | ref);
      st = ref;
    } else {
      uint32_t uniform = 0, major = 0;
      st = async_parse_header(static_cast<const uint8_t*>(g.fp.src) + r.offset, r.len, &uniform, &major);
      if (st == ST_OK && r.index_len < sizeof(IndexHeader)) st = PCO_B200_ASYNC_NO_INDEX;
      if (st == ST_OK && (uniform != g.fp.uniform_type || major != g.fp.format_major)) st = PCO_B200_ASYNC_HEADER_MISMATCH;
      if (st == ST_OK) {
        const uint8_t* ix = g.index + r.index_offset;
        IndexHeader ih;
        const uint64_t w0 = async_ld_u64(ix);
        ih.magic = uint32_t(w0);
        ih.version = uint32_t(w0 >> 32);
        ih.n_chunks = async_ld_u64(ix + 8);
        ih.n_total = async_ld_u64(ix + 16);
        ih.file_len = async_ld_u64(ix + 24);
        ih.chunks_offset = async_ld_u64(ix + 32);
        if (!index_header_ok(ih, r.len, r.index_len) || ih.chunks_offset % 8 != 0) {
          st = PCO_B200_ASYNC_INDEX_FOREIGN;
        } else {
          count = ih.n_total;
          n_chunks = ih.n_chunks;
          const uint64_t recs = r.index_offset + ih.chunks_offset;
          fc = FileCheck{recs, n_chunks, r.offset, r.len, r.index_offset, r.index_len, count, major, 0};
          fm = FileMerge{recs, 0, r.offset, r.index_offset, 0, n_chunks};  // list_at and out_add: af_place_kernel
        }
      }
    }
  }
  if (i < g.max_files) {
    fst[i] = st;
    fchk[i] = fc;
    merges[i] = fm;
  }
  CarrySum c_tot, k_tot;
  block_exscan<AF_THREADS>(carry_sum(count), &c_tot);
  block_exscan<AF_THREADS>(carry_sum(n_chunks), &k_tot);
  if (tid == 0) parts[blockIdx.x] = AfPart{c_tot, k_tot, s_bad, 0};
}

// One CTA: *n_files against max_files, the lowest ref refusal over all files (checked for every file before anything else, as
// decompress_files_impl does), and the CTA sums scanned into CTA offsets (in place).  Writes the AfState the next kernels read.
__global__ void __launch_bounds__(AF_SCAN_THREADS) af_scan_kernel(AfArgs g, AfPart* __restrict__ parts, AfState* __restrict__ state) {
  __shared__ unsigned long long s_bad;
  const uint32_t tid = threadIdx.x;
  if (tid == 0) s_bad = NONE64;
  __syncthreads();
  const uint64_t n_parts = ctas_of<AF_THREADS>(g.max_files);
  for (uint64_t c = tid; c < n_parts; c += AF_SCAN_THREADS)
    if (parts[c].bad_ref != NONE64) atomicMin(&s_bad, parts[c].bad_ref);
  auto sum = [&](uint64_t c, int k) -> CarrySum& { return k ? parts[c].chunks : parts[c].count; };
  CarrySum total[2] = {};
  cta_scan_inplace<AF_SCAN_THREADS, 1>(
      n_parts, [&](uint64_t c, int k) { return sum(c, k); }, [&](uint64_t c, int k, CarrySum v) { sum(c, k) = v; }, total);
  __syncthreads();
  if (tid != 0) return;
  AfState s;
  s.status = ST_OK;
  s.reserved = 0;
  s.n_read = *g.n_files;
  s.n_files = af_n_files(g);
  s.bad = NONE64;
  s.total = total[0];
  s.chunks = total[1];
  if (s.n_read > g.max_files) s.status = PCO_B200_ASYNC_TOO_MANY_FILES;
  else if (s_bad != NONE64) {
    s.status = uint32_t(s_bad);
    s.bad = s_bad;
  }
  *state = s;
}

// ceil(max_files / AF_THREADS) CTAs, one file per thread: its dst base and table base (exclusive scans), and its refusal, the first of
// decompress_files_impl's order that applies - header and index header (af_files_kernel), check_index_kernel's verdict (misaligned
// entries; records outside the file), placement (the running total passes dst_cap) - then the running chunk count past max_chunks.
// The lowest failing file wins (atomicMin of (file << 32) | status).
__global__ void __launch_bounds__(AF_THREADS) af_place_kernel(AfArgs g, const uint32_t* __restrict__ fst, const FileCheck* __restrict__ fchk,
                                                              const uint32_t* __restrict__ verdict, const AfPart* __restrict__ parts,
                                                              FileMerge* __restrict__ merges, AfState* __restrict__ state) {
  if (state->status != ST_OK) return;  // uniform: every thread leaves
  const uint32_t tid = threadIdx.x;
  const uint64_t n = state->n_files;
  const uint64_t i = uint64_t(blockIdx.x) * AF_THREADS + tid;
  const bool in = i < n;
  const uint64_t count = in ? fchk[i].n_total : 0, n_chunks = in ? fchk[i].n_chunks : 0;
  CarrySum tot;
  const CarrySum c_ex = carry_add(parts[blockIdx.x].count, block_exscan<AF_THREADS>(carry_sum(count), &tot));
  const CarrySum k_ex = carry_add(parts[blockIdx.x].chunks, block_exscan<AF_THREADS>(carry_sum(n_chunks), &tot));
  if (!in) return;
  merges[i].list_at = k_ex.s;
  merges[i].out_add = c_ex.s;
  const CarrySum c_inc = carry_add(c_ex, carry_sum(count)), k_inc = carry_add(k_ex, carry_sum(n_chunks));
  uint32_t st = fst[i];
  if (st == ST_OK && n_chunks > 0) {
    const uint32_t v = verdict[i];
    if (v == IDX_MISALIGNED) st = PCO_B200_ASYNC_ENTRIES_MISALIGNED;
    else if (v == IDX_OUTSIDE) st = PCO_B200_ASYNC_RECORDS_OUTSIDE;
  }
  if (st == ST_OK && (c_inc.ovf || c_inc.s > g.dst_cap)) st = PCO_B200_ASYNC_FILES_DST;
  if (st == ST_OK && (k_inc.ovf || k_inc.s > g.max_chunks)) st = PCO_B200_ASYNC_TOO_MANY_CHUNKS;
  if (st != ST_OK) atomicMin(reinterpret_cast<unsigned long long*>(&state->bad), (i << 32) | st);
}

// max(ceil(max_chunks / AF_THREADS), ceil(max_files / AF_THREADS)) CTAs: the gate.  Every thread reads the same decision from the state.
// *n_files above max_files or a ref refusal: nothing is decoded.  A file j refused by af_place_kernel: only the files before it are
// decoded, as pco_b200_decompress_files decodes only the files before its lowest failure, so that a decode failure in an earlier file
// is still the one reported.  FileMerge rows from the first file not decoded on are emptied, so merge_index_kernel writes nothing for
// them; table slots from the chunk count decoded to max_chunks get pads (chunk_offset = src_cap), which the decode kernels refuse
// without reading src.  chk->status keeps the refusal pending for af_finish_kernel.
__global__ void __launch_bounds__(AF_THREADS) af_table_kernel(AfArgs g, const AfState* __restrict__ state, AsyncCheck* __restrict__ chk,
                                                              FileMerge* __restrict__ merges, IndexChunk* __restrict__ table) {
  const uint64_t bad = state->bad, n = state->n_files;
  const uint32_t pre = state->status;
  // the files decoded: [0, limit), and their chunks: [0, accepted), at most max_chunks (a file before `limit` that took the running
  // count past max_chunks would have been refused itself)
  const uint64_t limit = pre != ST_OK ? 0 : bad != NONE64 ? bad >> 32 : n;
  const uint64_t accepted = limit == 0 ? 0 : limit < n ? merges[limit].list_at : state->chunks.s;
  const uint64_t k = uint64_t(blockIdx.x) * AF_THREADS + threadIdx.x;
  if (k < g.max_files && k >= limit) merges[k].n_chunks = 0;
  if (k < g.max_chunks && k >= accepted) table[k] = IndexChunk{g.fp.src_len, 0u, 0u, 0, 0};
  if (k == 0) {
    chk->status = pre != ST_OK ? pre : bad != NONE64 ? uint32_t(bad) : uint32_t(ST_OK);
    chk->n_chunks = uint32_t(accepted);
  }
}

// One CTA: the lowest failing table slot (its file: the last file whose table base is at most the slot), else the pending refusal, else
// success and file_ns.  Slots are in file order and only files before a pending refusal have chunks in the table, so the lowest failing
// slot lies in the lowest failing file.
__global__ void __launch_bounds__(AF_SCAN_THREADS) af_finish_kernel(const AfState* __restrict__ state, const AsyncCheck* __restrict__ chk,
                                                                    const FileMerge* __restrict__ merges, const FileCheck* __restrict__ fchk,
                                                                    const uint32_t* __restrict__ statuses, uint64_t* __restrict__ file_ns,
                                                                    PcoB200AsyncFilesStatus* __restrict__ out) {
  __shared__ uint32_t s_min;
  const uint32_t tid = threadIdx.x;
  if (tid == 0) s_min = 0xffffffffu;
  __syncthreads();
  const uint32_t pending = chk->status, n_chunks = chk->n_chunks;
  const uint64_t n = state->n_files;
  for (uint32_t k = tid; k < n_chunks; k += blockDim.x)
    if (statuses[k] != ST_OK) {
      atomicMin(&s_min, k);  // a thread's first failure is its lowest
      break;
    }
  __syncthreads();
  const bool ok = pending == ST_OK && s_min == 0xffffffffu;
  if (ok && file_ns)
    for (uint64_t i = tid; i < n; i += blockDim.x) file_ns[i] = fchk[i].n_total;
  if (tid != 0) return;
  PcoB200AsyncFilesStatus r;
  r.kind = PCO_B200_OK;
  r.device_status = ST_OK;
  r.file = NONE64;
  r.chunk = NONE64;
  r.n_written = pending == ST_OK ? state->total.s : 0;
  r.n_files = state->n_read;
  if (s_min != 0xffffffffu) {
    uint64_t a = 0, b = n;  // the last file whose list_at <= s_min
    while (b - a > 1) {
      const uint64_t m = a + (b - a) / 2;
      if (merges[m].list_at <= s_min) a = m;
      else b = m;
    }
    const uint32_t st = statuses[s_min];
    r.kind = async_kind_of(st);
    r.device_status = st;
    r.file = a;
    r.chunk = s_min - merges[a].list_at;
  } else if (pending != ST_OK) {
    r.kind = async_kind_of(pending);
    r.device_status = pending;
    if (pending != PCO_B200_ASYNC_TOO_MANY_FILES) r.file = state->bad >> 32;
  }
  *out = r;
}

}  // namespace pcob200
