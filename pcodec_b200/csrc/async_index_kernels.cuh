// Kernels of pco_b200_build_index_async: the side index of a standalone file without one (as pco writes them), built on the caller's
// stream with no host decision between launches, so a reader can queue it behind other GPU work or capture "build index, then
// pco_b200_decompress_async" in one CUDA graph.  It is the speculative walk of the blocking index-free decompress (host_api.cu,
// speculative_walk_rounds) with the host's steps moved to the device, over grids fixed by the plan's capacities:
//   ai_head_kernel      *src_len against src_cap, the header (async_parse_header) against the plan's flavour, the cursor on chunk 0;
//   two rounds of       (pco's EqualPagesUpTo writes chunks of at most two sizes, in two runs, so two rounds cover files paged that way)
//     ai_round_kernel     the 4-byte pattern at the cursor (type byte, n - 1); the round is idle on the terminator, on another type byte,
//                         once max_chunks chunks are indexed, and behind a round that took no chunk (its cursor and pattern would repeat);
//     ai_count_kernel     per CTA of the grid over src_cap, the positions behind the cursor that carry the pattern (CTAs outside leave);
//     ai_scan_kernel      the counts scanned into CTA bases, and the candidates kept: the first max_chunks - n + AI_SPARE_CANDS in
//                         position order (coincidences may lie in front of the last real chunk), as many as the round arena holds;
//     ai_scatter_kernel   the kept candidates in position order, each with a record and its entries' place in the round arena;
//     ai_walk_kernel<10>  every candidate walked as a chunk, one CTA each (walk_run, decode_kernels.cuh);
//     ai_walk_kernel<12>  again, the candidates that reported ST_UNSUPPORTED (tables of 2^11 or 2^12 states, level 9-12 files);
//     ai_chain_kernel     the chain of real chunks from the cursor (chunk_chain, codec_common.cuh), appended to the record list;
//   ai_serial_kernel    walk_run<12> in serial mode from the cursor: the rest of the file, with the reference's semantics for the
//                       terminator, corruption, truncation, chunks the walker declines (Unsupported) and files of three or more runs;
//                       its entries go to a region of their own, index_cap bytes, which holds the rest of any index that fits;
//   ai_place_kernel     the walk's verdict, and the chunks' entry offsets in the final layout (a scan of their sizes) and its fit;
//   ai_copy_kernel      one CTA per chunk: its record and its entries, padding zeroed, into the index (nothing when the verdict is not OK);
//   ai_finish_kernel    the index header and the PcoB200AsyncIndexStatus.
// The walks write records and entries into the workspace; the index is written only by the last three kernels, and only on success.
#pragma once
#include "async_kernels.cuh"
#include "cta_scan.cuh"
#include "decode_kernels.cuh"

namespace pcob200 {

constexpr int AI_THREADS = 256;         // the find grid and the per-chunk copy
constexpr int AI_FIND_PER_THREAD = 16;  // positions per thread of the find grid
constexpr uint64_t AI_FIND_SPAN = uint64_t(AI_THREADS) * AI_FIND_PER_THREAD;
constexpr int AI_SCAN_THREADS = 1024;   // the one-CTA scans
constexpr int AI_SCAN_PER_THREAD = 16;
constexpr uint32_t AI_SPARE_CANDS = 8;  // candidates kept beyond the chunks max_chunks still takes
constexpr int AI_ROUNDS = 2;

// what the kernels decide, at the start of the workspace
struct AiState {
  uint32_t status;       // ST_OK, a PCO_B200_ASYNC_* refusal or the failing chunk's status
  uint32_t active;       // the current round runs
  uint32_t stalled;      // a round ran and its chain took no chunk: the rounds are over
  uint32_t reserved;
  uint64_t src_len;      // *src_len as read
  uint64_t cursor;       // the first byte not yet indexed
  uint64_t n_chunks;     // chunks indexed so far (records in the list)
  uint64_t n_total;      // their numbers
  uint64_t arena_end;    // the first free byte of the round arena (a workspace offset)
  uint64_t n0, stride;   // the current round: its chunk size and each candidate's room for entries
  uint64_t pattern;      // its 4 bytes, little-endian
  uint64_t find_lo, find_hi;  // the find CTAs over [cursor, src_len - 3)
  uint64_t m;            // candidates kept
  uint64_t cand_at;      // candidate k's entries at cand_at + k * stride
  uint64_t serial_chunks, end_byte, fail_chunk, index_bytes;
  WalkResult tail;       // the serial walker's
};

// everything the launches take by value
struct AiArgs {
  const uint8_t* src;
  const uint64_t* src_len;
  uint8_t* index;
  uint8_t* ws;
  uint64_t src_cap, index_cap, max_chunks;
  uint32_t dtype, uniform_type, format_major;
};

// Chunk c's record `r` (chunk_offset as the index states it) and its walked entries at `from` (n_vars x batches of them, then anything)
// into the index: the entries at byte `at`, zeros up to the next 16-byte boundary, and the record with entries_offset = at.  Every
// thread of a CTA of AI_THREADS calls it.
__device__ __forceinline__ void index_copy_chunk(IndexChunk r, const uint32_t* from, uint8_t* index, uint64_t at, uint64_t c) {
  uint32_t* to = reinterpret_cast<uint32_t*>(index + at);
  const uint64_t words = uint64_t(r.n_vars) * n_batches_of(r.n) * (sizeof(BatchEntry) / 4), room = entries_bytes(r.n_vars, r.n) / 4;
  for (uint64_t w = threadIdx.x; w < room; w += AI_THREADS) to[w] = w < words ? from[w] : 0u;
  if (threadIdx.x == 0) {
    r.entries_offset = at;
    reinterpret_cast<IndexChunk*>(index + sizeof(IndexHeader))[c] = r;
  }
}

// The header of a side index of n_chunks records right behind it, for a file of file_len bytes whose terminator ends at end_byte.
__device__ __forceinline__ void write_index_header(uint8_t* index, uint64_t n_chunks, uint64_t n_total, uint64_t file_len, uint64_t end_byte) {
  IndexHeader h;
  memset(&h, 0, sizeof(h));
  h.magic = INDEX_MAGIC;
  h.version = 1;
  h.n_chunks = n_chunks;
  h.n_total = n_total;
  h.file_len = file_len;
  h.chunks_offset = sizeof(IndexHeader);
  h.end_byte = end_byte;
  *reinterpret_cast<IndexHeader*>(index) = h;
}

// Workspace of one in-flight call, byte offsets, each region 256-byte aligned: AiState | find CTA counts (8 bytes per AI_FIND_SPAN bytes
// of src_cap) | per candidate (max_chunks + AI_SPARE_CANDS): position, record, status, end | per chunk (max_chunks + 1, the one that
// tells a file of too many chunks): record, final entries offset | the round arena, the candidates' entries (2 x index_cap: a
// candidate's room is that of two vars, so every chunk of an index that fits index_cap has room at that stride) | the serial region,
// the serial walker's entries (index_cap: the coincidences' slots the rounds leave in the round arena never cost the walker room, so
// an index that fits index_cap always fits, and a walk that runs out of it has found an index larger than index_cap).
struct AiLayout {
  uint64_t parts, cand, crec, cst, cend, recs, offs, arena, arena_end, serial, serial_end, total;
};
__host__ __device__ inline uint64_t ai_find_ctas(uint64_t src_cap) {
  const uint64_t n = (src_cap + AI_FIND_SPAN - 1) / AI_FIND_SPAN;
  return n ? n : 1;
}
__host__ __device__ inline AiLayout ai_layout(uint64_t src_cap, uint64_t index_cap, uint64_t max_chunks) {
  const uint64_t cc = max_chunks + AI_SPARE_CANDS, rc = max_chunks + 1;
  AiLayout l;
  l.parts = async_align(sizeof(AiState));
  l.cand = l.parts + async_align(ai_find_ctas(src_cap) * sizeof(uint64_t));
  l.crec = l.cand + async_align(cc * sizeof(uint64_t));
  l.cst = l.crec + async_align(cc * sizeof(IndexChunk));
  l.cend = l.cst + async_align(cc * sizeof(uint32_t));
  l.recs = l.cend + async_align(cc * sizeof(uint64_t));
  l.offs = l.recs + async_align(rc * sizeof(IndexChunk));
  l.arena = l.offs + async_align(rc * sizeof(uint64_t));
  l.arena_end = l.arena + 2 * index_cap;
  l.serial = l.arena + async_align(2 * index_cap);
  l.serial_end = l.serial + index_cap;
  l.total = l.serial + async_align(index_cap);
  return l;
}

__device__ __forceinline__ FileParams ai_file(const AiArgs& g, const AiState& s) {
  return FileParams{g.src, s.src_len, g.dtype, g.uniform_type, g.format_major};
}

// One thread.  The file length against src_cap, the header against the plan's flavour; the cursor on the first chunk.
__global__ void ai_head_kernel(AiArgs g, AiState* __restrict__ state) {
  AiState s;
  memset(&s, 0, sizeof(s));
  s.src_len = *g.src_len;
  s.fail_chunk = ~uint64_t(0);
  s.arena_end = ai_layout(g.src_cap, g.index_cap, g.max_chunks).arena;
  uint32_t st = ST_OK;
  if (s.src_len > g.src_cap) {
    st = PCO_B200_ASYNC_FILE_OUTSIDE;
  } else {
    uint32_t uniform = 0, major = 0;
    st = async_parse_header(g.src, s.src_len, &uniform, &major, &s.cursor);
    if (st == ST_OK && (uniform != g.uniform_type || major != g.format_major)) st = PCO_B200_ASYNC_HEADER_MISMATCH;
  }
  s.status = st;
  *state = s;
}

// One thread: the round's pattern, or the round idle (the serial walker owns the terminator, another type byte, a cursor too close to
// the end for a chunk header, the chunk behind max_chunks, and the chunk a round before could not take - cold, corrupt or truncated).
__global__ void ai_round_kernel(AiArgs g, AiState* __restrict__ state) {
  AiState& s = *state;
  s.active = 0;
  s.m = 0;
  if (s.status != ST_OK || s.stalled || s.n_chunks >= g.max_chunks || s.cursor + 4 > s.src_len) return;
  const uint8_t* b = g.src + s.cursor;
  if (b[0] != g.dtype) return;
  s.pattern = uint64_t(b[0]) | (uint64_t(b[1]) << 8) | (uint64_t(b[2]) << 16) | (uint64_t(b[3]) << 24);
  s.n0 = (s.pattern >> 8) + 1;
  s.stride = entries_bytes(MAX_VARS, s.n0);
  s.find_lo = s.cursor / AI_FIND_SPAN;
  s.find_hi = (s.src_len - 3 + AI_FIND_SPAN - 1) / AI_FIND_SPAN;
  s.active = 1;
}

// The positions of thread threadIdx.x of CTA blockIdx.x inside [cursor, src_len - 3) whose 4 bytes are the pattern, as a bit mask.
__device__ __forceinline__ uint32_t ai_matches(const AiArgs& g, const AiState& s) {
  const uint64_t p0 = uint64_t(blockIdx.x) * AI_FIND_SPAN + uint64_t(threadIdx.x) * AI_FIND_PER_THREAD;
  const uint64_t lo = s.cursor, hi = s.src_len - 3;
  uint32_t mask = 0;
  if (p0 + AI_FIND_PER_THREAD <= lo || p0 >= hi) return 0;
  uint32_t w = 0;
  for (int i = 0; i < 3; i++) w |= (p0 + i < s.src_len ? uint32_t(g.src[p0 + i]) : 0u) << (8 * (i + 1));
#pragma unroll
  for (int q = 0; q < AI_FIND_PER_THREAD; q++) {
    const uint64_t p = p0 + q;
    w = (w >> 8) | ((p + 3 < s.src_len ? uint32_t(g.src[p + 3]) : 0u) << 24);
    if (p >= lo && p < hi && w == uint32_t(s.pattern)) mask |= 1u << q;
  }
  return mask;
}

// ai_find_ctas(src_cap) CTAs: each in [find_lo, find_hi) counts its positions.
__global__ void __launch_bounds__(AI_THREADS) ai_count_kernel(AiArgs g, const AiState* __restrict__ state, uint64_t* __restrict__ parts) {
  const AiState& s = *state;
  if (!s.active || blockIdx.x < s.find_lo || blockIdx.x >= s.find_hi) return;
  uint64_t total;
  block_exscan<AI_THREADS>(uint64_t(__popc(ai_matches(g, s))), &total);
  if (threadIdx.x == 0) parts[blockIdx.x] = total;
}

// One CTA: the counts scanned into CTA bases, and m, the candidates kept, with their place in the arena.
__global__ void __launch_bounds__(AI_SCAN_THREADS) ai_scan_kernel(AiArgs g, AiState* __restrict__ state, uint64_t* __restrict__ parts) {
  AiState& s = *state;
  if (!s.active) return;
  uint64_t* v = parts + s.find_lo;
  uint64_t found[1] = {};
  cta_scan_inplace<AI_SCAN_THREADS, AI_SCAN_PER_THREAD>(
      s.find_hi - s.find_lo, [&](uint64_t i, int) { return v[i]; }, [&](uint64_t i, int, uint64_t x) { v[i] = x; }, found);
  if (threadIdx.x != 0) return;
  const AiLayout l = ai_layout(g.src_cap, g.index_cap, g.max_chunks);
  const uint64_t at = (s.arena_end + 15) & ~uint64_t(15);
  const uint64_t room = at < l.arena_end ? l.arena_end - at : 0;
  s.m = min(min(found[0], g.max_chunks - s.n_chunks + AI_SPARE_CANDS), room / s.stride);
  s.cand_at = at;
}

// ai_find_ctas(src_cap) CTAs: the kept candidates at their rank in position order, each with a record for the walks.
__global__ void __launch_bounds__(AI_THREADS) ai_scatter_kernel(AiArgs g, const AiState* __restrict__ state, const uint64_t* __restrict__ parts,
                                                               uint64_t* __restrict__ cand, IndexChunk* __restrict__ crec) {
  const AiState& s = *state;
  if (!s.active || blockIdx.x < s.find_lo || blockIdx.x >= s.find_hi || parts[blockIdx.x] >= s.m) return;
  const uint32_t mask = ai_matches(g, s);
  uint64_t total;
  uint64_t rank = parts[blockIdx.x] + block_exscan<AI_THREADS>(uint64_t(__popc(mask)), &total);
  const uint64_t p0 = uint64_t(blockIdx.x) * AI_FIND_SPAN + uint64_t(threadIdx.x) * AI_FIND_PER_THREAD;
  for (uint32_t b = mask; b && rank < s.m; b &= b - 1, rank++) {
    const uint64_t p = p0 + __ffs(b) - 1;
    cand[rank] = p;
    crec[rank] = IndexChunk{p, uint32_t(s.n0), 0u, s.cand_at + rank * s.stride, 0};
  }
}

// max_chunks + AI_SPARE_CANDS CTAs launched as walk_kernel is: candidate blockIdx.x walked as a chunk (CAP_LOG 12: only one that the
// CAP_LOG 10 walk reported ST_UNSUPPORTED for); the others leave at once.
template <int CAP_LOG>
__global__ void __launch_bounds__(WALK_THREADS, PCOB_WALK_MIN_BLOCKS) ai_walk_kernel(AiArgs g, const AiState* __restrict__ state,
                                                                                    uint32_t* __restrict__ cst, uint64_t* __restrict__ cend) {
  const AiState& s = *state;
  if (!s.active || blockIdx.x >= s.m) return;
  if (CAP_LOG > SMALL_MAX_SIZE_LOG && cst[blockIdx.x] != ST_UNSUPPORTED) return;
  const AiLayout l = ai_layout(g.src_cap, g.index_cap, g.max_chunks);
  walk_run<CAP_LOG>(ai_file(g, s), g.ws, l.crec, uint32_t(s.m), 0, l.arena_end, 0, 0, ~uint64_t(0), cst, nullptr, 0, cend);
}

// One CTA: the chain of real chunks from the cursor, appended to the record list with their out_offset; the cursor behind them.  The
// chain is one thread's walk over the candidates; the CTA first pulls them towards L1.
__global__ void __launch_bounds__(AI_THREADS) ai_chain_kernel(AiArgs g, AiState* __restrict__ state) {
  AiState& s = *state;
  if (!s.active) return;
  const AiLayout l = ai_layout(g.src_cap, g.index_cap, g.max_chunks);
  const uint64_t* cand = reinterpret_cast<const uint64_t*>(g.ws + l.cand);
  const IndexChunk* crec = reinterpret_cast<const IndexChunk*>(g.ws + l.crec);
  const uint32_t* cst = reinterpret_cast<const uint32_t*>(g.ws + l.cst);
  const uint64_t* cend = reinterpret_cast<const uint64_t*>(g.ws + l.cend);
  IndexChunk* recs = reinterpret_cast<IndexChunk*>(g.ws + l.recs);
  const uint64_t m = s.m;
  for (uint64_t k = uint64_t(threadIdx.x) * 16; k < m; k += uint64_t(AI_THREADS) * 16) {
    asm volatile("prefetch.global.L1 [%0];" ::"l"(cand + k));
    asm volatile("prefetch.global.L1 [%0];" ::"l"(cend + k));
    asm volatile("prefetch.global.L1 [%0];" ::"l"(cst + k));
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  const uint64_t n = s.n_chunks, n0 = s.n0;
  uint64_t next = s.cursor, taken = 0, last = 0;
  // the cap counted in chunks (one unit per chunk): the chain stops at max_chunks, the serial walker finds out what lies behind
  chunk_chain(cand, cst, cend, uint32_t(m), s.cursor, 1, n, g.max_chunks, s.src_len, &next, [&](uint32_t k) {
    IndexChunk r = crec[k];
    r.out_offset = s.n_total + taken * n0;
    recs[n + taken] = r;
    taken++;
    last = k;
  });
  if (taken == 0) {
    s.stalled = 1;
    return;
  }
  s.n_chunks = n + taken;
  s.n_total += taken * n0;
  s.cursor = next;
  s.arena_end = crec[last].entries_offset + s.stride;
}

// One CTA launched as walk_kernel<12> is: the serial walk from the cursor to the terminator or the first chunk it cannot index, with
// records for up to max_chunks + 1 chunks in all.
__global__ void __launch_bounds__(WALK_THREADS, PCOB_WALK_MIN_BLOCKS) ai_serial_kernel(AiArgs g, AiState* __restrict__ state) {
  const AiState s = *state;
  if (s.status != ST_OK) return;
  const AiLayout l = ai_layout(g.src_cap, g.index_cap, g.max_chunks);
  const uint64_t limit = min(g.max_chunks + 1 - s.n_chunks, uint64_t(0xffffffffu));
  walk_run<12>(ai_file(g, s), g.ws, l.recs + s.n_chunks * sizeof(IndexChunk), uint32_t(limit), l.serial, l.serial_end,
               s.cursor, s.n_total, ~uint64_t(0), nullptr, &state->tail, 1, nullptr);
}

// One CTA: the serial walk's verdict (the terminator: done; records full: more than max_chunks chunks; entries full: the serial region,
// and so the index, is too small - whichever the walk meets first; anything else: that chunk's status), then each chunk's entries offset in the final layout - header, the
// n_chunks records, each chunk's entries at the next 16-byte boundary - and whether it fits index_cap.
__global__ void __launch_bounds__(AI_SCAN_THREADS) ai_place_kernel(AiArgs g, AiState* __restrict__ state) {
  __shared__ uint32_t s_ok;
  AiState& s = *state;
  const AiLayout l = ai_layout(g.src_cap, g.index_cap, g.max_chunks);
  if (threadIdx.x == 0) {
    if (s.status == ST_OK) {
      const WalkResult r = s.tail;
      const uint64_t n_all = s.n_chunks + r.n_chunks;
      s.serial_chunks = r.n_chunks;
      if (r.status == ST_TERMINATOR) {
        s.n_chunks = n_all;
        s.n_total += r.n_total;
        s.end_byte = r.next_byte;
      } else if (r.status == ST_INDEX_FULL) {
        s.status = n_all > g.max_chunks ? PCO_B200_ASYNC_TOO_MANY_CHUNKS : PCO_B200_ASYNC_FILES_INDEX_FULL;
        s.n_chunks = n_all;
      } else {
        s.status = r.status;
        s.fail_chunk = n_all;
        s.n_chunks = n_all;
      }
    }
    s_ok = s.status == ST_OK;
  }
  __syncthreads();
  if (!s_ok) return;
  const uint64_t n = s.n_chunks;
  const IndexChunk* recs = reinterpret_cast<const IndexChunk*>(g.ws + l.recs);
  uint64_t* offs = reinterpret_cast<uint64_t*>(g.ws + l.offs);
  for (uint64_t c = threadIdx.x; c < n; c += AI_SCAN_THREADS) offs[c] = entries_bytes(recs[c].n_vars, recs[c].n);
  __syncthreads();
  uint64_t end[1] = {sizeof(IndexHeader) + n * sizeof(IndexChunk)};
  cta_scan_inplace<AI_SCAN_THREADS, AI_SCAN_PER_THREAD>(
      n, [&](uint64_t i, int) { return offs[i]; }, [&](uint64_t i, int, uint64_t x) { offs[i] = x; }, end);
  if (threadIdx.x != 0) return;
  if (end[0] > g.index_cap) s.status = PCO_B200_ASYNC_FILES_INDEX_FULL;
  else s.index_bytes = end[0];
}

// max_chunks + 1 CTAs, one per chunk: its entries (the walked bytes, then zeros up to the 16-byte boundary) and its record into the index.
__global__ void __launch_bounds__(AI_THREADS) ai_copy_kernel(AiArgs g, const AiState* __restrict__ state) {
  const AiState& s = *state;
  const uint64_t c = blockIdx.x;
  if (s.status != ST_OK || c >= s.n_chunks) return;
  const AiLayout l = ai_layout(g.src_cap, g.index_cap, g.max_chunks);
  IndexChunk r = reinterpret_cast<const IndexChunk*>(g.ws + l.recs)[c];
  const uint64_t at = reinterpret_cast<const uint64_t*>(g.ws + l.offs)[c];
  index_copy_chunk(r, reinterpret_cast<const uint32_t*>(g.ws + r.entries_offset), g.index, at, c);
}

// One thread: the index header (on success) and the status.
__global__ void ai_finish_kernel(AiArgs g, const AiState* __restrict__ state, PcoB200AsyncIndexStatus* __restrict__ out) {
  const AiState& s = *state;
  PcoB200AsyncIndexStatus r;
  r.kind = async_kind_of(s.status);
  r.device_status = s.status;
  r.chunk = s.fail_chunk;
  r.n_chunks = s.n_chunks;
  r.n_total = s.n_total;
  r.index_bytes = s.status == ST_OK ? s.index_bytes : 0;
  r.serial_chunks = s.serial_chunks;
  if (s.status == ST_OK) write_index_header(g.index, s.n_chunks, s.n_total, s.src_len, s.end_byte);
  *out = r;
}

}  // namespace pcob200
