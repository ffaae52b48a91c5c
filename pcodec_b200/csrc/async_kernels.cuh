// Kernels of pco_b200_decompress_async beyond the ordinary decode kernels: an indexed standalone file decoded with no host decision
// between launches, so the call can be queued behind other work or captured in a CUDA graph.  Every launch has a grid fixed by the
// plan's capacities; what the file holds (its length, chunk count, n_total) is read from the side index on the device.
//   async_check_kernel   re-checks the standalone header against the plan and the index header against the capacities, copies the
//                        chunk records into the workspace table and fills it up to max_chunks with pad records that the decode
//                        kernels refuse without reading the file (chunk_offset = src_cap); computes the binomial table decode_kernel reads;
//   cold_chunks_kernel   decodes, one after another, the chunks the fast kernels reported ST_UNSUPPORTED for, with the catch-all decoder;
//   async_finish_kernel  finds the lowest failing chunk and writes the PcoB200AsyncStatus the host reads when it chooses.
// Between check and cold run the ordinary kernels, always launched: fused_narrow_kernel, symwalk_kernel<false>, decode_kernel<L, 1 / 2>.
#pragma once
#include "../../include/pco_b200.h"
#include "decode_cold.cuh"

namespace pcob200 {

constexpr int ASYNC_THREADS = 256;
constexpr uint32_t ASYNC_CHECK_RECS = ASYNC_THREADS / 4;  // chunk records per CTA of async_check_kernel (4 words each)
constexpr uint32_t ASYNC_COLD_WINDOW_LOG = 16;            // Lookback windows beyond 2^16 numbers are Unsupported on this path

// what async_check_kernel found, at the start of the workspace
struct AsyncCheck {
  uint32_t status;     // ST_OK or a PCO_B200_ASYNC_* refusal
  uint32_t n_chunks;   // the index's chunk count (0 when refused)
  uint64_t n_total, end_byte;
  uint64_t reserved;
  Binoms binoms;
};

// everything the launches take by value; fp.src_len is src_cap
struct AsyncArgs {
  FileParams fp;
  const uint8_t* index;
  uint64_t index_cap;
  uint64_t dst_cap;
  uint32_t max_chunks;
};

// The regions every asynchronous decompress workspace ends with, from byte offset `at`: the statuses and class bytes of `slots` decode
// slots | the general pair's `rows` symbol and offset rows | `stage_bytes` of staging (none but the ranges call's) | the catch-all
// decoder's scratch.  Byte offsets, each region 256-byte aligned.
struct AsyncDecodeTail {
  uint64_t st, cls, syms, offs, stage, cold, total;
};
__host__ __device__ inline uint64_t async_align(uint64_t x) { return (x + 255) & ~uint64_t(255); }
__host__ __device__ inline AsyncDecodeTail async_decode_tail(uint64_t at, uint64_t slots, uint64_t rows, uint64_t stage_bytes) {
  AsyncDecodeTail t;
  t.st = at;
  t.cls = t.st + async_align(slots * sizeof(uint32_t));
  t.syms = t.cls + async_align(slots);
  t.offs = t.syms + async_align(rows * BATCH_N);
  t.stage = t.offs + async_align(rows * sizeof(uint32_t));
  t.cold = t.stage + async_align(stage_bytes);
  t.total = t.cold + async_align(cold_scratch_bytes(ASYNC_COLD_WINDOW_LOG));
  return t;
}

// Workspace of one in-flight call: AsyncCheck | IndexChunk[max_chunks] | the decode tail.
struct AsyncLayout : AsyncDecodeTail {
  uint64_t table;
};
__host__ __device__ inline AsyncLayout async_layout(uint64_t dst_cap, uint32_t max_chunks) {
  AsyncLayout l;
  l.table = async_align(sizeof(AsyncCheck));
  static_cast<AsyncDecodeTail&>(l) =
      async_decode_tail(l.table + async_align(uint64_t(max_chunks) * sizeof(IndexChunk)), max_chunks, scratch_rows_total(dst_cap, max_chunks), 0);
  return l;
}

// The PcoB200Error kind of a chunk status (as status_to_error, host_common.hpp, gives it) or of any PCO_B200_ASYNC_* code (as its comment
// in pco_b200.h states it).  Every asynchronous call's status goes through this one table; the codes of the calls are disjoint.
__host__ __device__ inline uint32_t async_kind_of(uint32_t st) {
  switch (st) {
    case ST_OK: return PCO_B200_OK;
    case ST_INSUFFICIENT_DATA: case PCO_B200_ASYNC_HEADER_SHORT: return PCO_B200_INSUFFICIENT_DATA;
    case ST_INVALID_ARGUMENT: case PCO_B200_ASYNC_HEADER_MISMATCH: case PCO_B200_ASYNC_INDEX_FOREIGN: case PCO_B200_ASYNC_TOO_MANY_CHUNKS:
    case PCO_B200_ASYNC_INDEX_TILING: case PCO_B200_ASYNC_INDEX_TOTAL: case PCO_B200_ASYNC_TOO_MANY_RANGES: case PCO_B200_ASYNC_RANGE_PAST:
    case PCO_B200_ASYNC_RANGE_OVERFLOW: case PCO_B200_ASYNC_DST_SHORT: case PCO_B200_ASYNC_TOO_MANY_FILES: case PCO_B200_ASYNC_FILE_OUTSIDE:
    case PCO_B200_ASYNC_INDEX_OFFSET: case PCO_B200_ASYNC_INDEX_OUTSIDE: case PCO_B200_ASYNC_ENTRIES_MISALIGNED: case PCO_B200_ASYNC_RECORDS_OUTSIDE:
    case PCO_B200_ASYNC_FILE_TOO_LARGE: case PCO_B200_ASYNC_NUMS_CAP: case PCO_B200_ASYNC_TOO_MANY_PAGES: case PCO_B200_ASYNC_META_OUTSIDE:
    case PCO_B200_ASYNC_PAGE_OUTSIDE: case PCO_B200_ASYNC_PAGE_N: case PCO_B200_ASYNC_PAGES_DST: return PCO_B200_INVALID_ARGUMENT;
    case PCO_B200_ASYNC_DST_FULL: case PCO_B200_ASYNC_WINDOW: case PCO_B200_ASYNC_FILES_DST: case PCO_B200_ASYNC_FILES_DST_FULL:
    case PCO_B200_ASYNC_FILES_INDEX_FULL: case PCO_B200_ASYNC_FRAMES: return PCO_B200_IO;
    case ST_UNSUPPORTED: case PCO_B200_ASYNC_NO_INDEX: return PCO_B200_UNSUPPORTED;
    default: return PCO_B200_CORRUPTION;
  }
}

__device__ __forceinline__ uint64_t async_ld_u64(const uint8_t* p) {  // any alignment
  if ((reinterpret_cast<uintptr_t>(p) & 7) == 0) return *reinterpret_cast<const uint64_t*>(p);
  uint64_t v = 0;
  for (int i = 7; i >= 0; i--) v = (v << 8) | p[i];
  return v;
}

// parse_standalone_header (host_common.hpp) on the device, over the first bytes of a file of `file_len` bytes: ST_OK, or the refusal
// that gives the kind the host parse gives.  On ST_OK, *first_chunk_byte (when given) is where the first chunk starts.
__device__ inline uint32_t async_parse_header(const uint8_t* b, uint64_t file_len, uint32_t* uniform_type, uint32_t* format_major,
                                              uint64_t* first_chunk_byte = nullptr) {
  auto byte_at = [&](uint64_t i) -> uint32_t { return i < file_len ? b[i] : 0u; };
  if (file_len < 4) return PCO_B200_ASYNC_HEADER_SHORT;
  if (b[0] != 112 || b[1] != 99 || b[2] != 111 || b[3] != 33) return PCO_B200_ASYNC_HEADER_CORRUPT;  // "pco!"
  uint64_t pos = 4;
  const uint32_t ver = byte_at(pos);
  uint32_t uniform = 0;
  if (ver >= 2) {
    pos += 1;
    if (ver >= 3) {
      const uint32_t t = byte_at(pos);
      pos += 1;
      if (t != 0) {
        if (!nt_valid(t)) return PCO_B200_ASYNC_HEADER_CORRUPT;
        uniform = t;
      }
    }
    // varint: 6 bits (power - 1), then `power` bits; only its length and padding matter here
    const uint32_t power = 1 + (byte_at(pos) & 63);
    const uint32_t total_bits = 6 + power;
    const uint32_t nbytes = (total_bits + 7) / 8;
    if (pos + nbytes > file_len) return PCO_B200_ASYNC_HEADER_SHORT;
    const uint32_t pad = nbytes * 8 - total_bits;
    if (pad && (byte_at(pos + nbytes - 1) >> (8 - pad)) != 0) return PCO_B200_ASYNC_HEADER_CORRUPT;
    pos += nbytes;
  }
  if (pos > file_len) return PCO_B200_ASYNC_HEADER_SHORT;
  if (ver > 3) return PCO_B200_ASYNC_HEADER_CORRUPT;
  const uint32_t major = byte_at(pos);
  pos += major >= 4 ? 2 : 1;
  if (major > 4) return PCO_B200_ASYNC_HEADER_CORRUPT;
  if (pos > file_len) return PCO_B200_ASYNC_HEADER_SHORT;
  *uniform_type = uniform;
  *format_major = major;
  if (first_chunk_byte) *first_chunk_byte = pos;
  return ST_OK;
}

// C(n, j) mod 2^64 by Pascal additions, n = 0 .. 256 (ensure_device builds the same table on the host), by one thread, into the Binoms
// lvalue B.  A macro rather than a function: expanded in async_check_kernel, it compiles to the instructions the loop written there gave.
#define PCOB_ASYNC_FILL_BINOMS(B)                                                    \
  do {                                                                               \
    uint64_t row[MAX_ORDER] = {1, 0, 0, 0, 0, 0, 0};                                 \
    for (int n = 0; n <= 256; n++) {                                                 \
      if (n > 0)                                                                     \
        for (int j = MAX_ORDER - 1; j >= 1; j--) row[j] += row[j - 1];               \
      if ((n & 7) == 0 && n < 256)                                                   \
        for (int j = 0; j < MAX_ORDER; j++) (B).lane8[n >> 3][j] = row[j];           \
      if (n == 256)                                                                  \
        for (int j = 0; j < MAX_ORDER; j++) (B).full[j] = row[j];                    \
    }                                                                                \
  } while (0)

// ceil(max_chunks / ASYNC_CHECK_RECS) CTAs.  Each CTA checks the headers (a few dozen bytes, from L2 after the first CTA) and writes its
// share of the table; CTA 0 also writes the AsyncCheck.  The check is decompress_ex's (host_api.cu, decompress_fast) with
// file_len <= src_cap in place of equality, plus n_chunks <= max_chunks.  A refused file leaves a table of pads only.
__global__ void __launch_bounds__(ASYNC_THREADS) async_check_kernel(AsyncArgs a, AsyncCheck* __restrict__ chk, IndexChunk* __restrict__ table) {
  __shared__ uint32_t s_n;
  __shared__ uint64_t s_coff;
  const int tid = threadIdx.x;
  if (tid == 0) {
    uint64_t h[8] = {0, 0, 0, 0, 0, 0, 0, 0};  // IndexHeader: magic | version, n_chunks, n_total, file_len, chunks_offset, end_byte
    const bool ih_fits = a.index_cap >= sizeof(IndexHeader);
    if (ih_fits)
      for (int i = 0; i < 6; i++) h[i] = async_ld_u64(a.index + 8 * i);
    const uint32_t magic = uint32_t(h[0]), version = uint32_t(h[0] >> 32);
    const uint64_t n_chunks = h[1], file_len = h[3], coff = h[4];
    const bool len_ok = ih_fits && magic == INDEX_MAGIC && version == 1 && file_len <= a.fp.src_len;
    uint32_t uniform = 0, major = 0;
    uint32_t st = async_parse_header(static_cast<const uint8_t*>(a.fp.src), len_ok ? file_len : a.fp.src_len, &uniform, &major);
    if (st == ST_OK && (uniform != a.fp.uniform_type || major != a.fp.format_major)) st = PCO_B200_ASYNC_HEADER_MISMATCH;
    if (st == ST_OK && (!len_ok || coff > a.index_cap || n_chunks > (a.index_cap - coff) / sizeof(IndexChunk))) st = PCO_B200_ASYNC_INDEX_FOREIGN;
    if (st == ST_OK && n_chunks > a.max_chunks) st = PCO_B200_ASYNC_TOO_MANY_CHUNKS;
    s_n = st == ST_OK ? uint32_t(n_chunks) : 0u;
    s_coff = coff;
    if (blockIdx.x == 0) {
      chk->status = st;
      chk->n_chunks = s_n;
      chk->n_total = h[2];
      chk->end_byte = h[5];
      chk->reserved = 0;
    }
  } else if (tid == 32 && blockIdx.x == 0) {
    PCOB_ASYNC_FILL_BINOMS(chk->binoms);
  }
  __syncthreads();
  const uint64_t w = uint64_t(blockIdx.x) * ASYNC_THREADS + tid;  // word w of the table: record w / 4, field word w % 4
  const uint64_t k = w >> 2;
  if (k >= a.max_chunks) return;
  uint64_t v;
  if (k < s_n) v = async_ld_u64(a.index + s_coff + 8 * w);
  else v = (w & 3) == 0 ? a.fp.src_len : 0;  // pad: chunk_offset = src_cap, everything else 0
  reinterpret_cast<uint64_t*>(table)[w] = v;
}

// One CTA.  Its threads list the chunks in [0, n_chunks) whose status is ST_UNSUPPORTED, ASYNC_THREADS at a time; thread 0 decodes each
// with the catch-all decoder from its chunk_offset straight into dst + out_offset, bounded by its n and the destination.  The decoder
// stops behind the chunk (or inside it, when the destination ends there): the chunk is decoded once the decoder has counted it.
template <typename L>
__global__ void __launch_bounds__(ASYNC_THREADS) cold_chunks_kernel(FileParams fp, const IndexChunk* __restrict__ table, const AsyncCheck* __restrict__ chk,
                                                                    uint32_t* __restrict__ statuses, L* __restrict__ out, uint64_t out_len,
                                                                    uint8_t* __restrict__ scratch) {
  __shared__ uint32_t s_list[ASYNC_THREADS];
  __shared__ uint32_t s_count;
  const int tid = threadIdx.x;
  const uint32_t n_chunks = chk->n_chunks;
  for (uint32_t base = 0; base < n_chunks; base += ASYNC_THREADS) {
    if (tid == 0) s_count = 0;
    __syncthreads();
    const uint32_t k = base + tid;
    if (k < n_chunks && statuses[k] == ST_UNSUPPORTED) s_list[atomicAdd(&s_count, 1u)] = k;
    __syncthreads();
    if (tid == 0) {
      for (uint32_t i = 0; i < s_count; i++) {
        const uint32_t c = s_list[i];
        const IndexChunk rec = table[c];
        uint32_t st = ST_OK;  // a chunk that starts behind the destination is not decoded (as the whole-file catch-all stops before it)
        if (rec.out_offset < out_len) {
          ColdResult res;
          cold_decode_run<L>(fp, rec.chunk_offset, out + rec.out_offset, min(uint64_t(rec.n), out_len - rec.out_offset), scratch, ASYNC_COLD_WINDOW_LOG, &res);
          st = cold_status(res);
        }
        statuses[c] = st;
      }
    }
    __syncthreads();
  }
}

// One CTA: the lowest failing chunk in [0, n_chunks), or the file-level refusal, or the Progress decompress_ex reports.
__global__ void __launch_bounds__(1024) async_finish_kernel(uint64_t dst_cap, const AsyncCheck* __restrict__ chk, const uint32_t* __restrict__ statuses,
                                                            PcoB200AsyncStatus* __restrict__ out) {
  __shared__ uint32_t s_min;
  const uint32_t tid = threadIdx.x;
  if (tid == 0) s_min = 0xffffffffu;
  __syncthreads();
  const uint32_t check = chk->status, n_chunks = chk->n_chunks;
  if (check == ST_OK)
    for (uint32_t k = tid; k < n_chunks; k += blockDim.x)
      if (statuses[k] != ST_OK) {
        atomicMin(&s_min, k);  // a thread's first failure is its lowest
        break;
      }
  __syncthreads();
  if (tid != 0) return;
  PcoB200AsyncStatus r;
  r.kind = PCO_B200_OK;
  r.device_status = ST_OK;
  r.chunk = 0;
  r.n_processed = 0;
  r.finished = 0;
  r.n_chunks = n_chunks;
  if (check != ST_OK) {
    r.kind = async_kind_of(check);
    r.device_status = check;
    r.chunk = ~uint64_t(0);
  } else if (s_min != 0xffffffffu) {
    const uint32_t st = statuses[s_min];
    r.kind = async_kind_of(st);
    r.device_status = st;
    r.chunk = s_min;
  } else {
    const uint64_t n_total = chk->n_total;
    r.n_processed = min(n_total, dst_cap);
    r.finished = (chk->end_byte != 0 && n_total <= dst_cap) ? 1u : 0u;
  }
  *out = r;
}

}  // namespace pcob200
