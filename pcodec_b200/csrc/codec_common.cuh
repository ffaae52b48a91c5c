// Shared device-side definitions for the pco hot-path kernels (sm_90a).
//
// Format facts cited here are from the reference: docs/format.md and
// pco/src/metadata/*.rs (paths relative to /root/reference).  Nothing in this
// directory includes or links oracle/.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pcob200 {

constexpr int BATCH_N = 256;          // pco/src/constants.rs:62 FULL_BATCH_N
constexpr int ANS_INTERLEAVING = 4;   // pco/src/constants.rs:58
constexpr int MAX_ANS_BITS = 14;      // pco/src/constants.rs:32
constexpr int MAX_VARS = 2;           // primary + secondary (the lookback delta var is outside the GPU path)
constexpr int MAX_ORDER = 7;          // pco/src/constants.rs:36

// Per-chunk status written by the kernels (mirrors pco::errors::ErrorKind, pco/src/errors.rs:8-24)
enum : uint32_t {
  ST_OK = 0,
  ST_CORRUPTION = 1,
  ST_INSUFFICIENT_DATA = 2,
  ST_INVALID_ARGUMENT = 3,
  ST_UNSUPPORTED = 7,
  ST_TERMINATOR = 100,  // walker only: hit the 0x00 end-of-file byte
  ST_INDEX_FULL = 101,  // walker only: ran out of IndexChunk / BatchEntry space
  ST_DST_FULL = 102,    // walker only: indexed chunks already cover more numbers than the destination holds
};

enum : uint32_t { MODE_CLASSIC = 0, MODE_INT_MULT = 1, MODE_FLOAT_MULT = 2, MODE_FLOAT_QUANT = 3, MODE_DICT = 4 };
enum : uint32_t { DELTA_NONE = 0, DELTA_CONSECUTIVE = 1, DELTA_LOOKBACK = 2, DELTA_CONV1 = 3 };

// number type bytes (pco_c/include/cpcodec.h:10-20)
enum : uint32_t { NT_U32 = 1, NT_U64 = 2, NT_I32 = 3, NT_I64 = 4, NT_F32 = 5, NT_F64 = 6, NT_U16 = 7, NT_I16 = 8, NT_F16 = 9, NT_U8 = 10, NT_I8 = 11 };
__host__ __device__ inline bool nt_valid(uint32_t t) { return t >= 1 && t <= 11; }
__host__ __device__ inline uint32_t nt_bits(uint32_t t) {
  return (t == NT_U8 || t == NT_I8) ? 8 : (t == NT_U16 || t == NT_I16 || t == NT_F16) ? 16 : (t == NT_U32 || t == NT_I32 || t == NT_F32) ? 32 : 64;
}
__host__ __device__ inline bool nt_is_float(uint32_t t) { return t == NT_F16 || t == NT_F32 || t == NT_F64; }
__host__ __device__ inline bool nt_is_signed(uint32_t t) { return t == NT_I8 || t == NT_I16 || t == NT_I32 || t == NT_I64; }

// ---------------------------------------------------------------------------
// Side index (metadata beside the .pco bytes; see include/pco_b200.h)
// ---------------------------------------------------------------------------
constexpr uint32_t INDEX_MAGIC = 0x58444950u;  // "PIDX"
struct IndexHeader {
  uint32_t magic, version;
  uint64_t n_chunks, n_total, file_len;
  uint64_t chunks_offset;  // byte offset of IndexChunk[n_chunks] from the index start
  uint64_t end_byte;       // byte offset just past the terminator of the standalone file (0 if none seen)
  uint64_t reserved[2];
};
struct IndexChunk {
  uint64_t chunk_offset;   // byte offset of the chunk's type byte in the standalone file
  uint32_t n;              // numbers in the chunk
  uint32_t n_vars;         // latent vars with entries (file order)
  uint64_t entries_offset; // byte offset of this chunk's BatchEntry array from the index start
  uint64_t out_offset;     // element offset of the chunk's first number in the output
};
struct BatchEntry {
  uint32_t bit_pos;        // bit offset, from the chunk's type byte, of this (batch, var)'s ANS section
  uint16_t st[4];          // tANS state indices at the start of the batch
};
static_assert(sizeof(IndexHeader) == 64 && sizeof(IndexChunk) == 32 && sizeof(BatchEntry) == 12, "index layout");

// A side index header made for a file of `file_len` bytes, whose chunk table lies inside the index's `index_len` bytes (overflow-safe;
// the per-chunk fields are bounded on the device: entries inside the index, chunk_offset inside the file, writes inside the destination).
__host__ __device__ inline bool index_header_ok(const IndexHeader& ih, uint64_t file_len, uint64_t index_len) {
  return ih.magic == INDEX_MAGIC && ih.version == 1 && ih.file_len == file_len && ih.chunks_offset <= index_len &&
         ih.n_chunks <= (index_len - ih.chunks_offset) / sizeof(IndexChunk);
}

__host__ __device__ inline uint32_t n_batches_of(uint32_t n) { return (n + BATCH_N - 1) / BATCH_N; }
// latent slots of a chunk of `size` numbers in the encoder's per-number arrays: whole batches
__host__ __device__ inline uint64_t rows_of(uint64_t size) { return (size + BATCH_N - 1) / BATCH_N * BATCH_N; }
// A chunk's region of batch entries in a side index: n_vars x batches records of a chunk of n numbers, rounded up to 16 bytes.
__host__ __device__ inline uint64_t entries_bytes(uint32_t n_vars, uint64_t n) {
  return (uint64_t(n_vars) * n_batches_of(uint32_t(n)) * sizeof(BatchEntry) + 15) & ~uint64_t(15);
}

// PagingSpec::EqualPagesUpTo(max_page_n) over n numbers (pco/src/chunk_config.rs:134-183): n_chunks chunks, the first `rem` of
// low + 1 numbers, the others of low.  max_page_n 0 is the default, 2^18.
__host__ __device__ inline uint64_t page_cap(uint64_t max_page_n) { return max_page_n == 0 ? (uint64_t(1) << 18) : max_page_n; }
struct EqualPages {
  uint64_t n_chunks, low, rem;
  __host__ __device__ uint64_t start(uint64_t c) const { return c * low + (c < rem ? c : rem); }
  __host__ __device__ uint64_t size(uint64_t c) const { return low + (c < rem ? 1 : 0); }
  __host__ __device__ uint64_t row_start(uint64_t c) const {
    const uint64_t q = c < rem ? c : rem;
    return q * rows_of(low + 1) + (c - q) * rows_of(low);
  }
  // the side index compress_typed writes for these chunks: header, chunk records, then each chunk's entries of n_vars vars
  __host__ __device__ uint64_t entries_offset(uint32_t n_vars, uint64_t c) const {
    const uint64_t q = c < rem ? c : rem;
    return ((sizeof(IndexHeader) + n_chunks * sizeof(IndexChunk) + 15) & ~uint64_t(15)) + q * entries_bytes(n_vars, low + 1) +
           (c - q) * entries_bytes(n_vars, low);
  }
  __host__ __device__ uint64_t index_bytes(uint32_t n_vars) const { return entries_offset(n_vars, n_chunks); }
};
__host__ __device__ inline EqualPages equal_pages(uint64_t n, uint64_t max_page_n) {
  EqualPages p = {0, 0, 0};
  if (n == 0) return p;
  const uint64_t mp = page_cap(max_page_n);
  p.n_chunks = (n + mp - 1) / mp;
  p.low = n / p.n_chunks;
  p.rem = n % p.n_chunks;
  return p;
}

// The chain of real chunks among the candidates of a speculative walk of one index-free file: the host's rounds (follow_chunk_chain,
// host_common.hpp) and the device's (ai_chain_kernel, async_index_kernels.cuh).  `cand` (sorted, m entries) are the positions that look
// like a chunk start of `n0` numbers, `st` / `ends` what walking each of them as a chunk gave (status, first byte behind it).  Starting
// from `pos` - a real chunk start - the chunk at p is real, and the next real chunk starts where it ends: follow that for as long as the
// end is on the list, the walk succeeded, made progress and stayed inside the file (which ends at `src_len`), and the cap (`dst_len`
// units, `out_off` of them taken, `n0` per chunk) has room for another chunk.  take(k) gets the index (into cand) of each verified chunk
// in file order; returns their count and leaves the position behind the last one in *next_pos.  A candidate that no verified chunk ends
// on is a coincidence and is never reached.
#pragma nv_exec_check_disable
template <typename Take>
__host__ __device__ inline uint64_t chunk_chain(const uint64_t* cand, const uint32_t* st, const uint64_t* ends, uint32_t m, uint64_t pos, uint64_t n0,
                                                uint64_t out_off, uint64_t dst_len, uint64_t src_len, uint64_t* next_pos, Take take) {
  uint64_t p = pos, taken = 0;
  uint32_t lo = 0;  // the chain only moves forward: the lower bound of p is searched behind the last chunk taken, galloping
  for (;;) {
    uint32_t hi = lo, step = 1;
    while (hi < m && cand[hi] < p) {
      lo = hi + 1;
      hi = m - lo > step ? lo + step : m;
      step <<= 1;
    }
    while (lo < hi) {
      const uint32_t mid = lo + (hi - lo) / 2;
      if (cand[mid] < p) lo = mid + 1; else hi = mid;
    }
    if (lo == m || cand[lo] != p) break;
    if (st[lo] != ST_OK || ends[lo] <= p || ends[lo] > src_len) break;  // the serial walker reports what is wrong with this chunk
    if (out_off + (taken + 1) * n0 > dst_len) break;
    take(lo);
    taken++;
    p = ends[lo];
    lo++;
  }
  *next_pos = p;
  return taken;
}

// unoptimized_bins_log of var v of a chunk of n >= 1 numbers at compression level `level` (pco/src/wrapped/chunk_compressor.rs:362-371;
// the secondary var takes at most 6, LIMITED_UNOPTIMIZED_BINS_LOG, :238-248).
__host__ __device__ __forceinline__ uint32_t unoptimized_bins_log(uint32_t level, uint64_t n, int v) {
#ifdef __CUDA_ARCH__
  const uint32_t log_n = 63u - uint32_t(__clzll((long long)n));
#else
  const uint32_t log_n = 63u - uint32_t(__builtin_clzll(n));
#endif
  const uint32_t fast = log_n >= 4 ? log_n - 4 : 0;
  const uint32_t b = level <= fast ? level : fast + (level - fast) / 2;
  return v == 0 ? b : (b < 6u ? b : 6u);
}

// ---------------------------------------------------------------------------
// Bit stream view: a byte range addressed through 8-byte aligned words.
// ---------------------------------------------------------------------------
struct BitSrc {
  const uint64_t* words;  // 16-byte aligned base at or below the first byte (kernels also read it as 16-byte blocks)
  uint64_t n_bits;        // valid bits from `words` (i.e. (misalign + len) * 8)
  uint32_t mis_bits;      // bits between `words` and the first byte of the buffer
};

__host__ __device__ inline BitSrc make_bitsrc(const void* p, size_t len) {
  uintptr_t a = (uintptr_t)p;
  BitSrc s;
  s.words = (const uint64_t*)(a & ~uintptr_t(15));
  s.mis_bits = uint32_t(a & 15) * 8;
  s.n_bits = uint64_t(s.mis_bits) + uint64_t(len) * 8;
  return s;
}

// Zero-extended 64-bit window at absolute bit position `pos`: bytes past the end read as 0,
// like the reference's padded eof buffer (pco/src/bit_reader.rs:271-300).
__device__ inline uint64_t window64_safe(const BitSrc& s, uint64_t pos) {
  uint64_t w = pos >> 6;
  uint32_t r = uint32_t(pos & 63);
  uint64_t last = s.n_bits == 0 ? 0 : (s.n_bits - 1) >> 6;
  auto ld = [&](uint64_t i) -> uint64_t {
    if (s.n_bits == 0 || i > last) return 0;
    uint64_t v = s.words[i];
    if (i == last) {
      uint32_t valid = uint32_t(s.n_bits - (i << 6));  // 1..64
      if (valid < 64) v &= (uint64_t(1) << valid) - 1;
    }
    return v;
  };
  uint64_t lo = ld(w);
  if (r == 0) return lo;
  return (lo >> r) | (ld(w + 1) << (64 - r));
}
__device__ inline uint64_t read_bits_safe(const BitSrc& s, uint64_t pos, uint32_t n) {
  if (n == 0) return 0;
  uint64_t v = window64_safe(s, pos);
  return n >= 64 ? v : (v & ((uint64_t(1) << n) - 1));
}

// ---------------------------------------------------------------------------
// Parsed chunk header (built in shared memory by one CTA per chunk)
// ---------------------------------------------------------------------------
struct VarHdr {
  uint32_t ans_size_log;
  uint32_t n_bins;
  uint32_t latent_bits;
  uint32_t delta_order;     // consecutive order applied to this var (0 = none)
  uint64_t bins_bit;        // absolute bit position of bin 0
  uint32_t bin_stride;      // bits per bin: size_log + latent_bits + log2(latent_bits)+1
  uint32_t max_offset_bits; // filled while loading bins
};

struct ChunkHdr {
  uint32_t status;
  uint32_t n;               // numbers in this chunk (== page n in standalone)
  uint32_t mode;
  uint32_t mode_k;          // FloatQuant
  uint64_t mode_base;       // IntMult base / FloatMult base as ordered latent
  uint32_t delta_kind;
  uint32_t delta_order;
  uint32_t n_vars;
  uint32_t number_bits;
  VarHdr var[MAX_VARS];
  uint64_t page_bit;        // absolute bit position of the page (page meta start)
  uint64_t body_bit;        // absolute bit position of the first batch
  uint64_t moments[MAX_VARS][MAX_ORDER];
  uint32_t init_state[MAX_VARS][ANS_INTERLEAVING];
};

__host__ __device__ inline uint32_t offset_bits_bits(uint32_t latent_bits) {  // pco/src/bits.rs:24-26
  return latent_bits == 8 ? 4 : latent_bits == 16 ? 5 : latent_bits == 32 ? 6 : 7;
}

// Sequential parse of a chunk's fixed header fields by ONE thread.
//   standalone: [8b type][24b n-1] then wrapped chunk meta (pco/src/standalone/decompressor.rs:190-231)
//   wrapped chunk meta: docs/format.md:84-143, pco/src/metadata/{chunk,mode,delta_encoding,chunk_latent_var}.rs
// `pos` is the absolute bit position of the chunk's type byte (standalone) or of the chunk meta (wrapped,
// has_preamble = false, in which case h.n must be preset).  Returns the bit position after the chunk meta.
__device__ inline uint64_t parse_chunk_header(const BitSrc& s, uint64_t pos, uint32_t expected_type, uint32_t uniform_type,
                                              uint32_t format_major, bool has_preamble, ChunkHdr& h) {
  h.status = ST_OK;
  uint32_t number_bits = nt_bits(expected_type);
  h.number_bits = number_bits;
  if (has_preamble) {
    if (pos + 8 > s.n_bits) { h.status = ST_INSUFFICIENT_DATA; return pos; }
    uint32_t type_byte = uint32_t(read_bits_safe(s, pos, 8));
    pos += 8;
    if (type_byte == 0) { h.status = ST_TERMINATOR; return pos; }
    if (uniform_type != 0 && uniform_type != type_byte) { h.status = ST_CORRUPTION; return pos; }
    if (type_byte != expected_type) { h.status = ST_CORRUPTION; return pos; }
    h.n = uint32_t(read_bits_safe(s, pos, 24)) + 1;
    pos += 24;
    if (pos > s.n_bits) { h.status = ST_INSUFFICIENT_DATA; return pos; }
  }
  // ---- mode (metadata/mode.rs:102-167)
  h.mode = uint32_t(read_bits_safe(s, pos, 4));
  pos += 4;
  h.mode_base = 0;
  h.mode_k = 0;
  bool is_float = nt_is_float(expected_type);
  switch (h.mode) {
    case MODE_CLASSIC: break;
    case MODE_INT_MULT:
      if (format_major == 0) { h.status = ST_CORRUPTION; return pos; }
      h.mode_base = read_bits_safe(s, pos, number_bits);
      pos += number_bits;
      break;
    case MODE_FLOAT_MULT:
      h.mode_base = read_bits_safe(s, pos, number_bits);
      pos += number_bits;
      break;
    case MODE_FLOAT_QUANT:
      h.mode_k = uint32_t(read_bits_safe(s, pos, 8));
      pos += 8;
      break;
    case MODE_DICT:
      if (pos > s.n_bits) { h.status = ST_INSUFFICIENT_DATA; return pos; }
      h.status = ST_UNSUPPORTED;
      return pos;
    default:
      h.status = pos > s.n_bits ? ST_INSUFFICIENT_DATA : ST_CORRUPTION;
      return pos;
  }
  if (pos > s.n_bits) { h.status = ST_INSUFFICIENT_DATA; return pos; }
  // ---- delta encoding (metadata/delta_encoding.rs:118-202)
  h.delta_kind = DELTA_NONE;
  h.delta_order = 0;
  bool secondary_uses_delta = false;
  if (format_major < 3) {
    uint32_t order = uint32_t(read_bits_safe(s, pos, 3));
    pos += 3;
    if (order != 0) { h.delta_kind = DELTA_CONSECUTIVE; h.delta_order = order; }
  } else {
    uint32_t variant = uint32_t(read_bits_safe(s, pos, 4));
    pos += 4;
    if (variant == 1) {
      uint32_t order = uint32_t(read_bits_safe(s, pos, 3));
      pos += 3;
      if (order == 0) { h.status = ST_CORRUPTION; return pos; }
      h.delta_kind = DELTA_CONSECUTIVE;
      h.delta_order = order;
      secondary_uses_delta = read_bits_safe(s, pos, 1) != 0;
      pos += 1;
    } else if (variant == 2 || variant == 3) {
      h.status = ST_UNSUPPORTED;  // Lookback / Conv1: valid pco, outside the GPU hot path
      return pos;
    } else if (variant != 0) {
      h.status = ST_CORRUPTION;
      return pos;
    }
  }
  if (pos > s.n_bits) { h.status = ST_INSUFFICIENT_DATA; return pos; }
  // ---- mode validity for the number type (data_types/unsigned.rs:80-86, float.rs:372-384)
  {
    bool ok = true;
    if (is_float) {
      if (h.mode == MODE_INT_MULT) ok = false;
      if (h.mode == MODE_FLOAT_QUANT) {
        uint32_t precision = number_bits == 64 ? 52 : number_bits == 32 ? 23 : 10;
        ok = h.mode_k > 0 && h.mode_k <= precision;
      }
      if (h.mode == MODE_FLOAT_MULT) {
        // base = from_latent_ordered(mode_base) must be finite and nonzero
        uint64_t mid = uint64_t(1) << (number_bits - 1);
        uint64_t l = h.mode_base;
        uint64_t bits = (l & mid) ? (l ^ mid) : (~l & (number_bits == 64 ? ~uint64_t(0) : ((uint64_t(1) << number_bits) - 1)));
        uint32_t mant = number_bits == 64 ? 52 : number_bits == 32 ? 23 : 10;
        uint64_t abs_bits = bits & (mid - 1);
        uint64_t exp_mask = ((uint64_t(1) << (number_bits - 1 - mant)) - 1) << mant;
        ok = (abs_bits & exp_mask) != exp_mask && abs_bits != 0;
      }
    } else {
      if (h.mode == MODE_FLOAT_MULT || h.mode == MODE_FLOAT_QUANT) ok = false;
      if (h.mode == MODE_INT_MULT) ok = h.mode_base > 0;
    }
    if (!ok) { h.status = ST_CORRUPTION; return pos; }
  }
  // ---- latent vars (metadata/chunk_latent_var.rs:102-143)
  h.n_vars = (h.mode == MODE_CLASSIC) ? 1 : 2;
  for (uint32_t v = 0; v < h.n_vars; v++) {
    VarHdr& vh = h.var[v];
    vh.latent_bits = number_bits;
    vh.delta_order = (v == 0 || secondary_uses_delta) ? h.delta_order : 0;
    vh.ans_size_log = uint32_t(read_bits_safe(s, pos, 4));
    vh.n_bins = uint32_t(read_bits_safe(s, pos + 4, 15));
    pos += 19;
    if (pos > s.n_bits) { h.status = ST_INSUFFICIENT_DATA; return pos; }
    if ((1u << vh.ans_size_log) < vh.n_bins) { h.status = ST_CORRUPTION; return pos; }
    if (vh.n_bins == 1 && vh.ans_size_log > 0) { h.status = ST_CORRUPTION; return pos; }
    if (vh.ans_size_log > MAX_ANS_BITS) { h.status = ST_CORRUPTION; return pos; }
    vh.bins_bit = pos;
    vh.bin_stride = vh.ans_size_log + number_bits + offset_bits_bits(number_bits);
    vh.max_offset_bits = 0;
    pos += uint64_t(vh.n_bins) * vh.bin_stride;
    if (pos > s.n_bits) { h.status = ST_INSUFFICIENT_DATA; return pos; }
  }
  // byte-align; the padding must be zero (metadata/chunk.rs:166-168)
  uint32_t pad = uint32_t((8 - (pos & 7)) & 7);
  if (pad && read_bits_safe(s, pos, pad) != 0) { h.status = ST_CORRUPTION; return pos; }
  pos += pad;
  // ---- page meta (metadata/page.rs:36-57, page_latent_var.rs:28-49)
  h.page_bit = pos;
  for (uint32_t v = 0; v < h.n_vars; v++) {
    const VarHdr& vh = h.var[v];
    for (uint32_t k = 0; k < vh.delta_order; k++) {
      h.moments[v][k] = read_bits_safe(s, pos, vh.latent_bits);
      pos += vh.latent_bits;
    }
    for (int j = 0; j < ANS_INTERLEAVING; j++) {
      h.init_state[v][j] = uint32_t(read_bits_safe(s, pos, vh.ans_size_log));
      pos += vh.ans_size_log;
    }
  }
  if (pos > s.n_bits) { h.status = ST_INSUFFICIENT_DATA; return pos; }
  pad = uint32_t((8 - (pos & 7)) & 7);
  if (pad && read_bits_safe(s, pos, pad) != 0) { h.status = ST_CORRUPTION; return pos; }
  pos += pad;
  h.body_bit = pos;
  return pos;
}

// Stored latents of var v in a page of n numbers, and in batch b (docs/format.md:149-171;
// pco/src/wrapped/chunk_compressor.rs:185-191: a delta'd var stores n - order latents).
__host__ __device__ inline uint32_t var_stored_n(uint32_t n, uint32_t delta_order) { return n > delta_order ? n - delta_order : 0; }
__host__ __device__ inline uint32_t batch_count(uint32_t stored_n, uint32_t b) {
  uint32_t start = b * BATCH_N;
  return stored_n > start ? (stored_n - start < BATCH_N ? stored_n - start : BATCH_N) : 0;
}

}  // namespace pcob200
