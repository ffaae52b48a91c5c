// Encode-side kernels for the pco hot path on sm_90a (one launch handles many independent chunks):
//   split_delta_kernel  — K1+K2: mode split and consecutive delta encode, page moments, per-chunk min/max
//   sort_keys_kernel    — range-reduced copy of the stored latents (input of the planner's segmented sort)
//   plan_kernel         — bin training: equal-count histogram, bin-merge DP, tANS weight quantisation, tables
//   fallback_kernel     — size-guarantee check (Classic/NoOp/one wide bin fallback)
//   bin_kernel          — K3: branchless bin search -> symbol per latent, per-batch offset-bit sums
//   ans_encode_kernel   — K4: reverse 4-way interleaved tANS over the page, per-batch states (side index)
//   layout_kernel       — per-chunk scan of batch bit sizes -> bit offsets, chunk byte size
//   pack_kernel         — K5: header/meta/page-meta emission and the variable-width bit-pack of every batch
//
// Reference behaviour restated here (paths relative to /root/reference):
//   split                    pco/src/mode/classic.rs:6-12, float_mult.rs:38-60, int_mult.rs:20-36, float_quant.rs:41-73
//   delta encode             pco/src/delta/consecutive.rs:3-33, pco/src/wrapped/chunk_compressor.rs:142-217
//   histogram                pco/src/histograms.rs:87-298 (pivot-independent restatement on sorted data, see DESIGN.md)
//   bin optimisation         pco/src/bin_optimization.rs:19-198
//   weight quantisation      pco/src/ans/encoding.rs:95-175, pco/src/wrapped/chunk_compressor.rs:38-99
//   fallback                 pco/src/wrapped/chunk_compressor.rs:396-440,502-541
//   bin search / dissect     pco/src/compression_table.rs:51-74, pco/src/chunk_latent_compressor.rs:163-233
//   tANS encode              pco/src/ans/encoding.rs:28-92, pco/src/chunk_latent_compressor.rs:96-132
//   page / meta emission     pco/src/chunk_latent_compressor.rs:272-329, pco/src/metadata/{chunk,chunk_latent_var,page}.rs
#pragma once
#include <type_traits>

#include "decode_kernels.cuh"

namespace pcob200 {

#ifdef PCOB_ENC_TIMING
// experiment builds only: per-phase clock64 sums of CTA-level phases (thread 0 of every CTA), read by pco_b200_debug_enc_timing
__device__ unsigned long long g_enc_timing[32];
#define ENC_TICK_INIT() long long enc_t0_ = clock64()
#define ENC_TICK(idx) do { if (threadIdx.x == 0) { long long t_ = clock64(); atomicAdd(&g_enc_timing[idx], (unsigned long long)(t_ - enc_t0_)); enc_t0_ = t_; } } while (0)
#else
#define ENC_TICK_INIT() do { } while (0)
#define ENC_TICK(idx) do { } while (0)
#endif
constexpr int ENC_MAXB = 256;        // bins per latent var (compression level <= 8)
constexpr int ENC_MAX_SIZE_LOG = 10;

// Capacity of one latent var's plan.  Runs whose unoptimized_bins_log is at most 8 (every chunk at levels <= 8) use the narrow
// instantiation of every kernel below; a run with more unoptimized bins (levels 9-12: up to 4096 bins, estimated_ans_size_log <= 12,
// chunk_compressor.rs:63-79) uses the wide one: per-bin arrays of 4096, tables of 2^12 states, 16-bit symbols.
template <bool WIDE>
struct EncCap {
  static constexpr int MAXB = WIDE ? 4096 : ENC_MAXB;
  static constexpr int MAX_SIZE_LOG = WIDE ? 12 : ENC_MAX_SIZE_LOG;
  using Sym = typename std::conditional<WIDE, uint16_t, uint8_t>::type;  // bin index of a latent
};
constexpr uint32_t ENC_NARROW_BINS_LOG = 8;  // largest unoptimized_bins_log of the narrow instantiation

struct EncParams {
  const void* nums;
  uint64_t n_total;
  const uint64_t* chunk_starts;  // device, n_chunks + 1 element offsets
  const uint64_t* row_base;      // device, n_chunks + 1: first slot of each chunk in the latent / symbol / ans arrays
  uint32_t n_chunks;
  uint32_t max_chunk_n;
  uint32_t dtype;
  uint32_t mode;           // MODE_*
  uint64_t mode_base;      // IntMult base, or FloatMult base as ordered latent
  uint64_t base_bits;      // FloatMult: bits of base (as the number type)
  uint64_t inv_base_bits;  // FloatMult: bits of 1/base
  uint32_t mode_k;
  uint32_t order;          // consecutive delta order on the primary (0 = none)
  uint32_t n_vars;
  uint32_t bins_log[MAX_VARS];  // unoptimized_bins_log per var
  uint32_t uniform_type;   // header flavour
};

// The CHUNK_BINS instantiations of the planner kernels take the level in ep.bins_log[0] and compute each chunk's value with
// unoptimized_bins_log (codec_common.cuh), so one launch serves chunks whose sizes imply different values.

template <bool WIDE>
struct VarPlanT {
  static constexpr int MAXB = EncCap<WIDE>::MAXB;
  uint32_t n_bins, size_log, max_ob, n_lat;
  uint64_t wc_bits;            // sum over bins of count * worst-case bits per latent
  uint64_t est_bits;           // sum over bins of count * (offset bits + tANS bits at the bin's weight): size estimate for the Auto delta search
  uint64_t lower[MAXB];
  uint8_t ob[MAXB];
  uint16_t weight[MAXB];
  uint64_t syminfo[MAXB];  // cutoff (bits 0-15) | min_renorm_bits (16-23) | weight (24-39) | cum (40-55)
  uint16_t next_states[1 << EncCap<WIDE>::MAX_SIZE_LOG];
};
using VarPlan = VarPlanT<false>;
static_assert(sizeof(VarPlanT<false>) % 16 == 0 && sizeof(VarPlanT<true>) % 16 == 0, "plans are copied as 16-byte vectors");

struct ChunkEnc {              // per chunk, device
  uint64_t moments[MAX_VARS][MAX_ORDER];
  uint64_t vmin[MAX_VARS], vmax[MAX_VARS];
  uint64_t key_base[MAX_VARS];  // what the 16-bit keys of the counting path are relative to (mod 2^16): vmin, or the fused kernel's anchor
  uint32_t final_state[MAX_VARS][4];
  uint32_t fallback;           // 1 = Classic / NoOp / one bin of L::BITS offset bits
  uint32_t status;
  uint32_t meta_bytes, page_meta_bytes;
  uint64_t body_bits;
  uint64_t chunk_bytes;        // preamble + meta + page
  uint64_t out_offset;         // byte offset of the chunk in the output file
};

// ---------------------------------------------------------------------------
// f32 helpers with explicit rounding (never contracted to FMA)
// ---------------------------------------------------------------------------
__device__ __forceinline__ float log2_approx_dev(float x) {  // pco/src/bin_optimization.rs:19-43
  const float Z = 0.674f;
  const uint32_t SIGNIF_MASK = 0x7FFFFFu;
  const uint32_t Z_SIGNIF = __float_as_uint(Z) & SIGNIF_MASK;
  const float B = __fdiv_rn(2.0f, Z);
  const float Cc = __fdiv_rn(-B, __fmul_rn(6.0f, Z));
  const float A = __fsub_rn(-B, Cc);
  uint32_t bits = __float_as_uint(x);
  uint32_t exp = bits >> 23;
  uint32_t signif = bits & SIGNIF_MASK;
  uint32_t high_bit = signif > Z_SIGNIF ? 1u : 0u;
  uint32_t log_int = exp + high_bit - 127u;
  float normalized = __uint_as_float(((0x7Fu ^ high_bit) << 23) | signif);
  float t0 = __fadd_rn(__uint2float_rn(log_int), A);
  float t2 = __fadd_rn(B, __fmul_rn(Cc, normalized));
  return __fadd_rn(t0, __fmul_rn(normalized, t2));
}
__device__ __forceinline__ uint32_t bits_to_encode_u64(uint64_t x) { return x == 0 ? 0u : 64u - uint32_t(__clzll((long long)x)); }
__device__ __forceinline__ float bin_cost_dev(float bin_meta_cost, uint64_t range, uint32_t count, float total_log2) {  // bin_optimization.rs:46-57
  float cf = __uint2float_rn(count);
  float ans_cost = __fsub_rn(total_log2, log2_approx_dev(cf));
  float offset_cost = __uint2float_rn(bits_to_encode_u64(range));
  return __fadd_rn(bin_meta_cost, __fmul_rn(__fadd_rn(ans_cost, offset_cost), cf));
}

// ---------------------------------------------------------------------------
// K1 + K2: split into latents, delta encode the primary, moments, min/max of the stored latents
// ---------------------------------------------------------------------------
template <typename L>
__device__ __forceinline__ L round_mult_to_latent(L bits, const EncParams& ep, L* adj_out);

// int_float_to_latent (pco/src/data_types/float.rs:229-244) on bit patterns
__device__ __forceinline__ uint64_t int_float_to_latent_bits(uint64_t fbits) {
  const uint64_t MID = uint64_t(1) << 63;
  uint64_t abs_bits = fbits & ~MID;
  const uint64_t gpi = uint64_t(1) << 53;
  const uint64_t gpi_bits = 0x4340000000000000ull;
  double a = __longlong_as_double((long long)abs_bits);
  uint64_t abs_int = (a < 9007199254740992.0) ? (uint64_t)__double2ull_rz(a) : gpi + (abs_bits - gpi_bits);
  return (fbits & MID) ? (MID - 1 - abs_int) : (MID + abs_int);
}
__device__ __forceinline__ uint32_t int_float_to_latent_bits(uint32_t fbits) {
  const uint32_t MID = 1u << 31;
  uint32_t abs_bits = fbits & ~MID;
  const uint32_t gpi = 1u << 24;
  const uint32_t gpi_bits = 0x4b800000u;
  float a = __uint_as_float(abs_bits);
  uint32_t abs_int = (a < 16777216.0f) ? __float2uint_rz(a) : gpi + (abs_bits - gpi_bits);
  return (fbits & MID) ? (MID - 1 - abs_int) : (MID + abs_int);
}

// float_mult split of one number (pco/src/mode/float_mult.rs:38-60).  NaN operands follow the CPU rule
// (operand NaN propagates quieted), see float_mult_unadjusted in decode_kernels.cuh.
__device__ __forceinline__ void float_mult_split(uint64_t xbits, uint64_t base_bits, uint64_t inv_bits, uint64_t& primary, uint64_t& secondary) {
  const uint64_t MID = uint64_t(1) << 63, QUIET = 0x0008000000000000ull;
  double x = __longlong_as_double((long long)xbits);
  uint64_t mult_bits;
  if (x != x) mult_bits = xbits | QUIET;
  else {
    double q = __dmul_rn(x, __longlong_as_double((long long)inv_bits));
    mult_bits = (uint64_t)__double_as_longlong(round(q));  // round half away from zero
  }
  primary = int_float_to_latent_bits(mult_bits);
  double mult = __longlong_as_double((long long)mult_bits);
  uint64_t prod_bits = (mult != mult) ? (mult_bits | QUIET) : (uint64_t)__double_as_longlong(__dmul_rn(mult, __longlong_as_double((long long)base_bits)));
  uint64_t a = (xbits & MID) ? ~xbits : (xbits ^ MID);
  uint64_t b = (prod_bits & MID) ? ~prod_bits : (prod_bits ^ MID);
  secondary = (a - b) + MID;
}
__device__ __forceinline__ void float_mult_split(uint32_t xbits, uint32_t base_bits, uint32_t inv_bits, uint32_t& primary, uint32_t& secondary) {
  const uint32_t MID = 1u << 31, QUIET = 0x00400000u;
  float x = __uint_as_float(xbits);
  uint32_t mult_bits;
  if (x != x) mult_bits = xbits | QUIET;
  else {
    float q = __fmul_rn(x, __uint_as_float(inv_bits));
    mult_bits = __float_as_uint(roundf(q));
  }
  primary = int_float_to_latent_bits(mult_bits);
  float mult = __uint_as_float(mult_bits);
  uint32_t prod_bits = (mult != mult) ? (mult_bits | QUIET) : __float_as_uint(__fmul_rn(mult, __uint_as_float(base_bits)));
  uint32_t a = (xbits & MID) ? ~xbits : (xbits ^ MID);
  uint32_t b = (prod_bits & MID) ? ~prod_bits : (prod_bits ^ MID);
  secondary = (a - b) + MID;
}

template <typename L, int MODE>
__device__ __forceinline__ void split_one(L xbits, const EncParams& ep, bool is_float, bool is_signed, L& p, L& s) {
  constexpr L MID = L(L(1) << (LT<L>::BITS - 1));
  s = 0;
  if constexpr (MODE == MODE_CLASSIC) {
    p = to_latent_ordered<L>(xbits, is_float, is_signed);
  } else if constexpr (MODE == MODE_INT_MULT) {
    L u = to_latent_ordered<L>(xbits, is_float, is_signed);
    L base = L(ep.mode_base);
    p = L(u / base);
    s = L(u % base);
  } else if constexpr (MODE == MODE_FLOAT_QUANT) {
    L u = to_latent_ordered<L>(xbits, true, false);
    L kmax = L(L(L(1) << ep.mode_k) - 1);
    p = L(u >> ep.mode_k);
    L lowest = L(u & kmax);
    s = (xbits & MID) ? L(kmax - lowest) : lowest;
  } else {  // MODE_FLOAT_MULT
    if constexpr (sizeof(L) == 8) {
      uint64_t pp, ss;
      float_mult_split(uint64_t(xbits), ep.base_bits, ep.inv_base_bits, pp, ss);
      p = pp; s = ss;
    } else if constexpr (sizeof(L) == 4) {
      uint32_t pp, ss;
      float_mult_split(uint32_t(xbits), uint32_t(ep.base_bits), uint32_t(ep.inv_base_bits), pp, ss);
      p = pp; s = ss;
    } else {
      p = 0;
    }
  }
}

constexpr int SPLIT_THREADS = 256;
constexpr int SPLIT_PER_THREAD = 8;
constexpr int SPLIT_TILE = SPLIT_THREADS * SPLIT_PER_THREAD;

__device__ __forceinline__ void atomic_min_u64(uint64_t* a, uint64_t v) { atomicMin(reinterpret_cast<unsigned long long*>(a), (unsigned long long)v); }
__device__ __forceinline__ void atomic_max_u64(uint64_t* a, uint64_t v) { atomicMax(reinterpret_cast<unsigned long long*>(a), (unsigned long long)v); }

// grid: n_chunks * tiles_per_chunk.  The latent / symbol / ans arrays hold each chunk's STORED latents (the page minus the
// first `order` of the primary) from slot row_base[c] on, row_base a multiple of 256: every batch row starts on a
// 512-byte (u16) .. 2048-byte (u64) boundary and can be moved with 16-byte vector accesses.
// MODE is a template parameter and the difference stencil's signed binomials live in registers: the kernel must stay
// HBM-bound (read n, write n_vars * n latents), a generic per-element mode switch made it issue-bound.
template <typename L, int MODE>
__global__ void __launch_bounds__(SPLIT_THREADS) split_delta_kernel(EncParams ep, uint32_t tiles_per_chunk, L* __restrict__ lat0, L* __restrict__ lat1,
                                                                     ChunkEnc* __restrict__ chunks) {
  __shared__ L tile[SPLIT_TILE + MAX_ORDER];
  __shared__ uint64_t red_min[MAX_VARS][SPLIT_THREADS / 32], red_max[MAX_VARS][SPLIT_THREADS / 32];
  const uint32_t c = blockIdx.x / tiles_per_chunk, t = blockIdx.x % tiles_per_chunk;
  const uint64_t cs = ep.chunk_starts[c], ce = ep.chunk_starts[c + 1];
  const uint32_t n = uint32_t(ce - cs);
  const uint32_t tile_start = t * SPLIT_TILE;
  if (tile_start >= n) return;
  const L* nums = static_cast<const L*>(ep.nums) + cs;
  const uint64_t rb = ep.row_base[c];
  const bool is_float = nt_is_float(ep.dtype), is_signed = nt_is_signed(ep.dtype);
  const uint32_t order = ep.order;
  const bool two_vars = MODE != MODE_CLASSIC && ep.n_vars > 1;
  const int tid = threadIdx.x;
  constexpr L MID = L(L(1) << (LT<L>::BITS - 1));
  constexpr L LMAX = L(~L(0));
  // coef[j] = (-1)^j C(order, j) in wrapping arithmetic: the order-th backward difference is sum_j coef[j] x[i - j]
  // (== `order` passes of x[i] -= x[i-1], delta/consecutive.rs:19-33)
  L coef[MAX_ORDER + 1];
  {
    uint32_t binom = 1;
#pragma unroll
    for (uint32_t j = 0; j <= MAX_ORDER; j++) {
      coef[j] = j <= order ? ((j & 1) ? L(L(0) - L(binom)) : L(binom)) : L(0);
      if (j < order) binom = binom * (order - j) / (j + 1);
    }
  }
  // primary latents of [tile_start - order, tile_start + SPLIT_TILE) into shared memory (tile[0, order) is the halo)
  L mn1 = LMAX, mx1 = 0;
#pragma unroll
  for (int q = 0; q < SPLIT_PER_THREAD; q++) {
    const int i = q * SPLIT_THREADS + tid;
    const uint32_t idx = tile_start + uint32_t(i);
    L p = 0, s = 0;
    if (idx < n) {
      split_one<L, MODE>(nums[idx], ep, is_float, is_signed, p, s);
      if (two_vars) {
        lat1[rb + idx] = s;
        mn1 = min(mn1, s);
        mx1 = max(mx1, s);
      }
    }
    tile[order + i] = p;
  }
  if (tid < int(order)) {
    L p = 0, s = 0;
    if (tile_start + uint32_t(tid) >= order) split_one<L, MODE>(nums[tile_start + tid - order], ep, is_float, is_signed, p, s);
    tile[tid] = p;
  }
  __syncthreads();
  L mn0 = LMAX, mx0 = 0;
#pragma unroll
  for (int q = 0; q < SPLIT_PER_THREAD; q++) {
    const int i = q * SPLIT_THREADS + tid;
    const uint32_t idx = tile_start + uint32_t(i);
    L d = tile[order + i];
    if (order > 0) {
      L acc = d;  // coef[0] == 1
#pragma unroll
      for (uint32_t j = 1; j <= MAX_ORDER; j++) {
        if (j > order) break;
        acc = L(acc + L(coef[j] * tile[order + i - j]));
      }
      d = L(acc + MID);  // toggle_center (delta/mod.rs:29-33)
    }
    if (idx < n && idx >= order) {
      lat0[rb + idx - order] = d;
      mn0 = min(mn0, d);
      mx0 = max(mx0, d);
    }
  }
  // page moments: moment_j = (j-th backward difference)[j]  (delta/consecutive.rs:19-33)
  if (t == 0 && tid < int(order)) {
    uint32_t j = tid;
    L acc = 0;
    if (j < n) {
      uint32_t binom = 1;
      for (uint32_t q = 0; q <= j; q++) {
        L term = L(L(binom) * tile[order + j - q]);
        acc = (q & 1) ? L(acc - term) : L(acc + term);
        binom = binom * (j - q) / (q + 1);
      }
    }
    chunks[c].moments[0][j] = uint64_t(acc);
  }
  // block min/max -> per-chunk atomics (an empty range keeps min > max and is skipped)
  uint64_t a0 = mn0, b0 = mx0, a1 = mn1, b1 = mx1;
  bool any0 = mn0 <= mx0, any1 = mn1 <= mx1;
  if (!any0) { a0 = ~uint64_t(0); b0 = 0; }
  if (!any1) { a1 = ~uint64_t(0); b1 = 0; }
  for (int d = 16; d > 0; d >>= 1) {
    a0 = min(a0, __shfl_xor_sync(0xffffffffu, a0, d));
    b0 = max(b0, __shfl_xor_sync(0xffffffffu, b0, d));
    if (two_vars) {
      a1 = min(a1, __shfl_xor_sync(0xffffffffu, a1, d));
      b1 = max(b1, __shfl_xor_sync(0xffffffffu, b1, d));
    }
  }
  if ((tid & 31) == 0) { red_min[0][tid >> 5] = a0; red_max[0][tid >> 5] = b0; red_min[1][tid >> 5] = a1; red_max[1][tid >> 5] = b1; }
  __syncthreads();
  if (tid < int(ep.n_vars)) {
    uint64_t a = ~uint64_t(0), b = 0;
    for (int w = 0; w < SPLIT_THREADS / 32; w++) { a = min(a, red_min[tid][w]); b = max(b, red_max[tid][w]); }
    if (a <= b) { atomic_min_u64(&chunks[c].vmin[tid], a); atomic_max_u64(&chunks[c].vmax[tid], b); }
  }
}

// a chunk's record before the front end: zero, and an empty latent range
__device__ inline void reset_chunk_enc(ChunkEnc* ch) {
  ChunkEnc z;
  memset(&z, 0, sizeof(z));
  z.vmin[0] = z.vmin[1] = ~uint64_t(0);
  *ch = z;
}
__global__ void init_chunks_kernel(ChunkEnc* chunks, uint32_t n_chunks) {
  uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_chunks) return;
  reset_chunk_enc(&chunks[c]);
}

// Stored range of var v in chunk [cs, ce): [cs + order_v, ce)
__device__ __forceinline__ uint64_t stored_begin(uint64_t cs, uint64_t ce, uint32_t order_v) { return min(cs + order_v, ce); }

// keys = latent - min(chunk, var): order-preserving, and lets the planner's sort skip the constant high bits
// compact_base != nullptr: chunk c's keys go to keys[compact_base[c] ...) - the pages of one wrapped chunk as ONE gap-free
// segment (their rows in `lat` are padded to 256), for the sort over their union
template <typename L>
__global__ void sort_keys_kernel(EncParams ep, uint32_t tiles_per_chunk, const L* __restrict__ lat, L* __restrict__ keys,
                                 const ChunkEnc* __restrict__ chunks, int v, const uint64_t* __restrict__ compact_base = nullptr) {
  const uint32_t c = blockIdx.x / tiles_per_chunk, t = blockIdx.x % tiles_per_chunk;
  const uint64_t cs = ep.chunk_starts[c], ce = ep.chunk_starts[c + 1];
  const uint64_t sb = stored_begin(cs, ce, v == 0 ? ep.order : 0);
  const uint64_t rb = ep.row_base[c], n = ce - sb;
  const uint64_t ob = compact_base ? compact_base[c] : rb;
  const L mn = L(chunks[c].vmin[v]);
  for (int i = threadIdx.x; i < SPLIT_TILE; i += blockDim.x) {
    uint64_t k = uint64_t(t) * SPLIT_TILE + i;
    if (k < n) keys[ob + k] = L(lat[rb + k] - mn);
  }
}

// The pages of one wrapped chunk share their bins: one minimum / maximum for all of them (keys, bin lowers and lookup
// tables are relative to it).  flags[0] = range bits of the union.
__global__ void union_range_kernel(EncParams ep, uint32_t n_pages, ChunkEnc* __restrict__ chunks, uint32_t* __restrict__ flags) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  uint64_t a = ~uint64_t(0), b = 0;
  bool any = false;
  for (uint32_t p = 0; p < n_pages; p++) {
    const uint64_t cs = ep.chunk_starts[p], ce = ep.chunk_starts[p + 1];
    if (ce == stored_begin(cs, ce, ep.order)) continue;
    any = true;
    a = min(a, chunks[p].vmin[0]);
    b = max(b, chunks[p].vmax[0]);
  }
  if (!any) { a = 0; b = 0; }
  for (uint32_t p = 0; p < n_pages; p++) { chunks[p].vmin[0] = a; chunks[p].vmax[0] = b; chunks[p].key_base[0] = a; }
  flags[0] = b > a ? 64 - __clzll((long long)(b - a)) : 0;
}

// segment offsets for the segmented sort
__global__ void segment_offsets_kernel(EncParams ep, uint32_t order_v, uint64_t* begins, uint64_t* ends) {
  uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= ep.n_chunks) return;
  uint64_t cs = ep.chunk_starts[c], ce = ep.chunk_starts[c + 1];
  begins[c] = ep.row_base[c];
  ends[c] = ep.row_base[c] + (ce - stored_begin(cs, ce, order_v));
}

// ---------------------------------------------------------------------------
// radix_sort_segments_kernel: the wide-key-range planner's sort (histograms.rs:208-281 needs order statistics of the chunk's latents; a
// key range above 2^15 does not fit the shared-memory counting path).  One CTA per segment (= a chunk's stored keys, latent - minimum)
// sorts it by least-significant-digit passes of 11 bits over the `bits` significant bits, ping-ponging between the two key buffers:
//   count   : warp w owns a contiguous tile of the segment and histograms its digits - lanes with equal digits find each other with
//             match_any, one of them adds the group's size to the warp's own counter row (no atomics);
//   scan    : exclusive prefix over (digit, warp) - all keys of digit d from warp w go after those of smaller digits and of lower warps;
//   scatter : the warp walks its tile again in the same order; a key's place is its (digit, warp) offset plus its rank among the
//             equal-digit lanes of the step - a stable pass, so the passes compose into a sort.
// 6 passes for 64-bit keys, 3 for 32-bit ones, each two reads and one write of the segment: HBM-bound streaming, no library call.
// ---------------------------------------------------------------------------
constexpr int RS_THREADS = 512;
constexpr int RS_WARPS = RS_THREADS / 32;
constexpr int RS_BITS = 11;
constexpr int RS_BINS = 1 << RS_BITS;
constexpr int RS_UNROLL = 8;  // 256 keys of a warp in flight per iteration

template <typename L>
__global__ void __launch_bounds__(RS_THREADS, 1) radix_sort_segments_kernel(L* __restrict__ buf_a, L* __restrict__ buf_b, const uint64_t* __restrict__ seg_begin,
                                                                            const uint64_t* __restrict__ seg_end, uint32_t bits) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint32_t (*hist)[RS_BINS] = reinterpret_cast<uint32_t (*)[RS_BINS]>(smem_raw);  // [RS_WARPS][RS_BINS]
  __shared__ uint32_t part[RS_THREADS];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint64_t s0 = seg_begin[blockIdx.x];
  const uint64_t n64 = seg_end[blockIdx.x] - s0;
  const uint32_t n = uint32_t(n64);
  const uint32_t passes = (bits + RS_BITS - 1) / RS_BITS;
  if (n <= 1) {  // nothing to sort, but the caller reads the buffer an odd number of passes ends in
    if (n == 1 && (passes & 1) && threadIdx.x == 0) buf_b[s0] = buf_a[s0];
    return;
  }
  // tiles: multiples of 32 keys, so that every step of a warp is a full step except the last of the segment
  const uint32_t per = ((n + RS_WARPS - 1) / RS_WARPS + 31) & ~31u;
  const uint32_t lo = min(n, uint32_t(warp) * per), hi = min(n, lo + per);
  L* in = buf_a + s0;
  L* out = buf_b + s0;
  for (uint32_t p = 0; p < passes; p++) {
    const uint32_t shift = p * RS_BITS;
    const uint32_t dmask = (1u << min(uint32_t(RS_BITS), bits - shift)) - 1;
    for (uint32_t i = tid; i < uint32_t(RS_WARPS * RS_BINS); i += RS_THREADS) hist[0][i] = 0;
    __syncthreads();
    // ---- count: RS_UNROLL steps of 32 keys per iteration, their loads issued together (the pass is a latency chain otherwise: one
    // 256-byte load per warp in flight)
    for (uint32_t i = lo; i < hi; i += 32 * RS_UNROLL) {
      L k[RS_UNROLL];
#pragma unroll
      for (int u = 0; u < RS_UNROLL; u++) k[u] = i + 32 * u + lane < hi ? in[i + 32 * u + lane] : L(0);
#pragma unroll
      for (int u = 0; u < RS_UNROLL; u++) {
        const bool act = i + 32 * u + lane < hi;
        const uint32_t amask = __ballot_sync(0xffffffffu, act);
        if (act) {
          const uint32_t d = uint32_t(uint64_t(k[u]) >> shift) & dmask;
          const uint32_t m = __match_any_sync(amask, d);
          if (lane == __ffs(m) - 1) hist[warp][d] += __popc(m);
        }
        __syncwarp();
      }
    }
    __syncthreads();
    // ---- scan over (digit major, warp minor): thread t owns digits [4t, 4t + 4)
    {
      uint32_t sum = 0;
#pragma unroll
      for (int dd = 0; dd < RS_BINS / RS_THREADS; dd++)
        for (int w = 0; w < RS_WARPS; w++) sum += hist[w][tid * (RS_BINS / RS_THREADS) + dd];
      uint32_t inc = sum;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) { const uint32_t o = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += o; }
      part[tid] = inc;
      __syncthreads();
      uint32_t base = inc - sum;
      for (int w = 0; w < warp; w++) base += part[w * 32 + 31];
      __syncthreads();
#pragma unroll
      for (int dd = 0; dd < RS_BINS / RS_THREADS; dd++)
        for (int w = 0; w < RS_WARPS; w++) {
          const uint32_t c = hist[w][tid * (RS_BINS / RS_THREADS) + dd];
          hist[w][tid * (RS_BINS / RS_THREADS) + dd] = base;
          base += c;
        }
    }
    __syncthreads();
    // ---- scatter (same order as the count)
    for (uint32_t i = lo; i < hi; i += 32 * RS_UNROLL) {
      L k[RS_UNROLL];
#pragma unroll
      for (int u = 0; u < RS_UNROLL; u++) k[u] = i + 32 * u + lane < hi ? in[i + 32 * u + lane] : L(0);
#pragma unroll
      for (int u = 0; u < RS_UNROLL; u++) {
        const bool act = i + 32 * u + lane < hi;
        const uint32_t amask = __ballot_sync(0xffffffffu, act);
        if (act) {
          const uint32_t d = uint32_t(uint64_t(k[u]) >> shift) & dmask;
          const uint32_t m = __match_any_sync(amask, d);
          const uint32_t off = hist[warp][d];
          __syncwarp(amask);
          out[off + __popc(m & ((1u << lane) - 1))] = k[u];
          if (lane == __ffs(m) - 1) hist[warp][d] = off + __popc(m);
        }
        __syncwarp();
      }
    }
    __syncthreads();  // the pass's writes are visible to the whole CTA (same-CTA global writes are ordered by the barrier)
    L* t = in; in = out; out = t;
  }
}

// ---------------------------------------------------------------------------
// Bin training (train_infos, chunk_compressor.rs:52-99) in two kernels per latent var:
//   plan_probe_kernel — one 512-thread CTA per chunk, HBM-bound: order statistics at the 2^log equal-count boundaries
//                       (from shared-memory counters when the key range is narrow, else from the sorted keys)
//   plan_solve_kernel — one warp per chunk (SOLVE_THREADS; the code also runs with more), latency-bound and short: histogram
//                       state machine (one thread), bin-merge DP (the candidates of a step spread over the threads), weight
//                       quantisation, tANS tables.  All chunks are resident at once, so the serial parts overlap.
// ---------------------------------------------------------------------------
constexpr int PLAN_THREADS = 512;
constexpr int SOLVE_THREADS = 32;   // 128 (a barrier per DP step) measured slower with every chunk resident on C2
constexpr uint32_t PLAN_MAX_COUNT_BITS = 15;  // counting histogram (no sort) when the key range fits 2^15 shared-memory counters

// Order statistics handed from the probe kernel to the solver (per chunk and var, in HBM scratch)
template <bool WIDE>
struct PlanProbesT {
  static constexpr int MAXB = EncCap<WIDE>::MAXB;
  uint64_t vB1[MAXB], vB[MAXB], vLm1[MAXB], vR[MAXB];
  uint32_t runL[MAXB], runR[MAXB];
  uint64_t first;  // smallest key
  uint64_t pad;
};
using PlanProbes = PlanProbesT<false>;

struct PlanSmem {
  union {
    PlanProbes probes;  // dead once the unoptimized histogram exists
    struct {
      uint32_t o_count[ENC_MAXB];
      uint64_t o_lower[ENC_MAXB], o_upper[ENC_MAXB];
      uint32_t o_ob[ENC_MAXB];
      float fweights[ENC_MAXB];
      uint32_t weights[ENC_MAXB];
      uint32_t cum[ENC_MAXB + 1];
      uint16_t sym_of_state[1 << ENC_MAX_SIZE_LOG];
      uint32_t rank_counter[ENC_MAXB];
    };
  };
  // unoptimized bins
  uint32_t h_count[ENC_MAXB];
  uint64_t h_lower[ENC_MAXB], h_upper[ENC_MAXB];
  uint32_t n_hist;
  // DP
  uint32_t c_counts[ENC_MAXB + 1];
  float best_cost[ENC_MAXB + 1];
  uint32_t best_j[ENC_MAXB];
  uint32_t red_cost[2][SOLVE_THREADS / 32], red_j[2][SOLVE_THREADS / 32];  // per-warp argmin of a DP step
  uint32_t n_opt;
  uint32_t size_log;
};

// COUNTING = false: `keys` holds the var's stored latents minus the chunk minimum, sorted ascending per chunk.
// COUNTING = true : `keys` holds the raw (unsorted) latents and the key range is < 2^range_bits <= 2^15: the CTA counts
//                   every key into shared memory, prefix-sums the counters, and reads ranks / run extents off the
//                   cumulative counts -- the planner only ever needs order statistics, never the sorted array.
template <typename L, bool COUNTING, bool WIDE = false, bool CHUNK_BINS = false>
__global__ void __launch_bounds__(PLAN_THREADS) plan_probe_kernel(EncParams ep, const L* __restrict__ keys, const ChunkEnc* __restrict__ chunks,
                                                                   PlanProbesT<WIDE>* __restrict__ probes, int v, uint32_t range_bits,
                                                                   uint16_t* __restrict__ keys16, uint32_t n_override = 0) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint32_t* cum = reinterpret_cast<uint32_t*>(smem_raw);  // COUNTING: 2^range_bits + 1 entries
  __shared__ uint32_t scan_part[PLAN_THREADS / 32];
  const uint32_t c = blockIdx.x;
  const int tid = threadIdx.x;
  const uint64_t cs = ep.chunk_starts[c], ce = ep.chunk_starts[c + 1];
  const uint64_t sb = stored_begin(cs, ce, v == 0 ? ep.order : 0);
  // stored latents; n_override (sorted path only): `keys` is the gap-free sorted union of a wrapped chunk's pages
  const uint32_t n = n_override ? n_override : uint32_t(ce - sb);
  if (n == 0) return;
  const L* s = n_override ? keys : keys + ep.row_base[c];
  ENC_TICK_INIT();
  const uint32_t n_vals = COUNTING ? (1u << range_bits) : 0u;
  if (COUNTING) {
    const L mn = L(chunks[c].vmin[v]);  // (the host sets key_base = vmin for this path: range_bits_kernel)
    for (uint32_t i = tid; i <= n_vals; i += PLAN_THREADS) cum[i] = 0;
    __syncthreads();
    {
      // COUNTING also leaves the keys behind as 16 bits each (range < 2^15): binning and packing then read a quarter of
      // the bytes of the 64-bit latents
      uint16_t* k16 = keys16 + ep.row_base[c];
      // 4 consecutive latents per thread and step (rows are 256-aligned): vector loads in, one 8-byte store of keys out
      struct alignas(sizeof(L) * 4 > 16 ? 16 : sizeof(L) * 4) Vec4 { L v[4]; };
      const uint32_t n4 = n / 4;
      uint32_t q = tid;
      for (; q + PLAN_THREADS < n4; q += 2 * PLAN_THREADS) {  // two vectors in flight per thread
        const Vec4 a = *reinterpret_cast<const Vec4*>(s + 4 * size_t(q)), b = *reinterpret_cast<const Vec4*>(s + 4 * size_t(q + PLAN_THREADS));
        uint32_t ka[4], kb[4];
#pragma unroll
        for (int t = 0; t < 4; t++) { ka[t] = uint32_t(L(a.v[t] - mn)); kb[t] = uint32_t(L(b.v[t] - mn)); }
#pragma unroll
        for (int t = 0; t < 4; t++) { atomicAdd(&cum[ka[t]], 1u); atomicAdd(&cum[kb[t]], 1u); }
        *reinterpret_cast<uint2*>(k16 + 4 * size_t(q)) = make_uint2(ka[0] | (ka[1] << 16), ka[2] | (ka[3] << 16));
        *reinterpret_cast<uint2*>(k16 + 4 * size_t(q + PLAN_THREADS)) = make_uint2(kb[0] | (kb[1] << 16), kb[2] | (kb[3] << 16));
      }
      for (; q < n4; q += PLAN_THREADS) {
        const Vec4 a = *reinterpret_cast<const Vec4*>(s + 4 * size_t(q));
        uint32_t ka[4];
#pragma unroll
        for (int t = 0; t < 4; t++) { ka[t] = uint32_t(L(a.v[t] - mn)); atomicAdd(&cum[ka[t]], 1u); }
        *reinterpret_cast<uint2*>(k16 + 4 * size_t(q)) = make_uint2(ka[0] | (ka[1] << 16), ka[2] | (ka[3] << 16));
      }
      for (uint32_t i = 4 * n4 + tid; i < n; i += PLAN_THREADS) {
        const uint32_t k = uint32_t(L(s[i] - mn));
        atomicAdd(&cum[k], 1u);
        k16[i] = uint16_t(k);
      }
    }
    __syncthreads();
    ENC_TICK(0);  // zero + count
    // exclusive scan of the counters: warp w owns a contiguous span and walks it 32 counters at a time
    const int lane = tid & 31, warp = tid >> 5;
    const uint32_t span = (n_vals + PLAN_THREADS / 32 - 1) / (PLAN_THREADS / 32);
    const uint32_t w_lo = min(n_vals, warp * span), w_hi = min(n_vals, w_lo + span);
    uint32_t carry = 0;
    for (uint32_t base = w_lo; base < w_hi; base += 32) {
      const uint32_t idx = base + lane;
      const uint32_t cnt = idx < w_hi ? cum[idx] : 0u;
      uint32_t inc = cnt;
      for (int d = 1; d < 32; d <<= 1) { uint32_t o = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += o; }
      if (idx < w_hi) cum[idx] = carry + inc - cnt;
      carry += __shfl_sync(0xffffffffu, inc, 31);
    }
    if (lane == 0) scan_part[warp] = carry;
    __syncthreads();
    uint32_t wbase = 0;
    for (int w = 0; w < warp; w++) wbase += scan_part[w];
    for (uint32_t idx = w_lo + lane; idx < w_hi; idx += 32) cum[idx] += wbase;
    if (tid == 0) cum[n_vals] = n;
    __syncthreads();
    ENC_TICK(1);  // scan
  }
  // value at sorted rank idx
  auto s_at = [&](uint32_t idx) -> uint64_t {
    if (!COUNTING) return uint64_t(s[idx]);
    uint32_t lo = 0, hi = n_vals;  // invariant: cum[lo] <= idx < cum[hi]
    while (hi - lo > 1) { uint32_t m = (lo + hi) >> 1; if (cum[m] <= idx) lo = m; else hi = m; }
    return lo;
  };
  PlanProbesT<WIDE>& pr = probes[c];
  const uint32_t n_bins_log = CHUNK_BINS ? unoptimized_bins_log(ep.bins_log[0], ce - cs, v) : ep.bins_log[v];
  const uint32_t nbk = 1u << n_bins_log;
  auto c_count_of = [&](uint32_t b) -> uint32_t { return uint32_t((uint64_t(b + 1) * n + nbk - 1) >> n_bins_log); };
  if (tid == 0) pr.first = s_at(0);
  // probes at every equal-count boundary, in parallel (histograms.rs:132-140)
  for (uint32_t k = tid; k < nbk; k += PLAN_THREADS) {
    uint32_t B = c_count_of(k);
    uint64_t vb1 = 0, vb = 0, vlm1 = 0, vr = 0;
    uint32_t l = 0, r = 0;
    if (B >= 1 && B <= n) {
      vb1 = s_at(B - 1);
      if (B < n) vb = s_at(B);
      if (B < n && vb == vb1) {
        // extent [l, r) of the run of vb1
        if (COUNTING) {
          l = cum[uint32_t(vb1)];
          r = cum[uint32_t(vb1) + 1];
        } else {
          uint32_t lo = 0, hi = B - 1;  // first index with s[idx] >= vb1 is in [0, B-1]
          while (lo < hi) { uint32_t m = (lo + hi) >> 1; if (uint64_t(s[m]) < vb1) lo = m + 1; else hi = m; }
          l = lo;
          lo = B; hi = n;               // first index with s[idx] > vb1 is in [B+1, n]
          while (lo < hi) { uint32_t m = (lo + hi) >> 1; if (uint64_t(s[m]) <= vb1) lo = m + 1; else hi = m; }
          r = lo;
        }
        if (l > 0) vlm1 = s_at(l - 1);
        if (r < n) vr = s_at(r);
      }
    }
    pr.vB1[k] = vb1; pr.vB[k] = vb; pr.vLm1[k] = vlm1; pr.vR[k] = vr; pr.runL[k] = l; pr.runR[k] = r;
  }
  ENC_TICK(2);  // probes
}

// ---------------------------------------------------------------------------
// split_count_kernel: K1+K2 and the counting half of the planner in ONE pass over the numbers, for the case that
// dominates in practice - classic mode (one latent var) whose stored latents span < 2^15.  One CTA per chunk streams
// the chunk once: ordered latents, order-k backward difference (stencil of signed binomials over vector loads),
// min/max, shared-memory counters, 16-bit keys out.  The 64-bit latents are never written: split_delta_kernel +
// plan_probe_kernel move 6.8 GB per 2 GiB of u64 input (write and re-read of the latents), this kernel 2.6 GB.
// The chunk minimum is not known while counting, so everything is relative to an ANCHOR (the first stored latent):
//   key16   = (latent - anchor) mod 2^16          (consumers subtract key_base = anchor; offsets are differences)
//   counter = (latent - anchor) mod 2^15          (a range < 2^15 lies on an arc of the circle: no two values collide)
// and once min/max are known the counters are read through the rotation (min - anchor) mod 2^15.  A chunk whose range
// needs more than 15 bits raises flags[1]; the host then runs the two-kernel path for the whole call.
// ---------------------------------------------------------------------------
constexpr int SC_THREADS = 1024;
constexpr uint32_t SC_N = 1u << PLAN_MAX_COUNT_BITS, SC_MASK = SC_N - 1;

// The streaming pass of split_count_kernel for one delta order: SC_PER consecutive stored latents per thread and step.
// Stored index s holds the difference ending at number ORDER + s, which needs numbers s .. s + ORDER + SC_PER - 1:
// aligned 4-vectors from s on (the next thread's first vectors are this thread's last: those loads hit L1).
#ifndef PCOB_SC_PER
#define PCOB_SC_PER 8
#endif
constexpr int SC_PER = PCOB_SC_PER;
template <typename L, int ORDER>
__device__ __forceinline__ void sc_stream(const L* __restrict__ nums, uint32_t n, uint32_t stored, L anchor, bool is_float, bool is_signed,
                                          uint16_t* __restrict__ k16, uint32_t* __restrict__ cnt, L& mn, L& mx) {
  constexpr L MID = L(L(1) << (LT<L>::BITS - 1));
  constexpr int NX = SC_PER + (ORDER > 4 ? 8 : (ORDER > 0 ? 4 : 0));
  struct alignas(sizeof(L) * 4 > 16 ? 16 : sizeof(L) * 4) Vec4 { L v[4]; };
  const bool vec_ok = (reinterpret_cast<uintptr_t>(nums) & (sizeof(Vec4) - 1)) == 0;
  const uint32_t n_steps = (stored + SC_PER - 1) / SC_PER;
  const int tid = threadIdx.x;
  for (uint32_t q = tid; q < n_steps; q += SC_THREADS) {
    const uint32_t s = SC_PER * q;
    L x[NX];
    if (vec_ok && s + NX <= n) {
#pragma unroll
      for (int g = 0; g < NX / 4; g++) {
        const Vec4 a = *reinterpret_cast<const Vec4*>(nums + s + 4 * g);
#pragma unroll
        for (int u = 0; u < 4; u++) x[4 * g + u] = to_latent_ordered<L>(a.v[u], is_float, is_signed);
      }
    } else {
#pragma unroll
      for (int u = 0; u < NX; u++) x[u] = (u < ORDER + SC_PER && s + u < n) ? to_latent_ordered<L>(nums[s + u], is_float, is_signed) : L(0);
    }
    uint32_t kw[SC_PER];
#pragma unroll
    for (int u = 0; u < SC_PER; u++) {
      // d = sum_j (-1)^j C(ORDER, j) x[u + ORDER - j]  (== ORDER passes of x[i] -= x[i-1], delta/consecutive.rs:19-33)
      L d = x[u + ORDER];
      uint32_t binom = 1;
#pragma unroll
      for (int j = 1; j <= ORDER; j++) {
        binom = binom * uint32_t(ORDER - j + 1) / uint32_t(j);
        d = (j & 1) ? L(d - L(L(binom) * x[u + ORDER - j])) : L(d + L(L(binom) * x[u + ORDER - j]));
      }
      if (ORDER > 0) d = L(d + MID);  // toggle_center (delta/mod.rs:29-33)
      const bool live = s + u < stored;
      if (live) { mn = min(mn, d); mx = max(mx, d); }
      const uint32_t w = uint32_t(uint64_t(d) - uint64_t(anchor));  // zero-extended: the same modulus (2^16 / 2^15) for every number width
      kw[u] = w & 0xffffu;
      if (live) atomicAdd(&cnt[w & SC_MASK], 1u);
    }
    // rows are 256-aligned and padded: vector stores of the keys.  16-byte ones when SC_PER allows, so that a warp's stores fill
    // whole 32-byte sectors (two 8-byte stores would each leave every sector half written)
    if (SC_PER % 8 == 0) {
#pragma unroll
      for (int g = 0; g < SC_PER / 8; g++)
        *reinterpret_cast<uint4*>(k16 + s + 8 * g) = make_uint4(kw[8 * g] | (kw[8 * g + 1] << 16), kw[8 * g + 2] | (kw[8 * g + 3] << 16),
                                                               kw[8 * g + 4] | (kw[8 * g + 5] << 16), kw[8 * g + 6] | (kw[8 * g + 7] << 16));
    } else {
#pragma unroll
      for (int g = 0; g < SC_PER / 4; g++)
        *reinterpret_cast<uint2*>(k16 + s + 4 * g) = make_uint2(kw[4 * g] | (kw[4 * g + 1] << 16), kw[4 * g + 2] | (kw[4 * g + 3] << 16));
    }
  }
}

template <typename L, bool CHUNK_BINS = false>
__global__ void __launch_bounds__(SC_THREADS, 1) split_count_kernel(EncParams ep, ChunkEnc* __restrict__ chunks, PlanProbes* __restrict__ probes,
                                                                   uint16_t* __restrict__ keys16, uint32_t* __restrict__ flags) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint32_t* cnt = reinterpret_cast<uint32_t*>(smem_raw);  // SC_N counters, then their exclusive scan (rotated)
  __shared__ uint64_t red_min[SC_THREADS / 32], red_max[SC_THREADS / 32];
  __shared__ uint32_t scan_part[SC_THREADS / 32];
  __shared__ uint64_t sh_anchor, sh_min, sh_max;
  const uint32_t c = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint64_t cs = ep.chunk_starts[c], ce = ep.chunk_starts[c + 1];
  const uint32_t n = uint32_t(ce - cs);
  const uint32_t order = ep.order;
  const uint32_t stored = n > order ? n - order : 0;
  const L* __restrict__ nums = static_cast<const L*>(ep.nums) + cs;
  const bool is_float = nt_is_float(ep.dtype), is_signed = nt_is_signed(ep.dtype);
  constexpr L MID = L(L(1) << (LT<L>::BITS - 1));
  auto lat_at = [&](uint32_t idx) -> L { return idx < n ? to_latent_ordered<L>(nums[idx], is_float, is_signed) : L(0); };
  // coef[j] = (-1)^j C(order, j): the order-th backward difference is sum_j coef[j] x[i - j] (delta/consecutive.rs:19-33)
  L coef[MAX_ORDER + 1];
  {
    uint32_t binom = 1;
#pragma unroll
    for (uint32_t j = 0; j <= MAX_ORDER; j++) {
      coef[j] = j <= order ? ((j & 1) ? L(L(0) - L(binom)) : L(binom)) : L(0);
      if (j < order) binom = binom * (order - j) / (j + 1);
    }
  }
  for (uint32_t i = tid; i < SC_N; i += SC_THREADS) cnt[i] = 0;
  // page moments: moment_j = (j-th backward difference)[j]
  if (tid < int(order)) {
    const uint32_t j = tid;
    L acc = 0;
    if (j < n) {
      uint32_t binom = 1;
      for (uint32_t q = 0; q <= j; q++) {
        const L term = L(L(binom) * lat_at(j - q));
        acc = (q & 1) ? L(acc - term) : L(acc + term);
        binom = binom * (j - q) / (q + 1);
      }
    }
    chunks[c].moments[0][j] = uint64_t(acc);
  }
  if (tid == 0) {
    L a = 0;
    if (stored > 0) {
      a = lat_at(order);
      for (uint32_t j = 1; j <= order; j++) a = L(a + L(coef[j] * lat_at(order - j)));
      if (order > 0) a = L(a + MID);
    }
    sh_anchor = uint64_t(a);
  }
  __syncthreads();
  const L anchor = L(sh_anchor);
  uint16_t* __restrict__ k16 = keys16 + ep.row_base[c];
  L mn = L(~L(0)), mx = 0;
  switch (order) {  // the stencil's window offsets and binomials are compile-time per order
    case 0: sc_stream<L, 0>(nums, n, stored, anchor, is_float, is_signed, k16, cnt, mn, mx); break;
    case 1: sc_stream<L, 1>(nums, n, stored, anchor, is_float, is_signed, k16, cnt, mn, mx); break;
    case 2: sc_stream<L, 2>(nums, n, stored, anchor, is_float, is_signed, k16, cnt, mn, mx); break;
    case 3: sc_stream<L, 3>(nums, n, stored, anchor, is_float, is_signed, k16, cnt, mn, mx); break;
    case 4: sc_stream<L, 4>(nums, n, stored, anchor, is_float, is_signed, k16, cnt, mn, mx); break;
    case 5: sc_stream<L, 5>(nums, n, stored, anchor, is_float, is_signed, k16, cnt, mn, mx); break;
    case 6: sc_stream<L, 6>(nums, n, stored, anchor, is_float, is_signed, k16, cnt, mn, mx); break;
    default: sc_stream<L, 7>(nums, n, stored, anchor, is_float, is_signed, k16, cnt, mn, mx); break;
  }
  // chunk min / max
  {
    uint64_t a = mn <= mx ? uint64_t(mn) : ~uint64_t(0), b = mn <= mx ? uint64_t(mx) : 0;
    for (int d = 16; d > 0; d >>= 1) {
      a = min(a, __shfl_xor_sync(0xffffffffu, a, d));
      b = max(b, __shfl_xor_sync(0xffffffffu, b, d));
    }
    if (lane == 0) { red_min[warp] = a; red_max[warp] = b; }
    __syncthreads();
    if (tid == 0) {
      for (int w = 0; w < SC_THREADS / 32; w++) { a = min(a, red_min[w]); b = max(b, red_max[w]); }
      sh_min = a; sh_max = b;
      chunks[c].vmin[0] = a;
      chunks[c].vmax[0] = b;
      chunks[c].key_base[0] = uint64_t(anchor);
      const uint32_t bits = b > a ? 64 - __clzll((long long)(b - a)) : 0;
      atomicMax(&flags[0], bits);
      if (bits > PLAN_MAX_COUNT_BITS) atomicOr(&flags[1], 1u);
    }
    __syncthreads();
  }
  if (stored == 0) return;
  const uint64_t vmin = sh_min, vmax = sh_max;
  if (vmax - vmin > uint64_t(SC_MASK)) return;  // wide chunk: the host re-runs the call on the two-kernel path
  const uint32_t rot = uint32_t(vmin - uint64_t(anchor)) & SC_MASK;  // counter of key k (= latent - vmin) is cnt[(k + rot) & SC_MASK]
  // exclusive scan of the counters in key order: warp w owns a contiguous span of keys, 32 at a time
  {
    const uint32_t span = SC_N / (SC_THREADS / 32);
    const uint32_t w_lo = warp * span, w_hi = w_lo + span;
    uint32_t carry = 0;
    for (uint32_t base = w_lo; base < w_hi; base += 32) {
      const uint32_t pi = (base + lane + rot) & SC_MASK;
      const uint32_t v = cnt[pi];
      uint32_t inc = v;
      for (int d = 1; d < 32; d <<= 1) { uint32_t o = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += o; }
      cnt[pi] = carry + inc - v;
      carry += __shfl_sync(0xffffffffu, inc, 31);
    }
    if (lane == 0) scan_part[warp] = carry;
    __syncthreads();
    uint32_t wbase = 0;
    for (int w = 0; w < warp; w++) wbase += scan_part[w];
    for (uint32_t k = w_lo + lane; k < w_hi; k += 32) cnt[(k + rot) & SC_MASK] += wbase;
    __syncthreads();
  }
  auto cum = [&](uint32_t k) -> uint32_t { return k >= SC_N ? stored : cnt[(k + rot) & SC_MASK]; };
  // key at sorted rank idx
  auto s_at = [&](uint32_t idx) -> uint64_t {
    uint32_t lo = 0, hi = SC_N;  // invariant: cum(lo) <= idx < cum(hi)
    while (hi - lo > 1) { uint32_t m = (lo + hi) >> 1; if (cum(m) <= idx) lo = m; else hi = m; }
    return lo;
  };
  PlanProbes& pr = probes[c];
  const uint32_t n_bins_log = CHUNK_BINS ? unoptimized_bins_log(ep.bins_log[0], n, 0) : ep.bins_log[0];
  const uint32_t nbk = 1u << n_bins_log;
  auto c_count_of = [&](uint32_t b) -> uint32_t { return uint32_t((uint64_t(b + 1) * stored + nbk - 1) >> n_bins_log); };
  if (tid == 0) pr.first = s_at(0);
  // probes at every equal-count boundary (histograms.rs:132-140), as in plan_probe_kernel
  for (uint32_t k = tid; k < nbk; k += SC_THREADS) {
    const uint32_t B = c_count_of(k);
    uint64_t vb1 = 0, vb = 0, vlm1 = 0, vr = 0;
    uint32_t l = 0, r = 0;
    if (B >= 1 && B <= stored) {
      vb1 = s_at(B - 1);
      if (B < stored) vb = s_at(B);
      if (B < stored && vb == vb1) {
        l = cum(uint32_t(vb1));
        r = cum(uint32_t(vb1) + 1);
        if (l > 0) vlm1 = s_at(l - 1);
        if (r < stored) vr = s_at(r);
      }
    }
    pr.vB1[k] = vb1; pr.vB[k] = vb; pr.vLm1[k] = vlm1; pr.vR[k] = vr; pr.runL[k] = l; pr.runR[k] = r;
  }
}

// ---------------------------------------------------------------------------
// union_probe_kernel: the pages of ONE wrapped chunk share their bins (chunk_compressor.rs:129-140: deltas per page, one
// histogram over all stored latents).  split_count_kernel has run per page (keys relative to each page's anchor, per-page
// min / max); this kernel - one CTA, the multi-page wrapped path is not the bulk path - takes the minimum over the pages,
// counts every page's keys into one 2^15-counter histogram relative to it, scans, and leaves the union's probes in probes[0].
// Every page's vmin becomes the common minimum (the bins' lowers and the lookup tables are relative to it); key_base stays
// per page.  flags[0] = range bits of the union, flags[1] |= 1 when it needs more than 15.
// ---------------------------------------------------------------------------
template <typename L>
__global__ void __launch_bounds__(SC_THREADS, 1) union_probe_kernel(EncParams ep, uint32_t n_pages, ChunkEnc* __restrict__ chunks, PlanProbes* __restrict__ probes,
                                                                   const uint16_t* __restrict__ keys16, uint32_t* __restrict__ flags) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint32_t* cnt = reinterpret_cast<uint32_t*>(smem_raw);
  __shared__ uint32_t scan_part[SC_THREADS / 32];
  __shared__ uint64_t sh_min, sh_max;
  __shared__ uint32_t sh_total;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (uint32_t i = tid; i < SC_N; i += SC_THREADS) cnt[i] = 0;
  if (tid == 0) {
    uint64_t a = ~uint64_t(0), b = 0;
    uint32_t total = 0;
    for (uint32_t p = 0; p < n_pages; p++) {
      const uint64_t cs = ep.chunk_starts[p], ce = ep.chunk_starts[p + 1];
      const uint32_t stored = uint32_t(ce - stored_begin(cs, ce, ep.order));
      if (stored == 0) continue;
      total += stored;
      a = min(a, chunks[p].vmin[0]);
      b = max(b, chunks[p].vmax[0]);
    }
    sh_min = a; sh_max = b; sh_total = total;
    const uint32_t bits = (total && b > a) ? 64 - __clzll((long long)(b - a)) : 0;
    flags[0] = bits;
    if (bits > PLAN_MAX_COUNT_BITS) atomicOr(&flags[1], 1u);
  }
  __syncthreads();
  const uint64_t vmin = sh_min, vmax = sh_max;
  const uint32_t total = sh_total;
  if (total == 0 || vmax - vmin > uint64_t(SC_MASK)) return;
  for (uint32_t p = 0; p < n_pages; p++) {
    const uint64_t cs = ep.chunk_starts[p], ce = ep.chunk_starts[p + 1];
    const uint32_t stored = uint32_t(ce - stored_begin(cs, ce, ep.order));
    const uint16_t* k16 = keys16 + ep.row_base[p];
    const uint32_t shift = uint32_t(vmin - chunks[p].key_base[0]);  // key16 = latent - key_base (mod 2^16)
    for (uint32_t i = tid; i < stored; i += SC_THREADS) atomicAdd(&cnt[(uint32_t(k16[i]) - shift) & SC_MASK], 1u);
  }
  __syncthreads();
  if (tid < int(n_pages)) { chunks[tid].vmin[0] = vmin; chunks[tid].vmax[0] = vmax; }
  for (uint32_t p = SC_THREADS + tid; p < n_pages; p += SC_THREADS) { chunks[p].vmin[0] = vmin; chunks[p].vmax[0] = vmax; }
  {
    const uint32_t span = SC_N / (SC_THREADS / 32);
    const uint32_t w_lo = warp * span, w_hi = w_lo + span;
    uint32_t carry = 0;
    for (uint32_t base = w_lo; base < w_hi; base += 32) {
      const uint32_t v = cnt[base + lane];
      uint32_t inc = v;
      for (int d = 1; d < 32; d <<= 1) { uint32_t o = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += o; }
      cnt[base + lane] = carry + inc - v;
      carry += __shfl_sync(0xffffffffu, inc, 31);
    }
    if (lane == 0) scan_part[warp] = carry;
    __syncthreads();
    uint32_t wbase = 0;
    for (int w = 0; w < warp; w++) wbase += scan_part[w];
    for (uint32_t k = w_lo + lane; k < w_hi; k += 32) cnt[k] += wbase;
    __syncthreads();
  }
  auto cum = [&](uint32_t k) -> uint32_t { return k >= SC_N ? total : cnt[k]; };
  auto s_at = [&](uint32_t idx) -> uint64_t {
    uint32_t lo = 0, hi = SC_N;  // invariant: cum(lo) <= idx < cum(hi)
    while (hi - lo > 1) { uint32_t m = (lo + hi) >> 1; if (cum(m) <= idx) lo = m; else hi = m; }
    return lo;
  };
  PlanProbes& pr = probes[0];
  const uint32_t n_bins_log = ep.bins_log[0];
  const uint32_t nbk = 1u << n_bins_log;
  auto c_count_of = [&](uint32_t b) -> uint32_t { return uint32_t((uint64_t(b + 1) * total + nbk - 1) >> n_bins_log); };
  if (tid == 0) pr.first = s_at(0);
  for (uint32_t k = tid; k < nbk; k += SC_THREADS) {
    const uint32_t B = c_count_of(k);
    uint64_t vb1 = 0, vb = 0, vlm1 = 0, vr = 0;
    uint32_t l = 0, r = 0;
    if (B >= 1 && B <= total) {
      vb1 = s_at(B - 1);
      if (B < total) vb = s_at(B);
      if (B < total && vb == vb1) {
        l = cum(uint32_t(vb1));
        r = cum(uint32_t(vb1) + 1);
        if (l > 0) vlm1 = s_at(l - 1);
        if (r < total) vr = s_at(r);
      }
    }
    pr.vB1[k] = vb1; pr.vB[k] = vb; pr.vLm1[k] = vlm1; pr.vR[k] = vr; pr.runL[k] = l; pr.runR[k] = r;
  }
}

// plans[0] (trained on the union) -> the plan slot of every page; n_lat stays the union's (only fallback_kernel reads it)
template <bool WIDE = false>
__global__ void broadcast_plan_kernel(VarPlanT<WIDE>* __restrict__ plans, uint32_t n_pages) {
  const uint32_t p = blockIdx.x + 1;
  if (p >= n_pages) return;
  const uint4* src = reinterpret_cast<const uint4*>(&plans[0]);
  uint4* dst = reinterpret_cast<uint4*>(&plans[size_t(p) * MAX_VARS]);
  for (uint32_t i = threadIdx.x; i < sizeof(VarPlanT<WIDE>) / 16; i += blockDim.x) dst[i] = src[i];
}

template <typename L, bool CHUNK_BINS = false>
__global__ void __launch_bounds__(SOLVE_THREADS) plan_solve_kernel(EncParams ep, const PlanProbes* __restrict__ probes,
                                                                    const ChunkEnc* __restrict__ chunks, VarPlan* __restrict__ plans, int v,
                                                                    uint32_t n_override = 0) {
  __shared__ PlanSmem sm;
  const uint32_t c = blockIdx.x;
  const int tid = threadIdx.x;
  const uint64_t cs = ep.chunk_starts[c], ce = ep.chunk_starts[c + 1];
  const uint64_t sb = stored_begin(cs, ce, v == 0 ? ep.order : 0);
  // stored latents; n_override: the pages of one wrapped chunk share bins trained on all of them (union_probe_kernel)
  const uint32_t n = n_override ? n_override : uint32_t(ce - sb);
  VarPlan& plan = plans[size_t(c) * MAX_VARS + v];
  const uint64_t vmin = chunks[c].vmin[v];
  constexpr uint32_t LBITS = LT<L>::BITS;
  if (n == 0) {  // train_infos on an empty var (chunk_compressor.rs:56-58): zero bins
    if (tid == 0) { plan.n_bins = 0; plan.size_log = 0; plan.max_ob = 0; plan.n_lat = 0; plan.wc_bits = 0; plan.est_bits = 0; plan.next_states[0] = 0; }
    return;
  }
  ENC_TICK_INIT();
  const uint32_t n_bins_log = CHUNK_BINS ? unoptimized_bins_log(ep.bins_log[0], ce - cs, v) : ep.bins_log[v];
  const uint32_t nbk = 1u << n_bins_log;
  const bool small_n = n <= (1u << 20);  // (cc << n_bins_log) fits 32 bits (n_bins_log <= 8)
  // (cc << n_bins_log) / n, cc <= n: the quotient is at most 2^n_bins_log <= 256, so a float estimate is within 1 of it and one
  // remainder check makes it exact (an integer division is ~100 dependent cycles on the state machine's serial path)
  const float rcp_n = __frcp_rn(__uint2float_rn(n));
  auto bin_idx_of = [&](uint64_t cc) -> uint32_t {
    if (!small_n) return uint32_t((cc << n_bins_log) / n);
    const uint32_t num = uint32_t(cc) << n_bins_log;
    uint32_t q = __float2uint_rz(__fmul_rn(__uint2float_rz(num), rcp_n));
    const uint32_t r = num - q * n;
    if (int32_t(r) < 0) q -= 1;
    else if (r >= n) q += 1;
    return q;
  };
  auto c_count_of = [&](uint32_t b) -> uint32_t { return uint32_t((uint64_t(b + 1) * n + nbk - 1) >> n_bins_log); };
  {
    // stage this chunk's probes (coalesced 16-byte copies)
    const uint4* src = reinterpret_cast<const uint4*>(&probes[c]);
    uint4* dst = reinterpret_cast<uint4*>(&sm.probes);
    for (uint32_t i = tid; i < sizeof(PlanProbes) / 16; i += SOLVE_THREADS) dst[i] = src[i];
  }
  __syncthreads();
  // ---- 2. histogram state machine (HistogramBuilder), sequential over at most 2^log boundaries
  if (tid == 0) {
    uint32_t n_hist = 0, next_avail = 0, pos = 0;
    bool has_inc = false;
    uint32_t inc_count = 0;
    uint64_t inc_lower = 0, inc_upper = 0;
    uint64_t pos_val = sm.probes.first;
    auto apply_incomplete = [&](uint32_t cnt, uint64_t lo_v, uint64_t hi_v) {
      if (cnt == 0) return;
      if (has_inc) { inc_upper = hi_v; inc_count += cnt; }
      else { has_inc = true; inc_count = cnt; inc_lower = lo_v; inc_upper = hi_v; }
    };
    auto complete_bin = [&](uint32_t b) -> bool {
      if (!has_inc) return false;
      next_avail = b + 1;
      sm.h_count[n_hist] = inc_count; sm.h_lower[n_hist] = inc_lower; sm.h_upper[n_hist] = inc_upper;
      n_hist++;
      has_inc = false;
      return true;
    };
    while (pos < n) {
      uint32_t k = bin_idx_of(pos);
      uint32_t B = c_count_of(k);
      if (B >= n || sm.probes.vB1[k] != sm.probes.vB[k]) {
        apply_incomplete(B - pos, pos_val, sm.probes.vB1[k]);
        complete_bin(k);
        pos = B;
        pos_val = sm.probes.vB[k];
      } else {
        uint32_t l = sm.probes.runL[k], r = sm.probes.runR[k];
        uint64_t val = sm.probes.vB1[k];
        if (l > pos) apply_incomplete(l - pos, pos_val, sm.probes.vLm1[k]);
        // apply_constant_run (histograms.rs:142-161)
        uint32_t mid = l + (r - l) / 2;
        uint32_t b = bin_idx_of(mid);
        if (b > next_avail) {
          uint32_t spare = b - 1;
          if (!complete_bin(spare)) b = spare;
        }
        apply_incomplete(r - l, val, val);
        if (r >= c_count_of(b)) complete_bin(b);
        pos = r;
        pos_val = sm.probes.vR[k];
      }
    }
    sm.n_hist = n_hist;
  }
  __syncthreads();
  ENC_TICK(3);  // histogram state machine
  const uint32_t nh = sm.n_hist;
  // estimated_ans_size_log (chunk_compressor.rs:63-79)
  const uint32_t n_log_ceil = n <= 1 ? 0 : (32 - __clz(n - 1));
  const uint32_t est_size_log = min(min(n_bins_log + 2, 12u), n_log_ceil);
  // ---- 3. bin-merge DP (bin_optimization.rs:104-178)
  if (tid == 0) {
    uint32_t cc = 0;
    sm.c_counts[0] = 0;
    sm.best_cost[0] = 0.0f;
    for (uint32_t i = 0; i < nh; i++) { cc += sm.h_count[i]; sm.c_counts[i + 1] = cc; }
  }
  __syncthreads();
  const uint32_t total_count = sm.c_counts[nh];
  const float total_log2 = log2_approx_dev(__uint2float_rn(total_count));
  const float bin_meta_cost = __uint2float_rn(est_size_log + LBITS + offset_bits_bits(LBITS));
  for (uint32_t i = 0; i < nh; i++) {
    float my_cost = 3.402823466e+38f;
    uint32_t my_j = 0xffffffffu;
    const uint64_t upper = sm.h_upper[i];
    const uint32_t cci = sm.c_counts[i + 1];
    // each thread scans its js downward (strict <: the largest j wins ties)
    for (int j = int(i) - tid; j >= 0; j -= SOLVE_THREADS) {
      float cost = __fadd_rn(sm.best_cost[j], bin_cost_dev(bin_meta_cost, upper - sm.h_lower[j], cci - sm.c_counts[j], total_log2));
      if (cost < my_cost) { my_cost = cost; my_j = uint32_t(j); }
    }
    // argmin with "largest j among equal costs".  Costs are non-negative floats, so their bit patterns order like the values: per
    // warp two hardware reductions (REDUX) - the smallest cost, then the largest j among the lanes that hold it - and across the
    // warps one barrier per step (the per-warp results are double-buffered; thread 0, which writes best_cost[i + 1], is also the
    // only thread that reads it in step i + 1).
    const uint32_t cbits = my_j == 0xffffffffu ? 0xffffffffu : __float_as_uint(my_cost);
    const uint32_t cmin = __reduce_min_sync(0xffffffffu, cbits);
    const uint32_t jbest = __reduce_max_sync(0xffffffffu, (cbits == cmin && my_j != 0xffffffffu) ? my_j + 1u : 0u);
    if ((tid & 31) == 0) { sm.red_cost[i & 1][tid >> 5] = cmin; sm.red_j[i & 1][tid >> 5] = jbest; }
    __syncthreads();
    if (tid == 0) {
      uint32_t gmin = 0xffffffffu, gj = 0;
#pragma unroll
      for (int w = 0; w < SOLVE_THREADS / 32; w++) {
        const uint32_t cw = sm.red_cost[i & 1][w], jw = sm.red_j[i & 1][w];
        if (cw < gmin || (cw == gmin && jw > gj)) { gmin = cw; gj = jw; }
      }
      sm.best_cost[i + 1] = __uint_as_float(gmin);
      sm.best_j[i] = gj - 1u;
    }
  }
  ENC_TICK(4);  // DP
  // ---- 4. shortcuts, rewind, weights (thread 0: short sequential f32 sums whose order matters)
  if (tid == 0) {
    const float best = sm.best_cost[nh];
    const float slack = __fmul_rn(0.1f, __uint2float_rn(total_count));
    const float single = bin_cost_dev(bin_meta_cost, sm.h_upper[nh - 1] - sm.h_lower[0], total_count, total_log2);
    uint32_t n_opt = 0;
    bool done = false;
    if (single < __fadd_rn(best, slack)) {
      sm.o_lower[0] = sm.h_lower[0]; sm.o_upper[0] = sm.h_upper[nh - 1]; sm.o_count[0] = total_count;
      n_opt = 1;
      done = true;
    }
    if (!done) {
      bool all_trivial = true;
      for (uint32_t i = 0; i < nh; i++) if (sm.h_lower[i] != sm.h_upper[i]) { all_trivial = false; break; }
      if (all_trivial) {
        float cost = 0.0f;
        for (uint32_t i = 0; i < nh; i++) cost = __fadd_rn(cost, bin_cost_dev(bin_meta_cost, 0, sm.h_count[i], total_log2));
        if (cost < __fadd_rn(best, slack)) {
          for (uint32_t i = 0; i < nh; i++) { sm.o_lower[i] = sm.h_lower[i]; sm.o_upper[i] = sm.h_upper[i]; sm.o_count[i] = sm.h_count[i]; }
          n_opt = nh;
          done = true;
        }
      }
    }
    if (!done) {
      // rewind best_js into groups, last group first, then reverse
      uint32_t i = nh - 1;
      uint32_t cnt = 0;
      for (;;) {
        uint32_t j = sm.best_j[i];
        sm.o_lower[nh - 1 - cnt] = sm.h_lower[j];
        sm.o_upper[nh - 1 - cnt] = sm.h_upper[i];
        sm.o_count[nh - 1 - cnt] = sm.c_counts[i + 1] - sm.c_counts[j];
        cnt++;
        if (j > 0) i = j - 1; else break;
      }
      for (uint32_t q = 0; q < cnt; q++) {
        sm.o_lower[q] = sm.o_lower[nh - cnt + q]; sm.o_upper[q] = sm.o_upper[nh - cnt + q]; sm.o_count[q] = sm.o_count[nh - cnt + q];
      }
      n_opt = cnt;
    }
    for (uint32_t q = 0; q < n_opt; q++) sm.o_ob[q] = bits_to_encode_u64(sm.o_upper[q] - sm.o_lower[q]);
    sm.n_opt = n_opt;
    // ---- quantize_weights (ans/encoding.rs:95-175)
    uint32_t size_log;
    if (n_opt == 1) {
      size_log = 0;
      sm.weights[0] = 1;
    } else {
      uint32_t min_size_log = 32 - __clz(n_opt - 1);
      size_log = max(min_size_log, est_size_log);
      const uint32_t required = 1u << size_log;
      const float multiplier = __fdiv_rn(__uint2float_rn(required), __uint2float_rn(n));
      float desired_surplus = 0.0f;
      for (uint32_t q = 0; q < n_opt; q++) {
        float vv = __fsub_rn(__fmul_rn(__uint2float_rn(sm.o_count[q]), multiplier), 1.0f);
        vv = vv > 0.0f ? vv : 0.0f;
        sm.fweights[q] = vv;
        desired_surplus = __fadd_rn(desired_surplus, vv);
      }
      const uint32_t required_surplus = required - n_opt;
      const float surplus_mult = desired_surplus == 0.0f ? 0.0f : __fdiv_rn(__uint2float_rn(required_surplus), desired_surplus);
      uint32_t weight_sum = 0;
      for (uint32_t q = 0; q < n_opt; q++) {
        float fw = __fadd_rn(1.0f, __fmul_rn(sm.fweights[q], surplus_mult));
        sm.fweights[q] = fw;
        uint32_t w = __float2uint_rz(roundf(fw));
        sm.weights[q] = w;
        weight_sum += w;
      }
      uint32_t q = 0;
      while (weight_sum > required && q < n_opt) {
        if (sm.weights[q] > 1 && __uint2float_rn(sm.weights[q]) > sm.fweights[q]) { sm.weights[q] -= 1; weight_sum -= 1; }
        q += 1;
      }
      q = 0;
      while (weight_sum < required && q < n_opt) {
        if (__uint2float_rn(sm.weights[q]) < sm.fweights[q]) { sm.weights[q] += 1; weight_sum += 1; }
        q += 1;
      }
      uint32_t p2 = 32;
      for (uint32_t t = 0; t < n_opt; t++) p2 = min(p2, uint32_t(__ffs(sm.weights[t]) - 1));
      size_log -= p2;
      for (uint32_t t = 0; t < n_opt; t++) sm.weights[t] >>= p2;
    }
    sm.size_log = size_log;
    uint32_t cm = 0;
    uint64_t wc = 0;
    uint32_t max_ob = 0;
    float est = 0.0f;
    for (uint32_t t = 0; t < n_opt; t++) {
      sm.cum[t] = cm;
      cm += sm.weights[t];
      wc += uint64_t(sm.o_count[t]) * (sm.o_ob[t] + size_log - (31 - __clz(sm.weights[t])));  // bin.rs:25-27
      est += float(sm.o_count[t]) * (float(sm.o_ob[t] + size_log) - __log2f(float(sm.weights[t])));
      max_ob = max(max_ob, sm.o_ob[t]);
    }
    sm.cum[n_opt] = cm;
    plan.n_bins = n_opt;
    plan.size_log = size_log;
    plan.max_ob = max_ob;
    plan.n_lat = n;
    plan.wc_bits = wc;
    plan.est_bits = uint64_t(est);
  }
  __syncthreads();
  ENC_TICK(5);  // rewind + quantize
  const uint32_t n_opt = sm.n_opt, size_log = sm.size_log, size = 1u << size_log;
  const uint64_t lmask = LBITS == 64 ? ~uint64_t(0) : ((uint64_t(1) << LBITS) - 1);
  for (uint32_t q = tid; q < n_opt; q += SOLVE_THREADS) {
    plan.lower[q] = (sm.o_lower[q] + vmin) & lmask;
    plan.ob[q] = uint8_t(sm.o_ob[q]);
    plan.weight[q] = uint16_t(sm.weights[q]);
    sm.rank_counter[q] = 0;
    // SymbolInfo (ans/encoding.rs:36-49)
    uint32_t w = sm.weights[q];
    uint32_t max_x_s = 2 * w - 1;
    uint32_t min_renorm = size_log - (31 - __clz(max_x_s));
    uint32_t cutoff = (2 * w) << min_renorm;
    plan.syminfo[q] = uint64_t(cutoff) | (uint64_t(min_renorm) << 16) | (uint64_t(w) << 24) | (uint64_t(sm.cum[q]) << 40);
  }
  // spread (ans/spec.rs:37-59) and per-symbol ascending state lists (ans/encoding.rs:51-55)
  uint32_t stride = (3 * size) / 5;
  if ((stride & 1) == 0) stride += 1;
  for (uint32_t t = tid; t < size; t += SOLVE_THREADS) {
    uint32_t lo = 0, hi = n_opt;
    while (hi - lo > 1) { uint32_t m = (lo + hi) >> 1; if (sm.cum[m] <= t) lo = m; else hi = m; }
    sm.sym_of_state[(stride * t) & (size - 1)] = uint16_t(lo);
  }
  __syncthreads();
  if (tid < 32) {
    const uint32_t lane = tid;
    for (uint32_t base = 0; base < size; base += 32) {
      uint32_t st = base + lane;
      bool active = st < size;
      uint32_t sym = active ? sm.sym_of_state[st] : 0xffffffffu;
      uint32_t m = __match_any_sync(0xffffffffu, sym);
      uint32_t in_group = __popc(m & ((1u << lane) - 1));
      uint32_t prev = active ? sm.rank_counter[sym] : 0;
      __syncwarp();
      if (active && in_group == 0) sm.rank_counter[sym] = prev + __popc(m);
      __syncwarp();
      if (active) plan.next_states[sm.cum[sym] + prev + in_group] = uint16_t(st);  // state = size + st
    }
  }
  ENC_TICK(6);  // tables
}

// ---------------------------------------------------------------------------
// plan_solve_wide_kernel: plan_solve_kernel for runs with more than 256 unoptimized bins (levels 9-12: up to 4096 bins, tables of up
// to 2^12 states).  The same steps in the same f32 arithmetic and order; what differs is where the arrays live, since PlanSmem at 4096
// bins would not fit shared memory.  The DP's hot arrays (bin bounds, cumulative counts, best costs: 96 KB) are in dynamic shared
// memory.  The histogram state machine reads the probes from HBM (k only grows, so most loads hit L1), and once the histogram exists
// the chunk's probe slot is dead: it holds the rest (best_js, optimized bins, weights, spread) as WideSolveScratch.  WSOLVE_THREADS
// threads share each DP step's candidates (O(B^2) in all, like bin_optimization.rs:104-178).
// ---------------------------------------------------------------------------
constexpr int WSOLVE_THREADS = 256;
constexpr int WMAXB = EncCap<true>::MAXB;
struct WideSolveScratch {
  uint32_t best_j[WMAXB];
  uint32_t o_count[WMAXB];
  uint64_t o_lower[WMAXB];
  uint8_t o_ob[WMAXB];
  float fweights[WMAXB];
  uint32_t weights[WMAXB];
  uint32_t cum[WMAXB + 1];
  uint16_t sym_of_state[1 << EncCap<true>::MAX_SIZE_LOG];
  uint32_t rank_counter[WMAXB];
};
static_assert(sizeof(WideSolveScratch) <= sizeof(PlanProbesT<true>), "the wide solver's scratch reuses the chunk's probe slot");
struct WideSolveSmem {
  uint64_t h_lower[WMAXB], h_upper[WMAXB];
  uint32_t c_counts[WMAXB + 1];  // c_counts[i + 1] - c_counts[i] = count of unoptimized bin i
  float best_cost[WMAXB + 1];
  uint32_t red_cost[2][WSOLVE_THREADS / 32], red_j[2][WSOLVE_THREADS / 32];
  uint32_t n_hist, n_opt, size_log;
};

template <typename L>
__global__ void __launch_bounds__(WSOLVE_THREADS) plan_solve_wide_kernel(EncParams ep, PlanProbesT<true>* probes, const ChunkEnc* __restrict__ chunks,
                                                                         VarPlanT<true>* __restrict__ plans, int v, uint32_t n_override = 0) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  WideSolveSmem& sm = *reinterpret_cast<WideSolveSmem*>(smem_raw);
  const uint32_t c = blockIdx.x;
  const int tid = threadIdx.x;
  const uint64_t cs = ep.chunk_starts[c], ce = ep.chunk_starts[c + 1];
  const uint64_t sb = stored_begin(cs, ce, v == 0 ? ep.order : 0);
  const uint32_t n = n_override ? n_override : uint32_t(ce - sb);
  VarPlanT<true>& plan = plans[size_t(c) * MAX_VARS + v];
  const uint64_t vmin = chunks[c].vmin[v];
  constexpr uint32_t LBITS = LT<L>::BITS;
  if (n == 0) {
    if (tid == 0) { plan.n_bins = 0; plan.size_log = 0; plan.max_ob = 0; plan.n_lat = 0; plan.wc_bits = 0; plan.est_bits = 0; plan.next_states[0] = 0; }
    return;
  }
  const uint32_t n_bins_log = ep.bins_log[v];
  const uint32_t nbk = 1u << n_bins_log;
  // (cc << n_bins_log) < 2^36: plain 64-bit division (the narrow solver's float shortcut assumes n_bins_log <= 8)
  auto bin_idx_of = [&](uint64_t cc) -> uint32_t { return uint32_t((cc << n_bins_log) / n); };
  auto c_count_of = [&](uint32_t b) -> uint32_t { return uint32_t((uint64_t(b + 1) * n + nbk - 1) >> n_bins_log); };
  const PlanProbesT<true>& pr = probes[c];
  WideSolveScratch& ws = *reinterpret_cast<WideSolveScratch*>(&probes[c]);
  // ---- histogram state machine (HistogramBuilder), as in plan_solve_kernel
  if (tid == 0) {
    uint32_t n_hist = 0, next_avail = 0, pos = 0, cc = 0;
    bool has_inc = false;
    uint32_t inc_count = 0;
    uint64_t inc_lower = 0, inc_upper = 0;
    uint64_t pos_val = pr.first;
    sm.c_counts[0] = 0;
    sm.best_cost[0] = 0.0f;
    auto apply_incomplete = [&](uint32_t cnt, uint64_t lo_v, uint64_t hi_v) {
      if (cnt == 0) return;
      if (has_inc) { inc_upper = hi_v; inc_count += cnt; }
      else { has_inc = true; inc_count = cnt; inc_lower = lo_v; inc_upper = hi_v; }
    };
    auto complete_bin = [&](uint32_t b) -> bool {
      if (!has_inc) return false;
      next_avail = b + 1;
      cc += inc_count;
      sm.c_counts[n_hist + 1] = cc; sm.h_lower[n_hist] = inc_lower; sm.h_upper[n_hist] = inc_upper;
      n_hist++;
      has_inc = false;
      return true;
    };
    while (pos < n) {
      uint32_t k = bin_idx_of(pos);
      uint32_t B = c_count_of(k);
      if (B >= n || pr.vB1[k] != pr.vB[k]) {
        apply_incomplete(B - pos, pos_val, pr.vB1[k]);
        complete_bin(k);
        pos = B;
        pos_val = pr.vB[k];
      } else {
        uint32_t l = pr.runL[k], r = pr.runR[k];
        uint64_t val = pr.vB1[k];
        if (l > pos) apply_incomplete(l - pos, pos_val, pr.vLm1[k]);
        uint32_t mid = l + (r - l) / 2;
        uint32_t b = bin_idx_of(mid);
        if (b > next_avail) {
          uint32_t spare = b - 1;
          if (!complete_bin(spare)) b = spare;
        }
        apply_incomplete(r - l, val, val);
        if (r >= c_count_of(b)) complete_bin(b);
        pos = r;
        pos_val = pr.vR[k];
      }
    }
    sm.n_hist = n_hist;
  }
  __syncthreads();  // the probes are dead from here on: their slot becomes `ws`
  const uint32_t nh = sm.n_hist;
  const uint32_t n_log_ceil = n <= 1 ? 0 : (32 - __clz(n - 1));
  const uint32_t est_size_log = min(min(n_bins_log + 2, 12u), n_log_ceil);
  // ---- bin-merge DP (bin_optimization.rs:104-178); argmin per step with "largest j among equal costs", as in plan_solve_kernel
  const uint32_t total_count = sm.c_counts[nh];
  const float total_log2 = log2_approx_dev(__uint2float_rn(total_count));
  const float bin_meta_cost = __uint2float_rn(est_size_log + LBITS + offset_bits_bits(LBITS));
  for (uint32_t i = 0; i < nh; i++) {
    float my_cost = 3.402823466e+38f;
    uint32_t my_j = 0xffffffffu;
    const uint64_t upper = sm.h_upper[i];
    const uint32_t cci = sm.c_counts[i + 1];
    for (int j = int(i) - tid; j >= 0; j -= WSOLVE_THREADS) {
      float cost = __fadd_rn(sm.best_cost[j], bin_cost_dev(bin_meta_cost, upper - sm.h_lower[j], cci - sm.c_counts[j], total_log2));
      if (cost < my_cost) { my_cost = cost; my_j = uint32_t(j); }
    }
    const uint32_t cbits = my_j == 0xffffffffu ? 0xffffffffu : __float_as_uint(my_cost);
    const uint32_t cmin = __reduce_min_sync(0xffffffffu, cbits);
    const uint32_t jbest = __reduce_max_sync(0xffffffffu, (cbits == cmin && my_j != 0xffffffffu) ? my_j + 1u : 0u);
    if ((tid & 31) == 0) { sm.red_cost[i & 1][tid >> 5] = cmin; sm.red_j[i & 1][tid >> 5] = jbest; }
    __syncthreads();
    if (tid == 0) {
      uint32_t gmin = 0xffffffffu, gj = 0;
#pragma unroll
      for (int w = 0; w < WSOLVE_THREADS / 32; w++) {
        const uint32_t cw = sm.red_cost[i & 1][w], jw = sm.red_j[i & 1][w];
        if (cw < gmin || (cw == gmin && jw > gj)) { gmin = cw; gj = jw; }
      }
      sm.best_cost[i + 1] = __uint_as_float(gmin);
      ws.best_j[i] = gj - 1u;
    }
  }
  // ---- shortcuts, rewind, weights (thread 0, as in plan_solve_kernel)
  if (tid == 0) {
    const float best = sm.best_cost[nh];
    const float slack = __fmul_rn(0.1f, __uint2float_rn(total_count));
    const float single = bin_cost_dev(bin_meta_cost, sm.h_upper[nh - 1] - sm.h_lower[0], total_count, total_log2);
    uint32_t n_opt = 0;
    bool done = false;
    if (single < __fadd_rn(best, slack)) {
      ws.o_lower[0] = sm.h_lower[0]; ws.o_count[0] = total_count; ws.o_ob[0] = uint8_t(bits_to_encode_u64(sm.h_upper[nh - 1] - sm.h_lower[0]));
      n_opt = 1;
      done = true;
    }
    if (!done) {
      bool all_trivial = true;
      for (uint32_t i = 0; i < nh; i++) if (sm.h_lower[i] != sm.h_upper[i]) { all_trivial = false; break; }
      if (all_trivial) {
        float cost = 0.0f;
        for (uint32_t i = 0; i < nh; i++) cost = __fadd_rn(cost, bin_cost_dev(bin_meta_cost, 0, sm.c_counts[i + 1] - sm.c_counts[i], total_log2));
        if (cost < __fadd_rn(best, slack)) {
          for (uint32_t i = 0; i < nh; i++) { ws.o_lower[i] = sm.h_lower[i]; ws.o_count[i] = sm.c_counts[i + 1] - sm.c_counts[i]; ws.o_ob[i] = 0; }
          n_opt = nh;
          done = true;
        }
      }
    }
    if (!done) {
      uint32_t i = nh - 1;
      uint32_t cnt = 0;
      for (;;) {
        uint32_t j = ws.best_j[i];
        ws.o_lower[nh - 1 - cnt] = sm.h_lower[j];
        ws.o_ob[nh - 1 - cnt] = uint8_t(bits_to_encode_u64(sm.h_upper[i] - sm.h_lower[j]));
        ws.o_count[nh - 1 - cnt] = sm.c_counts[i + 1] - sm.c_counts[j];
        cnt++;
        if (j > 0) i = j - 1; else break;
      }
      for (uint32_t q = 0; q < cnt; q++) {
        ws.o_lower[q] = ws.o_lower[nh - cnt + q]; ws.o_ob[q] = ws.o_ob[nh - cnt + q]; ws.o_count[q] = ws.o_count[nh - cnt + q];
      }
      n_opt = cnt;
    }
    sm.n_opt = n_opt;
    // ---- quantize_weights (ans/encoding.rs:95-175)
    uint32_t size_log;
    if (n_opt == 1) {
      size_log = 0;
      ws.weights[0] = 1;
    } else {
      uint32_t min_size_log = 32 - __clz(n_opt - 1);
      size_log = max(min_size_log, est_size_log);
      const uint32_t required = 1u << size_log;
      const float multiplier = __fdiv_rn(__uint2float_rn(required), __uint2float_rn(n));
      float desired_surplus = 0.0f;
      for (uint32_t q = 0; q < n_opt; q++) {
        float vv = __fsub_rn(__fmul_rn(__uint2float_rn(ws.o_count[q]), multiplier), 1.0f);
        vv = vv > 0.0f ? vv : 0.0f;
        ws.fweights[q] = vv;
        desired_surplus = __fadd_rn(desired_surplus, vv);
      }
      const uint32_t required_surplus = required - n_opt;
      const float surplus_mult = desired_surplus == 0.0f ? 0.0f : __fdiv_rn(__uint2float_rn(required_surplus), desired_surplus);
      uint32_t weight_sum = 0;
      for (uint32_t q = 0; q < n_opt; q++) {
        float fw = __fadd_rn(1.0f, __fmul_rn(ws.fweights[q], surplus_mult));
        ws.fweights[q] = fw;
        uint32_t w = __float2uint_rz(roundf(fw));
        ws.weights[q] = w;
        weight_sum += w;
      }
      uint32_t q = 0;
      while (weight_sum > required && q < n_opt) {
        if (ws.weights[q] > 1 && __uint2float_rn(ws.weights[q]) > ws.fweights[q]) { ws.weights[q] -= 1; weight_sum -= 1; }
        q += 1;
      }
      q = 0;
      while (weight_sum < required && q < n_opt) {
        if (__uint2float_rn(ws.weights[q]) < ws.fweights[q]) { ws.weights[q] += 1; weight_sum += 1; }
        q += 1;
      }
      uint32_t p2 = 32;
      for (uint32_t t = 0; t < n_opt; t++) p2 = min(p2, uint32_t(__ffs(ws.weights[t]) - 1));
      size_log -= p2;
      for (uint32_t t = 0; t < n_opt; t++) ws.weights[t] >>= p2;
    }
    sm.size_log = size_log;
    uint32_t cm = 0;
    uint64_t wc = 0;
    uint32_t max_ob = 0;
    float est = 0.0f;
    for (uint32_t t = 0; t < n_opt; t++) {
      ws.cum[t] = cm;
      cm += ws.weights[t];
      wc += uint64_t(ws.o_count[t]) * (ws.o_ob[t] + size_log - (31 - __clz(ws.weights[t])));  // bin.rs:25-27
      est += float(ws.o_count[t]) * (float(ws.o_ob[t] + size_log) - __log2f(float(ws.weights[t])));
      max_ob = max(max_ob, uint32_t(ws.o_ob[t]));
    }
    ws.cum[n_opt] = cm;
    plan.n_bins = n_opt;
    plan.size_log = size_log;
    plan.max_ob = max_ob;
    plan.n_lat = n;
    plan.wc_bits = wc;
    plan.est_bits = uint64_t(est);
  }
  __syncthreads();
  const uint32_t n_opt = sm.n_opt, size_log = sm.size_log, size = 1u << size_log;
  const uint64_t lmask = LBITS == 64 ? ~uint64_t(0) : ((uint64_t(1) << LBITS) - 1);
  for (uint32_t q = tid; q < n_opt; q += WSOLVE_THREADS) {
    plan.lower[q] = (ws.o_lower[q] + vmin) & lmask;
    plan.ob[q] = ws.o_ob[q];
    plan.weight[q] = uint16_t(ws.weights[q]);
    ws.rank_counter[q] = 0;
    // SymbolInfo (ans/encoding.rs:36-49); cutoff <= 2^13 and cum < 2^12 fit their fields
    uint32_t w = ws.weights[q];
    uint32_t max_x_s = 2 * w - 1;
    uint32_t min_renorm = size_log - (31 - __clz(max_x_s));
    uint32_t cutoff = (2 * w) << min_renorm;
    plan.syminfo[q] = uint64_t(cutoff) | (uint64_t(min_renorm) << 16) | (uint64_t(w) << 24) | (uint64_t(ws.cum[q]) << 40);
  }
  // spread (ans/spec.rs:37-59) and per-symbol ascending state lists (ans/encoding.rs:51-55)
  uint32_t stride = (3 * size) / 5;
  if ((stride & 1) == 0) stride += 1;
  for (uint32_t t = tid; t < size; t += WSOLVE_THREADS) {
    uint32_t lo = 0, hi = n_opt;
    while (hi - lo > 1) { uint32_t m = (lo + hi) >> 1; if (ws.cum[m] <= t) lo = m; else hi = m; }
    ws.sym_of_state[(stride * t) & (size - 1)] = uint16_t(lo);
  }
  __syncthreads();
  if (tid < 32) {
    const uint32_t lane = tid;
    for (uint32_t base = 0; base < size; base += 32) {
      uint32_t st = base + lane;
      bool active = st < size;
      uint32_t sym = active ? ws.sym_of_state[st] : 0xffffffffu;
      uint32_t m = __match_any_sync(0xffffffffu, sym);
      uint32_t in_group = __popc(m & ((1u << lane) - 1));
      uint32_t prev = active ? ws.rank_counter[sym] : 0;
      __syncwarp();
      if (active && in_group == 0) ws.rank_counter[sym] = prev + __popc(m);
      __syncwarp();
      if (active) plan.next_states[ws.cum[sym] + prev + in_group] = uint16_t(st);  // state = size + st
    }
  }
}

// ---------------------------------------------------------------------------
// DeltaSpec::Auto on the GPU path: the reference (chunk_compressor.rs:310-360) trial-compresses a sample of each chunk -
// groups of 200 consecutive numbers at a regular stride (sampling.rs:21-60) - with consecutive orders 1, 2, ... until the
// estimated size stops shrinking (and with Lookback, which this path does not encode).  Here the same sample of every
// chunk's PRIMARY latents is gathered into a side array (gather_primary_sample_kernel, compress_host.cuh), the ordinary split/delta +
// planner kernels run on it per order, and the host evaluates the reference's f32 size formula per chunk (sample_cost): every chunk gets its
// own order.
// ---------------------------------------------------------------------------
struct SampleGeom { uint32_t group_n, n_groups, stride; };
__host__ __device__ inline SampleGeom delta_sample_geom(uint64_t n) {
  SampleGeom g{0, 0, 0};
  if (n < 10) return g;                                   // sampling.rs:14-20 calc_sample_n
  const uint64_t target = 10 + (n - 10) / 40;
  g.group_n = uint32_t(n < 200 ? n : 200);                // DELTA_TARGET_GROUP_N
  g.n_groups = uint32_t((target + 199) / 200);
  const uint64_t nominal = uint64_t(g.n_groups) * g.group_n;
  const uint64_t spare = n > nominal ? n - nominal : 0;
  g.stride = uint32_t(g.group_n + spare / ((g.n_groups > 2 ? g.n_groups : 2) - 1));
  return g;
}

// ---------------------------------------------------------------------------
// should_fallback (chunk_compressor.rs:502-541): one thread per chunk
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t var_meta_bits(uint32_t n_bins, uint32_t size_log, uint32_t lbits) {
  return 4 + 15 + n_bins * (size_log + lbits + offset_bits_bits(lbits));
}
__device__ __forceinline__ uint32_t mode_payload_bits(uint32_t mode, uint32_t lbits) {
  return mode == MODE_CLASSIC ? 0 : mode == MODE_FLOAT_QUANT ? 8 : lbits;
}

// shared_pages = 0: every chunk of the call is its own wrapped chunk with one page.  shared_pages = P > 0: the call's P
// "chunks" are the pages of ONE wrapped chunk (bins in plans[0], trained on all pages): one decision for all of them.
template <bool WIDE = false>
__global__ void fallback_kernel(EncParams ep, const VarPlanT<WIDE>* __restrict__ plans, ChunkEnc* __restrict__ chunks, uint32_t shared_pages = 0) {
  uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t lbits = nt_bits(ep.dtype);
  if (shared_pages) {
    if (c != 0) return;
    const uint64_t n = ep.chunk_starts[shared_pages] - ep.chunk_starts[0];
    uint32_t fb = 0;
    if (!(ep.order == 0 && ep.mode == MODE_CLASSIC)) {
      const VarPlanT<WIDE>& p = plans[0];
      const uint64_t wc_bits = 7ull * shared_pages + p.wc_bits;
      const uint64_t meta_bits = 4 + mode_payload_bits(ep.mode, lbits) + (4 + 5 + 5 + 64 + 32 * 32) + var_meta_bits(p.n_bins, p.size_log, lbits);
      const uint64_t page_meta_bits = 4 * p.size_log + uint64_t(lbits) * ep.order;
      const uint64_t worst = (meta_bits + 7) / 8 + shared_pages * ((page_meta_bits + 7) / 8) + (wc_bits + 7) / 8;
      const uint64_t baseline_meta_bits = 4 + (4 + 5 + 5 + 64 + 32 * 32) + 4 + 15 + (lbits + offset_bits_bits(lbits));
      const uint64_t baseline = (baseline_meta_bits + 7) / 8 + (n * lbits + 7) / 8;
      fb = worst > baseline ? 1 : 0;
    }
    for (uint32_t q = 0; q < shared_pages; q++) chunks[q].fallback = fb;
    return;
  }
  if (c >= ep.n_chunks) return;
  const uint64_t n = ep.chunk_starts[c + 1] - ep.chunk_starts[c];
  uint32_t fb = 0;
  if (!(ep.order == 0 && ep.mode == MODE_CLASSIC)) {
    uint64_t wc_bits = 7;  // 7 * n_pages
    uint64_t meta_bits = 4 + mode_payload_bits(ep.mode, lbits) + (4 + 5 + 5 + 64 + 32 * 32);  // mode.max_bit_size + DeltaEncoding::MAX_BIT_SIZE
    uint64_t page_meta_bits = 0;
    for (uint32_t v = 0; v < ep.n_vars; v++) {
      const VarPlanT<WIDE>& p = plans[size_t(c) * MAX_VARS + v];
      wc_bits += p.wc_bits;
      meta_bits += var_meta_bits(p.n_bins, p.size_log, lbits);
      page_meta_bits += 4 * p.size_log + uint64_t(lbits) * (v == 0 ? ep.order : 0);
    }
    uint64_t worst = (meta_bits + 7) / 8 + (page_meta_bits + 7) / 8 + (wc_bits + 7) / 8;
    uint64_t baseline_meta_bits = 4 + (4 + 5 + 5 + 64 + 32 * 32) + 4 + 15 + (lbits + offset_bits_bits(lbits));
    uint64_t baseline = (baseline_meta_bits + 7) / 8 + (n * lbits + 7) / 8;
    fb = worst > baseline ? 1 : 0;
  }
  chunks[c].fallback = fb;
}

// ---------------------------------------------------------------------------
// K3: bin search.  One warp per batch; writes the symbol of every stored latent and the batch's offset-bit sum.
// Batch b of var v covers stored latents [256 b, 256 b + 256) of the var's stored range.
// ---------------------------------------------------------------------------
constexpr int BIN_THREADS = 256;

template <typename L>
__device__ __forceinline__ L fallback_latent(const EncParams& ep, uint64_t g) {
  return to_latent_ordered<L>(static_cast<const L*>(ep.nums)[g], nt_is_float(ep.dtype), nt_is_signed(ep.dtype));
}

template <typename L, bool WIDE = false>
__global__ void __launch_bounds__(BIN_THREADS) bin_kernel(EncParams ep, uint32_t batches_per_chunk, const L* __restrict__ lat, const VarPlanT<WIDE>* __restrict__ plans,
                                                           const ChunkEnc* __restrict__ chunks, typename EncCap<WIDE>::Sym* __restrict__ sym,
                                                           uint32_t* __restrict__ ob_sum, int v) {
  __shared__ uint64_t lowers[EncCap<WIDE>::MAXB];
  __shared__ uint8_t obs[EncCap<WIDE>::MAXB];
  // one CTA handles 8 consecutive batches of one chunk
  const uint32_t groups_per_chunk = (batches_per_chunk + 7) / 8;
  const uint32_t c = blockIdx.x / groups_per_chunk, grp = blockIdx.x % groups_per_chunk;
  const uint64_t cs = ep.chunk_starts[c], ce = ep.chunk_starts[c + 1];
  const bool fb = chunks[c].fallback != 0;
  if (fb && v > 0) return;
  const uint64_t sb = fb ? cs : stored_begin(cs, ce, v == 0 ? ep.order : 0);
  const uint64_t rb = ep.row_base[c];
  const uint32_t n = uint32_t(ce - sb);
  const uint32_t b = grp * 8 + (threadIdx.x >> 5);
  const VarPlanT<WIDE>& plan = plans[size_t(c) * MAX_VARS + v];
  const uint32_t n_bins = fb ? 1 : plan.n_bins;
  for (int i = threadIdx.x; i < int(n_bins); i += BIN_THREADS) {
    lowers[i] = fb ? 0 : plan.lower[i];
    obs[i] = fb ? uint8_t(LT<L>::BITS) : plan.ob[i];
  }
  __syncthreads();
  if (uint64_t(b) * BATCH_N >= n) return;
  const int lane = threadIdx.x & 31;
  const uint32_t cnt = min(uint32_t(BATCH_N), n - b * BATCH_N);
  uint32_t search_log = n_bins <= 1 ? 0 : (32 - __clz(n_bins - 1));
  uint32_t bits = 0;
  uint32_t packed[2] = {0, 0};
#pragma unroll
  for (int e = 0; e < 8; e++) {
    uint32_t i = lane * 8 + e;
    uint32_t sidx = 0;
    if (i < cnt) {
      uint64_t k = uint64_t(b) * BATCH_N + i;
      uint64_t l = fb ? uint64_t(fallback_latent<L>(ep, cs + k)) : uint64_t(lat[rb + k]);
      // compression_table.rs:51-74: balanced search over lowers padded with MAX, then clamp
      for (uint32_t depth = 0; depth < search_log; depth++) {
        uint32_t bis = 1u << (search_log - 1 - depth);
        uint32_t cand = sidx + bis;
        // padding entries (L::MAX in the reference) can only move the index past n_bins - 1, which the clamp undoes
        bool ge = cand < n_bins && l >= lowers[cand];
        sidx += ge ? bis : 0;
      }
      if (n_bins > 0) sidx = min(sidx, n_bins - 1);
      bits += obs[sidx];
    }
    if constexpr (WIDE) {
      if (i < cnt) sym[rb + uint64_t(b) * BATCH_N + i] = uint16_t(sidx);  // 16-bit symbols
    } else {
      packed[e >> 2] |= sidx << (8 * (e & 3));
    }
  }
  if constexpr (!WIDE) {
    uint8_t* row = sym + rb + uint64_t(b) * BATCH_N;
#pragma unroll
    for (int e = 0; e < 8; e++) {
      uint32_t i = lane * 8 + e;
      if (i < cnt) row[i] = uint8_t(packed[e >> 2] >> (8 * (e & 3)));
    }
  }
  for (int d = 16; d > 0; d >>= 1) bits += __shfl_xor_sync(0xffffffffu, bits, d);
  if (lane == 0) ob_sum[(size_t(c) * MAX_VARS + v) * batches_per_chunk + b] = bits;
}

// Narrow key range (the counting-planner case, keys < 2^range_bits <= 2^15): the bin of a latent is a direct lookup in a
// per-chunk shared-memory table key -> bin (marks at every bin's lower bound, then a running max), instead of a
// search_log-deep binary search per latent.  One CTA bins BINL_BATCHES batches of one chunk, one warp per batch,
// lanes striding the batch so that every load is a fully used 256-byte line.
constexpr int BINL_THREADS = 256;
#ifndef PCOB_BINL_BATCHES
#define PCOB_BINL_BATCHES 512
#endif
constexpr int BINL_BATCHES = PCOB_BINL_BATCHES;  // batches per CTA: every CTA rebuilds the chunk's lookup table first (512 beat 128, 256 and 1024 on C2)

template <typename L>
__global__ void __launch_bounds__(BINL_THREADS) bin_lut_kernel(EncParams ep, uint32_t batches_per_chunk, uint32_t parts_per_chunk,
                                                                const uint16_t* __restrict__ keys16, const VarPlan* __restrict__ plans,
                                                                const ChunkEnc* __restrict__ chunks, uint8_t* __restrict__ sym,
                                                                uint32_t* __restrict__ ob_sum, int v, uint32_t range_bits) {
  extern __shared__ __align__(16) unsigned char binl_smem[];
  uint32_t* lut_w = reinterpret_cast<uint32_t*>(binl_smem);  // 2^range_bits bytes, 4 keys per word
  uint8_t* lut = binl_smem;
  __shared__ uint8_t obs[ENC_MAXB];
  __shared__ uint32_t warp_top[BINL_THREADS / 32];
  const uint32_t c = blockIdx.x / parts_per_chunk, part = blockIdx.x % parts_per_chunk;
  const uint64_t cs = ep.chunk_starts[c], ce = ep.chunk_starts[c + 1];
  const bool fb = chunks[c].fallback != 0;
  if (fb && v > 0) return;
  const uint64_t sb = fb ? cs : stored_begin(cs, ce, v == 0 ? ep.order : 0);
  const uint64_t rb = ep.row_base[c];
  const uint32_t n = uint32_t(ce - sb);
  const uint32_t b_begin = part * BINL_BATCHES;
  if (uint64_t(b_begin) * BATCH_N >= n) return;
  const uint32_t b_end = min(b_begin + BINL_BATCHES, n_batches_of(n));
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint32_t* sums = ob_sum + (size_t(c) * MAX_VARS + v) * batches_per_chunk;
  if (fb) {
    // one bin of L::BITS offset bits (chunk_compressor.rs:502-541): every symbol is 0
    for (uint32_t b = b_begin + warp; b < b_end; b += BINL_THREADS / 32) {
      const uint32_t cnt = min(uint32_t(BATCH_N), n - b * BATCH_N);
      uint8_t* row = sym + rb + uint64_t(b) * BATCH_N;
      for (uint32_t i = lane; i < cnt; i += 32) row[i] = 0;
      if (lane == 0) sums[b] = cnt * LT<L>::BITS;
    }
    return;
  }
  const VarPlan& plan = plans[size_t(c) * MAX_VARS + v];
  const uint32_t n_bins = plan.n_bins;
  const L vmin = L(chunks[c].vmin[v]);
  const uint32_t shift2 = (uint32_t(chunks[c].vmin[v] - chunks[c].key_base[v]) & 0xffffu) * 0x10001u;
  const uint32_t n_words = max(1u, (1u << range_bits) / 4);
  for (uint32_t i = tid; i < n_words; i += BINL_THREADS) lut_w[i] = 0;
  for (uint32_t i = tid; i < n_bins; i += BINL_THREADS) obs[i] = plan.ob[i];
  __syncthreads();
  for (uint32_t i = tid; i < n_bins; i += BINL_THREADS) lut[uint32_t(L(L(plan.lower[i]) - vmin))] = uint8_t(i);  // lowers are strictly increasing
  __syncthreads();
  {
    // running max over the marks: warp w owns a contiguous span of words and walks it 32 words at a time
    const uint32_t span = (n_words + BINL_THREADS / 32 - 1) / (BINL_THREADS / 32);
    const uint32_t w_lo = min(n_words, warp * span), w_hi = min(n_words, w_lo + span);
    uint32_t carry = 0;  // max bin index seen so far in this warp's span
    for (uint32_t base = w_lo; base < w_hi; base += 32) {
      const uint32_t idx = base + lane;
      uint32_t x = idx < w_hi ? lut_w[idx] : 0u;
      x = __vmaxu4(x, x << 8);
      x = __vmaxu4(x, x << 16);  // byte k = max of bytes 0..k
      uint32_t top = x >> 24;
      uint32_t inc = top;
      for (int d = 1; d < 32; d <<= 1) { uint32_t o = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc = max(inc, o); }
      uint32_t before = __shfl_up_sync(0xffffffffu, inc, 1);
      before = lane == 0 ? carry : max(before, carry);
      x = __vmaxu4(x, before * 0x01010101u);
      if (idx < w_hi) lut_w[idx] = x;
      carry = max(carry, __shfl_sync(0xffffffffu, inc, 31));
    }
    if (lane == 0) warp_top[warp] = carry;
    __syncthreads();
    uint32_t prev = 0;
    for (int w = 0; w < warp; w++) prev = max(prev, warp_top[w]);
    const uint32_t prev4 = prev * 0x01010101u;
    for (uint32_t idx = w_lo + lane; idx < w_hi; idx += 32) lut_w[idx] = __vmaxu4(lut_w[idx], prev4);
    __syncthreads();
  }
  for (uint32_t b = b_begin + warp; b < b_end; b += BINL_THREADS / 32) {
    const uint32_t cnt = min(uint32_t(BATCH_N), n - b * BATCH_N);
    // the keys the counting planner left behind (latent - chunk minimum, 16 bits): a lane owns 8 consecutive ones
    const uint4 k8 = *reinterpret_cast<const uint4*>(keys16 + rb + uint64_t(b) * BATCH_N + lane * 8);
    // stored keys are (latent - key_base) mod 2^16; the table is indexed by latent - vmin
    const uint32_t kw[4] = {__vsub2(k8.x, shift2), __vsub2(k8.y, shift2), __vsub2(k8.z, shift2), __vsub2(k8.w, shift2)};
    uint32_t bits = 0, lo = 0, hi = 0;
#pragma unroll
    for (int e = 0; e < 8; e++) {
      const uint32_t key = (kw[e >> 1] >> (16 * (e & 1))) & (n_words * 4 - 1);  // past the batch's count: stale bits, kept in range
      const uint32_t sidx = lut[key];
      if (uint32_t(lane * 8 + e) < cnt) bits += obs[sidx];
      if (e < 4) lo |= sidx << (8 * e); else hi |= sidx << (8 * (e - 4));
    }
    *reinterpret_cast<uint2*>(sym + rb + uint64_t(b) * BATCH_N + lane * 8) = make_uint2(lo, hi);  // rows are 256-aligned and padded
    for (int d = 16; d > 0; d >>= 1) bits += __shfl_xor_sync(0xffffffffu, bits, d);
    if (lane == 0) sums[b] = bits;
  }
}

// ---------------------------------------------------------------------------
// K4: reverse tANS.  One warp per (chunk, var); lanes 0-3 carry the 4 interleaved states over the whole page
// (latency-bound serial chains); all lanes stage symbols in and results out.
// Output per latent: u16 = ans_val | ans_bits << 12  (ans_bits <= ENC_MAX_SIZE_LOG = 10)
// ---------------------------------------------------------------------------
// The encoder state chain of a page is serial (each step's state feeds the next, 2^16 steps per chain), but a tANS
// step with a symbol of weight w maps all 2^size_log states onto w values, so two trajectories that start from different
// states over the same symbols merge after some steps (tens for typical bins) and are identical from there on.  The
// kernel uses that: the page is cut into up to 64 segments of whole batches, one group of 4 threads (the 4 interleaved
// chains) per segment, and every segment is encoded at once from a GUESSED input state - the state reached by replaying
// the last ANS_WARM_BATCHES batches of the preceding segment from an arbitrary state, which has almost always merged
// with the true trajectory by then.  Afterwards each segment compares its guess with its TRUE input (the output of the
// segment before it in encode order) and, if they differ, re-runs from the true input only until it meets the guessed
// trajectory.  A segment that never merges changes its output and the round iterates until no output moves (worst case:
// one segment per iteration, i.e. the serial order) - the result is always exactly the serial encoder's.
constexpr int ANS_THREADS = 256;
constexpr int ANS_SEGS = ANS_THREADS / 4;   // segments per round: one thread per (segment, interleaved chain)
constexpr int ANS_WARM_BATCHES = 2;         // batches of the preceding segment replayed to form the guess
constexpr uint32_t ANS_MAX_SEG_BATCHES = 16;
constexpr uint32_t ANS_TF_MAX = 8;          // largest pivot weight the transfer-function path enumerates (a quiet replay of the segment per slot, ~0.12 ms each)
constexpr int ANS_TF_LOOK = 4;              // it picks the lightest symbol among a chain's first ANS_TF_LOOK steps of the segment
// slots of the round counters ans_encode_kernel keeps when profiling (pco_b200_profile_ans_paths, include/pco_b200.h): by resolution,
// then the same four for the rounds after a page's first
enum : uint32_t { ANS_PATH_SPECULATION = 0, ANS_PATH_FIXUP = 1, ANS_PATH_TRANSFER = 2, ANS_PATH_IN_ORDER = 3, ANS_PATH_LATER_ROUND = 4, ANS_PATH_SLOTS = 8 };

template <bool WIDE>
struct AnsSmemT {
  uint32_t desc_tab[EncCap<WIDE>::MAXB];                 // per symbol: ((min_renorm_bits + 1) << 16 - cutoff) | B << 20 (see ans_step)
  uint16_t next_states[1 << EncCap<WIDE>::MAX_SIZE_LOG];  // full next state (size + slot), indexed cum + (x_s - weight)
  uint16_t out_state[ANS_SEGS][4];
  uint16_t carry[4];
  // transfer-function path (tables whose trajectories do not merge): per (segment, chain) the descriptors of its first steps, which of
  // them is the pivot (the lightest symbol) and its weight, the segment's output state for each slot the pivot step can land in, and the
  // resolved true input state
  uint16_t tf[ANS_SEGS][4][ANS_TF_MAX];
  uint32_t first_desc[ANS_SEGS][4][ANS_TF_LOOK];
  uint8_t pivot[ANS_SEGS][4];
  uint8_t pivot_w[ANS_SEGS][4];
  uint16_t true_in[ANS_SEGS][4];
};
using AnsSmem = AnsSmemT<false>;

// One tANS step (ans/encoding.rs:72-83) from a pre-resolved descriptor; returns the bit count, `o` = value | bits << 12.
// The descriptor holds the step as two additions (the FSE formulation of the same arithmetic) in one 32-bit word:
//   bits 0-19  A = (min_renorm_bits + 1) << 16 - cutoff :  bits = (state + A) >> 16       (= min_renorm_bits + (state >= cutoff))
//   bits 20-31 B = cum - weight + 1024                   :  next  = next_states[B - 1024 + (state >> bits)]
// (an 8-byte descriptor saves one more instruction per step but doubles the wavefronts of the lookups, and was slower)
// Wide tables (up to 2^12 states) keep B = (cum - weight) mod 2^12: the true index cum - weight + (state >> bits) lies in [0, 2^12),
// so the 12-bit sum recovers it.  A stays below 13 << 16 < 2^20 and state < 2^13: no carry into B either.
template <bool WIDE = false>
__device__ __forceinline__ uint32_t ans_next(uint32_t d, uint32_t x_s, const uint16_t* next_states) {
  if constexpr (WIDE) return next_states[((d >> 20) + x_s) & 0xfffu];
  else return (next_states - 1024)[(d >> 20) + x_s];
}
template <bool WIDE = false>
__device__ __forceinline__ uint32_t ans_step(uint32_t d, uint32_t& state, uint32_t& o, const uint16_t* next_states) {
  const uint32_t bits = ((state + d) >> 16) & 0xfu;  // state < 2^11 (2^13 wide) and B sits above bit 19: no carry into B
  o = (state & ~(0xffffffffu << bits)) | (bits << 12);  // bits <= 10 (12 wide): value in bits 0-11, width in bits 12-15
  state = ans_next<WIDE>(d, state >> bits, next_states);
  return bits;
}
// the same step without the output (warm-up, and the guessed trajectory replayed next to the true one)
template <bool WIDE = false>
__device__ __forceinline__ uint32_t ans_step_quiet(uint32_t d, uint32_t& state, const uint16_t* next_states) {
  const uint32_t bits = ((state + d) >> 16) & 0xfu;
  state = ans_next<WIDE>(d, state >> bits, next_states);
  return bits;
}

// Chain j's 64 steps over one FULL batch row (256 symbols, 16-byte aligned).  The 4 lanes of a segment read the same 16
// symbols per group of 4 steps (one LDG.128), and transpose their 4x4 outputs with two shuffles so that each lane stores
// 4 consecutive u16 (one STG.64).  `gmask` names the 4 lanes of the group; they execute this together.
// Wide tables (16-bit symbols) take the chain's 64 elements one by one.
template <bool QUIET, bool WIDE = false>
__device__ __forceinline__ uint32_t ans_full_batch(const AnsSmemT<WIDE>& sm, const typename EncCap<WIDE>::Sym* __restrict__ row_sym, uint16_t* __restrict__ row_out,
                                                   int j, uint32_t gmask, uint32_t& state) {
  if constexpr (WIDE) {
    uint32_t bits_total = 0;
    for (int m = BATCH_N / 4 - 1; m >= 0; m--) {
      const uint32_t d = sm.desc_tab[row_sym[4 * m + j]];
      if (QUIET) {
        ans_step_quiet<true>(d, state, sm.next_states);
      } else {
        uint32_t o;
        bits_total += ans_step<true>(d, state, o, sm.next_states);
        row_out[4 * m + j] = uint16_t(o);
      }
    }
    return bits_total;
  }
  const uint4* src = reinterpret_cast<const uint4*>(row_sym);
  const uint32_t pick = 0x4440u | uint32_t(j);  // __byte_perm selector: byte j of the word, zero-extended
  const uint32_t sel_send = (j & 1) ? 0x5410u : 0x7632u, sel_q01 = (j & 1) ? 0x3254u : 0x5410u, sel_q23 = (j & 1) ? 0x3276u : 0x7610u;
  uint32_t bits_total = 0;
  uint4 cur = src[15], nxt = cur;
#pragma unroll 2
  for (int q = 15; q >= 0; q--) {
    if (q > 0) nxt = src[q - 1];
    const uint32_t d3 = sm.desc_tab[__byte_perm(cur.w, 0, pick)], d2 = sm.desc_tab[__byte_perm(cur.z, 0, pick)];
    const uint32_t d1 = sm.desc_tab[__byte_perm(cur.y, 0, pick)], d0 = sm.desc_tab[__byte_perm(cur.x, 0, pick)];
    if (QUIET) {
      ans_step_quiet(d3, state, sm.next_states);
      ans_step_quiet(d2, state, sm.next_states);
      ans_step_quiet(d1, state, sm.next_states);
      ans_step_quiet(d0, state, sm.next_states);
    } else {
      uint32_t o0, o1, o2, o3;  // element 16 q + 4 k + j
      bits_total += ans_step(d3, state, o3, sm.next_states);
      bits_total += ans_step(d2, state, o2, sm.next_states);
      bits_total += ans_step(d1, state, o1, sm.next_states);
      bits_total += ans_step(d0, state, o0, sm.next_states);
      const uint32_t p01 = o0 | (o1 << 16), p23 = o2 | (o3 << 16);
      // 4x4 transpose over the group: lane t ends up with element k = t of lanes 0..3
      const uint32_t r2 = __shfl_xor_sync(gmask, (j & 2) ? p01 : p23, 2);
      const uint32_t a = (j & 2) ? r2 : p01, b = (j & 2) ? p23 : r2;
      const uint32_t r1 = __shfl_xor_sync(gmask, __byte_perm(a, b, sel_send), 1);
      uint2 w;
      w.x = __byte_perm(a, r1, sel_q01);
      w.y = __byte_perm(b, r1, sel_q23);
      *reinterpret_cast<uint2*>(row_out + 16 * q + 4 * j) = w;
    }
    cur = nxt;
  }
  return bits_total;
}

template <bool WIDE = false>
__global__ void __launch_bounds__(ANS_THREADS, 4) ans_encode_kernel(EncParams ep, uint32_t batches_per_chunk, const VarPlanT<WIDE>* __restrict__ plans,
                                                                     ChunkEnc* __restrict__ chunks, const typename EncCap<WIDE>::Sym* __restrict__ sym0,
                                                                     const typename EncCap<WIDE>::Sym* __restrict__ sym1, uint16_t* __restrict__ ans0,
                                                                     uint16_t* __restrict__ ans1, uint32_t* __restrict__ ans_sum,
                                                                     BatchEntry* __restrict__ entries, uint32_t* __restrict__ path_counts) {
  using Sym = typename EncCap<WIDE>::Sym;
  __shared__ AnsSmemT<WIDE> sm;
  const uint32_t c = blockIdx.x / MAX_VARS, v = blockIdx.x % MAX_VARS;
  if (v >= ep.n_vars) return;
  const int tid = threadIdx.x;
  const uint64_t cs = ep.chunk_starts[c], ce = ep.chunk_starts[c + 1];
  const bool fb = chunks[c].fallback != 0;
  if (fb && v > 0) return;
  const uint64_t sb = fb ? cs : stored_begin(cs, ce, v == 0 ? ep.order : 0);
  const uint32_t n = uint32_t(ce - sb);
  const uint32_t n_page = uint32_t(ce - cs);
  const uint32_t nb_page = n_batches_of(n_page);
  const VarPlanT<WIDE>& plan = plans[size_t(c) * MAX_VARS + v];
  const uint32_t n_bins = fb ? 1 : plan.n_bins;
  const uint32_t size_log = fb ? 0 : plan.size_log;
  const uint32_t size = 1u << size_log;
  uint32_t* sums = ans_sum + (size_t(c) * MAX_VARS + v) * batches_per_chunk;
  BatchEntry* ent = entries + (size_t(c) * MAX_VARS + v) * batches_per_chunk;
  if (size_log == 0) {
    // one symbol: no ANS bits, states stay at the default (chunk_latent_compressor.rs:103-108)
    for (uint32_t b = tid; b < nb_page; b += ANS_THREADS) {
      sums[b] = 0;
      BatchEntry e; e.bit_pos = 0; e.st[0] = e.st[1] = e.st[2] = e.st[3] = 0;
      ent[b] = e;
    }
    if (tid < 4) chunks[c].final_state[v][tid] = 0;
    return;
  }
  for (uint32_t i = tid; i < uint32_t(EncCap<WIDE>::MAXB); i += ANS_THREADS) {
    // entries past n_bins alias symbol 0 (never looked up: every staged symbol is < n_bins)
    const uint64_t info = plan.syminfo[i < n_bins ? i : 0];
    const uint32_t cutoff = uint32_t(info & 0xffff), mr = uint32_t(info >> 16) & 0xff, w = uint32_t(info >> 24) & 0xffff, cum = uint32_t(info >> 40) & 0xffff;
    sm.desc_tab[i] = (((mr + 1u) << 16) - cutoff) | ((WIDE ? (cum - w) & 0xfffu : cum + 1024u - w) << 20);
  }
  for (uint32_t i = tid; i < size; i += ANS_THREADS) sm.next_states[i] = uint16_t(size + plan.next_states[i]);
  const uint32_t nb = n_batches_of(n);
  for (uint32_t b = nb + tid; b < nb_page; b += ANS_THREADS) {  // page batches past the var's stored range: no symbols
    sums[b] = 0;
    BatchEntry e; e.bit_pos = 0; e.st[0] = e.st[1] = e.st[2] = e.st[3] = 0;
    ent[b] = e;
  }
  if (tid < 4) sm.carry[tid] = uint16_t(size);  // encoder.default_state()
  __syncthreads();
  const Sym* symp = (v == 0 ? sym0 : sym1) + ep.row_base[c];  // rows are 256-aligned (see split_delta_kernel)
  uint16_t* ansp = (v == 0 ? ans0 : ans1) + ep.row_base[c];
  const int j = tid & 3, s = tid >> 2;  // chain j of the s-th segment below the round's top
  const uint32_t gmask = 0xfu << ((tid & 31) & ~3);
  const uint32_t nb_full = n / BATCH_N;  // batches [0, nb_full) are full; batch nb_full (if any) is the short last one
  const uint32_t seg_b = min(max((nb + ANS_SEGS - 1) / ANS_SEGS, 2u), ANS_MAX_SEG_BATCHES);  // batches per segment
  const uint32_t n_segs = (nb + seg_b - 1) / seg_b;
  // chain j over a short batch, element by element (only the page's last batch can be short)
  auto short_batch = [&](uint32_t b, uint32_t& state) -> uint32_t {
    const uint32_t cnt = n - b * BATCH_N;
    const int steps = cnt > uint32_t(j) ? int((cnt - 1 - j) / 4 + 1) : 0;
    const Sym* rs = symp + uint64_t(b) * BATCH_N;
    uint16_t* ro = ansp + uint64_t(b) * BATCH_N;
    uint32_t bits_total = 0;
    for (int m = steps - 1; m >= 0; m--) {
      uint32_t o;
      bits_total += ans_step<WIDE>(sm.desc_tab[rs[4 * m + j]], state, o, sm.next_states);
      ro[4 * m + j] = uint16_t(o);
    }
    return bits_total;
  };
  // Last resort for tables on which neither the speculation nor the transfer functions work (every thread of the CTA calls it together):
  auto serial_pass = [&]() {
    // In-order pass over the whole page from the default state (idempotent: it overwrites what the rounds so far wrote).  The serial
    // part is the state chain alone: four lanes walk the four chains and leave every step's INPUT state in the output slot; the bits
    // and values follow from (state, symbol) per element, which the whole CTA then does in parallel.
    if (tid < 4) {
      uint32_t st = size;
      for (uint32_t b = nb; b > 0; b--) {
        const uint32_t bb = b - 1;
        const Sym* rs = symp + uint64_t(bb) * BATCH_N;
        uint16_t* ro = ansp + uint64_t(bb) * BATCH_N;
        if (!WIDE && bb < nb_full) {
          const uint4* src = reinterpret_cast<const uint4*>(rs);
          const uint32_t pick = 0x4440u | uint32_t(j);
          uint4 cur = src[15], nxt = cur;
#pragma unroll 2
          for (int q = 15; q >= 0; q--) {
            if (q > 0) nxt = src[q - 1];
            const uint32_t d3 = sm.desc_tab[__byte_perm(cur.w, 0, pick)], d2 = sm.desc_tab[__byte_perm(cur.z, 0, pick)];
            const uint32_t d1 = sm.desc_tab[__byte_perm(cur.y, 0, pick)], d0 = sm.desc_tab[__byte_perm(cur.x, 0, pick)];
            ro[16 * q + 12 + j] = uint16_t(st);
            ans_step_quiet<WIDE>(d3, st, sm.next_states);
            ro[16 * q + 8 + j] = uint16_t(st);
            ans_step_quiet<WIDE>(d2, st, sm.next_states);
            ro[16 * q + 4 + j] = uint16_t(st);
            ans_step_quiet<WIDE>(d1, st, sm.next_states);
            ro[16 * q + j] = uint16_t(st);
            ans_step_quiet<WIDE>(d0, st, sm.next_states);
            cur = nxt;
          }
        } else {  // the page's short last batch (every batch, 16-bit symbols)
          const uint32_t cnt = WIDE ? min(uint32_t(BATCH_N), n - bb * BATCH_N) : n - bb * BATCH_N;
          const int steps = cnt > uint32_t(j) ? int((cnt - 1 - j) / 4 + 1) : 0;
          for (int m = steps - 1; m >= 0; m--) {
            ro[4 * m + j] = uint16_t(st);
            ans_step_quiet<WIDE>(sm.desc_tab[rs[4 * m + j]], st, sm.next_states);
          }
        }
        if (j == 0) { sums[bb] = 0; ent[bb].bit_pos = 0; }
        ent[bb].st[j] = uint16_t(st - size);
      }
      chunks[c].final_state[v][j] = st - size;
    }
    __syncthreads();
    for (uint32_t bb = 0; bb < nb; bb++) {  // batch bb: one element per thread
      const uint32_t i = bb * BATCH_N + uint32_t(tid);
      uint32_t bits = 0;
      if (i < n) {
        const uint32_t st = ansp[i], d = sm.desc_tab[symp[i]];
        bits = ((st + d) >> 16) & 0xfu;
        ansp[i] = uint16_t((st & ~(0xffffffffu << bits)) | (bits << 12));
      }
      for (int dd = 16; dd > 0; dd >>= 1) bits += __shfl_xor_sync(0xffffffffu, bits, dd);
      if ((tid & 31) == 0 && bits) atomicAdd(&sums[bb], bits);
    }
  };
  for (uint32_t done = 0; done < n_segs; done += ANS_SEGS) {
    // this round: segments n_segs-1-done, n_segs-2-done, ... (encode order); thread group s takes the s-th of them
    const bool active = done + uint32_t(s) < n_segs;
    const uint32_t seg = active ? n_segs - 1 - done - uint32_t(s) : 0u;
    const uint32_t b_lo = seg * seg_b, b_hi = min(b_lo + seg_b, nb);
    uint32_t my_in = sm.carry[j];  // the round's first segment knows its input
    if (active && s > 0) {
      // guess: replay the tail of the preceding segment (full batches only) from an arbitrary state
      uint32_t g = size;
      const uint32_t w_hi = min(b_hi + ANS_WARM_BATCHES, nb_full);
      for (uint32_t b = w_hi; b > b_hi; b--)
        ans_full_batch<true, WIDE>(sm, symp + uint64_t(b - 1) * BATCH_N, nullptr, j, gmask, g);
      my_in = g;
    }
    // the segment's batches from input state `st` (the 4 lanes of the group together); returns the output state
    auto encode_segment = [&](uint32_t st) -> uint32_t {
      for (uint32_t b = b_hi; b > b_lo; b--) {
        const uint32_t bb = b - 1;
        uint32_t bits = bb < nb_full ? ans_full_batch<false, WIDE>(sm, symp + uint64_t(bb) * BATCH_N, ansp + uint64_t(bb) * BATCH_N, j, gmask, st)
                                     : short_batch(bb, st);
        bits += __shfl_xor_sync(gmask, bits, 1);
        bits += __shfl_xor_sync(gmask, bits, 2);
        // decoder state at the START of a batch == encoder state after encoding it (side index)
        if (j == 0) { sums[bb] = bits; ent[bb].bit_pos = 0; }
        ent[bb].st[j] = uint16_t(st - size);
      }
      return st;
    };
    uint32_t state = my_in;
    if (active) {
      state = encode_segment(my_in);
      sm.out_state[s][j] = uint16_t(state);
    }
    uint32_t my_out = state;
    __syncthreads();
    // The speculation rests on tANS trajectories merging (a symbol of weight w maps all states onto w values).  Tables that merge slowly
    // need other means, chosen by what they cost:
    //   fix-up        a wrong segment re-runs from its true input next to the old trajectory until the two meet.  Cheap when they meet
    //                 soon (C5 float64 order 0: a third of the guesses wrong, ~10 iterations); a correction that runs off its
    //                 segment moves the problem one segment on per iteration (as slow as a whole page in order).
    //   transfer fn   after a step with a symbol of weight w the state is one of w values (next_states[cum + slot], slot =
    //                 (state >> bits) - w) whatever it was before.  Each (segment, chain) takes the lightest symbol among its first
    //                 ANS_TF_LOOK steps as the pivot, replays the rest of the segment quietly once per slot (<= ANS_TF_MAX of them, ~0.12 ms
    //                 per replay), four threads chain the true inputs through the 64 transfer functions, every segment is encoded once
    //                 more from its true input.  For equal-weight tables (equal-count bins of smooth wide-range data: 3 guesses in 4
    //                 wrong, corrections never merge).
    //   in-order      serial_pass above, ~4.3 ms: tables with heavy symbols in long runs (C5 int64 order 0: weights 205 / 50 / 1).
    // One fix-up iteration always runs.  If more than a quarter of the round's (segment, chain) pairs ran off their segments in it, a
    // cascade is on its way: transfer functions if every pivot is light enough, else in-order.  Otherwise the fix-up goes on, and if it
    // has not converged after 24 iterations the same choice.
    const uint32_t n_round = min(n_segs - done, uint32_t(ANS_SEGS));
    uint32_t pv = 0, pw = 0xffffu;
    auto pivots_enumerable = [&]() -> bool {  // CTA-uniform
      const bool top_full = b_hi >= 1 && b_hi - 1 < nb_full;  // only the round's top segment (s == 0) can hold the page's short batch
      pv = 0;
      pw = 0xffffu;
      if (active && s > 0 && top_full) {
        // the chain's first steps in this segment: elements 252 + j, 248 + j, ... of batch b_hi - 1
        const Sym* rs = symp + uint64_t(b_hi - 1) * BATCH_N;
#pragma unroll
        for (int k = 0; k < ANS_TF_LOOK; k++) {
          const uint32_t sy = rs[4 * (63 - k) + j];
          sm.first_desc[s][j][k] = sm.desc_tab[sy];
          const uint32_t w = uint32_t(plan.syminfo[sy] >> 24) & 0xffff;
          if (w < pw) { pw = w; pv = uint32_t(k); }
        }
        sm.pivot[s][j] = uint8_t(pv);
        sm.pivot_w[s][j] = uint8_t(min(pw, 255u));
      }
      const bool enumerable = !(active && s > 0) || (top_full && pw <= ANS_TF_MAX);
      return __syncthreads_and(enumerable ? 1 : 0) != 0;
    };
    auto transfer_round = [&]() {  // after pivots_enumerable() == true; leaves the round's carry in sm.carry
      if (active && s > 0) {
        const Sym* rs = symp + uint64_t(b_hi - 1) * BATCH_N;
        const uint32_t dp = sm.first_desc[s][j][pv];
        for (uint32_t idx = 0; idx < pw; idx++) {
          uint32_t g = ans_next<WIDE>(dp, pw + idx, sm.next_states);  // the state after the pivot step landed in slot idx
          for (int m = 62 - int(pv); m >= 0; m--) ans_step_quiet<WIDE>(sm.desc_tab[rs[4 * m + j]], g, sm.next_states);  // rest of the top batch
          for (uint32_t b = b_hi - 1; b > b_lo; b--) ans_full_batch<true, WIDE>(sm, symp + uint64_t(b - 1) * BATCH_N, nullptr, j, gmask, g);
          sm.tf[s][j][idx] = uint16_t(g);
        }
      }
      __syncthreads();
      if (tid < 4) {  // chain tid: the true input of every segment of the round, in encode order
        uint32_t st = sm.out_state[0][tid];
        for (uint32_t s2 = 1; s2 < n_round; s2++) {
          sm.true_in[s2][tid] = uint16_t(st);
          const uint32_t pv2 = sm.pivot[s2][tid], pw2 = sm.pivot_w[s2][tid];
          for (uint32_t k = 0; k < pv2; k++) ans_step_quiet<WIDE>(sm.first_desc[s2][tid][k], st, sm.next_states);
          const uint32_t bits = ((st + sm.first_desc[s2][tid][pv2]) >> 16) & 0xfu;
          st = sm.tf[s2][tid][(st >> bits) - pw2];
        }
        sm.carry[tid] = uint16_t(st);
      }
      __syncthreads();
      if (active && s > 0) encode_segment(sm.true_in[s][j]);
      __syncthreads();
    };
    bool solved = false;
    {
      bool converged = false;
      int iter = 0;
      for (; iter < 24 && !converged; iter++) {
        const uint32_t in_true = (s == 0 || !active) ? my_in : uint32_t(sm.out_state[s - 1][j]);
        bool changed = false;
        if (in_true != my_in) {
          // re-run from the true input next to the old trajectory until they meet (element-wise path)
          uint32_t a = in_true, g = my_in;
          for (uint32_t b = b_hi; b > b_lo && a != g; b--) {
            const uint32_t bb = b - 1;
            const uint32_t cnt = min(uint32_t(BATCH_N), n - bb * BATCH_N);
            const int steps = cnt > uint32_t(j) ? int((cnt - 1 - j) / 4 + 1) : 0;
            const Sym* rs = symp + uint64_t(bb) * BATCH_N;
            uint16_t* ro = ansp + uint64_t(bb) * BATCH_N;
            int delta = 0;
            int m = steps - 1;
            for (; m >= 0 && a != g; m--) {
              const uint32_t d = sm.desc_tab[rs[4 * m + j]];
              uint32_t o;
              delta += int(ans_step<WIDE>(d, a, o, sm.next_states));
              delta -= int(ans_step_quiet<WIDE>(d, g, sm.next_states));
              ro[4 * m + j] = uint16_t(o);
            }
            if (delta != 0) atomicAdd(&sums[bb], uint32_t(delta));
            if (m < 0 && a != g) ent[bb].st[j] = uint16_t(a - size);  // the batch ended on the corrected trajectory
          }
          my_in = in_true;
          if (a != g) { changed = true; my_out = a; }  // ran off the segment without meeting the old trajectory
        }
        __syncthreads();  // every segment has read its predecessor's output
        if (changed) sm.out_state[s][j] = uint16_t(my_out);
        const uint32_t n_changed = uint32_t(__syncthreads_count(changed ? 1 : 0));
        converged = n_changed == 0;
        if (iter == 0 && n_changed > n_round) break;  // more than a quarter of the 4 n_round pairs (an eighth sent C5 float64 order 0 in-order, three times slower)
      }
      // test hook (pco_b200_profile_ans_paths; null unless profiling): one count per round by resolution, and again in the upper half
      // of the slots for rounds after the page's first
      auto count_round = [&](uint32_t path) {
        if (path_counts != nullptr && tid == 0) {
          atomicAdd(&path_counts[path], 1u);
          if (done > 0) atomicAdd(&path_counts[ANS_PATH_LATER_ROUND + path], 1u);
        }
      };
      if (!converged) {
        if (!pivots_enumerable()) {
          count_round(ANS_PATH_IN_ORDER);
          serial_pass();
          return;
        }
        count_round(ANS_PATH_TRANSFER);
        transfer_round();
        solved = true;
      } else {
        count_round(iter == 1 ? ANS_PATH_SPECULATION : ANS_PATH_FIXUP);  // iter: fix-up iterations run, the last one saw no output move
      }
    }
    if (solved) continue;  // transfer_round left the carry
    if (active && done + uint32_t(s) + 1 == min(n_segs, done + ANS_SEGS)) sm.carry[j] = uint16_t(my_out);  // the round's last segment
    __syncthreads();
  }
  if (tid < 4) chunks[c].final_state[v][tid] = uint32_t(sm.carry[tid]) - size;
}

// ---------------------------------------------------------------------------
// layout_kernel: one CTA per chunk.  Exclusive scan over (batch, var) bit sizes -> side-index bit positions,
// meta / page sizes, chunk byte size.
// ---------------------------------------------------------------------------
constexpr int LAYOUT_THREADS = 256;

template <bool WIDE = false>
__global__ void __launch_bounds__(LAYOUT_THREADS) layout_kernel(EncParams ep, uint32_t batches_per_chunk, const VarPlanT<WIDE>* __restrict__ plans,
                                                                 ChunkEnc* __restrict__ chunks, const uint32_t* __restrict__ ans_sum,
                                                                 const uint32_t* __restrict__ ob_sum, BatchEntry* __restrict__ entries) {
  __shared__ uint64_t warp_tot[LAYOUT_THREADS / 32];
  __shared__ uint64_t carry;
  const uint32_t c = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t lbits = nt_bits(ep.dtype);
  const uint64_t n = ep.chunk_starts[c + 1] - ep.chunk_starts[c];
  const bool fb = chunks[c].fallback != 0;
  const uint32_t n_vars = fb ? 1 : ep.n_vars;
  const uint32_t order = fb ? 0 : ep.order;
  const uint32_t mode = fb ? MODE_CLASSIC : ep.mode;
  const uint32_t nb = n_batches_of(uint32_t(n));
  // meta and page-meta sizes (metadata/chunk.rs:176-189, page.rs:22-34)
  uint32_t meta_bits = 4 + mode_payload_bits(mode, lbits) + 4 + (order > 0 ? 4 : 0);
  uint32_t page_meta_bits = 0;
  for (uint32_t v = 0; v < n_vars; v++) {
    const VarPlanT<WIDE>& p = plans[size_t(c) * MAX_VARS + v];
    uint32_t n_bins = fb ? 1 : p.n_bins, size_log = fb ? 0 : p.size_log;
    meta_bits += var_meta_bits(n_bins, size_log, lbits);
    page_meta_bits += 4 * size_log + lbits * (v == 0 ? order : 0);
  }
  const uint32_t meta_bytes = (meta_bits + 7) / 8, page_meta_bytes = (page_meta_bits + 7) / 8;
  const uint64_t body_bit0 = uint64_t(4 + meta_bytes + page_meta_bytes) * 8;  // relative to the chunk's type byte
  if (tid == 0) carry = 0;
  __syncthreads();
  // items in stream order: item = b * n_vars + v; size = ans bits + offset bits of that (batch, var)
  const uint32_t n_items = nb * n_vars;
  for (uint32_t base = 0; base < n_items; base += LAYOUT_THREADS) {
    uint32_t item = base + tid;
    uint64_t sz = 0;
    uint32_t b = 0, v = 0;
    if (item < n_items) {
      b = item / n_vars; v = item % n_vars;
      size_t k = (size_t(c) * MAX_VARS + v) * batches_per_chunk + b;
      const VarPlanT<WIDE>& p = plans[size_t(c) * MAX_VARS + v];
      bool trivial_ans = fb || p.n_bins <= 1;
      sz = uint64_t(trivial_ans ? 0 : ans_sum[k]) + ob_sum[k];
    }
    uint64_t inc = sz;
    for (int d = 1; d < 32; d <<= 1) {
      uint64_t o = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= d) inc += o;
    }
    if (lane == 31) warp_tot[warp] = inc;
    __syncthreads();
    uint64_t wbase = carry;
    for (int w = 0; w < warp; w++) wbase += warp_tot[w];
    if (item < n_items) {
      size_t k = (size_t(c) * MAX_VARS + v) * batches_per_chunk + b;
      entries[k].bit_pos = uint32_t(body_bit0 + wbase + inc - sz);
    }
    __syncthreads();
    if (tid == LAYOUT_THREADS - 1) carry = wbase + inc;
    __syncthreads();
  }
  if (tid == 0) {
    uint64_t body_bits = carry;
    chunks[c].meta_bytes = meta_bytes;
    chunks[c].page_meta_bytes = page_meta_bytes;
    chunks[c].body_bits = body_bits;
    chunks[c].chunk_bytes = 4 + meta_bytes + page_meta_bytes + (body_bits + 7) / 8;
  }
}

// exclusive scan of chunk sizes -> output offsets (one CTA; chunk counts are small)
__global__ void chunk_offsets_kernel(ChunkEnc* chunks, uint32_t n_chunks, uint64_t header_bytes, uint32_t footer_bytes, uint64_t* total_bytes) {
  __shared__ uint64_t part[1024];
  const int tid = threadIdx.x;
  uint32_t per = (n_chunks + blockDim.x - 1) / blockDim.x;
  uint32_t lo = min(n_chunks, tid * per), hi = min(n_chunks, lo + per);
  uint64_t s = 0;
  for (uint32_t c = lo; c < hi; c++) s += chunks[c].chunk_bytes;
  part[tid] = s;
  __syncthreads();
  if (tid == 0) {
    uint64_t acc = header_bytes;
    for (uint32_t t = 0; t < blockDim.x; t++) { uint64_t x = part[t]; part[t] = acc; acc += x; }
    *total_bytes = acc + footer_bytes;  // + terminator byte
  }
  __syncthreads();
  uint64_t off = part[tid];
  for (uint32_t c = lo; c < hi; c++) { chunks[c].out_offset = off; off += chunks[c].chunk_bytes; }
}

// ---------------------------------------------------------------------------
// K5: pack.  One CTA per chunk writes the chunk's bytes [out_offset, out_offset + chunk_bytes) with plain stores.
// Bits are OR-ed into a zeroed shared-memory staging window (32-bit atomics), then copied out; partial bytes at
// window boundaries are carried in shared memory, so no global atomics or pre-zeroed output are needed.
// ---------------------------------------------------------------------------
constexpr int PACK_THREADS = 256;
#ifndef PCOB_PACK_MIN_BLOCKS
#define PCOB_PACK_MIN_BLOCKS 4
#endif
constexpr int PACK_WINDOW_WORDS = 8192;  // 32 KiB staging window

// Wide plans: the head (chunk meta of up to 4096 bins of <= 83 bits each, plus the secondary var's) needs a larger window, and their
// vars never take the 16-bit-key path (no lowkey_ob table).
template <bool WIDE>
struct PackSmemT {
  static constexpr int WIN_WORDS = WIDE ? 3 * PACK_WINDOW_WORDS / 2 : PACK_WINDOW_WORDS;
  uint32_t win[WIN_WORDS + 8];
  uint64_t lowers[MAX_VARS][EncCap<WIDE>::MAXB];
  uint8_t obs[MAX_VARS][EncCap<WIDE>::MAXB];
  uint32_t lowkey_ob[MAX_VARS][WIDE ? 1 : EncCap<WIDE>::MAXB];  // 16-bit-key vars: (lower - chunk minimum) | offset_bits << 16
};
using PackSmem = PackSmemT<false>;

// OR `nbits` (<= 64) of `val` at bit position `pos` (relative to the window start) into the window
__device__ __forceinline__ void win_or(uint32_t* win, uint32_t pos, uint64_t val, uint32_t nbits) {
  if (nbits == 0) return;
  if (nbits < 64) val &= (uint64_t(1) << nbits) - 1;
  uint32_t w = pos >> 5, r = pos & 31;
  uint32_t lo = uint32_t(val) << r;
  if (lo) atomicOr(&win[w], lo);
  uint64_t rest = r ? (val >> (32 - r)) : (val >> 32);
  if (r + nbits > 32) {
    uint32_t mid = uint32_t(rest);
    if (mid) atomicOr(&win[w + 1], mid);
    if (r + nbits > 64) {
      uint32_t hi = uint32_t(rest >> 32);
      if (hi) atomicOr(&win[w + 2], hi);
    }
  }
}

// 8 consecutive latents of an aligned batch row as one vector access
template <typename L>
struct alignas(sizeof(L) * 8 > 16 ? 16 : sizeof(L) * 8) Vec8 { L v[8]; };

// Appends fields (<= 32 bits each, already masked to their width) at increasing bit positions of the shared window and
// ORs finished 32-bit words in; neighbouring lanes share at most the first and last word of a span.
struct BitAcc {
  uint32_t* win;
  uint64_t acc;
  uint32_t fill, w;
  __device__ __forceinline__ BitAcc(uint32_t* win_, uint32_t pos) : win(win_), acc(0), fill(pos & 31), w(pos >> 5) {}
  __device__ __forceinline__ void put(uint32_t val, uint32_t nbits) {
    acc |= uint64_t(val) << fill;
    fill += nbits;
    if (fill >= 32) {
      const uint32_t lo = uint32_t(acc);
      if (lo) atomicOr(&win[w], lo);
      w++;
      acc >>= 32;
      fill -= 32;
    }
  }
  __device__ __forceinline__ void flush() {
    if (fill > 0 && uint32_t(acc)) atomicOr(&win[w], uint32_t(acc));
  }
};

// 8 consecutive fields of <= 15 bits each (already masked) at bit `pos` of the window: a 3-level concatenation tree in
// registers (<= 120 bits), one shift to the word phase, then at most five 32-bit ORs into shared memory.
__device__ __forceinline__ void emit8_narrow(uint32_t* win, uint32_t pos, const uint32_t (&v)[8], const uint32_t (&nb)[8]) {
  const uint32_t p0 = v[0] | (v[1] << nb[0]), p1 = v[2] | (v[3] << nb[2]), p2 = v[4] | (v[5] << nb[4]), p3 = v[6] | (v[7] << nb[6]);
  const uint32_t l0 = nb[0] + nb[1], l1 = nb[2] + nb[3], l2 = nb[4] + nb[5];  // each <= 30
  const uint64_t q0 = uint64_t(p0) | (uint64_t(p1) << l0), q1 = uint64_t(p2) | (uint64_t(p3) << l2);  // each <= 60 bits
  const uint32_t m0 = l0 + l1;                                                                         // <= 60
  const uint64_t lo = q0 | (q1 << m0), hi = (q1 >> 1) >> (63 - m0);
  const uint32_t r = pos & 31, w = pos >> 5;
  const uint32_t x0 = uint32_t(lo), x1 = uint32_t(lo >> 32), x2 = uint32_t(hi), x3 = uint32_t(hi >> 32);
  const uint32_t w0 = x0 << r, w1 = __funnelshift_l(x0, x1, r), w2 = __funnelshift_l(x1, x2, r), w3 = __funnelshift_l(x2, x3, r);
  const uint32_t w4 = __funnelshift_l(x3, 0u, r);
  if (w0) atomicOr(&win[w], w0);
  if (w1) atomicOr(&win[w + 1], w1);
  if (w2) atomicOr(&win[w + 2], w2);
  if (w3) atomicOr(&win[w + 3], w3);
  if (w4) atomicOr(&win[w + 4], w4);
}

template <typename L, bool WIDE = false>
__global__ void __launch_bounds__(PACK_THREADS, PCOB_PACK_MIN_BLOCKS) pack_kernel(EncParams ep, uint32_t batches_per_chunk, const L* __restrict__ lat0, const L* __restrict__ lat1,
                                                             const VarPlanT<WIDE>* __restrict__ plans, const ChunkEnc* __restrict__ chunks,
                                                             const typename EncCap<WIDE>::Sym* __restrict__ sym0, const typename EncCap<WIDE>::Sym* __restrict__ sym1,
                                                             const uint16_t* __restrict__ ans0, const uint16_t* __restrict__ ans1,
                                                             const BatchEntry* __restrict__ entries, uint8_t* __restrict__ out, uint64_t out_cap,
                                                             const uint16_t* __restrict__ key0, const uint16_t* __restrict__ key1) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  PackSmemT<WIDE>& sm = *reinterpret_cast<PackSmemT<WIDE>*>(smem_raw);
  const uint32_t c = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const ChunkEnc& ch = chunks[c];
  if (ch.out_offset + ch.chunk_bytes > out_cap) return;  // host reports the Io error from the total size
  const uint64_t cs = ep.chunk_starts[c], ce = ep.chunk_starts[c + 1];
  const uint32_t n = uint32_t(ce - cs);
  const uint32_t lbits = LT<L>::BITS;
  const bool fb = ch.fallback != 0;
  const uint32_t n_vars = fb ? 1 : ep.n_vars;
  const uint32_t order = fb ? 0 : ep.order;
  const uint32_t mode = fb ? MODE_CLASSIC : ep.mode;
  const uint32_t nb = n_batches_of(n);
  uint8_t* dst = out + ch.out_offset;
  for (uint32_t v = 0; v < n_vars; v++) {
    const VarPlanT<WIDE>& p = plans[size_t(c) * MAX_VARS + v];
    uint32_t n_bins = fb ? 1 : p.n_bins;
    for (uint32_t i = tid; i < n_bins; i += PACK_THREADS) {
      sm.lowers[v][i] = fb ? 0 : p.lower[i];
      sm.obs[v][i] = fb ? uint8_t(lbits) : p.ob[i];
      // keys (key0/key1 non-null: the counting planner ran for this var) are (latent - key_base) mod 2^16, so is this table
      if constexpr (!WIDE) sm.lowkey_ob[v][i] = fb ? 0u : (uint32_t(p.lower[i] - ch.key_base[v]) & 0xffffu) | (uint32_t(p.ob[i]) << 16);
    }
  }
  // ---------------- head window: preamble + chunk meta + page meta ----------------
  const uint32_t head_bytes = 4 + ch.meta_bytes + ch.page_meta_bytes;
  for (uint32_t i = tid; i < (head_bytes + 3) / 4 + 2; i += PACK_THREADS) sm.win[i] = 0;
  __syncthreads();
  if (tid == 0) {
    uint32_t pos = 0;
    win_or(sm.win, pos, ep.dtype, 8); pos += 8;
    win_or(sm.win, pos, n - 1, 24); pos += 24;
    win_or(sm.win, pos, mode, 4); pos += 4;
    if (mode == MODE_INT_MULT || mode == MODE_FLOAT_MULT) { win_or(sm.win, pos, ep.mode_base, lbits); pos += lbits; }
    if (mode == MODE_FLOAT_QUANT) { win_or(sm.win, pos, ep.mode_k, 8); pos += 8; }
    if (order > 0) { win_or(sm.win, pos, 1, 4); win_or(sm.win, pos + 4, order, 3); pos += 8; }  // Consecutive, secondary_uses_delta = 0
    else { pos += 4; }
    // page meta (metadata/page_latent_var.rs:19-26): moments, then 4 final state indices per var
    uint32_t ppos = (4 + ch.meta_bytes) * 8;
    for (uint32_t v = 0; v < n_vars; v++) {
      const VarPlanT<WIDE>& p = plans[size_t(c) * MAX_VARS + v];
      uint32_t size_log = fb ? 0 : p.size_log;
      if (v == 0) for (uint32_t k = 0; k < order; k++) { win_or(sm.win, ppos, ch.moments[0][k], lbits); ppos += lbits; }
      for (int j = 0; j < 4; j++) { win_or(sm.win, ppos, ch.final_state[v][j], size_log); ppos += size_log; }
    }
  }
  {
    // bins of every var, in parallel (metadata/chunk_latent_var.rs:55-71)
    uint32_t pos = 32 + 4 + mode_payload_bits(mode, lbits) + 4 + (order > 0 ? 4 : 0);
    for (uint32_t v = 0; v < n_vars; v++) {
      const VarPlanT<WIDE>& p = plans[size_t(c) * MAX_VARS + v];
      uint32_t n_bins = fb ? 1 : p.n_bins, size_log = fb ? 0 : p.size_log;
      uint32_t stride = size_log + lbits + offset_bits_bits(lbits);
      if (tid == 0) { win_or(sm.win, pos, size_log, 4); win_or(sm.win, pos + 4, n_bins, 15); }
      pos += 19;
      for (uint32_t i = tid; i < n_bins; i += PACK_THREADS) {
        uint32_t bp = pos + i * stride;
        uint32_t w = fb ? 1 : p.weight[i];
        win_or(sm.win, bp, w - 1, size_log);
        win_or(sm.win, bp + size_log, sm.lowers[v][i], lbits);
        win_or(sm.win, bp + size_log + lbits, sm.obs[v][i], offset_bits_bits(lbits));
      }
      pos += n_bins * stride;
    }
  }
  __syncthreads();
  {
    const uint8_t* wb = reinterpret_cast<const uint8_t*>(sm.win);
    for (uint32_t i = tid; i < head_bytes; i += PACK_THREADS) dst[i] = wb[i];
  }
  __syncthreads();
  // ---------------- body: windows of whole batches ----------------
  // Window words mirror the destination's 4-byte words: stream bit X of the chunk sits at P(X) = X + skew from the
  // aligned-down chunk address, windows start on multiples of 32 in P, and finished words leave as 32-bit stores
  // (the chunk's first and last body words, which share bytes with the head / the next chunk, byte by byte).
  const uint64_t body_bit0 = uint64_t(head_bytes) * 8;
  const uint64_t body_end = body_bit0 + ch.body_bits;
  const uint32_t dst_mis = uint32_t(reinterpret_cast<uintptr_t>(dst) & 3);
  const uint64_t skew = 8ull * dst_mis;
  uint32_t* const dst_words = reinterpret_cast<uint32_t*>(dst - dst_mis);
  const uint64_t lo_byte = (body_bit0 + skew) / 8, hi_byte = (body_end + skew + 7) / 8;  // body bytes, in P
  auto entry_pos = [&](uint32_t b, uint32_t v) -> uint64_t {
    return entries[(size_t(c) * MAX_VARS + v) * batches_per_chunk + b].bit_pos + skew;
  };
  __shared__ uint32_t s_carry;
  if (tid == 0) s_carry = 0;
  // per-var constants of the chunk
  const uint64_t rb = ep.row_base[c];
  const VarPlanT<WIDE>& pl0 = plans[size_t(c) * MAX_VARS], &pl1 = plans[size_t(c) * MAX_VARS + (n_vars > 1 ? 1 : 0)];
  const bool ans_0 = !fb && pl0.n_bins != 1 && pl0.size_log > 0, ans_1 = !fb && pl1.n_bins != 1 && pl1.size_log > 0;
  const uint32_t mob_0 = fb ? lbits : pl0.max_ob, mob_1 = fb ? lbits : pl1.max_ob;
  const uint32_t stored_0 = uint32_t(ce - (fb ? cs : stored_begin(cs, ce, order))), stored_1 = uint32_t(ce - cs);
  const uint16_t* const keyp_0 = fb ? nullptr : key0;
  const uint16_t* const keyp_1 = fb ? nullptr : key1;
  const bool lean = !WIDE && n_vars == 1 && keyp_0 != nullptr && ans_0 && mob_0 > 0 && mob_0 <= 15;
  uint32_t b0 = 0;
  uint64_t win_p0 = (body_bit0 + skew) & ~uint64_t(31);
  while (b0 < nb) {
    // choose b1 > b0 so that [start(b0), end(b1 - 1)) fits the window; a single batch always fits (<= 2*256*78 bits)
    // (batch ends are monotone, so the batches that still fit form a prefix: every thread probes one candidate per round)
    uint32_t b1 = b0 + 1;
    const uint64_t win_cap_bits = uint64_t(PackSmemT<WIDE>::WIN_WORDS) * 32 - 96;
    for (;;) {
      const uint32_t cand = b1 + tid;
      bool fits = false;
      if (cand < nb) {
        const uint64_t endb = (cand + 1 < nb) ? entry_pos(cand + 1, 0) : body_end + skew;
        fits = endb - win_p0 <= win_cap_bits;
      }
      const uint32_t more = __syncthreads_count(fits ? 1 : 0);
      b1 += more;
      if (more < PACK_THREADS) break;
    }
    const uint64_t win_end_p = (b1 < nb) ? entry_pos(b1, 0) : body_end + skew;
    const uint32_t win_words = uint32_t((win_end_p - win_p0 + 31) / 32) + 1;
    for (uint32_t i = tid; i < win_words; i += PACK_THREADS) sm.win[i] = 0;
    __syncthreads();
    if (tid == 0 && s_carry) sm.win[0] = s_carry;
    __syncthreads();
    // the next batch's vectors (8 symbols, 8 tANS fields, 8 keys per lane) are requested while this one is packed
    const uint32_t bv_end = b1 * n_vars;
    using SymVec = typename std::conditional<WIDE, uint4, uint2>::type;  // 8 symbols
    SymVec nx_s8{};
    uint4 nx_a8 = make_uint4(0u, 0u, 0u, 0u), nx_k8 = make_uint4(0u, 0u, 0u, 0u);
    uint32_t nx_pos = 0;
    auto prefetch = [&](uint32_t bvn) {
      const uint32_t bn = n_vars == 1 ? bvn : bvn / n_vars, vn = n_vars == 1 ? 0u : bvn % n_vars;
      nx_pos = entries[(size_t(c) * MAX_VARS + vn) * batches_per_chunk + bn].bit_pos;
      const uint64_t row = rb + uint64_t(bn) * BATCH_N + lane * 8;
      nx_s8 = *reinterpret_cast<const SymVec*>((vn == 0 ? sym0 : sym1) + row);
      if (vn == 0 ? ans_0 : ans_1) nx_a8 = *reinterpret_cast<const uint4*>((vn == 0 ? ans0 : ans1) + row);
      const uint16_t* kp = vn == 0 ? keyp_0 : keyp_1;
      if (kp != nullptr) nx_k8 = *reinterpret_cast<const uint4*>(kp + row);
    };
    uint32_t bv = b0 * n_vars + warp;
    if (bv < bv_end) prefetch(bv);
    for (; bv < bv_end; bv += PACK_THREADS / 32) {
      const uint32_t b = n_vars == 1 ? bv : bv / n_vars, v = n_vars == 1 ? 0u : bv % n_vars;
      const SymVec s8 = nx_s8;
      const uint4 a8 = nx_a8, k8 = nx_k8;
      const uint32_t my_pos = nx_pos;
      if (bv + PACK_THREADS / 32 < bv_end) prefetch(bv + PACK_THREADS / 32);
      const uint32_t cnt = batch_count(v == 0 ? stored_0 : stored_1, b);
      if (cnt == 0) continue;
      if (lean && cnt == uint32_t(BATCH_N)) {
        // ---- the common case, without the generality: one var, tANS fields and 16-bit keys, a full batch.  Field widths
        // come ready-made (tANS: bits 12-15 of the field; offsets: the table entry), both lane totals go through ONE scan.
        const uint32_t p = uint32_t(my_pos + skew - win_p0);
        const uint32_t aw[4] = {a8.x, a8.y, a8.z, a8.w}, kw[4] = {k8.x, k8.y, k8.z, k8.w};
        uint32_t a_val[8], a_bits[8], o32[8], o_bits[8], tot = 0;
#pragma unroll
        for (int e = 0; e < 8; e++) {
          const uint32_t x = aw[e >> 1] >> (16 * (e & 1));
          a_bits[e] = (x >> 12) & 0xfu;
          a_val[e] = x & 0xfffu;
          const uint32_t t = sm.lowkey_ob[0][((e < 4 ? s8.x : s8.y) >> (8 * (e & 3))) & 0xffu];
          o_bits[e] = t >> 16;
          o32[e] = ((kw[e >> 1] >> (16 * (e & 1))) - t) & 0xffffu;
          tot += a_bits[e] + (o_bits[e] << 16);
        }
        uint32_t inc = tot;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t o = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += o; }
        const uint32_t ans_total = __shfl_sync(0xffffffffu, inc, 31) & 0xffffu;
        const uint32_t exc = inc - tot;
        if (tot & 0xffffu) emit8_narrow(sm.win, p + (exc & 0xffffu), a_val, a_bits);
        if (tot >> 16) emit8_narrow(sm.win, p + ans_total + (exc >> 16), o32, o_bits);
        continue;
      }
      const bool needs_ans = v == 0 ? ans_0 : ans_1;
      const uint32_t max_ob = v == 0 ? mob_0 : mob_1;
      const uint64_t sb = fb ? cs : stored_begin(cs, ce, v == 0 ? order : 0);
      const L* latp = (v == 0 ? lat0 : lat1) + rb + uint64_t(b) * BATCH_N;
      uint32_t pos = uint32_t(my_pos + skew - win_p0);
      // lane owns elements 8 lane .. 8 lane + 7: its fields are contiguous in the stream, so it assembles them in a
      // register and ORs whole 32-bit words into the window.  Rows are 256-aligned (split_delta_kernel): vector loads.
      const uint32_t first = lane * 8;
      uint32_t sy[8];
#pragma unroll
      for (int e = 0; e < 8; e++) {
        if constexpr (WIDE) sy[e] = ((&s8.x)[e >> 1] >> (16 * (e & 1))) & 0xffffu;
        else sy[e] = ((e < 4 ? s8.x : s8.y) >> (8 * (e & 3))) & 0xffu;
      }
      // --- ANS fields (chunk_latent_compressor.rs:285-297)
      uint32_t a_val[8], a_bits[8], a_tot = 0;
      if (needs_ans) {
        const uint32_t aw[4] = {a8.x, a8.y, a8.z, a8.w};
#pragma unroll
        for (int e = 0; e < 8; e++) {
          const uint32_t x = (aw[e >> 1] >> (16 * (e & 1))) & 0xffffu;
          const bool live = first + e < cnt;
          const uint32_t nbits = live ? x >> 12 : 0u;
          a_bits[e] = nbits;
          a_val[e] = live ? x & 0xfffu : 0u;
          a_tot += nbits;
        }
      } else {
#pragma unroll
        for (int e = 0; e < 8; e++) { a_val[e] = 0; a_bits[e] = 0; }
      }
      uint32_t inc = a_tot;
      for (int d = 1; d < 32; d <<= 1) { uint32_t o = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += o; }
      const uint32_t ans_total = __shfl_sync(0xffffffffu, inc, 31);
      if (a_tot) emit8_narrow(sm.win, pos + inc - a_tot, a_val, a_bits);  // a field is <= size_log <= 10 bits
      // --- offsets (chunk_latent_compressor.rs:299-327)
      if (!WIDE && max_ob > 0 && (v == 0 ? keyp_0 : keyp_1) != nullptr) {
        // 16-bit keys: offset = key - (lower - key_base) mod 2^16; offset_bits <= 15
        const uint32_t kw[4] = {k8.x, k8.y, k8.z, k8.w};
        uint32_t o_bits[8], o32[8], o_tot = 0;
#pragma unroll
        for (int e = 0; e < 8; e++) {
          const uint32_t t = sm.lowkey_ob[v][sy[e]];
          const bool live = first + e < cnt;
          o_bits[e] = live ? t >> 16 : 0u;
          o32[e] = live ? (((kw[e >> 1] >> (16 * (e & 1))) - t) & 0xffffu) : 0u;
          o_tot += o_bits[e];
        }
        uint32_t oinc = o_tot;
        for (int d = 1; d < 32; d <<= 1) { uint32_t o = __shfl_up_sync(0xffffffffu, oinc, d); if (lane >= d) oinc += o; }
        if (o_tot) emit8_narrow(sm.win, pos + ans_total + oinc - o_tot, o32, o_bits);  // a key-path offset is <= 15 bits
      } else if (max_ob > 0) {
        uint32_t o_bits[8], o_tot = 0;
        L o_val[8];
        if (fb) {
#pragma unroll
          for (int e = 0; e < 8; e++) o_val[e] = first + e < cnt ? fallback_latent<L>(ep, sb + uint64_t(b) * BATCH_N + first + e) : L(0);
        } else {
          const Vec8<L> l8 = *reinterpret_cast<const Vec8<L>*>(latp + first);
#pragma unroll
          for (int e = 0; e < 8; e++) o_val[e] = l8.v[e];
        }
#pragma unroll
        for (int e = 0; e < 8; e++) {
          const bool live = first + e < cnt;
          o_bits[e] = live ? uint32_t(sm.obs[v][sy[e]]) : 0u;
          o_val[e] = live ? L(o_val[e] - L(sm.lowers[v][sy[e]])) : L(0);
          o_tot += o_bits[e];
        }
        uint32_t oinc = o_tot;
        for (int d = 1; d < 32; d <<= 1) { uint32_t o = __shfl_up_sync(0xffffffffu, oinc, d); if (lane >= d) oinc += o; }
        if (max_ob <= 15) {
          uint32_t o32[8];
#pragma unroll
          for (int e = 0; e < 8; e++) o32[e] = uint32_t(o_val[e]);
          if (o_tot) emit8_narrow(sm.win, pos + ans_total + oinc - o_tot, o32, o_bits);
          continue;
        }
        BitAcc acc(sm.win, pos + ans_total + oinc - o_tot);
#pragma unroll
        for (int e = 0; e < 8; e++) {
          if constexpr (sizeof(L) == 8) {
            if (o_bits[e] > 32) { acc.put(uint32_t(o_val[e]), 32); acc.put(uint32_t(uint64_t(o_val[e]) >> 32), o_bits[e] - 32); }
            else acc.put(uint32_t(o_val[e]), o_bits[e]);
          } else {
            acc.put(uint32_t(o_val[e]), o_bits[e]);
          }
        }
        acc.flush();
      }
    }
    __syncthreads();
    // copy out whole words; a partially filled last word carries into the next window
    const uint64_t span_bits = win_end_p - win_p0;
    const uint32_t whole_words = (b1 < nb) ? uint32_t(span_bits / 32) : uint32_t((span_bits + 31) / 32);
    {
      uint32_t* gw = dst_words + (win_p0 >> 5);
      const uint64_t byte0 = win_p0 >> 3;
      if (byte0 >= lo_byte && byte0 + 4ull * whole_words <= hi_byte) {  // every word lies inside the body: plain copy
        for (uint32_t i = tid; i < whole_words; i += PACK_THREADS) gw[i] = sm.win[i];
      } else
      for (uint32_t i = tid; i < whole_words; i += PACK_THREADS) {
        const uint64_t wb0 = byte0 + 4ull * i;
        const uint32_t word = sm.win[i];
        if (wb0 >= lo_byte && wb0 + 4 <= hi_byte) gw[i] = word;
        else {
          uint8_t* g8 = reinterpret_cast<uint8_t*>(gw + i);
          for (uint32_t k = 0; k < 4; k++)
            if (wb0 + k >= lo_byte && wb0 + k < hi_byte) g8[k] = uint8_t(word >> (8 * k));
        }
      }
      if (tid == 0) s_carry = (b1 < nb && (span_bits & 31)) ? sm.win[whole_words] : 0;
    }
    __syncthreads();
    win_p0 += uint64_t(whole_words) * 32;
    b0 = b1;
  }
}

// standalone header + terminator (standalone/compressor.rs:85-105,157-163), written by one thread
__global__ void header_footer_kernel(uint8_t* out, uint64_t out_cap, const uint8_t* header, uint32_t header_bytes, const uint64_t* total_bytes) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    uint64_t total = *total_bytes;
    if (total > out_cap) return;
    for (uint32_t i = 0; i < header_bytes; i++) out[i] = header[i];
    out[total - 1] = 0;
  }
}

}  // namespace pcob200
