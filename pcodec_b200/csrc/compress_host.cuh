// Host orchestration of the compress path: validates the ChunkConfig like the reference, lays out the
// chunks, runs the encode kernels on one stream and returns the .pco bytes (+ optional side index).
#pragma once
#include <atomic>
#include <cmath>
#include <map>
#include <mutex>
#include <thread>

#include "encode_kernels.cuh"
#include "host_common.hpp"
#include "mode_search.hpp"

namespace pcob200 {

// internal flag of compress_typed (not in the public enum): the call's chunks are the PAGES of one wrapped chunk and share
// bins trained on all of them (pco/src/wrapped/chunk_compressor.rs:129-140)
constexpr uint32_t PCO_B200_INTERNAL_SHARED_BINS = 1u << 16;


struct CompressScratch {
  DevBuf lat0, lat1, keys_a, keys_b, sym0, sym1, ans0, ans1, ob_sum, ans_sum, entries, plans, chunks, starts, seg, out, small, index, probes, sample, sample_starts, key16_0, key16_1, idx_out, lb_vals, lb_resid, lb_scratch;
  // set_encode_attrs has run for [WIDE][log2(sizeof(L))]
  bool encode_attrs_set[2][4] = {};
  bool src_in_place = false;  // this call reads its numbers from the caller's page-locked host buffer (host_common.hpp, zero copy)
  // ans_encode_kernel's round counters of the last call, kept only while profiling is on (pco_b200_profile_ans_paths)
  DevBuf ans_paths;
  bool ans_paths_valid = false;
  void release() {
    for (DevBuf* b : {&lat0, &lat1, &keys_a, &keys_b, &sym0, &sym1, &ans0, &ans1, &ob_sum, &ans_sum, &entries, &plans, &chunks, &starts, &seg, &out, &small,
                      &index, &probes, &sample, &sample_starts, &key16_0, &key16_1, &idx_out, &lb_vals, &lb_resid, &lb_scratch, &ans_paths})
      b->release();
    ans_paths_valid = false;
  }
};

// pco/src/chunk_config.rs:134-183
inline PcoB200Error n_per_page(const PcoB200ChunkConfig& cfg, size_t n, std::vector<uint64_t>* out) {
  out->clear();
  if (cfg.paging_spec == PCO_B200_PAGING_EXACT) {
    out->assign(cfg.exact_page_ns, cfg.exact_page_ns + cfg.n_exact_pages);
  } else {
    const EqualPages ep = equal_pages(n, cfg.max_page_n);
    for (uint64_t c = 0; c < ep.n_chunks; c++) out->push_back(ep.size(c));
  }
  uint64_t summed = 0;
  for (uint64_t p : *out) summed += p;
  if (summed != n)
    return fail(PCO_B200_INVALID_ARGUMENT, "paging spec suggests " + std::to_string(summed) + " numbers but " + std::to_string(n) + " were given");
  for (uint64_t p : *out)
    if (p == 0) return fail(PCO_B200_INVALID_ARGUMENT, "cannot write data page of 0 numbers");
  return PCO_B200_OK;
}

// Scratch of one CHUNKS_ONLY pass of compress_typed over n numbers in chunks of the given sizes: the chunks' bytes (64, and each chunk's
// size guarantee plus 8 bytes of slack) and the side index.
struct ChunksScratch {
  size_t bytes, index;
};
inline ChunksScratch chunks_only_scratch(uint32_t lbits, uint64_t n, const std::vector<uint64_t>& chunk_ns) {
  ChunksScratch s{64, pco_b200_index_size_bound(size_t(n), chunk_ns.size()) + 64 * chunk_ns.size()};
  for (uint64_t p : chunk_ns) s.bytes += standalone_chunk_size_guarantee(lbits, size_t(p)) + 8;
  return s;
}

// standalone header bytes (pco/src/standalone/compressor.rs:12-16,85-105) into out[0 .. STANDALONE_HEADER_MAX); returns their count.
// The size hint is a varint: 6 bits (power - 1), then the `power` bits of n_hint.
constexpr uint32_t STANDALONE_HEADER_MAX = 17;
__host__ __device__ inline uint32_t size_hint_power(uint64_t n_hint) {
  uint32_t power = 1;
  while (power < 64 && (n_hint >> power) != 0) power++;
  return power;
}
__host__ __device__ inline uint32_t standalone_header_len(uint64_t n_hint) { return 8 + (6 + size_hint_power(n_hint) + 7) / 8; }
__host__ __device__ inline uint32_t standalone_header_into(uint64_t n_hint, uint8_t uniform_type, uint8_t* out) {
  const uint8_t magic[6] = {112, 99, 111, 33, 3, uniform_type};
  for (int i = 0; i < 6; i++) out[i] = magic[i];
  const uint32_t power = size_hint_power(n_hint), len = standalone_header_len(n_hint);
  for (uint32_t i = 0; i < len - 8; i++) out[6 + i] = uint8_t(i == 0 ? ((power - 1) | (n_hint << 6)) : (n_hint >> (8 * i - 6)));
  out[len - 2] = 4;
  out[len - 1] = 1;
  return len;
}
inline std::vector<uint8_t> make_standalone_header(uint64_t n_hint, uint8_t uniform_type) {
  uint8_t h[STANDALONE_HEADER_MAX];
  return std::vector<uint8_t>(h, h + standalone_header_into(n_hint, uniform_type, h));
}

__global__ void range_bits_kernel(ChunkEnc* chunks, uint32_t n_chunks, int v, uint32_t* out_bits) {
  uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_chunks) return;
  uint64_t a = chunks[c].vmin[v], b = chunks[c].vmax[v];
  uint32_t bits = b > a ? 64 - __clzll((long long)(b - a)) : 0;
  atomicMax(out_bits, bits);
  chunks[c].key_base[v] = a;  // plan_probe_kernel's keys are latent - vmin
}

// internal entries [(c, v)][batches_per_chunk] of one run -> its piece of the compact side index.  chunk_base / elem_base: index of the run's
// first chunk in the call and element offset of its first number; the file-level header fields are written by the call's last run.
__global__ void emit_index_kernel(EncParams ep, uint32_t batches_per_chunk, const ChunkEnc* chunks, const BatchEntry* entries, uint8_t* index,
                                  uint64_t chunks_offset, const uint64_t* entry_offsets, const uint64_t* total_bytes, uint32_t has_terminator, uint32_t chunk_base,
                                  uint64_t elem_base, uint32_t last_run) {
  const uint32_t c = blockIdx.x;
  if (c == 0 && threadIdx.x == 0 && last_run) {  // the file size is known on the device first: the host need not wait for it to write the header
    IndexHeader* ih = reinterpret_cast<IndexHeader*>(index);
    ih->file_len = *total_bytes;
    ih->end_byte = has_terminator ? *total_bytes : 0;
  }
  const uint64_t cs = ep.chunk_starts[c], ce = ep.chunk_starts[c + 1];
  const uint32_t n = uint32_t(ce - cs);
  const uint32_t nb = n_batches_of(n);
  const uint32_t n_vars = chunks[c].fallback ? 1 : ep.n_vars;
  if (threadIdx.x == 0) {
    IndexChunk ic;
    ic.chunk_offset = chunks[c].out_offset;
    ic.n = n;
    ic.n_vars = n_vars;
    ic.entries_offset = entry_offsets[c];
    ic.out_offset = elem_base + cs;
    reinterpret_cast<IndexChunk*>(index + chunks_offset)[chunk_base + c] = ic;
  }
  BatchEntry* dst = reinterpret_cast<BatchEntry*>(index + entry_offsets[c]);
  for (uint32_t i = threadIdx.x; i < n_vars * nb; i += blockDim.x) {
    uint32_t v = i / nb, b = i % nb;
    dst[size_t(v) * nb + b] = entries[(size_t(c) * MAX_VARS + v) * batches_per_chunk + b];
  }
}

// several runs: the first writes the standalone header, the last the terminator byte (standalone/compressor.rs:85-105,157-163)
__global__ void run_edge_kernel(uint8_t* out, uint64_t out_cap, const uint8_t* header, uint32_t header_bytes, const uint64_t* total_bytes, uint32_t footer) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    const uint64_t total = *total_bytes;
    if (total > out_cap) return;
    for (uint32_t i = 0; i < header_bytes; i++) out[i] = header[i];
    if (footer) out[total - 1] = 0;
  }
}

struct CompressResult {
  uint64_t total_bytes = 0;
  uint64_t index_bytes = 0;
};

// A chunk's resolved mode: what EncParams carries about it
struct ModeSel {
  uint32_t mode = MODE_CLASSIC;
  uint64_t mode_base = 0, base_bits = 0, inv_base_bits = 0;
  uint32_t mode_k = 0;
  bool operator==(const ModeSel& o) const {
    return mode == o.mode && mode_base == o.mode_base && base_bits == o.base_bits && inv_base_bits == o.inv_base_bits && mode_k == o.mode_k;
  }
};

inline void set_float_mult(ModeSel* ms, uint32_t lbits, double base_d, double inv_d) {
  ms->mode = MODE_FLOAT_MULT;
  if (lbits == 64) {
    std::memcpy(&ms->base_bits, &base_d, 8);
    std::memcpy(&ms->inv_base_bits, &inv_d, 8);
    ms->mode_base = (ms->base_bits >> 63) ? ~ms->base_bits : (ms->base_bits ^ (uint64_t(1) << 63));
  } else {
    const float base = float(base_d), inv = float(inv_d);
    uint32_t bb, ib;
    std::memcpy(&bb, &base, 4);
    std::memcpy(&ib, &inv, 4);
    ms->base_bits = bb;
    ms->inv_base_bits = ib;
    ms->mode_base = (bb >> 31) ? uint32_t(~bb) : (bb ^ 0x80000000u);
  }
}

// The EncParams of a pass: the number type, the header flavour (uniform_type: the dtype or 0), the mode, the delta order and the primary
// var's unoptimized_bins_log (the CHUNK_BINS kernels read the level there).  The caller fills the chunk fields.
inline EncParams enc_params(uint32_t dtype, uint32_t uniform_type, const ModeSel& ms, uint32_t order, uint32_t bins_log) {
  EncParams ep;
  std::memset(&ep, 0, sizeof(ep));
  ep.dtype = dtype;
  ep.uniform_type = uniform_type;
  ep.mode = ms.mode;
  ep.mode_base = ms.mode_base;
  ep.base_bits = ms.base_bits;
  ep.inv_base_bits = ms.inv_base_bits;
  ep.mode_k = ms.mode_k;
  ep.order = order;
  ep.n_vars = ms.mode == MODE_CLASSIC ? 1 : 2;
  ep.bins_log[0] = bins_log;
  ep.bins_log[1] = std::min<uint32_t>(bins_log, 6);  // LIMITED_UNOPTIMIZED_BINS_LOG (chunk_compressor.rs:238-248)
  return ep;
}

// The shared-memory size and carveout attributes of the encode kernels of latent type L: the narrow instantiations (the planner's in
// their CHUNK_BINS form when CHUNK_BINS), or the wide ones when WIDE.
template <typename L, bool WIDE, bool CHUNK_BINS = false>
inline cudaError_t set_encode_attrs() {
  const int count_smem = int(((size_t(1) << PLAN_MAX_COUNT_BITS) + 1) * 4 + 16), max_shared = int(cudaSharedmemCarveoutMaxShared);
  cudaError_t err = cudaSuccess;
  auto set = [&](const void* f, cudaFuncAttribute attr, int value) {
    if (err == cudaSuccess) err = cudaFuncSetAttribute(f, attr, value);
  };
  if constexpr (WIDE) {
    set((const void*)plan_probe_kernel<L, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, count_smem);
    set((const void*)plan_solve_wide_kernel<L>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(sizeof(WideSolveSmem)));
    set((const void*)pack_kernel<L, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(sizeof(PackSmemT<true>)));
    set((const void*)plan_probe_kernel<L, true, true>, cudaFuncAttributePreferredSharedMemoryCarveout, max_shared);
    set((const void*)plan_solve_wide_kernel<L>, cudaFuncAttributePreferredSharedMemoryCarveout, max_shared);
    set((const void*)pack_kernel<L, true>, cudaFuncAttributePreferredSharedMemoryCarveout, max_shared);
  } else {
    set((const void*)plan_probe_kernel<L, true, false, CHUNK_BINS>, cudaFuncAttributeMaxDynamicSharedMemorySize, count_smem);
    set((const void*)split_count_kernel<L, CHUNK_BINS>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(size_t(SC_N) * 4));
    set((const void*)union_probe_kernel<L>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(size_t(SC_N) * 4));
    set((const void*)pack_kernel<L>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(sizeof(PackSmem)));
    set((const void*)radix_sort_segments_kernel<L>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(size_t(RS_WARPS) * RS_BINS * sizeof(uint32_t)));
    // several counting CTAs per SM: ask for the largest shared-memory carveout
    set((const void*)plan_probe_kernel<L, true, false, CHUNK_BINS>, cudaFuncAttributePreferredSharedMemoryCarveout, max_shared);
    set((const void*)pack_kernel<L>, cudaFuncAttributePreferredSharedMemoryCarveout, max_shared);
    set((const void*)bin_lut_kernel<L>, cudaFuncAttributePreferredSharedMemoryCarveout, max_shared);
  }
  return err;
}

// the numbers of every chunk at the positions choose_mode_sample visits (sampling.rs:73-95): positions depend on the chunk's n only
template <typename L>
__global__ void gather_positions_kernel(const L* __restrict__ nums, const uint64_t* __restrict__ chunk_starts, const uint32_t* __restrict__ chunk_ids,
                                        const uint32_t* __restrict__ pos, uint32_t m, L* __restrict__ out) {
  const uint32_t c = chunk_ids[blockIdx.x];
  const L* src = nums + chunk_starts[c];
  L* dst = out + size_t(blockIdx.x) * m;
  for (uint32_t j = threadIdx.x; j < m; j += blockDim.x) dst[j] = src[pos[j]];
}

// the delta sample (sampling.rs:21-60) of every chunk's PRIMARY latents under the chunk's own mode, as unsigned numbers of width L
struct ModeSelDev { uint32_t mode, mode_k; uint64_t mode_base, base_bits, inv_base_bits; };
template <typename L>
__global__ void gather_primary_sample_kernel(const L* __restrict__ nums, const uint64_t* __restrict__ chunk_starts, const uint64_t* __restrict__ sample_starts,
                                             const ModeSelDev* __restrict__ modes, uint32_t dtype, L* __restrict__ sample) {
  const uint32_t c = blockIdx.x;
  const uint64_t cs = chunk_starts[c], n = chunk_starts[c + 1] - cs;
  const SampleGeom g = delta_sample_geom(n);
  const uint32_t ns = g.n_groups * g.group_n;
  L* dst = sample + sample_starts[c];
  const ModeSelDev ms = modes[c];
  EncParams ep;
  ep.dtype = dtype; ep.mode = ms.mode; ep.mode_k = ms.mode_k; ep.mode_base = ms.mode_base; ep.base_bits = ms.base_bits; ep.inv_base_bits = ms.inv_base_bits;
  const bool is_float = nt_is_float(dtype), is_signed = nt_is_signed(dtype);
  for (uint32_t i = threadIdx.x; i < ns; i += blockDim.x) {
    const L x = nums[cs + uint64_t(i / g.group_n) * g.stride + i % g.group_n];
    L pr, se;
    switch (ms.mode) {
      case MODE_INT_MULT: split_one<L, MODE_INT_MULT>(x, ep, is_float, is_signed, pr, se); break;
      case MODE_FLOAT_MULT: split_one<L, MODE_FLOAT_MULT>(x, ep, is_float, is_signed, pr, se); break;
      case MODE_FLOAT_QUANT: split_one<L, MODE_FLOAT_QUANT>(x, ep, is_float, is_signed, pr, se); break;
      default: split_one<L, MODE_CLASSIC>(x, ep, is_float, is_signed, pr, se); break;
    }
    dst[i] = pr;
  }
}

// The Lookback candidate of the Auto delta search (chunk_compressor.rs:326-338) on every chunk's delta sample: choose_lookbacks
// (delta/lookback.rs:96-159: brute-force, repeating and hashed proposals, the best by goodness = leading zeros of the difference + a
// popularity bonus) and encode_in_place (:166-187), by ONE thread per chunk - the search is a serial state machine (hash table of last
// positions, running popularity counts).  Outputs per chunk, len - 1 entries each at out_starts[c]: the lookbacks as u32 numbers and
// the residuals (latent - latent[i - lookback] + MID) as numbers of width L; both then go through the ordinary planner as trial vars.
constexpr uint32_t LB_PROPOSED = 16, LB_BRUTE = 6, LB_REPEATING = 4;
__host__ __device__ inline uint32_t lookback_window_n_log(uint64_t n) {  // delta::new_lookback (delta/mod.rs:37-48): state_n_log = 0
  const uint32_t x = uint32_t(n - 1);
  const uint32_t bits = x == 0 ? 0u : 32u -
#ifdef __CUDA_ARCH__
                                     uint32_t(__clz(x));
#else
                                     uint32_t(__builtin_clz(x));
#endif
  return bits < 4 ? 4u : bits > 15 ? 15u : bits;
}
template <typename L>
__global__ void lookback_trial_kernel(const L* __restrict__ sample, const uint64_t* __restrict__ sample_starts, const uint64_t* __restrict__ out_starts,
                                      uint32_t* __restrict__ lookbacks, L* __restrict__ resid, uint32_t* __restrict__ hash_scratch,
                                      uint32_t* __restrict__ count_scratch, uint32_t hash_stride, uint32_t count_stride) {
  const uint32_t c = blockIdx.x;
  const uint64_t len = sample_starts[c + 1] - sample_starts[c];
  if (len <= 1) return;
  const L* lat = sample + sample_starts[c];
  uint32_t* lb_out = lookbacks + out_starts[c];
  L* r_out = resid + out_starts[c];
  const uint32_t wlog = lookback_window_n_log(len);
  const uint32_t window_n = 1u << wlog, hash_table_n = 1u << (wlog + 1), hash_mask = hash_table_n - 1;
  uint32_t* table = hash_scratch + size_t(c) * hash_stride;   // [2][hash_table_n] last position of a bucket
  uint32_t* counts = count_scratch + size_t(c) * count_stride;  // [min(window_n, len)] how often a lookback was used
  const uint32_t n_counts = uint32_t(min(uint64_t(window_n), len));
  for (uint32_t i = threadIdx.x; i < 2 * hash_table_n; i += blockDim.x) table[i] = 0;
  for (uint32_t i = threadIdx.x; i < n_counts; i += blockDim.x) counts[i] = 1;
  __syncthreads();
  if (threadIdx.x != 0) return;
  constexpr L MID = L(L(1) << (sizeof(L) * 8 - 1));
  uint32_t proposed[LB_PROPOSED];
#pragma unroll
  for (uint32_t i = 0; i < LB_PROPOSED; i++) proposed[i] = 1;  // (i + 1).min(state_n), state_n = 1
  uint32_t best_lookback = 1, repeating_idx = 0;
  auto hash_fn = [&](uint64_t x) -> uint32_t {
    x = (x ^ (x >> 32)) * 11400714819323197441ull;
    x = x ^ (x >> 32);
    return uint32_t(x) & hash_mask;
  };
  for (uint32_t i = 1; i < uint32_t(len); i++) {
    const L l = lat[i];
    const uint32_t new_brute = min(i, LB_PROPOSED);
    proposed[new_brute - 1] = new_brute;
    uint32_t proposal_idx = LB_BRUTE + LB_REPEATING, offset = 0;
#pragma unroll
    for (uint32_t coarse = 0; coarse < 2; coarse++) {  // COARSENESSES = [0, 8]
      const uint64_t bucket = uint64_t(l) >> (coarse * 8);
      const uint32_t h0 = hash_fn(bucket - 1), h1 = hash_fn(bucket), h2 = hash_fn(bucket + 1);
      const uint32_t hs[3] = {h0, h1, h2};
#pragma unroll
      for (int t = 0; t < 3; t++) {
        const uint32_t last = i - table[offset + hs[t]];
        proposed[proposal_idx] = last <= window_n ? last : min(proposal_idx, i);
        proposal_idx++;
      }
      table[offset + h1] = i;
      offset += hash_table_n;
    }
    uint32_t best_goodness = 0, new_best = 0;
#pragma unroll
    for (uint32_t t = 0; t < LB_PROPOSED; t++) {
      const uint32_t lookback = proposed[t];
      const uint32_t cnt = counts[lookback - 1];
      const L other = lat[i - lookback];
      const uint32_t lookback_goodness = 32 - uint32_t(__clz(cnt));
      const L d0 = L(l - other), d1 = L(other - l);
      const L delta = d0 < d1 ? d0 : d1;
      const uint32_t lz = sizeof(L) == 8 ? uint32_t(__clzll((long long)uint64_t(delta))) : uint32_t(__clz(uint32_t(delta))) - uint32_t(32 - sizeof(L) * 8);
      const uint32_t goodness = lookback_goodness + lz;
      if (goodness > best_goodness) { best_goodness = goodness; new_best = lookback; }
    }
    if (new_best != best_lookback) repeating_idx += 1;
    proposed[LB_BRUTE + repeating_idx % LB_REPEATING] = new_best;
    best_lookback = new_best;
    lb_out[i - 1] = new_best;
    r_out[i - 1] = L(L(l - lat[i - new_best]) + MID);
    counts[new_best - 1] += 1;
  }
}

// what the Auto delta search needs of a trial plan: bin count, table size and per bin (weight, offset bits) - 772 bytes per chunk
// (12 KB for wide plans)
template <bool WIDE>
struct PlanSummaryT { uint32_t n_bins, size_log; uint16_t weight[EncCap<WIDE>::MAXB]; uint8_t ob[EncCap<WIDE>::MAXB]; };
using PlanSummary = PlanSummaryT<false>;
template <bool WIDE = false>
__global__ void plan_summary_kernel(const VarPlanT<WIDE>* __restrict__ plans, uint32_t n_chunks, PlanSummaryT<WIDE>* __restrict__ out) {
  const uint32_t c = blockIdx.x;
  if (c >= n_chunks) return;
  const VarPlanT<WIDE>& p = plans[size_t(c) * MAX_VARS];
  if (threadIdx.x == 0) { out[c].n_bins = p.n_bins; out[c].size_log = p.size_log; }
  for (uint32_t i = threadIdx.x; i < uint32_t(EncCap<WIDE>::MAXB); i += blockDim.x) { out[c].weight[i] = p.weight[i]; out[c].ob[i] = p.ob[i]; }
}
// calculate_compressed_sample_size (chunk_compressor.rs:289-307): meta_size_hint() + page_size_hint_inner(0, 1.0) of a Classic one-page
// chunk holding the sample, as f32.  avg_bits_per_latent: metadata/bins.rs:23-32 (f64, bins in order).
template <typename Summary>
inline float sample_cost(const Summary& p, uint32_t lbits, uint32_t order, uint64_t sample_n) {
  const uint64_t meta_bits = 4 + (4 + 5 + 5 + 64 + 32 * 32) + 4 + 15 + uint64_t(p.n_bins) * (p.size_log + lbits + offset_bits_bits(lbits));
  const uint64_t page_bits = uint64_t(order) * lbits + 4ull * p.size_log;
  const double total_weight = double(uint64_t(1) << p.size_log);
  double acc = 0.0;
  for (uint32_t b = 0; b < p.n_bins; b++) {
    const double ans_bits = double(p.size_log) - std::log2(double(p.weight[b]));
    acc += (ans_bits + double(p.ob[b])) * double(p.weight[b]) / total_weight;
  }
  const uint64_t n_stored = sample_n > order ? sample_n - order : 0;
  const uint64_t body_bits = uint64_t(std::ceil(double(n_stored) * acc * 1.0));
  return float((meta_bits + 7) / 8 + (page_bits + 7) / 8 + (body_bits + 7) / 8);
}

// the same for the Lookback trial chunk: delta var (the lookbacks, u32) + primary (residuals, one latent of delta state per page)
template <typename Summary>
inline float lookback_sample_cost(const Summary& d, const Summary& p, uint32_t lbits, uint64_t n_stored) {
  const uint64_t meta_bits = 4 + (4 + 5 + 5 + 64 + 32 * 32) + (4 + 15 + uint64_t(d.n_bins) * (d.size_log + 32 + offset_bits_bits(32))) +
                             (4 + 15 + uint64_t(p.n_bins) * (p.size_log + lbits + offset_bits_bits(lbits)));
  const uint64_t page_bits = 4ull * d.size_log + (uint64_t(lbits) + 4ull * p.size_log);
  auto avg_bits = [](const Summary& v) {
    const double total_weight = double(uint64_t(1) << v.size_log);
    double acc = 0.0;
    for (uint32_t b = 0; b < v.n_bins; b++) acc += ((double(v.size_log) - std::log2(double(v.weight[b]))) + double(v.ob[b])) * double(v.weight[b]) / total_weight;
    return acc;
  };
  const uint64_t body_bits = uint64_t(std::ceil(double(n_stored) * avg_bits(d))) + uint64_t(std::ceil(double(n_stored) * avg_bits(p)));
  return float((meta_bits + 7) / 8 + (page_bits + 7) / 8 + (body_bits + 7) / 8);
}

// mode sample positions per chunk size (host, computed once per distinct n; sampling.rs:73-95)
inline const std::vector<uint32_t>& mode_sample_positions(size_t n) {
  static std::mutex mu;
  static std::map<size_t, std::vector<uint32_t>> cache;
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find(n);
  if (it == cache.end()) {
    std::vector<uint32_t> v;
    for (size_t p : mode_search::sample_positions(n)) v.push_back(uint32_t(p));
    if (cache.size() > 64) cache.clear();
    it = cache.emplace(n, std::move(v)).first;
  }
  return it->second;
}

// K1+K2 and the planner for one set of chunks (a run of a call's chunks, the chunks' samples during the Auto delta search, or a trial
// latent var of that search).  `e` describes the set (its own chunk_starts / row_base, counted from 0); plans and probes land in slots
// 0 .. e.n_chunks - 1 of the scratch.  T is the latent width the set is planned in (the number's, or u32 for lookback indices).
// WIDE: the set's unoptimized_bins_log is above 8 (levels 9-12).  Those sets take the two-kernel front end (split_delta_kernel, then
// the counting or sorting probe kernel) and plan_solve_wide_kernel; binning and packing then read the 64-bit latents.
template <typename L, bool WIDE = false>
static PcoB200Error plan_front(CompressScratch& S, cudaStream_t stream, EncParams& e, uint32_t tiles, size_t slots, uint32_t (&vrb)[MAX_VARS],
                               const std::vector<uint64_t>& sizes, bool shared, L* (&d_lat)[2]) {
  constexpr int LW = sizeof(L) == 1 ? 0 : sizeof(L) == 2 ? 1 : sizeof(L) == 4 ? 2 : 3;
  constexpr size_t RS_SMEM = size_t(RS_WARPS) * RS_BINS * sizeof(uint32_t);
  ChunkEnc* d_chunks = S.chunks.as<ChunkEnc>();
  VarPlanT<WIDE>* d_plans = S.plans.as<VarPlanT<WIDE>>();
  PlanProbesT<WIDE>* d_probes = S.probes.as<PlanProbesT<WIDE>>();
  uint32_t* d_small = S.small.as<uint32_t>();
  // the solver of the set's capacity, over `grid` chunks (n_override: see plan_solve_kernel)
  auto solve = [&](uint32_t grid, int v, uint32_t n_override) {
    if constexpr (WIDE) {
      profiler().begin("plan_solve_wide_kernel", stream);
      plan_solve_wide_kernel<L><<<grid, WSOLVE_THREADS, sizeof(WideSolveSmem), stream>>>(e, d_probes, d_chunks, d_plans, v, n_override);
    } else {
      profiler().begin("plan_solve_kernel", stream);
      plan_solve_kernel<L><<<grid, SOLVE_THREADS, 0, stream>>>(e, d_probes, d_chunks, d_plans, v, n_override);
    }
    profiler().end(stream);
  };

    const uint32_t n_chunks = e.n_chunks;
    PCOB_CUDA_TRY(S.lat0.reserve(slots * sizeof(L) + 64));
    if (e.n_vars > 1) PCOB_CUDA_TRY(S.lat1.reserve(slots * sizeof(L) + 64));
    d_lat[0] = S.lat0.as<L>();
    d_lat[1] = S.lat1.as<L>();
    init_chunks_kernel<<<(n_chunks + 255) / 256, 256, 0, stream>>>(d_chunks, n_chunks);
    for (const bool wide : {false, WIDE}) {
      if (S.encode_attrs_set[wide][LW]) continue;
      S.encode_attrs_set[wide][LW] = true;
      PCOB_CUDA_TRY((wide ? set_encode_attrs<L, true>() : set_encode_attrs<L, false>()));
    }
    if constexpr (!WIDE) {  // (wide sets: the two-kernel path below)
    if (e.mode == MODE_CLASSIC && e.n_vars == 1) {
      // one-pass front end: split + delta + counting histogram + 16-bit keys, no 64-bit latents (split_count_kernel).
      // It assumes every chunk's stored latents span < 2^15; a chunk that does not raises flags[1] and the call is redone
      // on the two-kernel path below (the speculation costs one read of the input).
      PCOB_CUDA_TRY(S.key16_0.reserve(slots * 2 + 64));
      PCOB_CUDA_TRY(cudaMemsetAsync(d_small, 0, 8, stream));
      profiler().begin("split_count_kernel", stream);
      split_count_kernel<L><<<n_chunks, SC_THREADS, size_t(SC_N) * 4, stream>>>(e, d_chunks, d_probes, S.key16_0.as<uint16_t>(), d_small);
      profiler().end(stream);
      PCOB_CUDA_TRY(cudaGetLastError());  // a failed launch must not read as "no chunk raised a flag"
      uint32_t fl[2] = {0, 0};
      PCOB_CUDA_TRY(readback_small_sync(fl, d_small, 8, stream));
      call_trace().mark("c.flags");
      if (fl[1] == 0 && shared) {
        // pages of one chunk: one histogram over all of them, one plan, copied to every page's slot
        PCOB_CUDA_TRY(cudaMemsetAsync(d_small, 0, 8, stream));
        profiler().begin("union_probe_kernel", stream);
        union_probe_kernel<L><<<1, SC_THREADS, size_t(SC_N) * 4, stream>>>(e, n_chunks, d_chunks, d_probes, S.key16_0.as<uint16_t>(), d_small);
        profiler().end(stream);
        PCOB_CUDA_TRY(cudaMemcpyAsync(fl, d_small, 8, cudaMemcpyDeviceToHost, stream));
        PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
        if (fl[1] == 0) {
          vrb[0] = fl[0];
          uint64_t stored_total = 0;
          for (uint64_t pn : sizes) stored_total += pn > e.order ? pn - e.order : 0;
          profiler().begin("plan_solve_kernel", stream);
          plan_solve_kernel<L><<<1, SOLVE_THREADS, 0, stream>>>(e, d_probes, d_chunks, d_plans, 0, uint32_t(stored_total));
          profiler().end(stream);
          broadcast_plan_kernel<<<n_chunks, 128, 0, stream>>>(d_plans, n_chunks);
          return PCO_B200_OK;
        }
        fl[1] = 1;  // every page is narrow but their union is not: the two-kernel path below (it needs the 64-bit latents)
      }
      if (fl[1] == 0) {
        vrb[0] = fl[0];
        profiler().begin("plan_solve_kernel", stream);
        plan_solve_kernel<L><<<n_chunks, SOLVE_THREADS, 0, stream>>>(e, d_probes, d_chunks, d_plans, 0);
        profiler().end(stream);
        return PCO_B200_OK;
      }
      init_chunks_kernel<<<(n_chunks + 255) / 256, 256, 0, stream>>>(d_chunks, n_chunks);
      if (S.src_in_place) {
        // the speculation read the numbers in place over PCIe; the two-kernel path would read them again: bring this set into HBM
        // first (the in-place pointer of a page-locked buffer is also its host address)
        PCOB_CUDA_TRY(S.index.reserve(size_t(e.n_total) * sizeof(L) + 64));
        PCOB_CUDA_TRY(copy_sliced(S.index.p, e.nums, size_t(e.n_total) * sizeof(L), cudaMemcpyHostToDevice, stream));
        e.nums = S.index.p;
      }
    }
    }
    profiler().begin("split_delta_kernel", stream);
    switch (e.mode) {
      case MODE_CLASSIC: split_delta_kernel<L, MODE_CLASSIC><<<n_chunks * tiles, SPLIT_THREADS, 0, stream>>>(e, tiles, d_lat[0], d_lat[1], d_chunks); break;
      case MODE_INT_MULT: split_delta_kernel<L, MODE_INT_MULT><<<n_chunks * tiles, SPLIT_THREADS, 0, stream>>>(e, tiles, d_lat[0], d_lat[1], d_chunks); break;
      case MODE_FLOAT_QUANT: split_delta_kernel<L, MODE_FLOAT_QUANT><<<n_chunks * tiles, SPLIT_THREADS, 0, stream>>>(e, tiles, d_lat[0], d_lat[1], d_chunks); break;
      default: split_delta_kernel<L, MODE_FLOAT_MULT><<<n_chunks * tiles, SPLIT_THREADS, 0, stream>>>(e, tiles, d_lat[0], d_lat[1], d_chunks); break;
    }
    profiler().end(stream);
    // ---- planner per var: range-reduced keys -> segmented radix sort over the significant bits -> plan
    if (shared) {
      // pages of one wrapped chunk on the sort path: common minimum, the pages' keys as one gap-free segment, one sort,
      // the union's probes and plan, copied to every page's slot (classic mode: one latent var)
      PCOB_CUDA_TRY(cudaMemsetAsync(d_small, 0, 4, stream));
      profiler().begin("union_range_kernel", stream);
      union_range_kernel<<<1, 32, 0, stream>>>(e, n_chunks, d_chunks, d_small);
      profiler().end(stream);
      uint32_t range_bits = 0;
      PCOB_CUDA_TRY(cudaMemcpyAsync(&range_bits, d_small, 4, cudaMemcpyDeviceToHost, stream));
      PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
      vrb[0] = std::max<uint32_t>(range_bits, PLAN_MAX_COUNT_BITS + 1);  // binning and packing read the 64-bit latents on this path
      std::vector<uint64_t> prefix(sizes.size() + 1, 0);
      for (size_t i = 0; i < sizes.size(); i++) prefix[i + 1] = prefix[i] + (sizes[i] > e.order ? sizes[i] - e.order : 0);
      const uint64_t stored_total = prefix.back();
      PCOB_CUDA_TRY(S.keys_a.reserve(slots * sizeof(L) + 64));
      PCOB_CUDA_TRY(S.keys_b.reserve(slots * sizeof(L) + 64));
      PCOB_CUDA_TRY(S.seg.reserve((prefix.size() + 2) * 8 + 64));
      uint64_t* d_prefix = S.seg.as<uint64_t>();  // [0 .. n_pages]: compaction offsets; then {segment begin, segment end}
      PCOB_CUDA_TRY(cudaMemcpyAsync(d_prefix, prefix.data(), prefix.size() * 8, cudaMemcpyHostToDevice, stream));
      const uint64_t seg_host[2] = {0, stored_total};
      uint64_t* d_seg = d_prefix + prefix.size();
      PCOB_CUDA_TRY(cudaMemcpyAsync(d_seg, seg_host, 16, cudaMemcpyHostToDevice, stream));
      // (span names prefixed union_: one segment holding every page, told apart from the per-chunk sort below)
      profiler().begin("union_sort_keys_kernel", stream);
      sort_keys_kernel<L><<<n_chunks * tiles, 256, 0, stream>>>(e, tiles, d_lat[0], S.keys_a.as<L>(), d_chunks, 0, d_prefix);
      profiler().end(stream);
      const L* sorted = S.keys_a.as<L>();
      if (stored_total > 1) {
        const uint32_t sort_bits = std::max<uint32_t>(range_bits, 1);
        profiler().begin("union_radix_sort_kernel", stream);
        radix_sort_segments_kernel<L><<<1, RS_THREADS, RS_SMEM, stream>>>(S.keys_a.as<L>(), S.keys_b.as<L>(), d_seg, d_seg + 1, sort_bits);
        profiler().end(stream);
        if (((sort_bits + RS_BITS - 1) / RS_BITS) & 1) sorted = S.keys_b.as<L>();
      }
      profiler().begin("union_plan_probe_kernel_sorted", stream);
      plan_probe_kernel<L, false, WIDE><<<1, PLAN_THREADS, 16, stream>>>(e, sorted, d_chunks, d_probes, 0, range_bits, nullptr, uint32_t(stored_total));
      profiler().end(stream);
      solve(1, 0, uint32_t(stored_total));
      broadcast_plan_kernel<WIDE><<<n_chunks, 128, 0, stream>>>(d_plans, n_chunks);
      return PCO_B200_OK;
    }
    for (uint32_t v = 0; v < e.n_vars; v++) {
      const uint32_t order_v = v == 0 ? e.order : 0;
      PCOB_CUDA_TRY(cudaMemsetAsync(d_small, 0, 4, stream));
      range_bits_kernel<<<(n_chunks + 255) / 256, 256, 0, stream>>>(d_chunks, n_chunks, int(v), d_small);
      uint32_t range_bits = 0;
      PCOB_CUDA_TRY(cudaMemcpyAsync(&range_bits, d_small, 4, cudaMemcpyDeviceToHost, stream));
      PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
      vrb[v] = range_bits;
      if (range_bits <= PLAN_MAX_COUNT_BITS) {
        // small key range (the usual case once the chunk minimum is subtracted): counting histogram, no sort
        const size_t smem = ((size_t(1) << range_bits) + 1) * 4 + 16;
        profiler().begin("plan_probe_kernel_counting", stream);
        PCOB_CUDA_TRY((v == 0 ? S.key16_0 : S.key16_1).reserve(slots * 2 + 64));
        plan_probe_kernel<L, true, WIDE><<<n_chunks, PLAN_THREADS, smem, stream>>>(e, d_lat[v], d_chunks, d_probes, int(v), range_bits,
                                                                                    (v == 0 ? S.key16_0 : S.key16_1).as<uint16_t>());
        profiler().end(stream);
        solve(n_chunks, int(v), 0);
        continue;
      }
      // wide key range: sort the range-reduced keys (the two key buffers exist only on this path)
      PCOB_CUDA_TRY(S.keys_a.reserve(slots * sizeof(L) + 64));
      PCOB_CUDA_TRY(S.keys_b.reserve(slots * sizeof(L) + 64));
      profiler().begin("sort_keys_kernel", stream);
      sort_keys_kernel<L><<<n_chunks * tiles, 256, 0, stream>>>(e, tiles, d_lat[v], S.keys_a.as<L>(), d_chunks, int(v));
      profiler().end(stream);
      uint64_t* seg_begin = S.seg.as<uint64_t>();
      uint64_t* seg_end = seg_begin + n_chunks;
      segment_offsets_kernel<<<(n_chunks + 255) / 256, 256, 0, stream>>>(e, order_v, seg_begin, seg_end);
      const L* sorted = S.keys_a.as<L>();
      {
        const uint32_t sort_bits = std::max<uint32_t>(range_bits, 1);
        profiler().begin("radix_sort_segments_kernel", stream);
        radix_sort_segments_kernel<L><<<n_chunks, RS_THREADS, RS_SMEM, stream>>>(S.keys_a.as<L>(), S.keys_b.as<L>(), seg_begin, seg_end, sort_bits);
        profiler().end(stream);
        if (((sort_bits + RS_BITS - 1) / RS_BITS) & 1) sorted = S.keys_b.as<L>();  // an odd number of passes ends in the second buffer
      }
      profiler().begin("plan_probe_kernel_sorted", stream);
      plan_probe_kernel<L, false, WIDE><<<n_chunks, PLAN_THREADS, 16, stream>>>(e, sorted, d_chunks, d_probes, int(v), range_bits, nullptr);
      profiler().end(stream);
      solve(n_chunks, int(v), 0);
    }
    return PCO_B200_OK;
}

// What a ChunkConfig resolves to for an array of n numbers before any device work: the chunk sizes, the explicit mode and delta order, and
// whether Auto searches run.  pco_b200_compress_files checks every file with it before the pipeline runs.
struct ConfigCheck {
  std::vector<uint64_t> pages;
  ModeSel explicit_mode;
  bool auto_mode = false, auto_delta = false;
  uint32_t explicit_order = 0;
};

// config validation (pco/src/chunk_config.rs:269-314)
inline PcoB200Error check_config(const PcoB200ChunkConfig& cfg, uint32_t dtype, size_t n, ConfigCheck* out) {
  const uint32_t lbits = nt_bits(dtype);
  const bool is_float = nt_is_float(dtype);
  std::vector<uint64_t>& pages = out->pages;
  ModeSel& explicit_mode = out->explicit_mode;
  bool& auto_mode = out->auto_mode;
  bool& auto_delta = out->auto_delta;
  uint32_t& explicit_order = out->explicit_order;
  if (cfg.compression_level > 12) return fail(PCO_B200_INVALID_ARGUMENT, "compression level may not exceed 12");
  if (cfg.delta_spec == PCO_B200_DELTA_TRY_CONSECUTIVE && cfg.delta_order > 7)
    return fail(PCO_B200_INVALID_ARGUMENT, "consecutive delta order may not exceed 7");
  if (lbits == 8 && !cfg.enable_8_bit)
    return fail(PCO_B200_INVALID_ARGUMENT, "compressing 8-bit types with Pco is often a mistake; enable them on the ChunkConfig if you know what you're doing");
  if (PcoB200Error e = n_per_page(cfg, n, &pages)) return e;
  for (uint64_t p : pages)
    if (p > (uint64_t(1) << 24)) return fail(PCO_B200_INVALID_ARGUMENT, "count may not exceed 16777216 per chunk");
  // ---- the explicit mode, if any (Auto is resolved per chunk by compress_typed)
  switch (cfg.mode_spec) {
    case PCO_B200_MODE_CLASSIC: break;
    case PCO_B200_MODE_TRY_INT_MULT:
      if (is_float) return fail(PCO_B200_INVALID_ARGUMENT, "unable to use int mult mode on floats");
      explicit_mode.mode = MODE_INT_MULT;
      explicit_mode.mode_base = lbits == 64 ? cfg.int_mult_base : (cfg.int_mult_base & ((uint64_t(1) << lbits) - 1));
      if (explicit_mode.mode_base == 0) return fail(PCO_B200_INVALID_ARGUMENT, "The chosen mode of IntMult(0) was invalid");
      break;
    case PCO_B200_MODE_TRY_FLOAT_QUANT: {
      if (!is_float) return fail(PCO_B200_INVALID_ARGUMENT, "unable to use float mode for ints");
      uint32_t precision = lbits == 64 ? 52 : lbits == 32 ? 23 : 10;
      if (cfg.float_quant_k == 0 || cfg.float_quant_k > precision) return fail(PCO_B200_INVALID_ARGUMENT, "The chosen mode of FloatQuant was invalid");
      explicit_mode.mode = MODE_FLOAT_QUANT;
      explicit_mode.mode_k = cfg.float_quant_k;
      break;
    }
    case PCO_B200_MODE_TRY_FLOAT_MULT: {
      if (!is_float) return fail(PCO_B200_INVALID_ARGUMENT, "unable to use float mode for ints");
      if (lbits == 16) return fail(PCO_B200_UNSUPPORTED, "f16 FloatMult is outside the GPU hot path");
      const bool finite_nonzero = lbits == 64 ? (std::isfinite(cfg.float_mult_base) && cfg.float_mult_base != 0.0)
                                              : (std::isfinite(float(cfg.float_mult_base)) && float(cfg.float_mult_base) != 0.0f);
      if (!finite_nonzero) return fail(PCO_B200_INVALID_ARGUMENT, "The chosen mode of FloatMult was invalid");
      if (lbits == 64) set_float_mult(&explicit_mode, 64, cfg.float_mult_base, 1.0 / cfg.float_mult_base);
      else set_float_mult(&explicit_mode, 32, double(float(cfg.float_mult_base)), double(1.0f / float(cfg.float_mult_base)));
      break;
    }
    case PCO_B200_MODE_AUTO: auto_mode = true; break;
    default: return fail(PCO_B200_UNSUPPORTED, "ModeSpec::TryDict is outside the GPU hot path");
  }
  switch (cfg.delta_spec) {
    case PCO_B200_DELTA_NOOP: break;
    case PCO_B200_DELTA_TRY_CONSECUTIVE: explicit_order = cfg.delta_order; break;
    case PCO_B200_DELTA_AUTO: auto_delta = true; break;  // resolved per chunk by compress_typed's sampled search
    case PCO_B200_DELTA_TRY_CONV1:
      if (cfg.delta_order == 0) break;
      return fail(PCO_B200_UNSUPPORTED, "DeltaSpec::TryConv1 is outside the GPU hot path");
    default: return fail(PCO_B200_UNSUPPORTED, "DeltaSpec::TryLookback is outside the GPU hot path");
  }
  return PCO_B200_OK;
}

template <typename L>
static PcoB200Error compress_typed(CompressScratch& S, const void* nums, size_t n, uint32_t dtype, const PcoB200ChunkConfig& cfg, bool uniform_type,
                                   void* dst, size_t dst_cap, void* index_dst, size_t index_cap, uint32_t flags, cudaStream_t stream,
                                   CompressResult* res) {
  const bool src_dev = flags & PCO_B200_SRC_ON_DEVICE, dst_dev = flags & PCO_B200_DST_ON_DEVICE;
  const uint32_t lbits = sizeof(L) * 8;
  constexpr int LW = sizeof(L) == 1 ? 0 : sizeof(L) == 2 ? 1 : sizeof(L) == 4 ? 2 : 3;
  const bool is_float = nt_is_float(dtype);
  ConfigCheck checked;
  if (PcoB200Error e = check_config(cfg, dtype, n, &checked)) return e;
  const std::vector<uint64_t>& pages = checked.pages;
  const ModeSel explicit_mode = checked.explicit_mode;
  const bool auto_mode = checked.auto_mode, auto_delta = checked.auto_delta;
  const uint32_t explicit_order = checked.explicit_order;
  const bool chunks_only = flags & PCO_B200_CHUNKS_ONLY;
  S.ans_paths_valid = false;
  std::vector<uint8_t> header = make_standalone_header(n, uint8_t(uniform_type ? dtype : 0));
  if (chunks_only) header.clear();
  // empty input: header + terminator only (standalone/simple.rs:62-91)
  if (n == 0) {
    if (!chunks_only) header.push_back(0);
    if (header.size() > dst_cap) return fail(PCO_B200_IO, "failed to write whole buffer");
    if (dst_dev && !header.empty()) PCOB_CUDA_TRY(cudaMemcpyAsync(dst, header.data(), header.size(), cudaMemcpyHostToDevice, stream));
    else if (!header.empty()) std::memcpy(dst, header.data(), header.size());
    PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
    res->total_bytes = header.size();
    if (index_dst && index_cap >= sizeof(IndexHeader)) {
      IndexHeader ih;
      std::memset(&ih, 0, sizeof(ih));
      ih.magic = INDEX_MAGIC; ih.version = 1; ih.file_len = header.size(); ih.chunks_offset = sizeof(IndexHeader); ih.end_byte = header.size();
      std::memcpy(index_dst, &ih, sizeof(ih));
      res->index_bytes = sizeof(ih);
    }
    return PCO_B200_OK;
  }
  const uint32_t n_chunks_all = uint32_t(pages.size());
  std::vector<uint64_t> starts(pages.size() + 1, 0);
  uint64_t max_chunk_n = 0;
  for (size_t i = 0; i < pages.size(); i++) { starts[i + 1] = starts[i] + pages[i]; max_chunk_n = std::max<uint64_t>(max_chunk_n, pages[i]); }
  // unoptimized_bins_log is a function of each chunk's n (chunk_compressor.rs:362-371); the kernels take one value per launch, so chunks
  // that disagree (small chunks on either side of a power of two) go through the pipeline in separate runs below.  The Auto searches plan
  // all chunks' samples in one launch: they still need one value.
  const bool shared_bins = (flags & PCO_B200_INTERNAL_SHARED_BINS) && pages.size() > 1;
  const uint32_t bins_log = unoptimized_bins_log(cfg.compression_level, shared_bins ? n : pages[0], 0);
  std::vector<uint32_t> chunk_bins_log(pages.size(), bins_log);
  bool bins_log_uniform = true;
  if (!shared_bins)
    for (size_t i = 0; i < pages.size(); i++) {
      chunk_bins_log[i] = unoptimized_bins_log(cfg.compression_level, pages[i], 0);
      if (chunk_bins_log[i] != bins_log) bins_log_uniform = false;
    }
  if (!bins_log_uniform && (auto_mode || auto_delta))
    return fail(PCO_B200_UNSUPPORTED, "ModeSpec::Auto / DeltaSpec::Auto over chunks whose sizes imply different unoptimized_bins_log in one call");
  // levels 9-12 train up to 4096 unoptimized bins: runs with more than 256 take the wide instantiation of the kernels
  bool any_wide = false;
  for (uint32_t bl : chunk_bins_log) any_wide = any_wide || bl > ENC_NARROW_BINS_LOG;

  // ---- the numbers in HBM
  const void* d_nums = nums;
  DevBuf& in_stage = S.index;  // a dedicated input staging buffer when nums live on the host (kept apart from the sort buffers)
  S.src_in_place = false;
  if (!src_dev) {
    // explicit classic configs read a page-locked input in place (one pass of split_count_kernel over PCIe, no staging); the Auto
    // searches gather samples from all over the array and the two-latent modes take the two-kernel front end: those stage as before
    void* in_place = nullptr;
    if ((zero_copy_mask().load(std::memory_order_relaxed) & 1) && !auto_mode && !auto_delta && explicit_mode.mode == MODE_CLASSIC && !shared_bins)
      in_place = mapped_host_ptr(nums);
    call_trace().mark("c.begin");
    if (in_place) {
      d_nums = in_place;
      S.src_in_place = true;
    } else {
      PCOB_CUDA_TRY(in_stage.reserve(n * sizeof(L) + 64));
      PCOB_CUDA_TRY(copy_sliced(in_stage.p, nums, n * sizeof(L), cudaMemcpyHostToDevice, stream));
      d_nums = in_stage.p;
    }
    call_trace().mark("c.h2d_submitted");
  }
  // scratch sized for the whole call; every run below (and the Auto searches) indexes it from 0
  PCOB_CUDA_TRY(S.plans.reserve(size_t(n_chunks_all) * MAX_VARS * (any_wide ? sizeof(VarPlanT<true>) : sizeof(VarPlan))));
  PCOB_CUDA_TRY(S.chunks.reserve(size_t(n_chunks_all) * sizeof(ChunkEnc)));
  PCOB_CUDA_TRY(S.starts.reserve((starts.size() + 1) * 32));
  PCOB_CUDA_TRY(S.seg.reserve(size_t(n_chunks_all) * 16));
  PCOB_CUDA_TRY(S.small.reserve(256 + header.size()));
  PCOB_CUDA_TRY(S.probes.reserve(size_t(n_chunks_all) * (any_wide ? sizeof(PlanProbesT<true>) : sizeof(PlanProbes))));
  ChunkEnc* d_chunks = S.chunks.as<ChunkEnc>();
  uint32_t* d_small = S.small.as<uint32_t>();  // [0]: range bits, [2..3]: total bytes (u64), header at byte 64
  uint64_t* d_total = reinterpret_cast<uint64_t*>(d_small + 2);
  uint8_t* d_header = reinterpret_cast<uint8_t*>(d_small) + 64;
  if (!header.empty()) PCOB_CUDA_TRY(cudaMemcpyAsync(d_header, header.data(), header.size(), cudaMemcpyHostToDevice, stream));
  uint32_t* d_ans_paths = nullptr;  // non-null only while profiling: the timed path launches ans_encode_kernel without counters
  if (profiler_enabled().load(std::memory_order_relaxed)) {
    PCOB_CUDA_TRY(S.ans_paths.reserve(ANS_PATH_SLOTS * sizeof(uint32_t)));
    PCOB_CUDA_TRY(cudaMemsetAsync(S.ans_paths.p, 0, ANS_PATH_SLOTS * sizeof(uint32_t), stream));
    d_ans_paths = S.ans_paths.as<uint32_t>();
    S.ans_paths_valid = true;
  }

  // ---- K1+K2 and the planner for one set of chunks (a run of the call's chunks, or the chunks' samples during the Auto delta search).
  // `e` describes the set (its own chunk_starts / row_base, counted from 0); plans and probes land in slots 0 .. e.n_chunks - 1.
  // `wide` is std::true_type for sets whose unoptimized_bins_log is above 8, else std::false_type.
  L* d_lat[2] = {nullptr, nullptr};
  auto front = [&](auto wide, EncParams& e, uint32_t tiles, size_t slots, uint32_t (&vrb)[MAX_VARS], const std::vector<uint64_t>& sizes, bool shared) -> PcoB200Error {
    return plan_front<L, decltype(wide)::value>(S, stream, e, tiles, slots, vrb, sizes, shared, d_lat);
  };

  // ---- ModeSpec::Auto and DeltaSpec::Auto are the reference's PER-CHUNK searches (chunk_compressor.rs:396-440): every chunk of the
  // call gets its own answer; with shared bins (the pages of ONE wrapped chunk) the whole input is the unit.
  const size_t n_units = shared_bins ? 1 : pages.size();
  auto unit_begin = [&](size_t u) -> uint64_t { return shared_bins ? 0 : starts[u]; };
  auto unit_n = [&](size_t u) -> uint64_t { return shared_bins ? uint64_t(n) : pages[u]; };
  std::vector<ModeSel> unit_mode(n_units, explicit_mode);
  std::vector<uint32_t> unit_order(n_units, explicit_order);
  if (auto_mode) {
    // the reference's search (mode_search.hpp) reads ~n/40 numbers per chunk at positions that depend on n only: the device gathers
    // every chunk's sample, the host (one task per chunk on its worker threads) runs the scalar analysis
    std::map<uint64_t, std::vector<uint32_t>> by_n;
    for (size_t u = 0; u < n_units; u++) by_n[unit_n(u)].push_back(uint32_t(u));
    std::vector<uint64_t> ustarts(n_units + 1, 0);
    for (size_t u = 0; u < n_units; u++) ustarts[u] = unit_begin(u);
    ustarts[n_units] = n;
    PCOB_CUDA_TRY(S.sample_starts.reserve((n_units + 1) * 8 + n_units * 4 + 64));
    uint64_t* d_ustarts = S.sample_starts.as<uint64_t>();
    PCOB_CUDA_TRY(cudaMemcpyAsync(d_ustarts, ustarts.data(), ustarts.size() * 8, cudaMemcpyHostToDevice, stream));
    for (auto& kv : by_n) {
      const std::vector<uint32_t>& pos = mode_sample_positions(size_t(kv.first));
      const uint32_t m = uint32_t(pos.size());
      if (m == 0) continue;  // fewer than MIN_SAMPLE numbers: Classic (sampling.rs:14-20)
      const std::vector<uint32_t>& ids = kv.second;
      PCOB_CUDA_TRY(S.sample.reserve(ids.size() * size_t(m) * sizeof(L) + 64));
      PCOB_CUDA_TRY(S.seg.reserve((ids.size() + m) * 4 + 64));
      uint32_t* d_ids = S.seg.as<uint32_t>();
      uint32_t* d_pos = d_ids + ids.size();
      PCOB_CUDA_TRY(cudaMemcpyAsync(d_ids, ids.data(), ids.size() * 4, cudaMemcpyHostToDevice, stream));
      PCOB_CUDA_TRY(cudaMemcpyAsync(d_pos, pos.data(), size_t(m) * 4, cudaMemcpyHostToDevice, stream));
      gather_positions_kernel<L><<<uint32_t(ids.size()), 256, 0, stream>>>(static_cast<const L*>(d_nums), d_ustarts, d_ids, d_pos, m, S.sample.as<L>());
      std::vector<L> h_sample(ids.size() * size_t(m));
      PCOB_CUDA_TRY(cudaMemcpyAsync(h_sample.data(), S.sample.p, h_sample.size() * sizeof(L), cudaMemcpyDeviceToHost, stream));
      PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
      std::vector<mode_search::Choice> choices(ids.size());
      auto work = [&](size_t i) {
        const L* sp = h_sample.data() + i * size_t(m);
        mode_search::Choice c;
        if constexpr (sizeof(L) == 8) c = is_float ? mode_search::choose_float_from_sample<double>(sp, m) : mode_search::choose_int_from_sample<L>(sp, m, nt_is_signed(dtype));
        else if constexpr (sizeof(L) == 4) c = is_float ? mode_search::choose_float_from_sample<float>(sp, m) : mode_search::choose_int_from_sample<L>(sp, m, nt_is_signed(dtype));
        else if constexpr (sizeof(L) == 2) c = is_float ? mode_search::choose_float_from_sample<mode_search::Half>(sp, m) : mode_search::choose_int_from_sample<L>(sp, m, nt_is_signed(dtype));
        else c = mode_search::choose_int_from_sample<L>(sp, m, nt_is_signed(dtype));
        choices[i] = c;
      };
      const size_t n_threads = std::max<size_t>(1, std::min<size_t>(ids.size(), std::min<size_t>(std::thread::hardware_concurrency(), 32)));
      if (n_threads <= 1) {
        for (size_t i = 0; i < ids.size(); i++) work(i);
      } else {
        std::atomic<size_t> next{0};
        std::vector<std::thread> pool;
        for (size_t t = 0; t < n_threads; t++)
          pool.emplace_back([&] { for (size_t i = next.fetch_add(1); i < ids.size(); i = next.fetch_add(1)) work(i); });
        for (auto& th : pool) th.join();
      }
      for (size_t i = 0; i < ids.size(); i++) {
        const mode_search::Choice& c = choices[i];
        ModeSel ms;
        if (c.kind == 1) { ms.mode = MODE_INT_MULT; ms.mode_base = c.int_base; }
        else if (c.kind == 3) { ms.mode = MODE_FLOAT_QUANT; ms.mode_k = c.k; }
        else if (c.kind == 2) {
          if (lbits == 16) return fail(PCO_B200_UNSUPPORTED, "ModeSpec::Auto chose FloatMult for an f16 chunk: f16 FloatMult is outside the GPU hot path");
          set_float_mult(&ms, lbits, c.base, c.inv_base);
        }
        unit_mode[ids[i]] = ms;
      }
    }
  }
  if (shared_bins && unit_mode[0].mode != MODE_CLASSIC)
    return fail(PCO_B200_UNSUPPORTED, "wrapped chunks with several pages: classic mode only, for now");
  if (auto_delta) {
    // choose_auto_delta_encoding (chunk_compressor.rs:310-360) per chunk: the sample of the chunk's primary latents (sampling.rs:21-60) is
    // trial-compressed in Classic mode with NoOp, then consecutive orders 1, 2, ... while the cost keeps falling.  Every order is planned
    // for all chunks at once by the ordinary front end + planner kernels; the costs are the reference's f32 formula (sample_cost).
    // The Lookback candidate (chunk_compressor.rs:326-338) is weighed like the reference does; this path does not ENCODE Lookback, so a
    // chunk on which it wins makes the call fail with PCO_B200_UNSUPPORTED rather than write bytes the reference would not.
    std::vector<uint64_t> s_starts(n_units + 1, 0), s_rows(n_units + 1, 0), s_sizes(n_units, 0), ustarts(n_units + 1, 0);
    uint64_t max_ns = 0;
    for (size_t u = 0; u < n_units; u++) {
      const SampleGeom g = delta_sample_geom(unit_n(u));
      const uint64_t ns = uint64_t(g.n_groups) * g.group_n;
      s_starts[u + 1] = s_starts[u] + ns;
      s_sizes[u] = ns;
      s_rows[u + 1] = s_rows[u] + ((ns + BATCH_N - 1) / BATCH_N) * BATCH_N;
      max_ns = std::max(max_ns, ns);
      ustarts[u] = unit_begin(u);
    }
    ustarts[n_units] = n;
    // the trial plans use the chunks' bins_log (calculate_compressed_sample_size): wide plans at levels 9-12
    auto search = [&](auto wide) -> PcoB200Error {
      constexpr bool W = decltype(wide)::value;
      using Summary = PlanSummaryT<W>;
      const VarPlanT<W>* d_plans = S.plans.as<VarPlanT<W>>();
      std::vector<ModeSelDev> hm(n_units);
      for (size_t u = 0; u < n_units; u++) hm[u] = ModeSelDev{unit_mode[u].mode, unit_mode[u].mode_k, unit_mode[u].mode_base, unit_mode[u].base_bits, unit_mode[u].inv_base_bits};
      PCOB_CUDA_TRY(S.sample.reserve(s_starts.back() * sizeof(L) + 64));
      const size_t words = 3 * (n_units + 1);
      PCOB_CUDA_TRY(S.sample_starts.reserve(words * 8 + n_units * sizeof(ModeSelDev) + n_units * sizeof(Summary) + 256));
      uint64_t* d_ss = S.sample_starts.as<uint64_t>();
      uint64_t* d_srows = d_ss + (n_units + 1);
      uint64_t* d_ustarts = d_srows + (n_units + 1);
      ModeSelDev* d_modes = reinterpret_cast<ModeSelDev*>(d_ustarts + (n_units + 1));
      Summary* d_sum = reinterpret_cast<Summary*>(d_modes + n_units);
      PCOB_CUDA_TRY(cudaMemcpyAsync(d_ss, s_starts.data(), s_starts.size() * 8, cudaMemcpyHostToDevice, stream));
      PCOB_CUDA_TRY(cudaMemcpyAsync(d_srows, s_rows.data(), s_rows.size() * 8, cudaMemcpyHostToDevice, stream));
      PCOB_CUDA_TRY(cudaMemcpyAsync(d_ustarts, ustarts.data(), ustarts.size() * 8, cudaMemcpyHostToDevice, stream));
      PCOB_CUDA_TRY(cudaMemcpyAsync(d_modes, hm.data(), hm.size() * sizeof(ModeSelDev), cudaMemcpyHostToDevice, stream));
      gather_primary_sample_kernel<L><<<uint32_t(n_units), 256, 0, stream>>>(static_cast<const L*>(d_nums), d_ustarts, d_ss, d_modes, dtype, S.sample.as<L>());
      // the sample holds latents: unsigned numbers of the same width
      EncParams es = enc_params(lbits == 8 ? NT_U8 : lbits == 16 ? NT_U16 : lbits == 32 ? NT_U32 : NT_U64, 0, ModeSel{}, 0, bins_log);
      es.nums = S.sample.p;
      es.chunk_starts = d_ss;
      es.row_base = d_srows;
      es.n_total = s_starts.back();
      es.n_chunks = uint32_t(n_units);
      es.max_chunk_n = uint32_t(max_ns);
      const uint32_t s_tiles = uint32_t((max_ns + SPLIT_TILE - 1) / SPLIT_TILE);
      std::vector<Summary> h_sum(n_units);
      std::vector<float> best_cost(n_units, 0.f);
      std::vector<uint8_t> open(n_units, 1), lookback_best(n_units, 0);
      size_t n_open = n_units;
      for (uint32_t k = 0; k <= MAX_ORDER && n_open > 0; k++) {
        es.order = k;
        uint32_t vrb[MAX_VARS] = {64, 64};
        if (PcoB200Error e = front(wide, es, s_tiles, size_t(s_rows.back()), vrb, s_sizes, false)) return e;
        PCOB_CUDA_TRY(cudaGetLastError());
        plan_summary_kernel<W><<<uint32_t(n_units), 128, 0, stream>>>(d_plans, uint32_t(n_units), d_sum);
        PCOB_CUDA_TRY(cudaMemcpyAsync(h_sum.data(), d_sum, n_units * sizeof(Summary), cudaMemcpyDeviceToHost, stream));
        PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
        for (size_t u = 0; u < n_units; u++) {
          if (!open[u]) continue;
          if (s_sizes[u] == 0) { open[u] = 0; n_open--; continue; }  // no sample: NoOp (chunk_compressor.rs:314-316)
          const float cost = sample_cost(h_sum[u], lbits, k, s_sizes[u]);
          if (k == 0) best_cost[u] = cost;
          else if (cost < best_cost[u]) { best_cost[u] = cost; unit_order[u] = k; lookback_best[u] = 0; }
          else { open[u] = 0; n_open--; }  // "it's almost always convex" (chunk_compressor.rs:347-357)
        }
        if (k == 0 && n_open > 0) {
          // ---- the Lookback candidate (chunk_compressor.rs:326-338), weighed right after NoOp: the sample is lookback-encoded on the
          // device (lookback_trial_kernel), its two latent vars - the lookbacks as u32, the residuals in the number's width - are
          // planned by the ordinary kernels, and the cost is the same f32 formula plus the required-savings penalty
          bool any = false;
          for (size_t u = 0; u < n_units; u++) any = any || (open[u] && best_cost[u] > 0.25f * float(s_sizes[u]));
          if (any) {
            std::vector<uint64_t> lb_starts(n_units + 1, 0), lb_rows(n_units + 1, 0), lb_sizes(n_units, 0);
            uint64_t max_lb = 0;
            for (size_t u = 0; u < n_units; u++) {
              lb_sizes[u] = s_sizes[u] > 0 ? s_sizes[u] - 1 : 0;  // state_n = 1
              lb_starts[u + 1] = lb_starts[u] + lb_sizes[u];
              lb_rows[u + 1] = lb_rows[u] + ((lb_sizes[u] + BATCH_N - 1) / BATCH_N) * BATCH_N;
              max_lb = std::max(max_lb, lb_sizes[u]);
            }
            const uint32_t wlog_max = lookback_window_n_log(std::max<uint64_t>(max_ns, 2));
            const uint32_t hash_stride = 2u << (wlog_max + 1), count_stride = 1u << wlog_max;
            PCOB_CUDA_TRY(S.lb_vals.reserve(lb_starts.back() * 4 + 64));
            PCOB_CUDA_TRY(S.lb_resid.reserve(lb_starts.back() * sizeof(L) + 64));
            PCOB_CUDA_TRY(S.lb_scratch.reserve(n_units * (size_t(hash_stride) + count_stride) * 4 + 3 * (n_units + 1) * 8 + 64));
            uint32_t* d_hash = S.lb_scratch.as<uint32_t>();
            uint32_t* d_cnt = d_hash + n_units * size_t(hash_stride);
            uint64_t* d_lbs = reinterpret_cast<uint64_t*>(d_cnt + n_units * size_t(count_stride));
            uint64_t* d_lbrows = d_lbs + (n_units + 1);
            PCOB_CUDA_TRY(cudaMemcpyAsync(d_lbs, lb_starts.data(), lb_starts.size() * 8, cudaMemcpyHostToDevice, stream));
            PCOB_CUDA_TRY(cudaMemcpyAsync(d_lbrows, lb_rows.data(), lb_rows.size() * 8, cudaMemcpyHostToDevice, stream));
            lookback_trial_kernel<L><<<uint32_t(n_units), 128, 0, stream>>>(S.sample.as<L>(), d_ss, d_lbs, S.lb_vals.as<uint32_t>(), S.lb_resid.as<L>(), d_hash, d_cnt,
                                                                            hash_stride, count_stride);
            PCOB_CUDA_TRY(cudaGetLastError());
            EncParams el = es;
            el.order = 0;
            el.chunk_starts = d_lbs;
            el.row_base = d_lbrows;
            el.n_total = lb_starts.back();
            el.max_chunk_n = uint32_t(max_lb);
            const uint32_t l_tiles = uint32_t((max_lb + SPLIT_TILE - 1) / SPLIT_TILE);
            std::vector<Summary> sum_d(n_units), sum_p(n_units);
            {  // the delta var: lookbacks, planned as u32 with the chunk's unoptimized_bins_log (chunk_compressor.rs:238-248)
              EncParams ed = el;
              ed.dtype = NT_U32;
              ed.nums = S.lb_vals.p;
              uint32_t vrb[MAX_VARS] = {64, 64};
              uint32_t* lat32[2] = {nullptr, nullptr};
              if (PcoB200Error e = plan_front<uint32_t, W>(S, stream, ed, l_tiles, size_t(lb_rows.back()), vrb, lb_sizes, false, lat32)) return e;
              PCOB_CUDA_TRY(cudaGetLastError());
              plan_summary_kernel<W><<<uint32_t(n_units), 128, 0, stream>>>(d_plans, uint32_t(n_units), d_sum);
              PCOB_CUDA_TRY(cudaMemcpyAsync(sum_d.data(), d_sum, n_units * sizeof(Summary), cudaMemcpyDeviceToHost, stream));
              PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
            }
            {  // the primary: residuals
              EncParams epr = el;
              epr.nums = S.lb_resid.p;
              uint32_t vrb[MAX_VARS] = {64, 64};
              if (PcoB200Error e = front(wide, epr, l_tiles, size_t(lb_rows.back()), vrb, lb_sizes, false)) return e;
              PCOB_CUDA_TRY(cudaGetLastError());
              plan_summary_kernel<W><<<uint32_t(n_units), 128, 0, stream>>>(d_plans, uint32_t(n_units), d_sum);
              PCOB_CUDA_TRY(cudaMemcpyAsync(sum_p.data(), d_sum, n_units * sizeof(Summary), cudaMemcpyDeviceToHost, stream));
              PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
            }
            for (size_t u = 0; u < n_units; u++) {
              const float penalty = 0.25f * float(s_sizes[u]);  // LOOKBACK_REQUIRED_BYTE_SAVINGS_PER_N * sample_n
              if (!open[u] || !(best_cost[u] > penalty) || lb_sizes[u] == 0) continue;
              const float cost = lookback_sample_cost(sum_d[u], sum_p[u], lbits, lb_sizes[u]) + penalty;
              if (cost < best_cost[u]) { best_cost[u] = cost; lookback_best[u] = 1; }
            }
          }
        }
      }
      for (size_t u = 0; u < n_units; u++)
        if (lookback_best[u])
          return fail(PCO_B200_UNSUPPORTED, "DeltaSpec::Auto: the Lookback delta wins on chunk " + std::to_string(u) + "; the GPU hot path does not encode Lookback (pass a consecutive DeltaSpec)");
      return PCO_B200_OK;
    };
    if (s_starts.back() > 0)
      if (PcoB200Error e = bins_log > ENC_NARROW_BINS_LOG ? search(std::true_type{}) : search(std::false_type{})) return e;
  }

  // ---- runs of consecutive chunks with the same resolved (mode, order): each is one pass of the pipeline; a call with explicit specs
  // (and the usual homogeneous array under Auto) is a single run
  struct Run { size_t c0, c1; ModeSel ms; uint32_t order, bins_log; };
  std::vector<Run> runs;
  if (shared_bins) runs.push_back(Run{0, pages.size(), unit_mode[0], unit_order[0], bins_log});
  else
    for (size_t c = 0; c < pages.size(); c++) {
      if (!runs.empty() && runs.back().ms == unit_mode[c] && runs.back().order == unit_order[c] && runs.back().bins_log == chunk_bins_log[c]) runs.back().c1 = c + 1;
      else runs.push_back(Run{c, c + 1, unit_mode[c], unit_order[c], chunk_bins_log[c]});
    }
  // side index layout (host): entries of chunk c take n_vars(c) x batches(c) records
  const uint64_t chunks_offset = sizeof(IndexHeader);
  std::vector<uint64_t> eoff(n_chunks_all, 0);
  uint64_t index_total = 0;
  if (index_dst != nullptr) {
    uint64_t off = (chunks_offset + uint64_t(n_chunks_all) * sizeof(IndexChunk) + 15) & ~uint64_t(15);
    for (const Run& r : runs)
      for (size_t c = r.c0; c < r.c1; c++) {
        eoff[c] = off;
        off += entries_bytes(r.ms.mode == MODE_CLASSIC ? 1 : 2, pages[c]);
      }
    if (off > index_cap) return fail(PCO_B200_IO, "index buffer too small (need " + std::to_string(off) + " bytes)");
    index_total = off;
    PCOB_CUDA_TRY(S.idx_out.reserve(off + 64));  // assembled on the device run by run, one copy out
    // the 16-byte padding behind a chunk's entries is written by no kernel: zero, so that the index is a function of the numbers
    PCOB_CUDA_TRY(cudaMemsetAsync(S.idx_out.p, 0, off, stream));
  }
  uint64_t file_off = header.size();  // bytes of the file in front of the next run's first chunk
  uint8_t* d_out = static_cast<uint8_t*>(dst);
  // a page-locked host destination is written in place by pack_kernel (word stores, every byte once), exactly like a device destination:
  // no staging, no file-size round trip in front of the pack (host_common.hpp, zero copy)
  bool dst_direct = dst_dev;
  if (!dst_dev && (zero_copy_mask().load(std::memory_order_relaxed) & 4)) {
    if (void* in_place = mapped_host_ptr(dst)) {
      d_out = static_cast<uint8_t*>(in_place);
      dst_direct = true;
    }
  }
  for (size_t ri = 0; ri < runs.size(); ri++) {
    const Run& run = runs[ri];
    const bool first_run = ri == 0, last_run = ri + 1 == runs.size();
    const uint32_t n_chunks = uint32_t(run.c1 - run.c0);
    std::vector<uint64_t> rpages(pages.begin() + run.c0, pages.begin() + run.c1);
    std::vector<uint64_t> rstarts(n_chunks + 1, 0), rrows(n_chunks + 1, 0);
    uint64_t run_max_n = 0;
    for (uint32_t i = 0; i < n_chunks; i++) {
      rstarts[i + 1] = rstarts[i] + rpages[i];
      rrows[i + 1] = rrows[i] + ((rpages[i] + BATCH_N - 1) / BATCH_N) * BATCH_N;
      run_max_n = std::max(run_max_n, rpages[i]);
    }
    EncParams ep = enc_params(dtype, uniform_type ? dtype : 0, run.ms, run.order, run.bins_log);
    ep.n_total = rstarts.back();
    ep.n_chunks = n_chunks;
    ep.max_chunk_n = uint32_t(run_max_n);
    ep.nums = static_cast<const L*>(d_nums) + starts[run.c0];
    const uint32_t bpc = n_batches_of(uint32_t(run_max_n));
    const uint32_t tiles_per_chunk = uint32_t((run_max_n + SPLIT_TILE - 1) / SPLIT_TILE);
    const size_t n_slots = size_t(rrows.back());
    const bool wide_run = run.bins_log > ENC_NARROW_BINS_LOG;
    const size_t sym_bytes = wide_run ? 2 : 1;  // symbols are bin indices: 16 bits when a var can have more than 256 bins
    PCOB_CUDA_TRY(S.sym0.reserve(n_slots * sym_bytes + 64));
    PCOB_CUDA_TRY(S.ans0.reserve(n_slots * 2 + 64));
    if (ep.n_vars > 1) { PCOB_CUDA_TRY(S.sym1.reserve(n_slots * sym_bytes + 64)); PCOB_CUDA_TRY(S.ans1.reserve(n_slots * 2 + 64)); }
    const size_t n_cvb = size_t(n_chunks) * MAX_VARS * bpc;
    PCOB_CUDA_TRY(S.ob_sum.reserve(n_cvb * 4));
    PCOB_CUDA_TRY(S.ans_sum.reserve(n_cvb * 4));
    PCOB_CUDA_TRY(S.entries.reserve(n_cvb * sizeof(BatchEntry)));
    uint64_t* d_rstarts = S.starts.as<uint64_t>();
    PCOB_CUDA_TRY(cudaMemcpyAsync(d_rstarts, rstarts.data(), rstarts.size() * 8, cudaMemcpyHostToDevice, stream));
    PCOB_CUDA_TRY(cudaMemcpyAsync(d_rstarts + rstarts.size(), rrows.data(), rrows.size() * 8, cudaMemcpyHostToDevice, stream));
    ep.chunk_starts = d_rstarts;
    ep.row_base = d_rstarts + rstarts.size();
    uint16_t* d_ans[2] = {S.ans0.as<uint16_t>(), S.ans1.as<uint16_t>()};
    PCOB_CUDA_TRY(cudaMemsetAsync(S.ob_sum.p, 0, n_cvb * 4, stream));
    uint32_t var_range_bits[MAX_VARS] = {64, 64};
    // planner, fallback, K3, K4 and layout in the run's capacity (`wide`: std::true_type when the run trains more than 256 bins)
    auto encode_run = [&](auto wide) -> PcoB200Error {
      constexpr bool W = decltype(wide)::value;
      using Sym = typename EncCap<W>::Sym;
      const VarPlanT<W>* d_plans = S.plans.as<VarPlanT<W>>();
      Sym* d_sym[2] = {S.sym0.as<Sym>(), S.sym1.as<Sym>()};
      if (PcoB200Error e = front(wide, ep, tiles_per_chunk, n_slots, var_range_bits, rpages, shared_bins)) return e;
      PCOB_CUDA_TRY(cudaGetLastError());
      fallback_kernel<W><<<(n_chunks + 255) / 256, 256, 0, stream>>>(ep, d_plans, d_chunks, shared_bins ? n_chunks : 0u);
      // ---- K3, K4
      const uint32_t groups_per_chunk = (bpc + 7) / 8;
      for (uint32_t v = 0; v < ep.n_vars; v++) {
        if constexpr (!W) {  // wide runs bin by search over the 64-bit latents (their front end writes no 16-bit keys to look up)
          if (var_range_bits[v] <= PLAN_MAX_COUNT_BITS) {
            const uint32_t parts = (bpc + BINL_BATCHES - 1) / BINL_BATCHES;
            profiler().begin("bin_lut_kernel", stream);
            bin_lut_kernel<L><<<n_chunks * parts, BINL_THREADS, (size_t(1) << var_range_bits[v]) + 16, stream>>>(ep, bpc, parts, (v == 0 ? S.key16_0 : S.key16_1).as<uint16_t>(), d_plans, d_chunks, d_sym[v],
                                                                                                                 S.ob_sum.as<uint32_t>(), int(v), var_range_bits[v]);
            profiler().end(stream);
            continue;
          }
        }
        profiler().begin("bin_kernel", stream);
        bin_kernel<L, W><<<n_chunks * groups_per_chunk, BIN_THREADS, 0, stream>>>(ep, bpc, d_lat[v], d_plans, d_chunks, d_sym[v], S.ob_sum.as<uint32_t>(), int(v));
        profiler().end(stream);
      }
      // the ans kernel indexes (chunk, var) by blockIdx; both vars share the launch via separate symbol arrays
      profiler().begin("ans_encode_kernel", stream);
      ans_encode_kernel<W><<<n_chunks * MAX_VARS, ANS_THREADS, 0, stream>>>(ep, bpc, d_plans, d_chunks, d_sym[0], d_sym[1], d_ans[0], d_ans[1], S.ans_sum.as<uint32_t>(),
                                                                            S.entries.as<BatchEntry>(), d_ans_paths);
      profiler().end(stream);
      // ---- layout, offsets, K5
      profiler().begin("layout_kernel", stream);
      layout_kernel<W><<<n_chunks, LAYOUT_THREADS, 0, stream>>>(ep, bpc, d_plans, d_chunks, S.ans_sum.as<uint32_t>(), S.ob_sum.as<uint32_t>(), S.entries.as<BatchEntry>());
      profiler().end(stream);
      return PCO_B200_OK;
    };
    if (PcoB200Error e = wide_run ? encode_run(std::true_type{}) : encode_run(std::false_type{})) return e;
    const uint32_t footer = (last_run && !chunks_only) ? 1u : 0u;
    chunk_offsets_kernel<<<1, 1024, 0, stream>>>(d_chunks, n_chunks, file_off, footer, d_total);
    uint64_t total = 0;
    const bool need_total_now = !dst_direct || !last_run;  // a host destination is staged (sized from the file size); a later run starts where this one ends
    if (need_total_now) {
      PCOB_CUDA_TRY(readback_small_sync(&total, d_total, 8, stream));
      PCOB_CUDA_TRY(cudaGetLastError());
      call_trace().mark("c.total");
      if (total > dst_cap) return fail(PCO_B200_IO, "failed to write whole buffer (need " + std::to_string(total) + " bytes, dst_cap " + std::to_string(dst_cap) + ")");
    }
    if (!dst_direct) {
      PCOB_CUDA_TRY(S.out.reserve(total - (first_run ? 0 : file_off) + 64));
      // the run's bytes are staged at their file offsets relative to the run's first byte (the header belongs to the first run)
      d_out = S.out.as<uint8_t>() - (first_run ? 0 : file_off);
    }
    // device destination: no host round trip for the last run - pack_kernel leaves out any chunk that would not fit dst_cap, and the size
    // is checked when it is read back behind the kernel
    const uint64_t out_cap = dst_direct ? uint64_t(dst_cap) : total;
    profiler().begin("pack_kernel", stream);
    if (wide_run) {
      pack_kernel<L, true><<<n_chunks, PACK_THREADS, sizeof(PackSmemT<true>), stream>>>(ep, bpc, d_lat[0], d_lat[1], S.plans.as<VarPlanT<true>>(), d_chunks, S.sym0.as<uint16_t>(),
                                                                                       S.sym1.as<uint16_t>(), d_ans[0], d_ans[1], S.entries.as<BatchEntry>(), d_out, out_cap,
                                                                                       nullptr, nullptr);
    } else {
      pack_kernel<L><<<n_chunks, PACK_THREADS, sizeof(PackSmem), stream>>>(ep, bpc, d_lat[0], d_lat[1], S.plans.as<VarPlan>(), d_chunks, S.sym0.as<uint8_t>(),
                                                                          S.sym1.as<uint8_t>(), d_ans[0], d_ans[1], S.entries.as<BatchEntry>(), d_out, out_cap,
                                                                          var_range_bits[0] <= PLAN_MAX_COUNT_BITS ? S.key16_0.as<uint16_t>() : nullptr,
                                                                          (ep.n_vars > 1 && var_range_bits[1] <= PLAN_MAX_COUNT_BITS) ? S.key16_1.as<uint16_t>() : nullptr);
    }
    profiler().end(stream);
    if (!chunks_only && (first_run || last_run)) {
      if (runs.size() == 1) header_footer_kernel<<<1, 32, 0, stream>>>(d_out, out_cap, d_header, uint32_t(header.size()), d_total);
      else run_edge_kernel<<<1, 32, 0, stream>>>(d_out, out_cap, d_header, first_run ? uint32_t(header.size()) : 0u, d_total, last_run ? 1u : 0u);
    }
    PCOB_CUDA_TRY(cudaGetLastError());
    if (!dst_direct) {
      const uint64_t from = first_run ? 0 : file_off;
      PCOB_CUDA_TRY(copy_sliced(static_cast<uint8_t*>(dst) + from, d_out + from, total - from, cudaMemcpyDeviceToHost, stream));
    }
    // ---- this run's piece of the side index
    if (index_dst != nullptr) {
      DevBuf& idx = S.idx_out;
      PCOB_CUDA_TRY(S.seg.reserve(size_t(n_chunks) * 16));
      PCOB_CUDA_TRY(cudaMemcpyAsync(S.seg.p, eoff.data() + run.c0, size_t(n_chunks) * 8, cudaMemcpyHostToDevice, stream));
      if (first_run) {
        IndexHeader ih;
        std::memset(&ih, 0, sizeof(ih));
        ih.magic = INDEX_MAGIC; ih.version = 1; ih.n_chunks = n_chunks_all; ih.n_total = n; ih.chunks_offset = chunks_offset;  // file_len, end_byte: emit_index_kernel
        PCOB_CUDA_TRY(cudaMemcpyAsync(idx.p, &ih, sizeof(ih), cudaMemcpyHostToDevice, stream));
      }
      emit_index_kernel<<<n_chunks, 256, 0, stream>>>(ep, bpc, d_chunks, S.entries.as<BatchEntry>(), idx.as<uint8_t>(), chunks_offset, S.seg.as<uint64_t>(), d_total,
                                                      chunks_only ? 0u : 1u, uint32_t(run.c0), starts[run.c0], last_run ? 1u : 0u);
      PCOB_CUDA_TRY(cudaGetLastError());
    }
    if (!last_run || !dst_direct) {
      // the scratch is reused by the next run, and a host destination must be complete before the call returns
      PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
      PCOB_CUDA_TRY(cudaGetLastError());
      call_trace().mark("c.run_done");
      file_off = total - footer;
      res->total_bytes = total;
    } else {
      PCOB_CUDA_TRY(cudaMemcpyAsync(&total, d_total, 8, cudaMemcpyDeviceToHost, stream));  // read back behind the kernels
      if (index_dst != nullptr)
        PCOB_CUDA_TRY(cudaMemcpyAsync(index_dst, S.idx_out.p, index_total, (flags & PCO_B200_INDEX_ON_DEVICE) ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, stream));
      PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
      PCOB_CUDA_TRY(cudaGetLastError());
      if (total > dst_cap) return fail(PCO_B200_IO, "failed to write whole buffer (need " + std::to_string(total) + " bytes, dst_cap " + std::to_string(dst_cap) + ")");
      res->total_bytes = total;
      res->index_bytes = index_total;
      return PCO_B200_OK;
    }
  }
  if (index_dst != nullptr) {
    PCOB_CUDA_TRY(cudaMemcpyAsync(index_dst, S.idx_out.p, index_total, (flags & PCO_B200_INDEX_ON_DEVICE) ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, stream));
    PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
    res->index_bytes = index_total;
  }
  call_trace().mark("c.end");
  call_trace().flush("compress");
  return PCO_B200_OK;
}

}  // namespace pcob200
