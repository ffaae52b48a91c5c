// The multi-CTA prefix scan every asynchronous pipeline plans its batch with, in three launches over grids fixed by the plan:
//   a multi-CTA kernel    per CTA, the sums of its items (block_exscan's total), ctas_of<NT>(n) CTAs;
//   a one-CTA kernel      those CTA sums scanned in place into CTA offsets (cta_scan_inplace), tile after tile with a carry;
//   a multi-CTA kernel    each item's offset: its CTA's offset plus block_exscan's exclusive result.
// Sums of untrusted counts are CarrySums: the flag records a carry out of 64 bits anywhere in the sum, so a refusal names exactly the
// first item where the running sum passes 2^64 (an item whose exclusive sum has no flag and whose inclusive sum has one).
#pragma once
#include "codec_common.cuh"

namespace pcob200 {

constexpr uint64_t NONE64 = ~uint64_t(0);

struct CarrySum {  // a sum with a flag for a carry out of 64 bits anywhere in it
  uint64_t s;
  uint32_t ovf, reserved;
};
static_assert(sizeof(CarrySum) == 16, "part structs and workspace regions embed it");

template <int NT>
__host__ __device__ inline uint64_t ctas_of(uint64_t n) { return (n + NT - 1) / NT; }

__device__ __forceinline__ CarrySum carry_sum(uint64_t s) { return CarrySum{s, 0u, 0u}; }

// The one addition of the scans.  The flag is sticky, so the CarrySum sum is associative and any scan order flags the same items.
__device__ __forceinline__ uint64_t carry_add(uint64_t a, uint64_t b) { return a + b; }
__device__ __forceinline__ CarrySum carry_add(CarrySum a, CarrySum b) {
  CarrySum r;
  r.s = a.s + b.s;
  r.ovf = a.ovf | b.ovf | (r.s < a.s ? 1u : 0u);
  r.reserved = 0;
  return r;
}
__device__ __forceinline__ uint64_t carry_shfl_up(uint64_t v, int d) { return __shfl_up_sync(0xffffffffu, v, d); }
__device__ __forceinline__ CarrySum carry_shfl_up(CarrySum v, int d) {
  return CarrySum{__shfl_up_sync(0xffffffffu, v.s, d), __shfl_up_sync(0xffffffffu, v.ovf, d), 0u};
}

// Exclusive scan of one value per thread over a CTA of NT threads (a multiple of 32, at most 1024); *total = the CTA's sum, in every
// thread.  V is uint64_t or CarrySum.  Every thread calls it; it ends on a barrier, so calls may follow each other.
template <int NT, typename V>
__device__ __forceinline__ V block_exscan(V v, V* total) {
  __shared__ V s_warp[NT / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  V inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const V o = carry_shfl_up(inc, d);
    if (lane >= d) inc = carry_add(o, inc);
  }
  V ex = carry_shfl_up(inc, 1);
  if (lane == 0) ex = V{};
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    V w = lane < NT / 32 ? s_warp[lane] : V{};
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const V o = carry_shfl_up(w, d);
      if (lane >= d) w = carry_add(o, w);
    }
    if (lane < NT / 32) s_warp[lane] = w;
  }
  __syncthreads();
  const V r = warp ? carry_add(s_warp[warp - 1], ex) : ex;
  *total = s_warp[NT / 32 - 1];
  __syncthreads();  // s_warp may be reused by the next call
  return r;
}

// One CTA of NT threads: n items of K sums each, every sum k replaced by its exclusive prefix sum over the items, in tiles of NT x PER
// items (PER consecutive items per thread).  load(i, k) reads sum k of item i, store(i, k, v) writes its prefix; neither is called for
// i >= n.  carry[k] is the value before item 0 on entry and that plus the sum of all items on return, in every thread.
template <int NT, int PER, int K, typename V, typename Load, typename Store>
__device__ __forceinline__ void cta_scan_inplace(uint64_t n, Load load, Store store, V (&carry)[K]) {
  for (uint64_t t0 = 0; t0 < n; t0 += uint64_t(NT) * PER) {
    const uint64_t i0 = t0 + uint64_t(threadIdx.x) * PER;
#pragma unroll
    for (int k = 0; k < K; k++) {
      V run = V{};
      for (int q = 0; q < PER; q++)
        if (i0 + q < n) run = carry_add(run, load(i0 + q, k));
      V tot;
      run = carry_add(carry[k], block_exscan<NT>(run, &tot));
      for (int q = 0; q < PER; q++)
        if (i0 + q < n) {  // loaded again rather than held: PER values per thread would cost as many registers
          const V x = load(i0 + q, k);
          store(i0 + q, k, run);
          run = carry_add(run, x);
        }
      carry[k] = carry_add(carry[k], tot);
    }
  }
}

}  // namespace pcob200
