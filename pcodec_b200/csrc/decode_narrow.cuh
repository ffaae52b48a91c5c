// decode_narrow_kernel: the lean instantiation of K7b+K8+K9 for the chunks that delta coding usually produces -
// classic mode, consecutive order 0 or 1, 2..256 bins whose lowers lie within 2^16 of the first bin and whose offsets
// take <= 15 bits (32- and 64-bit number types).  symwalk_kernel classifies every chunk (it has parsed and validated
// the header and bins anyway) and leaves a NarrowInfo record for the chunks of this class; everything else goes to
// decode_kernel.  Same unit of work as decode_kernel (CTA per chunk, warp per batch, 8 consecutive latents per lane),
// but the narrow ranges allow:
//   * one 4-byte table entry per bin, q = offset_bits | (lower - lower_0) << 7: the running sums of a lane's 8 entries
//     give, in one pass of adds, every field's bit position (low 7 bits: <= 8 * 15 = 120) and the prefix sums of the
//     bin lowers (high bits);
//   * the order-1 un-delta (delta/consecutive.rs:35-50) as ONE 32-bit warp scan of (lower - lower_0 + offset) - a
//     batch sums to < 2^25 - with lower_0 (+ MID, mod/delta toggle) folded in as i * base, instead of 64-bit scans;
//   * the batch's offset bits staged by one 16-byte cp.async per lane (512 bytes per warp, double-buffered), the
//     lane's 8 fields peeled off two 64-bit register windows;
//   * a prologue that is one 1 KiB coalesced load - no header parse, no table build.
// Reference behaviour restated: pco/src/page_latent_decompressor.rs:15-44 (offsets), delta/consecutive.rs:35-50,
// delta/mod.rs:29-33 (toggle), mode/classic.rs:14-24 (join), wrapped/page_decompressor.rs:115-221 (batch driver).
#pragma once
#include "decode_kernels.cuh"

namespace pcob200 {

#ifndef PCOB_NW_THREADS
#define PCOB_NW_THREADS 256
#endif
// warps of a chunk's CTA.  More warps per chunk would mean shorter CTAs and a smaller tail wave (1024 chunks on 132 SMs x 4 = 528 slots = 1.94
// waves), but the carry chain hands over once per batch (~290 cycles per link), and 8 warps were faster than 16 or 32.
constexpr int NW_THREADS = PCOB_NW_THREADS;
constexpr int NW_WARPS = NW_THREADS / 32;
constexpr int NW_RING = 2 * NW_WARPS < 32 ? 32 : 2 * NW_WARPS;  // carry-chain slots: more than the batches in flight
constexpr int NW_WIN_WORDS = 128 + 4;  // 512 staged bytes + 16 of slack for the 3-word lane windows

#ifndef PCOB_NW_MIN_BLOCKS
#define PCOB_NW_MIN_BLOCKS (1024 / PCOB_NW_THREADS)
#endif

// one step of an inclusive warp scan: v += (value of lane - d) for lanes >= d; the shuffle's own range predicate guards the add
__device__ __forceinline__ uint32_t scan_step_up(uint32_t v, int d) {
  uint32_t r;
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .u32 t;\n\t"
      "shfl.sync.up.b32 t|p, %1, %2, 0, 0xffffffff;\n\t"
      "mov.u32 %0, %1;\n\t"
      "@p add.u32 %0, %1, t;\n\t}"
      : "=r"(r) : "r"(v), "r"(d));
  return r;
}
// shifts that take the amount from the low 5 bits of `s` (the table entry itself: its bits 4..6 are zero)
__device__ __forceinline__ uint32_t shr_wrap(uint32_t lo, uint32_t hi, uint32_t s) {
  uint32_t r;
  asm("shf.r.wrap.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(lo), "r"(hi), "r"(s));
  return r;
}
__device__ __forceinline__ uint32_t ones_shl_wrap(uint32_t s) {  // 0xffffffff << (s & 31)
  uint32_t r;
  asm("shf.l.wrap.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(0u), "r"(0xffffffffu), "r"(s));
  return r;
}
struct NarrowSmem {
  uint32_t q[SMALL_MAX_BINS];
  alignas(16) uint32_t win[NW_WARPS][2][NW_WIN_WORDS];
  // delta carry chain: link[b % NW_RING] = {first number of batch b, b + 1}, written with ONE 16-byte store and read
  // with one 16-byte load, so the record is never seen half-written and the hand-over needs no fence
  alignas(16) uint64_t link[NW_RING][2];
  uint32_t err;
};

template <typename L, int K>
__device__ __forceinline__ void narrow_chunk(NarrowSmem& sm, const FileParams& fp, const IndexChunk& task, const NarrowInfo* __restrict__ inf,
                                             uint32_t* __restrict__ statuses, L* __restrict__ out, uint64_t out_len,
                                             const uint8_t* __restrict__ d_syms, const uint32_t* __restrict__ d_offs) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid < SMALL_MAX_BINS) sm.q[tid] = inf->q[tid];
  if (tid < NW_RING) {
    sm.link[tid][0] = tid == 0 ? inf->moment0 : 0;
    sm.link[tid][1] = (K == 1 && tid == 0) ? 1u : 0u;
  }
  if (tid == 0) sm.err = 0;
  __syncthreads();
  const BitSrc src = make_bitsrc(fp.src, fp.src_len);
  const uint64_t max_blk = (src.n_bits == 0 ? 0 : (src.n_bits - 1) >> 6) >> 1;
  const uint64_t chunk_bit0 = src.mis_bits + task.chunk_offset * 8;
  // 16-byte blocks of the stream, addressed relative to the chunk's first block so that the loop works in 32 bits
  const uint64_t cblk0 = chunk_bit0 >> 7;
  const uint32_t cbr = uint32_t(chunk_bit0 & 127);
  const uint32_t max_rel = max_blk > cblk0 ? uint32_t(min(max_blk - cblk0, uint64_t(0xffffffffu))) : 0u;
  const ulonglong2* __restrict__ chunk_blk = reinterpret_cast<const ulonglong2*>(src.words) + min(cblk0, max_blk);
  const uint32_t n = inf->n;
  // pco::standalone::simple_decompress_into semantics: emit only what fits in the destination
  const uint32_t n_out = task.out_offset >= out_len ? 0u : uint32_t(min(uint64_t(n), out_len - task.out_offset));
  const uint32_t nb_total = n_batches_of(n), nb_out = n_batches_of(n_out);
  const uint32_t stored = var_stored_n(n, K);
  const L base = L(inf->base);
  const uint64_t row0 = scratch_row0(task.out_offset, blockIdx.x);
  const int kind = nt_is_float(fp.dtype) ? 2 : (nt_is_signed(fp.dtype) ? 1 : 0);
  const uint32_t q_sa = smem_addr(sm.q);
  const uint32_t win_sa = smem_addr(sm.win[warp][0]);
  const uint32_t link_sa = smem_addr(&sm.link[0][0]);
  uint32_t end_err = 0;
  // running pointers of this warp's next batch (b + NW_WARPS)
  const uint2* __restrict__ sy_ptr = reinterpret_cast<const uint2*>(d_syms + (row0 + warp) * BATCH_N) + lane;
  const uint32_t* __restrict__ off_ptr = d_offs + row0 + warp;
  L* __restrict__ dst = out + task.out_offset + size_t(warp) * BATCH_N + lane * 8;

  auto issue_window = [&](uint32_t off, uint32_t bufi) {
    const uint32_t rel = min(((cbr + off) >> 7) + uint32_t(lane), max_rel);
    const void* gp = chunk_blk + rel;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(win_sa + bufi * uint32_t(NW_WIN_WORDS * 4) + uint32_t(lane) * 16u), "l"(gp));
    asm volatile("cp.async.commit_group;");
  };
  // (one cp.async.bulk of the 512 bytes per batch, signalled on an mbarrier, instead of 32 LDGSTS: correct, but slightly slower)

  // a batch's section start is requested two batches ahead, its symbols and its window one batch ahead (symbols two ahead were
  // slower; a __nanosleep back-off in the chain poll changed nothing once the hand-over was one record)
  constexpr int SY_STEP = NW_WARPS * (BATCH_N / 8);  // uint2 per round of NW_WARPS batches
  uint32_t off_cur = 0, off_nxt = 0;
  uint2 sy_nxt = make_uint2(0u, 0u);
  if (uint32_t(warp) < nb_out) {
    off_cur = __ldg(off_ptr);
    issue_window(off_cur, 0);
    sy_nxt = __ldg(sy_ptr);
    if (uint32_t(warp) + NW_WARPS < nb_out) off_nxt = __ldg(off_ptr + NW_WARPS);
  }
  uint32_t buf = 0;
  for (uint32_t b = warp; b < nb_out; b += NW_WARPS) {
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncwarp();  // this batch's window is visible to the warp; every lane is done with the other buffer
    const uint2 sy = sy_nxt;
    uint32_t off_n2 = 0;
    sy_ptr += SY_STEP;
    off_ptr += NW_WARPS;
    if (b + NW_WARPS < nb_out) {
      issue_window(off_nxt, buf ^ 1u);
      sy_nxt = __ldg(sy_ptr);
      if (b + 2 * NW_WARPS < nb_out) off_n2 = __ldg(off_ptr + NW_WARPS);
    }
    const uint32_t cnt = batch_count(stored, b);
    // ---- bins of the lane's 8 latents
    uint32_t q[8];
    q[0] = lds_u32(q_sa + ((sy.x << 2) & 0x3fcu));
    q[1] = lds_u32(q_sa + ((sy.x >> 6) & 0x3fcu));
    q[2] = lds_u32(q_sa + ((sy.x >> 14) & 0x3fcu));
    q[3] = lds_u32(q_sa + ((sy.x >> 22) & 0x3fcu));
    q[4] = lds_u32(q_sa + ((sy.y << 2) & 0x3fcu));
    q[5] = lds_u32(q_sa + ((sy.y >> 6) & 0x3fcu));
    q[6] = lds_u32(q_sa + ((sy.y >> 14) & 0x3fcu));
    q[7] = lds_u32(q_sa + ((sy.y >> 22) & 0x3fcu));
    if (cnt != uint32_t(BATCH_N)) {  // the page's last batch: latents past the stored ones read no bits and add nothing
#pragma unroll
      for (int e = 0; e < 8; e++)
        if (uint32_t(lane * 8 + e) >= cnt) q[e] = 0;
    }
    // running sums: low 7 bits = bits before field e + 1, high bits = sum of (lower - lower_0) up to e
    uint32_t P[8];
    P[0] = q[0];
#pragma unroll
    for (int e = 1; e < 8; e++) P[e] = P[e - 1] + q[e];
    const uint32_t lane_bits = P[7] & 127u;
    uint32_t inc = lane_bits;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) inc = scan_step_up(inc, d);
    const uint32_t sec_rel = cbr + off_cur;  // bit position of the section, from the chunk's first 16-byte block
    // ---- the 8 offsets: two 64-bit register windows (4 fields <= 60 bits each) out of the staged bytes
    uint32_t f[8];
    {
      const uint32_t wbase = win_sa + buf * uint32_t(NW_WIN_WORDS * 4);
      const uint32_t pa = (sec_rel & 127u) + (inc - lane_bits);
      const uint32_t pb = pa + (P[3] & 127u);
      const uint32_t wa = wbase + ((pa >> 5) << 2), wb = wbase + ((pb >> 5) << 2);
      const uint32_t a0 = lds_u32(wa), a1 = lds_u32(wa + 4), a2 = lds_u32(wa + 8);
      const uint32_t b0 = lds_u32(wb), b1 = lds_u32(wb + 4), b2 = lds_u32(wb + 8);
      uint32_t lo = shr_wrap(a0, a1, pa), hi = shr_wrap(a1, a2, pa);
#pragma unroll
      for (int e = 0; e < 4; e++) {  // q[e]'s low 5 bits are the field width
        f[e] = lo & ~ones_shl_wrap(q[e]);
        if (e < 3) {
          lo = shr_wrap(lo, hi, q[e]);
          hi = shr_wrap(hi, 0u, q[e]);
        }
      }
      lo = shr_wrap(b0, b1, pb);
      hi = shr_wrap(b1, b2, pb);
#pragma unroll
      for (int e = 4; e < 8; e++) {
        f[e] = lo & ~ones_shl_wrap(q[e]);
        if (e < 7) {
          lo = shr_wrap(lo, hi, q[e]);
          hi = shr_wrap(hi, 0u, q[e]);
        }
      }
    }
    L res[8];
    if (K == 0) {
#pragma unroll
      for (int e = 0; e < 8; e++) res[e] = L(base + L((q[e] >> 7) + f[e]));
    } else {
      // ---- order-1 un-delta: exclusive prefix sums of (lower - lower_0 + offset) in 32 bits, + i * base + first number
      uint32_t F[8];
      F[0] = f[0];
#pragma unroll
      for (int e = 1; e < 8; e++) F[e] = F[e - 1] + f[e];
      const uint32_t T = (P[7] >> 7) + F[7];
      uint32_t incT = T;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) incT = scan_step_up(incT, d);
      const uint32_t totT = __shfl_sync(0xffffffffu, incT, 31);
      const uint32_t slot = b % NW_RING, nslot = (b + 1) % NW_RING;
      uint64_t m64, fl;
      do {
        asm volatile("ld.volatile.shared.v2.u64 {%0, %1}, [%2];" : "=l"(m64), "=l"(fl) : "r"(link_sa + 16 * slot) : "memory");
      } while (fl != b + 1);
      const L m = L(m64);
      if (lane == 0)
        asm volatile("st.volatile.shared.v2.u64 [%0], {%1, %2};" ::"r"(link_sa + 16 * nslot), "l"(uint64_t(L(L(m + L(base << 8)) + L(totT)))),
                     "l"(uint64_t(b + 2)) : "memory");
      L D = L(L(m + L(base * L(lane * 8))) + L(incT - T));
      res[0] = D;
#pragma unroll
      for (int e = 1; e < 8; e++) {
        D = L(D + base);
        res[e] = L(D + L((P[e - 1] >> 7) + F[e - 1]));
      }
    }
    if (kind != 0) {
#pragma unroll
      for (int e = 0; e < 8; e++) res[e] = from_latent_kind<L>(res[e], kind);
    }
    const uint32_t out_cnt = min(uint32_t(BATCH_N), n_out - b * BATCH_N);  // numbers this batch emits
    if (out_cnt == uint32_t(BATCH_N) && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
      store8<L>(dst, res);  // 16-byte vector stores when aligned
    } else {
#pragma unroll
      for (int e = 0; e < 8; e++)
        if (uint32_t(lane * 8 + e) < out_cnt) dst[e] = res[e];
    }
    dst += NW_WARPS * BATCH_N;
    // ---- end-of-page checks by the warp that owns the last batch (page_decompressor.rs:184-188)
    if (b == nb_total - 1) {
      const uint32_t total_bits = __shfl_sync(0xffffffffu, inc, 31);
      const uint64_t bit = (cblk0 << 7) + sec_rel + total_bits;
      if (lane == 0) {
        if (bit > src.n_bits) end_err = ST_INSUFFICIENT_DATA;
        else {
          const uint32_t pad = uint32_t((8 - (bit & 7)) & 7);
          if (pad && read_bits_safe(src, bit, pad) != 0) end_err = ST_CORRUPTION;
        }
      }
    }
    off_cur = off_nxt;
    off_nxt = off_n2;
    buf ^= 1u;
  }
  if (end_err) atomicMax(&sm.err, end_err);
  __syncthreads();
  if (tid == 0) statuses[blockIdx.x] = sm.err;
}

template <typename L>
__global__ void __launch_bounds__(NW_THREADS, PCOB_NW_MIN_BLOCKS)
decode_narrow_kernel(FileParams fp, const IndexChunk* __restrict__ chunks, uint32_t* __restrict__ statuses, L* __restrict__ out, uint64_t out_len,
                     const uint8_t* __restrict__ d_syms, const uint32_t* __restrict__ d_offs, const uint8_t* __restrict__ d_cls,
                     const NarrowInfo* __restrict__ infos) {
  const uint32_t cls = d_cls[blockIdx.x];
  if (cls != CLS_NARROW0 && cls != CLS_NARROW1) return;
  __shared__ NarrowSmem sm;
  const IndexChunk task = chunks[blockIdx.x];
  if (cls == CLS_NARROW1) narrow_chunk<L, 1>(sm, fp, task, infos + blockIdx.x, statuses, out, out_len, d_syms, d_offs);
  else narrow_chunk<L, 0>(sm, fp, task, infos + blockIdx.x, statuses, out, out_len, d_syms, d_offs);
}

}  // namespace pcob200
