// cold_decode_kernel: EVERY valid standalone pco stream, decoded on the device by one thread that reads the stream the way the
// reference's decompressor does - chunk after chunk, batch after batch, latent var after latent var.  It is the catch-all behind the
// fast kernels (fused_narrow_kernel, symwalk_kernel + decode_kernel), which serve Classic / IntMult / FloatMult / FloatQuant with no or
// consecutive deltas and tables of <= 2^10 states / 256 bins: files with Dict mode, Lookback or Conv1 deltas, secondary_uses_delta,
// larger tANS tables (ans_size_log <= 14, up to 2^15 bins: compression levels 9..12) or f16 FloatMult come here instead of being
// refused.  Throughput is that of one GPU thread (a few MB/s); what matters on this path is that valid pco is never turned away and that
// no byte of it is decoded on the CPU.
// Reference behaviour restated (paths relative to /root/reference):
//   chunk meta          pco/src/metadata/{chunk.rs:127-174, mode.rs:102-167, delta_encoding.rs:118-202, chunk_latent_var.rs:102-143}
//   page meta           pco/src/metadata/{page.rs:36-57, page_latent_var.rs:28-49}
//   tANS tables, walk   pco/src/ans/{spec.rs:24-59, decoding.rs:27-48}, pco/src/page_latent_decompressor.rs:89-177
//   offsets             pco/src/page_latent_decompressor.rs:15-44
//   deltas              pco/src/delta/{consecutive.rs:35-50, lookback.rs:201-246, conv1.rs:149-160,464-483, mod.rs:29-33,125-159}
//   joins               pco/src/mode/{classic.rs:14-24, int_mult.rs:38-54, float_mult.rs:17-36, float_quant.rs:13-39, dict.rs:70-90}
//   batch / page driver pco/src/wrapped/page_decompressor.rs:33-69,115-221; standalone loop pco/src/standalone/decompressor.rs:190-273
#pragma once
#include <cuda_fp16.h>

#include "decode_kernels.cuh"

namespace pcob200 {

constexpr int COLD_MAX_SIZE_LOG = 14;                 // pco/src/constants.rs:32
constexpr uint32_t COLD_MAX_BINS = 1u << 15;          // 15-bit bin count (constants.rs:20)
constexpr uint32_t COLD_MAX_WINDOW_LOG = 24;          // MAX_DELTA_LOOKBACK_WINDOW_N_LOG (constants.rs:45)

// per latent var (delta, primary, secondary): tables and page state in global scratch
struct ColdVar {
  uint32_t present, latent_bits, ans_size_log, n_bins, max_ob;
  uint32_t delta_kind;      // how THIS var is delta coded (DELTA_*); the lookback var itself is never delta coded
  uint32_t n_state;         // latents of delta state per page
  uint32_t st[4];
  uint64_t dpos;            // lookback: position in the window buffer
  uint32_t* node;           // [2^14] next_state_idx_base (0-15) | bits_to_read (24-31)
  uint16_t* sym;            // [2^14] bin of the state
  uint64_t* lower;          // [2^15]
  uint8_t* ob;              // [2^15]
  uint32_t* weight;         // [2^15] (build only)
  uint64_t* dstate;         // consecutive moments / conv1 state (<= 32) / lookback window buffer (2 * max(window_n, 256))
  uint64_t* lat;            // [256 + 32] the batch's latents
  uint32_t* obits;          // [256] offset bits per latent
};

struct ColdResult {
  uint32_t status;          // ST_OK, ST_TERMINATOR (clean end), ST_DST_FULL, or an error kind
  uint32_t n_chunks;
  uint64_t n_total;         // numbers in the chunks seen (a chunk that only partly fits counts in full)
  uint64_t next_byte;
};

// The status of one chunk the catch-all decoder was run on: ST_OK once the decoder has counted the chunk, else its error, where a run
// that ended cleanly (or at the destination's end) before the chunk is corrupt data.
__device__ __forceinline__ uint32_t cold_status(const ColdResult& res) {
  return res.n_chunks > 0 ? uint32_t(ST_OK) : (res.status == ST_OK || res.status == ST_TERMINATOR || res.status == ST_DST_FULL) ? uint32_t(ST_CORRUPTION) : res.status;
}

__host__ __device__ inline size_t cold_scratch_bytes(uint32_t window_n_log_cap) {
  const size_t per_var = (size_t(1) << COLD_MAX_SIZE_LOG) * (4 + 2) + size_t(COLD_MAX_BINS) * (8 + 1 + 4) + (256 + 32) * 8 + 256 * 4 + 64;
  const size_t win = 2 * (size_t(1) << (window_n_log_cap > 8 ? window_n_log_cap : 8)) * 8;  // buffer_n = 2 max(window_n, 256) for each delta-coded var
  return 3 * per_var + 2 * win + 8192;
}

struct ColdReader {  // the reference's BitReader over the padded stream: reads past the end give zeros, bounds are checked after a section
  BitSrc s;
  uint64_t bit;
  __device__ __forceinline__ uint64_t read(uint32_t n) {
    const uint64_t v = read_bits_safe(s, bit < s.n_bits ? bit : s.n_bits, n);
    bit += n;
    return v;
  }
  __device__ __forceinline__ bool in_bounds() const { return bit <= s.n_bits; }
  __device__ __forceinline__ bool drain_empty_byte() {  // false: non-zero padding
    const uint32_t pad = uint32_t((8 - (bit & 7)) & 7);
    if (pad == 0) return true;
    const bool ok = read_bits_safe(s, bit < s.n_bits ? bit : s.n_bits, pad) == 0;
    bit += pad;
    return ok;
  }
};

struct ColdChunk {
  uint32_t mode, mode_k, delta_kind, order, window_n_log, state_n_log, quant, conv_order, number_bits;
  bool secondary_uses_delta;
  uint64_t mode_base;
  uint64_t dict_bit;   // absolute bit position of dict value 0
  uint32_t dict_len;
  int64_t bias;
  int64_t w[32];
};

__device__ inline uint32_t cold_build_var(ColdReader& r, ColdVar& v, uint32_t latent_bits) {
  v.latent_bits = latent_bits;
  v.ans_size_log = uint32_t(r.read(4));
  v.n_bins = uint32_t(r.read(15));
  if (!r.in_bounds()) return ST_INSUFFICIENT_DATA;
  if ((1u << v.ans_size_log) < v.n_bins) return ST_CORRUPTION;
  if (v.n_bins == 1 && v.ans_size_log > 0) return ST_CORRUPTION;
  if (v.ans_size_log > uint32_t(COLD_MAX_SIZE_LOG)) return ST_CORRUPTION;
  const uint32_t obb = offset_bits_bits(latent_bits);
  v.max_ob = 0;
  uint32_t total = 0;
  for (uint32_t i = 0; i < v.n_bins; i++) {
    const uint32_t wgt = uint32_t(r.read(v.ans_size_log)) + 1;
    const uint64_t lower = r.read(latent_bits);
    const uint32_t ob = uint32_t(r.read(obb));
    if (ob > latent_bits) return r.in_bounds() ? ST_CORRUPTION : ST_INSUFFICIENT_DATA;
    v.weight[i] = wgt;
    v.lower[i] = lower;
    v.ob[i] = uint8_t(ob);
    v.max_ob = max(v.max_ob, ob);
    total += wgt;
    if ((i & 127) == 127 && !r.in_bounds()) return ST_INSUFFICIENT_DATA;
  }
  if (!r.in_bounds()) return ST_INSUFFICIENT_DATA;
  const uint32_t size = 1u << v.ans_size_log;
  if (v.n_bins == 0) {  // one implicit symbol of weight 1 (ans/spec.rs:61-66)
    if (v.ans_size_log != 0) return ST_CORRUPTION;
    v.weight[0] = 1; v.lower[0] = 0; v.ob[0] = 0;
    total = 1;
  }
  if (total != size) return ST_CORRUPTION;  // ans/spec.rs:38-44
  // spread (ans/spec.rs:24-59) and decoder nodes (ans/decoding.rs:27-48)
  uint32_t stride = (3 * size) / 5;
  if ((stride & 1) == 0) stride += 1;
  const uint32_t nb = v.n_bins == 0 ? 1 : v.n_bins;
  uint32_t step = 0;
  for (uint32_t b = 0; b < nb; b++)
    for (uint32_t k = 0; k < v.weight[b]; k++, step++) v.sym[(stride * step) & (size - 1)] = uint16_t(b);
  // x_s counts up from the weight in state order; reuse `weight` as the running counter
  for (uint32_t sidx = 0; sidx < size; sidx++) {
    const uint32_t b = v.sym[sidx];
    const uint32_t x_s = v.weight[b]++;
    const uint32_t btr = __clz(x_s) - __clz(size);
    v.node[sidx] = ((x_s << btr) - size) | (btr << 24);
  }
  return ST_OK;
}

// One batch of a var before its delta: tANS symbols, then offsets (page_latent_decompressor.rs:181-235)
__device__ inline void cold_read_pre_delta(ColdReader& r, ColdVar& v, uint32_t n) {
  if (n == 0) return;
  const uint64_t lmask = v.latent_bits == 64 ? ~uint64_t(0) : ((uint64_t(1) << v.latent_bits) - 1);
  if (v.n_bins > 1) {
    uint32_t st[4] = {v.st[0], v.st[1], v.st[2], v.st[3]};
    for (uint32_t i = 0; i < n; i++) {
      const uint32_t j = i & 3;
      const uint32_t nd = v.node[st[j]];
      const uint32_t btr = nd >> 24;
      const uint32_t b = v.sym[st[j]];
      const uint32_t val = uint32_t(r.read(btr));
      v.lat[i] = v.lower[b];
      v.obits[i] = v.ob[b];
      st[j] = (nd & 0xffffu) + val;
    }
    v.st[0] = st[0]; v.st[1] = st[1]; v.st[2] = st[2]; v.st[3] = st[3];
  } else {
    for (uint32_t i = 0; i < n; i++) { v.lat[i] = v.lower[0]; v.obits[i] = v.ob[0]; }
  }
  if (v.max_ob > 0)
    for (uint32_t i = 0; i < n; i++) v.lat[i] = (v.lat[i] + r.read(v.obits[i])) & lmask;
}

// delta decode of the batch in v.lat[0 .. dst_len) (delta/mod.rs:125-159); lookbacks: the delta var's latents of this batch
__device__ inline uint32_t cold_undelta(const ColdChunk& ch, ColdVar& v, const uint64_t* lookbacks, uint32_t dst_len) {
  const uint64_t lmask = v.latent_bits == 64 ? ~uint64_t(0) : ((uint64_t(1) << v.latent_bits) - 1);
  const uint64_t mid = uint64_t(1) << (v.latent_bits - 1);
  if (v.delta_kind == DELTA_CONSECUTIVE) {
    for (uint32_t i = 0; i < dst_len; i++) v.lat[i] = (v.lat[i] + mid) & lmask;  // toggle_center (delta/mod.rs:29-33)
    for (int k = int(ch.order) - 1; k >= 0; k--) {                                // consecutive.rs:35-50
      uint64_t m = v.dstate[k];
      for (uint32_t i = 0; i < dst_len; i++) {
        const uint64_t t = v.lat[i];
        v.lat[i] = m;
        m = (m + t) & lmask;
      }
      v.dstate[k] = m;
    }
  } else if (v.delta_kind == DELTA_CONV1) {  // conv1.rs:149-160,464-483: wrapping arithmetic in the conv type (i16 / i32 / i64)
    const uint32_t conv_bits = v.latent_bits == 8 ? 16 : v.latent_bits == 16 ? 32 : 64;
    const uint64_t cmask = conv_bits == 64 ? ~uint64_t(0) : ((uint64_t(1) << conv_bits) - 1);
    const uint32_t order = ch.conv_order;
    // residual window: state (order) then the batch
    for (uint32_t i = 0; i < dst_len; i++) {
      const uint64_t latent = (v.lat[i] + mid) & lmask;
      uint64_t s = uint64_t(ch.bias) & cmask;
      for (uint32_t j = 0; j < order; j++) {
        // residuals[i + j] of the window = state / already decoded latents, as a signed conv-type value (zero-extended L)
        const uint64_t rv = (i + j < order) ? v.dstate[i + j] : v.lat[i + j - order];
        s = (s + (uint64_t(ch.w[j]) & cmask) * (rv & lmask)) & cmask;
      }
      int64_t ss = conv_bits == 64 ? int64_t(s) : (s & (uint64_t(1) << (conv_bits - 1))) ? int64_t(s | ~cmask) : int64_t(s);
      if (ss < 0) ss = 0;
      const uint64_t pred = uint64_t(ss >> ch.quant) & lmask;
      v.lat[i] = (latent + pred) & lmask;
    }
    // the window is (state ++ decoded batch): its last `order` entries are the next state, its FIRST dst_len entries are the batch's output
    // (conv1.rs:464-483: the decoded values come out `order` positions late, the page's first numbers being the state itself)
    uint64_t ns[32];
    for (uint32_t j = 0; j < order; j++) {
      const uint32_t idx = dst_len + j;  // position in the window of length order + dst_len
      ns[j] = idx < order ? v.dstate[idx] : v.lat[idx - order];
    }
    for (uint32_t i = dst_len; i-- > 0;) v.lat[i] = i < order ? v.dstate[i] : v.lat[i - order];
    for (uint32_t j = 0; j < order; j++) v.dstate[j] = ns[j];
  } else if (v.delta_kind == DELTA_LOOKBACK) {  // lookback.rs:201-246
    const uint64_t window_n = uint64_t(1) << ch.window_n_log, state_n = uint64_t(1) << ch.state_n_log;
    const uint64_t buffer_n = max(window_n, uint64_t(BATCH_N)) * 2;
    uint64_t start = v.dpos;
    if (start + dst_len > buffer_n) {
      for (uint64_t i = 0; i < window_n; i++) v.dstate[i] = v.dstate[start - window_n + i];
      start = window_n;
    }
    bool oob = false;
    for (uint32_t i = 0; i < dst_len; i++) {
      const uint64_t lb = lookbacks[i] & 0xffffffffull;
      uint64_t lookback = lb;
      if (lb > window_n || lb == 0) { oob = oob || lb > window_n; lookback = lb == 0 ? 0 : 1; }
      v.dstate[start + i] = (((v.lat[i] + mid) & lmask) + v.dstate[start + i - lookback]) & lmask;
    }
    for (uint32_t i = 0; i < dst_len; i++) v.lat[i] = v.dstate[start - state_n + i];
    v.dpos = start + dst_len;
    if (oob) return ST_CORRUPTION;
  }
  return ST_OK;
}

template <typename L>
__device__ inline uint32_t cold_join(const ColdChunk& ch, const ColdReader& r0, uint32_t dtype, const ColdVar& pv, const ColdVar& sv, L* dst, uint32_t n_emit) {
  const bool is_float = nt_is_float(dtype), is_signed = nt_is_signed(dtype);
  constexpr L MID = L(L(1) << (LT<L>::BITS - 1));
  for (uint32_t i = 0; i < n_emit; i++) {
    const L p = L(pv.lat[i]);
    L outv;
    switch (ch.mode) {
      case MODE_CLASSIC: outv = from_latent_ordered<L>(p, is_float, is_signed); break;
      case MODE_DICT: {
        const uint64_t idx = pv.lat[i] & 0xffffffffull;
        if (idx >= ch.dict_len) return ST_CORRUPTION;
        const uint64_t pos = ch.dict_bit + idx * LT<L>::BITS;
        outv = from_latent_ordered<L>(L(read_bits_safe(r0.s, pos < r0.s.n_bits ? pos : r0.s.n_bits, LT<L>::BITS)), is_float, is_signed);
        break;
      }
      case MODE_INT_MULT: outv = from_latent_ordered<L>(L(L(p * L(ch.mode_base)) + L(sv.lat[i])), is_float, is_signed); break;
      case MODE_FLOAT_MULT: {
        L un;
        if constexpr (sizeof(L) == 2) {
          // f16 as the half crate computes: widen to f32, multiply, round back to nearest-even (data_types/float.rs:254-366)
          const uint16_t l = uint16_t(p);
          const bool neg = l < 0x8000u;
          const uint16_t abs_int = neg ? uint16_t(0x7fffu - l) : uint16_t(l - 0x8000u);
          const uint16_t gpi = 1u << 11;
          const uint16_t base_bits = from_latent_ordered<uint16_t>(uint16_t(ch.mode_base), true, false);
          if (abs_int >= gpi && uint16_t(0x6800u + (abs_int - gpi)) > 0x7c00u) {
            // int_float_from_latent gave a NaN: widened to f32, multiplied and narrowed again it keeps its sign and payload and comes
            // back quiet (half's conversions and the CPU's multiply; a GPU multiply would return the canonical NaN)
            un = L(uint16_t((neg ? 0x8000u : 0u) | uint16_t(0x6800u + (abs_int - gpi)) | 0x0200u));
          } else {
            const uint16_t hb = abs_int < gpi ? __half_as_ushort(__float2half_rn(float(abs_int))) : uint16_t(0x6800u + (abs_int - gpi));  // an f16
            const float f = __half2float(__ushort_as_half(uint16_t(hb | (neg ? 0x8000u : 0u))));  // the sign as a bit, not as a negation
            const float prod = __fmul_rn(f, __half2float(__ushort_as_half(base_bits)));
            un = L(__half_as_ushort(__float2half_rn(prod)));
          }
        } else if constexpr (sizeof(L) >= 4) {
          un = float_mult_unadjusted(p, from_latent_ordered<L>(L(ch.mode_base), true, false));
        } else {
          un = 0;
        }
        const L u = to_latent_ordered<L>(un, true, false);
        outv = from_latent_ordered<L>(L(L(u + L(sv.lat[i])) + MID), true, false);
        break;
      }
      default: {  // MODE_FLOAT_QUANT
        const uint32_t k = ch.mode_k;
        const L sign_cutoff = L(MID >> k);
        const L kmax = L(L(L(1) << k) - 1);
        const L s = L(sv.lat[i]);
        const L lowest = p >= sign_cutoff ? s : L(kmax - s);
        outv = from_latent_ordered<L>(L(L(p << k) + lowest), true, false);
        break;
      }
    }
    dst[i] = outv;
  }
  return ST_OK;
}

// The decoder one thread runs: the chunks from `first_chunk_byte` on, into out[0, out_len).  scratch: cold_scratch_bytes(COLD window cap)
// bytes.  cold_decode_kernel runs it over a whole file; cold_chunks_kernel (async_kernels.cuh) over one chunk at a time.
template <typename L>
__device__ __forceinline__ void cold_decode_run(const FileParams& fp, uint64_t first_chunk_byte, L* __restrict__ out, uint64_t out_len,
                                                uint8_t* __restrict__ scratch, uint32_t window_log_cap, ColdResult* __restrict__ result) {
  const BitSrc src = make_bitsrc(fp.src, fp.src_len);
  ColdReader r{src, src.mis_bits + first_chunk_byte * 8};
  // carve the scratch
  ColdVar vars[3];
  {
    uint8_t* p = scratch;
    const size_t win_bytes = 2 * (size_t(1) << (window_log_cap > 8 ? window_log_cap : 8)) * 8;
    for (int v = 0; v < 3; v++) {
      vars[v].lower = reinterpret_cast<uint64_t*>(p); p += size_t(COLD_MAX_BINS) * 8;
      vars[v].lat = reinterpret_cast<uint64_t*>(p); p += (256 + 32) * 8;
      vars[v].dstate = reinterpret_cast<uint64_t*>(p); p += v == 0 ? 64 * 8 : win_bytes;  // the lookback var itself carries no delta state
      vars[v].node = reinterpret_cast<uint32_t*>(p); p += (size_t(1) << COLD_MAX_SIZE_LOG) * 4;
      vars[v].weight = reinterpret_cast<uint32_t*>(p); p += size_t(COLD_MAX_BINS) * 4;
      vars[v].obits = reinterpret_cast<uint32_t*>(p); p += 256 * 4;
      vars[v].sym = reinterpret_cast<uint16_t*>(p); p += (size_t(1) << COLD_MAX_SIZE_LOG) * 2;
      vars[v].ob = p; p += size_t(COLD_MAX_BINS);
      p = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(p) + 15) & ~uintptr_t(15));
    }
  }
  uint64_t out_off = 0;
  uint32_t n_chunks = 0;
  uint32_t status = ST_OK;
  const uint32_t number_bits = nt_bits(fp.dtype);
  for (;;) {
    // ---- chunk preamble (standalone/decompressor.rs:190-231)
    if (r.bit + 8 > src.n_bits) { status = ST_INSUFFICIENT_DATA; break; }
    const uint64_t chunk_byte = (r.bit - src.mis_bits) >> 3;
    const uint32_t type_byte = uint32_t(r.read(8));
    if (type_byte == 0) { status = ST_TERMINATOR; break; }
    if ((fp.uniform_type != 0 && fp.uniform_type != type_byte) || type_byte != fp.dtype) { status = ST_CORRUPTION; break; }
    const uint32_t n = uint32_t(r.read(24)) + 1;
    if (!r.in_bounds()) { status = ST_INSUFFICIENT_DATA; break; }
    // ---- chunk meta
    ColdChunk ch;
    ch.number_bits = number_bits;
    ch.mode = uint32_t(r.read(4));
    ch.mode_base = 0; ch.mode_k = 0; ch.dict_len = 0; ch.dict_bit = 0;
    bool bad = false;
    switch (ch.mode) {
      case MODE_CLASSIC: break;
      case MODE_INT_MULT: if (fp.format_major == 0) bad = true; ch.mode_base = r.read(number_bits); break;
      case MODE_FLOAT_MULT: ch.mode_base = r.read(number_bits); break;
      case MODE_FLOAT_QUANT: ch.mode_k = uint32_t(r.read(8)); break;
      case MODE_DICT:
        ch.dict_len = uint32_t(r.read(25));
        if (!r.drain_empty_byte()) bad = true;
        break;
      default: bad = true;
    }
    if (!r.in_bounds()) { status = ST_INSUFFICIENT_DATA; break; }
    if (bad) { status = ST_CORRUPTION; break; }
    if (ch.mode == MODE_DICT) {
      ch.dict_bit = r.bit;
      r.bit += uint64_t(ch.dict_len) * number_bits;
      if (!r.in_bounds()) { status = ST_INSUFFICIENT_DATA; break; }
    }
    ch.delta_kind = DELTA_NONE; ch.order = 0; ch.secondary_uses_delta = false; ch.window_n_log = 0; ch.state_n_log = 0; ch.quant = 0; ch.conv_order = 0; ch.bias = 0;
    if (fp.format_major < 3) {
      const uint32_t order = uint32_t(r.read(3));
      if (order) { ch.delta_kind = DELTA_CONSECUTIVE; ch.order = order; }
    } else {
      const uint32_t variant = uint32_t(r.read(4));
      if (variant == 1) {
        ch.order = uint32_t(r.read(3));
        if (ch.order == 0) bad = true;
        ch.delta_kind = DELTA_CONSECUTIVE;
        ch.secondary_uses_delta = r.read(1) != 0;
      } else if (variant == 2) {
        ch.window_n_log = 1 + uint32_t(r.read(5));
        ch.state_n_log = uint32_t(r.read(4));
        if (ch.window_n_log > COLD_MAX_WINDOW_LOG || ch.state_n_log > ch.window_n_log) bad = true;
        ch.delta_kind = DELTA_LOOKBACK;
        ch.secondary_uses_delta = r.read(1) != 0;
      } else if (variant == 3) {
        ch.delta_kind = DELTA_CONV1;
        ch.quant = uint32_t(r.read(5));
        ch.bias = int64_t(r.read(64) ^ (uint64_t(1) << 63));
        ch.conv_order = 1 + uint32_t(r.read(5));
        for (uint32_t i = 0; i < ch.conv_order; i++) ch.w[i] = int64_t(int32_t(uint32_t(r.read(32)) ^ 0x80000000u));
      } else if (variant != 0) bad = true;
    }
    if (!r.in_bounds()) { status = ST_INSUFFICIENT_DATA; break; }
    if (bad) { status = ST_CORRUPTION; break; }
    if (ch.delta_kind == DELTA_LOOKBACK && ch.window_n_log > window_log_cap) { status = ST_UNSUPPORTED; break; }  // window larger than this launch's scratch
    // mode validity for the number type (data_types/unsigned.rs:80-86, float.rs:372-384)
    {
      const bool is_float = nt_is_float(fp.dtype);
      bool ok = true;
      if (is_float) {
        if (ch.mode == MODE_INT_MULT) ok = false;
        if (ch.mode == MODE_FLOAT_QUANT) { const uint32_t prec = number_bits == 64 ? 52 : number_bits == 32 ? 23 : 10; ok = ch.mode_k > 0 && ch.mode_k <= prec; }
        if (ch.mode == MODE_FLOAT_MULT) {
          const uint64_t mid = uint64_t(1) << (number_bits - 1);
          const uint64_t l = ch.mode_base;
          const uint64_t bits = (l & mid) ? (l ^ mid) : (~l & (number_bits == 64 ? ~uint64_t(0) : ((uint64_t(1) << number_bits) - 1)));
          const uint32_t mant = number_bits == 64 ? 52 : number_bits == 32 ? 23 : 10;
          const uint64_t abs_bits = bits & (mid - 1);
          const uint64_t exp_mask = ((uint64_t(1) << (number_bits - 1 - mant)) - 1) << mant;
          ok = (abs_bits & exp_mask) != exp_mask && abs_bits != 0;
        }
      } else {
        if (ch.mode == MODE_FLOAT_MULT || ch.mode == MODE_FLOAT_QUANT) ok = false;
        if (ch.mode == MODE_INT_MULT) ok = ch.mode_base > 0;
      }
      if (!ok) { status = ST_CORRUPTION; break; }
    }
    // ---- latent vars: [delta (Lookback only, u32)], primary (u32 indices in Dict mode), [secondary]
    ColdVar& dv = vars[0];
    ColdVar& pv = vars[1];
    ColdVar& sv = vars[2];
    dv.present = ch.delta_kind == DELTA_LOOKBACK;
    pv.present = 1;
    sv.present = ch.mode == MODE_INT_MULT || ch.mode == MODE_FLOAT_MULT || ch.mode == MODE_FLOAT_QUANT;
    for (int vi = 0; vi < 3; vi++)
      for (int i = 0; i < 256 + 32; i++) vars[vi].lat[i] = 0;  // the reference's per-chunk batch scratch starts zeroed (stale entries feed the last batch of a page)
    if (dv.present) { status = cold_build_var(r, dv, 32); if (status != ST_OK) break; }
    status = cold_build_var(r, pv, ch.mode == MODE_DICT ? 32u : number_bits);
    if (status != ST_OK) break;
    if (sv.present) { status = cold_build_var(r, sv, number_bits); if (status != ST_OK) break; }
    if (!r.drain_empty_byte()) { status = ST_CORRUPTION; break; }
    if (!r.in_bounds()) { status = ST_INSUFFICIENT_DATA; break; }
    // validate_chunk_meta (metadata/chunk.rs:32-92)
    if (ch.delta_kind == DELTA_LOOKBACK) {
      const uint64_t window_n = uint64_t(1) << ch.window_n_log;
      for (uint32_t i = 0; i < dv.n_bins; i++)
        if (dv.lower[i] < 1 || dv.lower[i] > window_n) bad = true;
    } else if (ch.delta_kind == DELTA_CONV1) {
      const uint32_t lb = pv.latent_bits;
      if (lb == 64) bad = true;
      else {
        const uint32_t conv_bits = lb == 8 ? 16 : lb == 16 ? 32 : 64;
        if (ch.quant > min(31u, conv_bits - 1)) bad = true;
        double wsum = 0.0;
        for (uint32_t i = 0; i < ch.conv_order; i++) wsum += double(ch.w[i] < 0 ? -ch.w[i] : ch.w[i]);
        const double max_pred = fabs(double(ch.bias)) + exp2(double(lb)) * wsum;
        if (max_pred >= exp2(double(conv_bits - 1))) bad = true;
      }
    }
    if (bad) { status = ST_CORRUPTION; break; }
    dv.delta_kind = DELTA_NONE;
    pv.delta_kind = ch.delta_kind;
    sv.delta_kind = ((ch.delta_kind == DELTA_CONSECUTIVE || ch.delta_kind == DELTA_LOOKBACK) && ch.secondary_uses_delta) ? ch.delta_kind : uint32_t(DELTA_NONE);
    auto n_state_of = [&](uint32_t kind) -> uint32_t {
      return kind == DELTA_CONSECUTIVE ? ch.order : kind == DELTA_LOOKBACK ? (1u << ch.state_n_log) : kind == DELTA_CONV1 ? ch.conv_order : 0u;
    };
    dv.n_state = 0;
    pv.n_state = n_state_of(pv.delta_kind);
    sv.n_state = n_state_of(sv.delta_kind);
    // ---- page meta (metadata/page.rs:36-57): per var its delta state, then 4 tANS state indices
    for (int vi = 0; vi < 3; vi++) {
      ColdVar& v = vars[vi];
      if (!v.present) continue;
      if (v.delta_kind == DELTA_LOOKBACK) {
        const uint64_t window_n = uint64_t(1) << ch.window_n_log;
        const uint64_t buffer_n = max(window_n, uint64_t(BATCH_N)) * 2;
        for (uint64_t i = 0; i < buffer_n; i++) v.dstate[i] = 0;
        for (uint32_t i = 0; i < v.n_state; i++) v.dstate[window_n - v.n_state + i] = r.read(v.latent_bits);
        v.dpos = window_n;
      } else {
        for (uint32_t i = 0; i < v.n_state; i++) v.dstate[i] = r.read(v.latent_bits);
      }
      for (int j = 0; j < 4; j++) v.st[j] = uint32_t(r.read(v.ans_size_log));
    }
    if (!r.drain_empty_byte()) { status = ST_CORRUPTION; break; }
    if (!r.in_bounds()) { status = ST_INSUFFICIENT_DATA; break; }
    const uint32_t n_state = pv.n_state;  // n_latents_per_delta_state: the primary's (page_decompressor.rs:38)
    const uint32_t n_in_body = n > n_state ? n - n_state : 0;
    for (int vi = 0; vi < 3; vi++)
      if (vars[vi].present && vars[vi].n_bins == 0 && n_in_body > 0) bad = true;  // page_decompressor.rs:52-57
    if (bad) { status = ST_CORRUPTION; break; }
    // ---- batches (page_decompressor.rs:115-221); pco::standalone::simple_decompress_into semantics for a short destination
    const uint64_t room = out_off < out_len ? out_len - out_off : 0;
    const uint32_t n_emit_chunk = uint32_t(min(uint64_t(n), room));
    uint32_t remaining = n;
    uint32_t done = 0;
    const bool decode_all = n_emit_chunk == n;  // a chunk that does not fit is decoded as far as the destination reaches, then the walk stops
    while (remaining > 0 && (decode_all || done < n_emit_chunk)) {
      const uint32_t batch_n = min(uint32_t(BATCH_N), remaining);
      const uint64_t* lookbacks = nullptr;
      if (dv.present) {
        const uint32_t limit = min(remaining > n_state ? remaining - n_state : 0u, batch_n);
        cold_read_pre_delta(r, dv, limit);
        if (!r.in_bounds()) { status = ST_INSUFFICIENT_DATA; break; }
        lookbacks = dv.lat;
      }
      for (int vi = 1; vi < 3; vi++) {
        ColdVar& v = vars[vi];
        if (!v.present) continue;
        const uint32_t pre = min(uint32_t(BATCH_N), remaining > v.n_state ? remaining - v.n_state : 0u);
        cold_read_pre_delta(r, v, pre);
        if (!r.in_bounds()) { status = ST_INSUFFICIENT_DATA; break; }
        const uint32_t st2 = cold_undelta(ch, v, lookbacks, batch_n);
        if (st2 != ST_OK) { status = st2; break; }
      }
      if (status != ST_OK) break;
      const uint32_t n_emit = done < n_emit_chunk ? min(batch_n, n_emit_chunk - done) : 0u;
      if (n_emit) {
        const uint32_t st3 = cold_join<L>(ch, r, fp.dtype, pv, sv, out + out_off + done, n_emit);
        if (st3 != ST_OK) { status = st3; break; }
      }
      done += batch_n;
      remaining -= batch_n;
      if (remaining == 0 && !r.drain_empty_byte()) { status = ST_CORRUPTION; break; }
    }
    if (status != ST_OK) break;
    (void)chunk_byte;
    out_off += n;
    n_chunks += 1;
    if (!decode_all) { status = ST_DST_FULL; break; }
    if (out_off > out_len) { status = ST_DST_FULL; break; }
  }
  result->status = status;
  result->n_chunks = n_chunks;
  result->n_total = out_off;
  result->next_byte = (r.bit - src.mis_bits) >> 3;
}

// One thread decodes the file from `first_chunk_byte` on.  scratch: cold_scratch_bytes(COLD window cap) bytes.
template <typename L>
__global__ void cold_decode_kernel(FileParams fp, uint64_t first_chunk_byte, L* __restrict__ out, uint64_t out_len, uint8_t* __restrict__ scratch,
                                   uint32_t window_log_cap, ColdResult* __restrict__ result) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  cold_decode_run<L>(fp, first_chunk_byte, out, out_len, scratch, window_log_cap, result);
}

}  // namespace pcob200
