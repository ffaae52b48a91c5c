// ORACLE — TEST INFRASTRUCTURE ONLY (see pco_core.hpp header).
// Mode split/join, delta encode/decode, per-latent-var page (de)compression,
// chunk compressor (planner driver) and the standalone/wrapped entry points.
#pragma once
#include "pco_planner.hpp"

namespace pco_oracle {

// ===========================================================================
// Config (pco/src/chunk_config.rs:15-224)
// ===========================================================================
enum class ModeSpecKind : int { Auto = 0, Classic = 1, TryFloatMult = 2, TryFloatQuant = 3, TryIntMult = 4, TryDict = 5 };
enum class DeltaSpecKind : int { Auto = 0, NoOp = 1, TryConsecutive = 2, TryLookback = 3, TryConv1 = 4 };
enum class PagingKind : int { EqualPagesUpTo = 0, Exact = 1 };

struct ChunkConfig {
  size_t compression_level = DEFAULT_COMPRESSION_LEVEL;
  ModeSpecKind mode_kind = ModeSpecKind::Auto;
  double float_mult_base = 0.0;
  Bitlen float_quant_k = 0;
  uint64_t int_mult_base = 0;
  DeltaSpecKind delta_kind = DeltaSpecKind::Auto;
  size_t delta_order = 0;
  PagingKind paging_kind = PagingKind::EqualPagesUpTo;
  size_t max_page_n = DEFAULT_MAX_PAGE_N;
  std::vector<size_t> exact_pages;
  bool enable_8_bit = false;
};

// chunk_config.rs:134-183
inline std::vector<size_t> n_per_page(const ChunkConfig& c, size_t n) {
  std::vector<size_t> res;
  if (c.paging_kind == PagingKind::EqualPagesUpTo) {
    if (n == 0) return res;
    if (c.max_page_n == 0) invalid_argument("max_page_n must be positive");  // Rust would panic on div by zero
    size_t n_pages = (n + c.max_page_n - 1) / c.max_page_n;
    size_t low = n / n_pages, high = low + 1, r = n % n_pages;
    res.assign(n_pages, low);
    for (size_t i = 0; i < r; i++) res[i] = high;
  } else {
    res = c.exact_pages;
  }
  size_t summed = 0;
  for (size_t p : res) summed += p;
  if (summed != n) invalid_argument("paging spec suggests " + std::to_string(summed) + " numbers but " + std::to_string(n) + " were given");
  for (size_t p : res) if (p == 0) invalid_argument("cannot write data page of 0 numbers");
  return res;
}

// chunk_config.rs:269-314
inline void validate_config(const ChunkConfig& c, Bitlen latent_bits) {
  if (c.compression_level > MAX_COMPRESSION_LEVEL) invalid_argument("compression level may not exceed 12");
  if (c.delta_kind == DeltaSpecKind::TryConsecutive && c.delta_order > MAX_CONSECUTIVE_DELTA_ORDER)
    invalid_argument("consecutive delta order may not exceed 7");
  if (c.delta_kind == DeltaSpecKind::TryConv1) {
    if (c.delta_order > MAX_CONV1_DELTA_ORDER) invalid_argument("conv1 delta order may not exceed 32");
    if (latent_bits > 32) invalid_argument("Conv1 delta encoding is only supported for types with 32 or fewer bits");
  }
  if (latent_bits == 8 && !c.enable_8_bit) invalid_argument("compressing 8-bit types with Pco is often a mistake");
}

// ===========================================================================
// Float helpers (pco/src/data_types/float.rs:130-252)
// ===========================================================================
template <typename L> struct FloatOps;
template <> struct FloatOps<uint32_t> {
  using F = float;
  static constexpr int MANTISSA_DIGITS = 24;
  static F from_bits(uint32_t b) { F f; std::memcpy(&f, &b, 4); return f; }
  static uint32_t to_bits(F f) { uint32_t b; std::memcpy(&b, &f, 4); return b; }
  static F mul(F a, F b) { return a * b; }
  static F round_(F a) { return std::round(a); }
  static F from_f64(double x) { return F(x); }
  static F inv(F a) { return 1.0f / a; }
  static F from_uint(uint32_t x) { return F(x); }
  static uint32_t to_uint(F x) { return uint32_t(x); }
  static bool lt(F a, F b) { return a < b; }
};
template <> struct FloatOps<uint64_t> {
  using F = double;
  static constexpr int MANTISSA_DIGITS = 53;
  static F from_bits(uint64_t b) { F f; std::memcpy(&f, &b, 8); return f; }
  static uint64_t to_bits(F f) { uint64_t b; std::memcpy(&b, &f, 8); return b; }
  static F mul(F a, F b) { return a * b; }
  static F round_(F a) { return std::round(a); }
  static F from_f64(double x) { return x; }
  static F inv(F a) { return 1.0 / a; }
  static F from_uint(uint64_t x) { return F(x); }
  static uint64_t to_uint(F x) { return uint64_t(x); }
  static bool lt(F a, F b) { return a < b; }
};
// f16 via the half crate's semantics: every op widens to f32 and rounds back (RNE).
struct F16 { uint16_t bits; };
template <> struct FloatOps<uint16_t> {
  using F = F16;
  static constexpr int MANTISSA_DIGITS = 11;
  static F from_bits(uint16_t b) { return F16{b}; }
  static uint16_t to_bits(F f) { return f.bits; }
  static F mul(F a, F b) { return F16{f32_to_f16_bits(f16_bits_to_f32(a.bits) * f16_bits_to_f32(b.bits))}; }
  static F round_(F a) { return F16{f32_to_f16_bits(std::round(f16_bits_to_f32(a.bits)))}; }
  static F from_uint(uint16_t x) { return F16{f32_to_f16_bits(float(x))}; }
  static F from_f64(double x);                                                                      // half::f16::from_f64, defined with the mode search
  static F inv(F a) { return F16{f32_to_f16_bits(1.0f / f16_bits_to_f32(a.bits))}; }               // f16::ONE / a
  static uint16_t to_uint(F x) { return uint16_t(f16_bits_to_f32(x.bits)); }
  static bool lt(F a, F b) { return f16_bits_to_f32(a.bits) < f16_bits_to_f32(b.bits); }
};
template <> struct FloatOps<uint8_t> {};  // no 8-bit floats

// float.rs:208-226
template <typename L>
inline typename FloatOps<L>::F int_float_from_latent(L l) {
  using FO = FloatOps<L>;
  constexpr L MID = LatentTraits<L>::MID;
  bool negative;
  L abs_int;
  if (l >= MID) { negative = false; abs_int = L(l - MID); } else { negative = true; abs_int = L(MID - 1 - l); }
  L gpi = L(L(1) << FO::MANTISSA_DIGITS);
  L abs_bits;
  if (abs_int < gpi) abs_bits = FO::to_bits(FO::from_uint(abs_int));
  else abs_bits = L(FO::to_bits(FO::from_uint(gpi)) + (abs_int - gpi));
  if (negative) abs_bits = L(abs_bits ^ MID);  // unary minus flips the sign bit
  return FO::from_bits(abs_bits);
}
// float.rs:229-244
template <typename L>
inline L int_float_to_latent(typename FloatOps<L>::F x) {
  using FO = FloatOps<L>;
  constexpr L MID = LatentTraits<L>::MID;
  L bits = FO::to_bits(x);
  L abs_bits = L(bits & ~MID);
  typename FloatOps<L>::F abs = FO::from_bits(abs_bits);
  L gpi = L(L(1) << FO::MANTISSA_DIGITS);
  typename FloatOps<L>::F gpi_float = FO::from_uint(gpi);
  L abs_int;
  if (FO::lt(abs, gpi_float)) abs_int = FO::to_uint(abs);
  else abs_int = L(gpi + (abs_bits - FO::to_bits(gpi_float)));
  bool sign_positive = (bits & MID) == 0;
  return sign_positive ? L(MID + abs_int) : L(MID - 1 - abs_int);
}

// ===========================================================================
// Delta (pco/src/delta/{mod,consecutive,lookback,conv1}.rs)
// ===========================================================================
// delta/mod.rs:29-33
template <typename L>
inline void toggle_center_in_place(L* v, size_t n) {
  for (size_t i = 0; i < n; i++) v[i] = L(v[i] + LatentTraits<L>::MID);
}

// delta/consecutive.rs:3-33
template <typename L>
inline std::vector<L> consecutive_encode_in_place(size_t order, L* latents, size_t len) {
  std::vector<L> moments;
  moments.reserve(order);
  L* v = latents;
  size_t n = len;
  for (size_t k = 0; k < order; k++) {
    moments.push_back(n > 0 ? v[0] : L(0));
    if (n > 0)
      for (size_t i = n - 1; i >= 1; i--) v[i] = L(v[i] - v[i - 1]);
    size_t trunc = std::min<size_t>(n, 1);
    v += trunc;
    n -= trunc;
  }
  toggle_center_in_place(v, n);
  return moments;
}

// delta/consecutive.rs:35-50
template <typename L>
inline void consecutive_decode_in_place(std::vector<L>& moments, L* latents, size_t len) {
  toggle_center_in_place(latents, len);
  for (size_t k = moments.size(); k-- > 0;) {
    L m = moments[k];
    for (size_t i = 0; i < len; i++) {
      L tmp = latents[i];
      latents[i] = m;
      m = L(m + tmp);
    }
    moments[k] = m;
  }
}

// ----- lookback (delta/lookback.rs) -----------------------------------------
constexpr size_t LB_PROPOSED = 16, LB_BRUTE = 6, LB_REPEATING = 4;
constexpr Bitlen LB_COARSENESSES[2] = {0, 8};
constexpr Bitlen ENCODING_LOOKBACK_MAX_WINDOW_N_LOG = 15, ENCODING_LOOKBACK_MIN_WINDOW_N_LOG = 4;

// delta/mod.rs:37-49
inline DeltaEncoding new_lookback(size_t n) {
  DeltaEncoding d;
  d.kind = DeltaKind::Lookback;
  Bitlen w = bits_to_encode_offset<uint32_t>(uint32_t(n) - 1);
  d.window_n_log = std::min(std::max(w, ENCODING_LOOKBACK_MIN_WINDOW_N_LOG), ENCODING_LOOKBACK_MAX_WINDOW_N_LOG);
  d.state_n_log = 0;
  d.secondary_uses_delta = false;
  return d;
}

// delta/lookback.rs:23-159
template <typename L>
inline std::vector<DeltaLookback> choose_lookbacks(const DeltaEncoding& cfg, const L* latents, size_t len) {
  size_t state_n = size_t(1) << cfg.state_n_log;
  if (len <= state_n) return {};
  size_t hash_table_n = size_t(1) << (cfg.window_n_log + 1);
  size_t window_n = size_t(1) << cfg.window_n_log;
  if (window_n < LB_PROPOSED) invalid_argument("we do not support tiny windows during compression");
  std::vector<uint32_t> lookback_counts(std::min(window_n, len), 1);
  std::vector<DeltaLookback> lookbacks(len - state_n);
  std::vector<size_t> idx_hash_table(2 * hash_table_n, 0);
  size_t proposed[LB_PROPOSED];
  for (size_t i = 0; i < LB_PROPOSED; i++) proposed[i] = std::min(i + 1, state_n);
  size_t best_lookback = 1;
  size_t repeating_idx = 0;
  size_t hash_mask = hash_table_n - 1;
  auto hash_fn = [&](uint64_t x) {
    x = (x ^ (x >> 32)) * 11400714819323197441ull;
    x = x ^ (x >> 32);
    return size_t(x) & hash_mask;
  };
  for (size_t i = state_n; i < len; i++) {
    L l = latents[i];
    size_t new_brute = std::min(i, LB_PROPOSED);
    proposed[new_brute - 1] = new_brute;
    // hash_lookup
    {
      size_t proposal_idx = LB_BRUTE + LB_REPEATING;
      size_t offset = 0;
      for (Bitlen coarseness : LB_COARSENESSES) {
        uint64_t bucket = uint64_t(l) >> coarseness;
        uint64_t buckets[3] = {bucket - 1, bucket, bucket + 1};
        size_t hashes[3];
        for (int t = 0; t < 3; t++) hashes[t] = hash_fn(buckets[t]);
        for (int t = 0; t < 3; t++) {
          size_t lb_last = i - idx_hash_table[offset + hashes[t]];
          proposed[proposal_idx] = lb_last <= window_n ? lb_last : std::min(proposal_idx, i);
          proposal_idx++;
        }
        idx_hash_table[offset + hashes[1]] = i;
        offset += hash_table_n;
      }
    }
    // find_best_lookback
    size_t new_best = 0;
    {
      Bitlen best_goodness = 0;
      for (size_t t = 0; t < LB_PROPOSED; t++) {
        size_t lookback = proposed[t];
        uint32_t count = lookback_counts[lookback - 1];
        L other = latents[i - lookback];
        Bitlen lookback_goodness = 32 - (count == 0 ? 32 : Bitlen(__builtin_clz(count)));
        L d0 = L(l - other), d1 = L(other - l);
        L delta = std::min(d0, d1);
        Bitlen goodness = lookback_goodness + leading_zeros<L>(delta);
        if (goodness > best_goodness) { best_goodness = goodness; new_best = lookback; }
      }
    }
    if (new_best != best_lookback) repeating_idx += 1;
    proposed[LB_BRUTE + repeating_idx % LB_REPEATING] = new_best;
    best_lookback = new_best;
    lookbacks[i - state_n] = DeltaLookback(best_lookback);
    lookback_counts[best_lookback - 1] += 1;
  }
  return lookbacks;
}

// delta/lookback.rs:166-187
template <typename L>
inline std::vector<L> lookback_encode_in_place(const DeltaEncoding& cfg, const DeltaLookback* lookbacks, L* latents, size_t len) {
  size_t state_n = size_t(1) << cfg.state_n_log;
  size_t real_state_n = std::min(len, state_n);
  for (size_t i = len; i-- > real_state_n;) {
    size_t lookback = lookbacks[i - state_n];
    latents[i] = L(latents[i] - latents[i - lookback]);
  }
  std::vector<L> state(state_n, 0);
  for (size_t i = 0; i < real_state_n; i++) state[state_n - real_state_n + i] = latents[i];
  toggle_center_in_place(latents, len);
  return state;
}

// ----- conv1 decode (delta/conv1.rs:149-160,191-253,464-483) ----------------
template <typename L> struct ConvType;
template <> struct ConvType<uint8_t> { using S = int16_t; };
template <> struct ConvType<uint16_t> { using S = int32_t; };
template <> struct ConvType<uint32_t> { using S = int64_t; };
template <> struct ConvType<uint64_t> { using S = int64_t; };

template <typename L>
inline void conv1_decode_in_place(const DeltaEncoding& cfg, std::vector<L>& state, L* latents, size_t len) {
  using S = typename ConvType<L>::S;
  using US = typename std::make_unsigned<S>::type;
  size_t order = cfg.weights.size();
  std::vector<S> weights(order);
  for (size_t i = 0; i < order; i++) weights[i] = S(cfg.weights[i]);
  S bias = S(cfg.bias);
  Bitlen q = cfg.quantization;
  toggle_center_in_place(latents, len);
  // The reference's order-6 specialisation computes the same sums in a
  // different association order; integer wrapping arithmetic is associative,
  // so one general implementation covers both.
  std::vector<L> residuals(len + order);
  for (size_t i = 0; i < order; i++) residuals[i] = state[i];
  for (size_t i = 0; i < len; i++) residuals[order + i] = latents[i];
  for (size_t i = order; i < residuals.size(); i++) {
    US s = US(bias);
    for (size_t j = 0; j < order; j++) s = US(s + US(US(weights[j]) * US(S(residuals[i - order + j]))));
    S ss = S(s);
    if (ss < 0) ss = 0;
    L pred = L(ss >> q);
    residuals[i] = L(residuals[i] + pred);
  }
  for (size_t i = 0; i < len; i++) latents[i] = residuals[i];
  for (size_t i = 0; i < order; i++) state[i] = residuals[len + i];
}

// ----- conv1 encode (delta/conv1.rs:12-147 the small matrix type, :256-461 fit + encode) --------------------------------
// All of the fit is f64 with the reference's exact operation order: plain multiply-adds where it writes `a * b + c`, fused ones
// (std::fma) where it calls mul_add.  Pinned by its unit tests (:503-583) and by re-encoding v1_0_0_conv1.pco byte for byte.
struct ConvMatrix {  // column-major (conv1.rs:16-52)
  std::vector<double> data;
  size_t h = 0, w = 0;
  ConvMatrix(double value, size_t h_, size_t w_) : data(h_ * w_, value), h(h_), w(w_) {}
  double& at(size_t i, size_t j) { return data[i + j * h]; }
  double at(size_t i, size_t j) const { return data[i + j * h]; }
};
inline ConvMatrix conv_cholesky(ConvMatrix m) {  // :54-93 Cholesky-Crout, L of X = L L*
  const size_t h = m.h;
  for (size_t j = 0; j < h; j++) {
    for (size_t i = 0; i < j; i++) m.at(i, j) = 0.0;
    double s = 0.0;
    for (size_t k = 0; k < j; k++) {
      const double value = m.at(j, k);
      s = std::fma(value, value, s);
    }
    const double diag_value = std::sqrt(std::fmax(m.at(j, j) - s, 0.0));  // safe_sqrt; f64::max returns the non-NaN operand like fmax
    m.at(j, j) = diag_value;
    const double scale = diag_value == 0.0 ? 0.0 : 1.0 / diag_value;
    for (size_t i = j + 1; i < h; i++) {
      double t = 0.0;
      for (size_t k = 0; k < j; k++) t = std::fma(m.at(i, k), m.at(j, k), t);
      m.at(i, j) = scale * (m.at(i, j) - t);
    }
  }
  return m;
}
inline ConvMatrix conv_forward_sub(const ConvMatrix& l, ConvMatrix y) {  // :122-146 solves L x = y
  for (size_t k = 0; k < y.w; k++)
    for (size_t j = 0; j < l.h; j++) {
      const double diag_value = y.at(j, k) / l.at(j, j);
      y.at(j, k) = diag_value;
      for (size_t i = j + 1; i < l.h; i++) y.at(i, k) = y.at(i, k) - diag_value * l.at(i, j);
    }
  return y;
}
inline ConvMatrix conv_transposed_backward_sub(const ConvMatrix& l, ConvMatrix y) {  // :96-119 solves L^T x = y
  for (size_t k = 0; k < y.w; k++)
    for (size_t j = l.h; j-- > 0;) {
      const double diag_value = y.at(j, k) / l.at(j, j);
      y.at(j, k) = diag_value;
      for (size_t i = 0; i < j; i++) y.at(i, k) = y.at(i, k) - diag_value * l.at(j, i);
    }
  return y;
}
constexpr size_t CONV1_ENCODE_BATCH_SIZE = 512;  // :11
// Test knob: pco 1.0.0 (which wrote pco/assets/v1_0_0_conv1.pco) fitted without the L2 term and kept one more bit of quantization
// than 1.0.3 does; with this set the asset re-encodes byte for byte, which pins everything else in the conv1 path and the planner.
inline bool& conv1_v1_0_0_parameters() { static bool on = false; return on; }
inline std::vector<double> conv_initial_autocov_dots(const std::vector<double>& v, size_t order) {  // :256-287
  const size_t n = v.size();
  std::vector<double> dots(order + 1, 0.0);
  const size_t almost_n = (n - order) / CONV1_ENCODE_BATCH_SIZE * CONV1_ENCODE_BATCH_SIZE;
  for (size_t start = 0; start < almost_n; start += CONV1_ENCODE_BATCH_SIZE)
    for (size_t sep = 0; sep <= order; sep++) {
      double dot0 = 0.0, dot1 = 0.0, dot2 = 0.0, dot3 = 0.0;
      for (size_t i = start; i < start + CONV1_ENCODE_BATCH_SIZE; i += 4) {
        dot0 += v[i] * v[i + sep];
        dot1 += v[i + 1] * v[i + sep + 1];
        dot2 += v[i + 2] * v[i + sep + 2];
        dot3 += v[i + 3] * v[i + sep + 3];
      }
      dots[sep] += (dot0 + dot1) + (dot2 + dot3);
    }
  for (size_t i = almost_n; i < n - order; i++)
    for (size_t sep = 0; sep <= order; sep++) dots[sep] += v[i] * v[i + sep];
  return dots;
}
inline void conv_autocov_mats(const std::vector<double>& v, size_t order, double regularization, ConvMatrix* xtx_out, ConvMatrix* xty_out) {  // :290-346
  const size_t n = v.size();
  double initial_sum = 0.0;
  for (size_t i = 0; i < n - order; i++) initial_sum += v[i];
  const std::vector<double> initial_dots = conv_initial_autocov_dots(v, order);
  ConvMatrix xtx(0.0, order + 1, order + 1), xty(0.0, order + 1, 1);
  for (size_t i = 0; i < order; i++) {
    xtx.at(i, 0) = initial_dots[i];
    xtx.at(0, i) = initial_dots[i];
  }
  xtx.at(order, 0) = initial_sum;
  xtx.at(0, order) = initial_sum;
  xty.at(0, 0) = initial_dots[order];
  for (size_t i = 1; i < order; i++) {
    for (size_t j = 1; j <= i; j++) {
      const double dot = xtx.at(i - 1, j - 1) + (v[n - order + i - 1] * v[n - order + j - 1] - v[i - 1] * v[j - 1]);
      xtx.at(i, j) = dot;
      xtx.at(j, i) = dot;
    }
    const double sum = xtx.at(order, i - 1) + (v[n - order + i - 1] - v[i - 1]);
    xtx.at(order, i) = sum;
    xtx.at(i, order) = sum;
  }
  for (size_t i = 1; i < order; i++) xty.at(i, 0) = xtx.at(order - 1, i - 1) + (v[n - order + i - 1] * v[n - 1] - v[i - 1] * v[order - 1]);
  xtx.at(order, order) = double(n - order);
  xty.at(order, 0) = xtx.at(order, order - 1) + (v[n - 1] - v[order - 1]);
  for (size_t i = 0; i <= order; i++) xtx.at(i, i) = xtx.at(i, i) + regularization;
  *xtx_out = std::move(xtx);
  *xty_out = std::move(xty);
}
inline std::vector<double> conv_autocorr_least_squares(const std::vector<double>& v, size_t order) {  // :348-361
  ConvMatrix xtx(0.0, 0, 0), xty(0.0, 0, 0);
  conv_autocov_mats(v, order, conv1_v1_0_0_parameters() ? 0.0 : 0.1, &xtx, &xty);  // L2_REGULARIZATION
  const ConvMatrix chol = conv_cholesky(std::move(xtx));
  return conv_transposed_backward_sub(chol, conv_forward_sub(chol, std::move(xty))).data;
}
inline int64_t f64_as_i64(double x) {  // Rust `as i64`: saturating, NaN -> 0
  if (std::isnan(x)) return 0;
  if (x >= 9223372036854775808.0) return std::numeric_limits<int64_t>::max();
  if (x <= -9223372036854775808.0) return std::numeric_limits<int64_t>::min();
  return int64_t(x);
}
// conv1.rs:363-421 choose_config; false = None (the caller falls back to NoOp, chunk_compressor.rs:387-391)
template <typename L>
inline bool conv1_choose_config(size_t order, const L* latents, size_t n, DeltaEncoding* out) {
  using S = typename ConvType<L>::S;
  if (n < order + 1) return false;
  const L center = choose_pivot<L>(latents, n);
  std::vector<double> v(n);
  for (size_t i = 0; i < n; i++) v[i] = latents[i] < center ? -double(uint64_t(L(center - latents[i]))) : double(uint64_t(L(latents[i] - center)));
  const std::vector<double> beta = conv_autocorr_least_squares(v, order);
  double total_weight = 0.0, total_abs_weight = 0.0;
  for (size_t i = 0; i < order; i++) {
    total_abs_weight += std::fabs(beta[i]);
    total_weight += beta[i];
  }
  if (!std::isfinite(total_weight) || !std::isfinite(total_abs_weight)) return false;
  const double float_bias = ((1.0 - total_weight) * double(uint64_t(center))) + beta[order];
  const double conv_max = double(std::numeric_limits<S>::max()), l_max = double(uint64_t(std::numeric_limits<L>::max()));
  const double lg = std::floor(std::log2(conv_max / (total_abs_weight * l_max + std::fabs(float_bias) + 1.0)));
  int64_t q64 = std::isnan(lg) ? 0 : (lg >= 2147483647.0 ? 2147483647 : (lg <= -2147483648.0 ? -2147483648ll : int64_t(lg)));  // `as i32`
  int32_t quantization = int32_t(std::max<int64_t>(q64 - (conv1_v1_0_0_parameters() ? 0 : 1), -2147483648ll));
  quantization = std::min<int32_t>(quantization, int32_t(MAX_CONV1_DELTA_QUANTIZATION));
  quantization = std::min<int32_t>(quantization, int32_t(8 * sizeof(S)) - 1);
  if (quantization < 0) return false;
  const double quantize_factor = std::ldexp(1.0, quantization);
  DeltaEncoding d;
  d.kind = DeltaKind::Conv1;
  d.quantization = Bitlen(quantization);
  for (size_t i = 0; i < order; i++) d.weights.push_back(f64_as_i64(std::round(beta[i] * quantize_factor)));
  d.bias = f64_as_i64(float_bias * quantize_factor);
  *out = d;
  return true;
}
// conv1.rs:423-461 encode_in_place: residual_i = latent_i - predict(latent_{i-order..i}) + MID from the ORIGINAL latents; the first
// `order` entries become junk (latent + MID, the reference's zero-initialised predictions) and are not stored
template <typename L>
inline std::vector<L> conv1_encode_in_place(const DeltaEncoding& cfg, L* latents, size_t len) {
  using S = typename ConvType<L>::S;
  using US = typename std::make_unsigned<S>::type;
  const size_t order = cfg.weights.size();
  std::vector<L> initial_state(latents, latents + std::min(order, len));
  std::vector<L> original(latents, latents + len);
  const S bias = S(cfg.bias);
  for (size_t i = 0; i < len; i++) {
    L prediction = 0;
    if (i >= order) {
      US s = US(bias);
      for (size_t j = 0; j < order; j++) s = US(s + US(US(S(cfg.weights[j])) * US(S(original[i - order + j]))));
      S ss = S(s);
      if (ss < 0) ss = 0;
      prediction = L(ss >> cfg.quantization);
    }
    latents[i] = L(L(original[i] - prediction) + LatentTraits<L>::MID);
  }
  return initial_state;
}

// ===========================================================================
// Per-latent-var decompression
// (pco/src/chunk_latent_decompressor.rs, page_latent_decompressor.rs)
// ===========================================================================
struct VarDecoderBase {
  virtual ~VarDecoderBase() {}
  virtual void init_page(const PageVarMeta& pv) = 0;
  virtual void read_batch_pre_delta(BitReader& r, size_t batch_n) = 0;
  virtual void read_batch(BitReader& r, const uint32_t* delta_latents, size_t n_remaining_in_page) = 0;
  virtual const void* latents() const = 0;
  size_t n_bins = 0;
};

template <typename L>
struct VarDecoder : VarDecoderBase {
  LatentVarDelta delta;
  Bitlen max_offset_bits = 0;
  std::vector<L> state_lowers;
  std::vector<AnsNode> nodes;
  alignas(64) uint32_t offset_bits_csum[FULL_BATCH_N];
  alignas(64) uint32_t offset_bits[FULL_BATCH_N];
  alignas(64) L lat[FULL_BATCH_N];
  // page state (page_latent_decompressor.rs:65-87)
  AnsState ans_state_idxs[ANS_INTERLEAVING];
  std::vector<L> delta_state;
  size_t delta_state_pos = 0;

  // chunk_latent_decompressor.rs:30-75
  VarDecoder(const LatentVarMeta& vm, LatentVarDelta d) : delta(d) {
    n_bins = vm.bins.size();
    max_offset_bits = vm.max_offset_bits();
    std::vector<Weight> weights;
    std::vector<Bitlen> bin_offset_bits;
    for (const Bin& b : vm.bins) { weights.push_back(b.weight); bin_offset_bits.push_back(b.offset_bits); }
    AnsSpec spec = ans_spec_from_weights(vm.ans_size_log, weights);
    state_lowers.reserve(spec.state_symbols.size());
    for (Symbol s : spec.state_symbols) state_lowers.push_back(s < vm.bins.size() ? L(vm.bins[s].lower) : L(0));
    nodes = ans_decoder_nodes(spec, bin_offset_bits);
    for (size_t i = 0; i < FULL_BATCH_N; i++) { offset_bits_csum[i] = 0; offset_bits[i] = 0; lat[i] = 0; }
    if (vm.bins.size() == 1) {
      uint32_t csum = 0;
      for (size_t i = 0; i < FULL_BATCH_N; i++) {
        offset_bits[i] = vm.bins[0].offset_bits;
        offset_bits_csum[i] = csum;
        lat[i] = L(vm.bins[0].lower);
        csum += vm.bins[0].offset_bits;
      }
    }
  }

  // page_latent_decompressor.rs:72-87 + delta/mod.rs:86-99, lookback.rs:189-199
  void init_page(const PageVarMeta& pv) override {
    for (size_t j = 0; j < ANS_INTERLEAVING; j++) ans_state_idxs[j] = pv.ans_final_state_idxs[j];
    std::vector<L> stored(pv.delta_state.size());
    for (size_t i = 0; i < stored.size(); i++) stored[i] = L(pv.delta_state[i]);
    if (delta.kind == DeltaKind::Lookback) {
      size_t window_n = size_t(1) << delta.enc->window_n_log;
      size_t buffer_n = std::max(window_n, FULL_BATCH_N) * 2;
      delta_state.assign(buffer_n, 0);
      for (size_t i = 0; i < stored.size(); i++) delta_state[window_n - stored.size() + i] = stored[i];
      delta_state_pos = window_n;
    } else {
      delta_state = std::move(stored);
      delta_state_pos = 0;
    }
  }

  // page_latent_decompressor.rs:89-177 (one loop covers the full and partial batch variants)
  inline void read_ans_symbols(BitReader& r, size_t batch_n) {
    size_t bit = r.bit_idx;
    uint32_t offset_bit_idx = 0;
    AnsState st[ANS_INTERLEAVING] = {ans_state_idxs[0], ans_state_idxs[1], ans_state_idxs[2], ans_state_idxs[3]};
    const AnsNode* nd = nodes.data();
    const L* lowers = state_lowers.data();
    for (size_t i = 0; i < batch_n; i++) {
      size_t j = i % ANS_INTERLEAVING;
      AnsState s = st[j];
      uint64_t packed = r.u64_at(bit / 8);
      AnsNode node = nd[s];
      Bitlen btr = node.bits_to_read;
      AnsState ans_val = AnsState(packed >> (bit % 8)) & ((AnsState(1) << btr) - 1);
      offset_bits_csum[i] = offset_bit_idx;
      offset_bits[i] = node.offset_bits;
      lat[i] = lowers[s];
      bit += btr;
      offset_bit_idx += node.offset_bits;
      st[j] = AnsState(node.next_state_idx_base) + ans_val;
    }
    r.bit_idx = bit;
    for (size_t j = 0; j < ANS_INTERLEAVING; j++) ans_state_idxs[j] = st[j];
  }

  // page_latent_decompressor.rs:15-44
  inline void read_offsets(BitReader& r, size_t n) {
    size_t base = r.bit_idx;
    for (size_t i = 0; i < n; i++) {
      Bitlen ob = offset_bits[i];
      size_t bit = base + offset_bits_csum[i];
      size_t byte = bit / 8;
      Bitlen bpb = Bitlen(bit % 8);
      uint64_t w = r.u64_at(byte) >> bpb;
      if (sizeof(L) == 8 && bpb + ob > 64) w |= r.u64_at(byte + 8) << (64 - bpb);
      lat[i] = L(lat[i] + L(lowest_bits_u64(w, ob)));
    }
    r.bit_idx = base + offset_bits_csum[n - 1] + offset_bits[n - 1];
  }

  // page_latent_decompressor.rs:181-235
  void read_batch_pre_delta(BitReader& r, size_t batch_n) override {
    if (batch_n == 0) return;
    if (n_bins > 1) read_ans_symbols(r, batch_n);
    else for (size_t i = 0; i < batch_n; i++) lat[i] = state_lowers[0];
    if (max_offset_bits > 0) read_offsets(r, batch_n);
  }

  // page_latent_decompressor.rs:237-257 + delta/mod.rs:125-159
  void read_batch(BitReader& r, const uint32_t* delta_latents, size_t n_remaining_in_page) override {
    size_t n_state = delta.n_latents_per_state();
    size_t n_remaining_pre_delta = n_remaining_in_page > n_state ? n_remaining_in_page - n_state : 0;
    size_t pre_delta_len = std::min(FULL_BATCH_N, n_remaining_pre_delta);
    read_batch_pre_delta(r, pre_delta_len);
    size_t dst_len = std::min(n_remaining_in_page, FULL_BATCH_N);
    switch (delta.kind) {
      case DeltaKind::NoOp: break;
      case DeltaKind::Consecutive: consecutive_decode_in_place(delta_state, lat, dst_len); break;
      case DeltaKind::Conv1: conv1_decode_in_place(*delta.enc, delta_state, lat, dst_len); break;
      case DeltaKind::Lookback: {
        // delta/lookback.rs:201-246
        toggle_center_in_place(lat, dst_len);
        size_t window_n = size_t(1) << delta.enc->window_n_log, state_n = size_t(1) << delta.enc->state_n_log;
        size_t start_pos = delta_state_pos;
        if (start_pos + dst_len > delta_state.size()) {
          std::memmove(delta_state.data(), delta_state.data() + (start_pos - window_n), window_n * sizeof(L));
          start_pos = window_n;
        }
        bool oob = false;
        // zip(latents, lookbacks): lookbacks hold pre_delta_len valid entries; the
        // reference zips against the delta var's 256-entry scratch, so stale
        // entries beyond pre_delta_len are consumed too.
        for (size_t i = 0; i < dst_len; i++) {
          size_t pos = start_pos + i;
          uint32_t lb = delta_latents[i];
          size_t lookback;
          if (lb <= uint32_t(window_n)) lookback = lb; else { oob = true; lookback = 1; }
          delta_state[pos] = L(lat[i] + delta_state[pos - lookback]);
        }
        size_t end_pos = start_pos + dst_len;
        for (size_t i = 0; i < dst_len; i++) lat[i] = delta_state[start_pos - state_n + i];
        delta_state_pos = end_pos;
        if (oob) corruption("delta lookback exceeded window n");
        break;
      }
    }
  }
  const void* latents() const override { return lat; }
};

inline std::unique_ptr<VarDecoderBase> make_var_decoder(const LatentVarMeta& vm, LatentVarDelta d) {
  switch (vm.latent_bits) {
    case 8: return std::unique_ptr<VarDecoderBase>(new VarDecoder<uint8_t>(vm, d));
    case 16: return std::unique_ptr<VarDecoderBase>(new VarDecoder<uint16_t>(vm, d));
    case 32: return std::unique_ptr<VarDecoderBase>(new VarDecoder<uint32_t>(vm, d));
    default: return std::unique_ptr<VarDecoderBase>(new VarDecoder<uint64_t>(vm, d));
  }
}

// ===========================================================================
// Mode split / join (pco/src/mode/*.rs)
// ===========================================================================
template <typename L>
inline void join_latents(const ChunkMeta& cm, uint8_t number_type, const void* primary_v, const void* secondary_v, L* dst, size_t n) {
  bool isf = number_type_is_float(number_type), iss = number_type_is_signed(number_type);
  const Mode& mode = cm.mode;
  switch (mode.kind) {
    case ModeKind::Classic: {  // mode/classic.rs:14-24
      const L* p = static_cast<const L*>(primary_v);
      for (size_t i = 0; i < n; i++) dst[i] = from_latent_ordered_bits<L>(p[i], isf, iss);
      break;
    }
    case ModeKind::Dict: {  // mode/dict.rs:70-90
      const uint32_t* idxs = static_cast<const uint32_t*>(primary_v);
      for (size_t i = 0; i < n; i++)
        if (idxs[i] >= uint32_t(mode.dict.size())) corruption("dict index exceeded dict length " + std::to_string(mode.dict.size()));
      for (size_t i = 0; i < n; i++) dst[i] = from_latent_ordered_bits<L>(L(mode.dict[idxs[i]]), isf, iss);
      break;
    }
    case ModeKind::IntMult: {  // mode/int_mult.rs:38-54
      const L* p = static_cast<const L*>(primary_v);
      const L* s = static_cast<const L*>(secondary_v);
      L base = L(mode.base_latent);
      for (size_t i = 0; i < n; i++) dst[i] = from_latent_ordered_bits<L>(L(L(p[i] * base) + s[i]), isf, iss);
      break;
    }
    case ModeKind::FloatMult: {  // mode/float_mult.rs:17-36
      if constexpr (sizeof(L) >= 2) {
        using FO = FloatOps<L>;
        const L* p = static_cast<const L*>(primary_v);
        const L* s = static_cast<const L*>(secondary_v);
        auto base = FO::from_bits(from_latent_ordered_bits<L>(L(mode.base_latent), true, false));
        for (size_t i = 0; i < n; i++) {
          auto unadjusted = FO::mul(int_float_from_latent<L>(p[i]), base);
          L u = to_latent_ordered_bits<L>(FO::to_bits(unadjusted), true, false);
          dst[i] = from_latent_ordered_bits<L>(L(L(u + s[i]) + LatentTraits<L>::MID), true, false);
        }
      }
      break;
    }
    case ModeKind::FloatQuant: {  // mode/float_quant.rs:13-39
      const L* p = static_cast<const L*>(primary_v);
      const L* s = static_cast<const L*>(secondary_v);
      Bitlen k = mode.k;
      L sign_cutoff = L(LatentTraits<L>::MID >> k);
      L lowest_k_bits_max = L(L(L(1) << k) - 1);
      for (size_t i = 0; i < n; i++) {
        bool pos = p[i] >= sign_cutoff;
        L lowest = pos ? s[i] : L(lowest_k_bits_max - s[i]);
        dst[i] = from_latent_ordered_bits<L>(L(L(p[i] << k) + lowest), true, false);
      }
      break;
    }
  }
}

// ===========================================================================
// Page decompression (pco/src/wrapped/page_decompressor.rs)
// ===========================================================================
struct ChunkDecoder {
  ChunkMeta meta;
  uint8_t number_type;
  std::unique_ptr<VarDecoderBase> delta_var, primary, secondary;

  // wrapped/chunk_decompressor.rs:17-72
  ChunkDecoder(ChunkMeta m, uint8_t nt) : meta(std::move(m)), number_type(nt) {
    if (!mode_is_valid(meta.mode, nt)) corruption("invalid mode for number type");
    if (meta.has_delta_var) delta_var = make_var_decoder(meta.delta_var, delta_for_latent_var(meta.delta, VarKey::Delta));
    primary = make_var_decoder(meta.primary, delta_for_latent_var(meta.delta, VarKey::Primary));
    if (meta.has_secondary) secondary = make_var_decoder(meta.secondary, delta_for_latent_var(meta.delta, VarKey::Secondary));
  }
  size_t n_latents_per_delta_state() const { return delta_for_latent_var(meta.delta, VarKey::Primary).n_latents_per_state(); }
};

struct Progress {
  size_t n_processed = 0;
  bool finished = false;
};

// State of one page being decoded: PageDecompressorState (page_decompressor.rs:22-221)
template <typename L>
struct PageDecoder {
  ChunkDecoder& cd;
  BitReader& r;
  size_t n_remaining;

  PageDecoder(ChunkDecoder& cd_, BitReader& r_, size_t n) : cd(cd_), r(r_), n_remaining(n) {
    PageMeta pm = read_page_meta(r, cd.meta);
    r.check_in_bounds();
    size_t n_state = cd.n_latents_per_delta_state();
    size_t n_in_body = n > n_state ? n - n_state : 0;
    auto init = [&](VarDecoderBase* vd, const PageVarMeta& pv) {
      if (vd->n_bins == 0 && n_in_body > 0)
        corruption("unable to decompress chunk with no bins and " + std::to_string(n_in_body) + " latents");
      vd->init_page(pv);
    };
    if (cd.delta_var) init(cd.delta_var.get(), pm.delta_var);
    init(cd.primary.get(), pm.primary);
    if (cd.secondary) init(cd.secondary.get(), pm.secondary);
  }

  // page_decompressor.rs:115-191
  void read_batch(L* dst, size_t batch_n) {
    const uint32_t* delta_latents = nullptr;
    if (cd.delta_var) {
      size_t n_state = cd.n_latents_per_delta_state();
      size_t limit = std::min(n_remaining > n_state ? n_remaining - n_state : 0, batch_n);
      cd.delta_var->read_batch_pre_delta(r, limit);
      r.check_in_bounds();
      delta_latents = static_cast<const uint32_t*>(cd.delta_var->latents());
    }
    cd.primary->read_batch(r, delta_latents, n_remaining);
    r.check_in_bounds();
    const void* sec = nullptr;
    if (cd.secondary) {
      cd.secondary->read_batch(r, delta_latents, n_remaining);
      r.check_in_bounds();
      sec = cd.secondary->latents();
    }
    join_latents<L>(cd.meta, cd.number_type, cd.primary->latents(), sec, dst, batch_n);
    n_remaining -= batch_n;
    if (n_remaining == 0) r.drain_empty_byte("expected trailing bits at end of page to be empty");
  }

  // page_decompressor.rs:193-221
  Progress read(L* dst, size_t dst_len) {
    if (dst_len % FULL_BATCH_N != 0 && dst_len < n_remaining)
      invalid_argument("num_dst's length must either be a multiple of 256 or be at least the count of numbers remaining");
    size_t n_to_process = std::min(dst_len, n_remaining);
    size_t n_processed = 0;
    while (n_processed < n_to_process) {
      size_t end = std::min(n_processed + FULL_BATCH_N, n_to_process);
      read_batch(dst + n_processed, end - n_processed);
      n_processed = end;
    }
    Progress p;
    p.n_processed = n_processed;
    p.finished = n_remaining == 0;
    return p;
  }
};

// ===========================================================================
// Per-latent-var compression
// (pco/src/compression_table.rs, chunk_latent_compressor.rs)
// ===========================================================================
template <typename L>
struct PageDissectedVar {
  std::vector<AnsState> ans_vals;
  std::vector<Bitlen> ans_bits;
  std::vector<L> offsets;
  std::vector<Bitlen> offset_bits;
  AnsState ans_final_states[ANS_INTERLEAVING];
};

template <typename L>
struct VarCompressor {
  // compression_table.rs:9-33
  size_t search_size_log = 0;
  std::vector<L> search_lowers;
  std::vector<BinCompressionInfo<L>> infos;  // sorted by lower
  AnsEncoder encoder;
  double avg_bits_per_latent = 0.0;
  bool is_trivial = false, needs_ans = false;
  Bitlen max_bits_per_offset = 0;
  std::vector<L> latents;
  alignas(64) L scratch_lowers[FULL_BATCH_N];
  alignas(64) Symbol scratch_symbols[FULL_BATCH_N];

  // chunk_latent_compressor.rs:135-161
  VarCompressor(const TrainedBins<L>& trained, const LatentVarMeta& vm, std::vector<L> lat) : latents(std::move(lat)) {
    needs_ans = vm.bins.size() != 1;
    infos = trained.infos;
    search_size_log = infos.size() <= 1 ? 0 : 1 + ilog2_u64(infos.size() - 1);
    // sort_unstable_by_key(lower): lowers are distinct for trained bins
    std::sort(infos.begin(), infos.end(), [](const BinCompressionInfo<L>& a, const BinCompressionInfo<L>& b) { return a.lower < b.lower; });
    for (auto& i : infos) search_lowers.push_back(i.lower);
    while (search_lowers.size() < (size_t(1) << search_size_log)) search_lowers.push_back(LatentTraits<L>::MAX);
    std::vector<Weight> weights;
    for (const Bin& b : vm.bins) weights.push_back(b.weight);
    AnsSpec spec = ans_spec_from_weights(trained.ans_size_log, weights);
    encoder = AnsEncoder(spec);
    max_bits_per_offset = vm.max_offset_bits();
    // metadata/bins.rs:23-32
    double total_weight = double(uint64_t(1) << trained.ans_size_log);
    double acc = 0.0;
    for (const Bin& b : vm.bins) {
      double ans_bits = double(trained.ans_size_log) - std::log2(double(b.weight));
      acc += (ans_bits + double(b.offset_bits)) * double(b.weight) / total_weight;
    }
    avg_bits_per_latent = acc;
    is_trivial = vm.are_trivial();
    L default_lower = infos.size() == 1 ? infos[0].lower : L(0);
    for (size_t i = 0; i < FULL_BATCH_N; i++) { scratch_lowers[i] = default_lower; scratch_symbols[i] = 0; }
  }

  // chunk_latent_compressor.rs:194-233 (binary_search compression_table.rs:51-74, dissect_bins :163-182,
  // set_offsets :185-192, encode_ans_in_reverse :96-132)
  void dissect_batch(size_t page_start, size_t rel_start, size_t rel_end, PageDissectedVar<L>& dst) {
    size_t batch_n = rel_end - rel_start;
    const L* lat = latents.data() + page_start + rel_start;
    size_t search_idxs[FULL_BATCH_N];
    for (size_t i = 0; i < batch_n; i++) search_idxs[i] = 0;
    for (size_t depth = 0; depth < search_size_log; depth++) {
      size_t bisection = size_t(1) << (search_size_log - 1 - depth);
      for (size_t i = 0; i < batch_n; i++) {
        size_t cand = search_idxs[i] + bisection;
        search_idxs[i] += (lat[i] >= search_lowers[cand]) ? bisection : 0;
      }
    }
    size_t n_bins = infos.size();
    if (n_bins < (size_t(1) << search_size_log))
      for (size_t i = 0; i < batch_n; i++) search_idxs[i] = std::min(search_idxs[i], n_bins - 1);
    Bitlen* ob = dst.offset_bits.data() + rel_start;
    if (infos.size() <= 1) {
      Bitlen d = infos.size() == 1 ? infos[0].offset_bits : 0;
      for (size_t i = 0; i < batch_n; i++) ob[i] = d;
    } else {
      for (size_t i = 0; i < batch_n; i++) {
        const auto& info = infos[search_idxs[i]];
        scratch_lowers[i] = info.lower;
        scratch_symbols[i] = info.symbol;
        ob[i] = info.offset_bits;
      }
    }
    L* offs = dst.offsets.data() + rel_start;
    for (size_t i = 0; i < batch_n; i++) offs[i] = L(lat[i] - scratch_lowers[i]);
    // reverse tANS
    AnsState* ans_vals = dst.ans_vals.data() + rel_start;
    Bitlen* ans_bits = dst.ans_bits.data() + rel_start;
    if (encoder.size_log == 0) {
      for (size_t i = 0; i < batch_n; i++) ans_bits[i] = 0;
      return;
    }
    for (size_t i = batch_n; i-- > 0;) {
      size_t j = i % ANS_INTERLEAVING;
      Bitlen bitlen;
      AnsState st = dst.ans_final_states[j];
      AnsState ns = encoder.encode(st, scratch_symbols[i], &bitlen);
      ans_vals[i] = AnsState(lowest_bits_u64(st, bitlen));
      ans_bits[i] = bitlen;
      dst.ans_final_states[j] = ns;
    }
  }

  // chunk_latent_compressor.rs:246-270
  PageDissectedVar<L> dissect_page(size_t start, size_t end) {
    PageDissectedVar<L> d;
    for (size_t j = 0; j < ANS_INTERLEAVING; j++) d.ans_final_states[j] = encoder.default_state();
    if (is_trivial) return d;
    size_t page_n = end - start;
    d.ans_vals.resize(page_n);
    d.ans_bits.resize(page_n);
    d.offsets.resize(page_n);
    d.offset_bits.resize(page_n);
    size_t n_batches = (page_n + FULL_BATCH_N - 1) / FULL_BATCH_N;
    for (size_t b = n_batches; b-- > 0;) dissect_batch(start, b * FULL_BATCH_N, std::min((b + 1) * FULL_BATCH_N, page_n), d);
    return d;
  }

  // chunk_latent_compressor.rs:272-329
  void write_dissected_batch(const PageDissectedVar<L>& d, size_t batch_start, BitWriter& w) const {
    if (batch_start >= d.offsets.size()) return;
    size_t end = std::min(batch_start + FULL_BATCH_N, d.offsets.size());
    if (needs_ans)
      for (size_t i = batch_start; i < end; i++) w.write_uint(d.ans_vals[i], d.ans_bits[i]);
    if (max_bits_per_offset > 0)
      for (size_t i = batch_start; i < end; i++) w.write_uint(uint64_t(d.offsets[i]), d.offset_bits[i]);
  }
};

// ===========================================================================
// Chunk compressor (pco/src/wrapped/chunk_compressor.rs)
// ===========================================================================
struct VarCompressorBase {
  virtual ~VarCompressorBase() {}
};

template <typename L>
struct PageInfoVar {
  std::vector<uint64_t> delta_state;
  size_t start = 0, end = 0;  // stored range in the var's latent array
};

// (worst_case_size, baseline) in bytes of each should_fallback decision of this thread's last compress, one per chunk in chunk
// order.  Every compress clears it first: simple_compress (the standalone file of every caller, dictionary chunks included, and
// each chunk of pco_oracle_bench_roundtrip) and pco_oracle_chunk_compressor_new (one wrapped chunk), so it never holds more than
// one call's chunks.  Test infrastructure: the tests build chunks a byte either side of the size guarantee and check how far off
// they are.
inline std::vector<std::pair<uint64_t, uint64_t>>& fallback_margins() {
  static thread_local std::vector<std::pair<uint64_t, uint64_t>> margins;
  return margins;
}

template <typename L>  // L = number's latent type
struct ChunkCompressor {
  ChunkMeta meta;
  uint8_t number_type;
  std::vector<size_t> page_ns;
  // per page, per var
  std::vector<PageInfoVar<L>> pi_delta, pi_primary, pi_secondary;
  std::unique_ptr<VarCompressor<uint32_t>> vc_delta;
  std::unique_ptr<VarCompressor<L>> vc_primary, vc_secondary;
  std::vector<Weight> counts_delta, counts_primary, counts_secondary;

  size_t n_pages() const { return page_ns.size(); }

  // chunk_compressor.rs:502-541
  bool should_fallback(size_t n) const {
    size_t worst_case_body_bit_size = 7 * n_pages();
    auto add = [&](const LatentVarMeta& vm, const std::vector<Weight>& counts) {
      for (size_t i = 0; i < vm.bins.size() && i < counts.size(); i++) {
        const Bin& b = vm.bins[i];
        Bitlen wc = b.offset_bits + vm.ans_size_log - ilog2_u64(b.weight);
        worst_case_body_bit_size += size_t(counts[i]) * size_t(wc);
      }
    };
    if (meta.has_delta_var) add(meta.delta_var, counts_delta);
    add(meta.primary, counts_primary);
    if (meta.has_secondary) add(meta.secondary, counts_secondary);
    size_t worst_case_size = meta.max_size() + n_pages() * meta.exact_page_meta_size() + (worst_case_body_bit_size + 7) / 8;
    // wrapped/guarantee.rs:11-37
    ChunkMeta base;
    base.number_bits = meta.number_bits;
    base.primary.latent_bits = meta.number_bits;
    base.primary.ans_size_log = 0;
    base.primary.bins = {Bin{1, 0, meta.number_bits}};
    size_t baseline = base.max_size() + (n * size_t(meta.number_bits) + 7) / 8;
    fallback_margins().emplace_back(uint64_t(worst_case_size), uint64_t(baseline));
    if (meta.delta.kind == DeltaKind::NoOp && meta.mode.kind == ModeKind::Classic) return false;  // already the fallback's layout
    return worst_case_size > baseline;
  }

  // chunk_compressor.rs:575-603 (page_size_hint_inner)
  size_t page_size_hint_inner(size_t page_idx, double overestimation) const {
    size_t body_bit_size = 0;
    auto add = [&](double avg_bits, size_t n_stored) {
      double nums_bit_size = double(n_stored) * avg_bits;
      body_bit_size += size_t(std::ceil(nums_bit_size * overestimation));
    };
    if (vc_delta) add(vc_delta->avg_bits_per_latent, pi_delta[page_idx].end - pi_delta[page_idx].start);
    add(vc_primary->avg_bits_per_latent, pi_primary[page_idx].end - pi_primary[page_idx].start);
    if (vc_secondary) add(vc_secondary->avg_bits_per_latent, pi_secondary[page_idx].end - pi_secondary[page_idx].start);
    return meta.exact_page_meta_size() + (body_bit_size + 7) / 8;
  }
  size_t meta_size_hint() const { return meta.max_size(); }
  size_t page_size_hint(size_t page_idx) const { return page_size_hint_inner(page_idx, 1.2); }

  void write_meta(std::vector<uint8_t>& dst) const { write_chunk_meta(meta, dst); }

  // chunk_compressor.rs:624-705
  void write_page(size_t page_idx, std::vector<uint8_t>& dst) {
    if (page_idx >= n_pages()) invalid_argument("page idx exceeds num pages");
    PageDissectedVar<uint32_t> dd;
    PageDissectedVar<L> dp, ds;
    if (vc_delta) dd = vc_delta->dissect_page(pi_delta[page_idx].start, pi_delta[page_idx].end);
    dp = vc_primary->dissect_page(pi_primary[page_idx].start, pi_primary[page_idx].end);
    if (vc_secondary) ds = vc_secondary->dissect_page(pi_secondary[page_idx].start, pi_secondary[page_idx].end);
    PageMeta pm;
    auto fill = [&](PageVarMeta& pv, const std::vector<uint64_t>& state, const AnsState* finals, AnsState default_state) {
      pv.delta_state = state;
      for (size_t j = 0; j < ANS_INTERLEAVING; j++) pv.ans_final_state_idxs[j] = finals[j] - default_state;
    };
    if (vc_delta) fill(pm.delta_var, pi_delta[page_idx].delta_state, dd.ans_final_states, vc_delta->encoder.default_state());
    fill(pm.primary, pi_primary[page_idx].delta_state, dp.ans_final_states, vc_primary->encoder.default_state());
    if (vc_secondary) fill(pm.secondary, pi_secondary[page_idx].delta_state, ds.ans_final_states, vc_secondary->encoder.default_state());
    BitWriter w(dst);
    write_page_meta(meta, pm, w);
    size_t page_n = page_ns[page_idx];
    for (size_t batch_start = 0; batch_start < page_n; batch_start += FULL_BATCH_N) {
      if (vc_delta) vc_delta->write_dissected_batch(dd, batch_start, w);
      vc_primary->write_dissected_batch(dp, batch_start, w);
      if (vc_secondary) vc_secondary->write_dissected_batch(ds, batch_start, w);
    }
    w.finish();
  }
};

// ----- sampling for Auto delta (pco/src/sampling.rs:9-60) -------------------
inline bool calc_sample_n(size_t n, size_t* out) {
  if (n >= 10) { *out = 10 + (n - 10) / 40; return true; }
  return false;
}
template <typename L>
inline bool choose_delta_sample(const std::vector<L>& primary, std::vector<L>* sample) {
  size_t n = primary.size();
  size_t target;
  if (!calc_sample_n(n, &target)) return false;
  size_t group_n = std::min<size_t>(200, n);
  size_t n_groups = (target + 199) / 200;
  size_t nominal = n_groups * group_n;
  size_t stride = group_n + ((n > nominal ? n - nominal : 0) / (std::max<size_t>(n_groups, 2) - 1));
  sample->clear();
  sample->reserve(nominal);
  for (size_t i = 0; i < n_groups; i++) {
    size_t gs = stride * i;
    sample->insert(sample->end(), primary.begin() + gs, primary.begin() + gs + group_n);
  }
  return true;
}

// ----- sampling for the Auto MODE search (pco/src/sampling.rs:62-103) ---------------------------------------------
// rand_xoshiro 0.6.0 Xoroshiro128PlusPlus::seed_from_u64 (Cargo.lock:2682-2685): the two state words are the first two
// outputs of SplitMix64 started at the seed.  Not in /root/reference (a crates.io dependency): restated from the published
// algorithm and pinned by the reference's own KAT (sampling.rs:186-201, tests/test_oracle_kats.py::test_choose_mode_sample).
struct Xoroshiro128PlusPlus {
  uint64_t s0, s1;
  static uint64_t rotl(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }
  explicit Xoroshiro128PlusPlus(uint64_t seed) {
    auto splitmix = [&seed]() {
      seed += 0x9e3779b97f4a7c15ull;
      uint64_t z = seed;
      z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
      z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
      return z ^ (z >> 31);
    };
    s0 = splitmix();
    s1 = splitmix();
  }
  uint64_t next_u64() {
    const uint64_t r = rotl(s0 + s1, 17) + s0;
    s1 ^= s0;
    s0 = rotl(s0, 49) ^ s1 ^ (s1 << 21);
    s1 = rotl(s1, 28);
    return r;
  }
};
// choose_mode_sample's index draw (Floyd's algorithm, sampling.rs:73-95): the indices it visits, in visiting order; the
// caller applies its filter to nums[idx].  Returns false when n < MIN_SAMPLE (the reference also returns None when fewer
// than MIN_SAMPLE numbers pass the filter - the caller's check).
inline bool choose_mode_sample_indices(size_t n, std::vector<size_t>* out) {
  size_t target;
  if (!calc_sample_n(n, &target)) return false;
  Xoroshiro128PlusPlus rng(0);
  std::vector<uint8_t> visited((n + 7) / 8, 0);
  out->clear();
  out->reserve(target);
  for (size_t j = n - target; j < n; j++) {
    const size_t t = size_t(rng.next_u64() % (uint64_t(j) + 1));
    const size_t idx = (visited[t / 8] >> (t % 8)) & 1 ? j : t;
    visited[idx / 8] |= uint8_t(1u << (idx % 8));
    out->push_back(idx);
  }
  return true;
}

// ----- ModeSpec::Auto for integer types: IntMult base detection (pco/src/mode/int_mult.rs:57-235) ---------------------
// data_types/unsigned.rs:28-35: Auto bids int mult alone when choose_base finds a base, else classic alone.
// Where the reference iterates a std HashMap (most_prominent_gcd :187-204, est_bits_saved_per_num sampling.rs:110-141) its
// order is per-process random: ties between equally scored gcds and the last ulp of the f64 sum are not defined by the
// reference itself.  This restatement visits keys in ascending order (ties -> the larger gcd, like max_by_key over an
// ascending iteration) - any result it gives is one the reference can give.
template <typename L>
inline L calc_gcd(L x, L y) {  // int_mult.rs:57-70
  if (x == 0) return y;
  for (;;) {
    if (y == 0) return x;
    x = L(x % y);
    std::swap(x, y);
  }
}

template <typename F>
inline bool solve_root_by_false_position(F f, double lb, double ub, double* root) {  // int_mult.rs:72-97
  const double X_TOLERANCE = 1E-4;
  double flb = f(lb), fub = f(ub);
  if (flb > 0.0 || fub < 0.0) return false;
  while (ub - lb > X_TOLERANCE && fub - flb > 0.0) {
    const double lb_prop = 0.001 + 0.998 * fub / (fub - flb);
    const double mid = lb_prop * lb + (1.0 - lb_prop) * ub;
    const double fmid = f(mid);
    if (fmid < 0.0) {
      lb = mid;
      flb = fmid;
    } else {
      ub = mid;
      fub = fmid;
    }
  }
  *root = (lb + ub) / 2.0;
  return true;
}

template <typename L>
inline L calc_triple_gcd(const L* triple) {  // int_mult.rs:99-115
  L a = triple[0], b = triple[1], c = triple[2];
  if (a > b) std::swap(a, b);
  if (b > c) std::swap(b, c);
  if (a > b) std::swap(a, b);
  return calc_gcd<L>(L(b - a), L(c - a));
}

inline double single_category_entropy(double p) { return (p == 0.0 || p == 1.0) ? 0.0 : -p * std::log2(p); }  // mode/mod.rs:7-13
inline double worst_case_categorical_entropy(double concentrated_p, double n_categories_m1) {                // mode/mod.rs:15-18
  return single_category_entropy(concentrated_p) + n_categories_m1 * single_category_entropy((1.0 - concentrated_p) / n_categories_m1);
}

const double MULT_REQUIRED_BITS_SAVED_PER_NUM = 0.5;  // constants.rs:48

inline bool filter_score_triple_gcd(double gcd, size_t triples_w_gcd_, size_t total_triples_, double* score) {  // int_mult.rs:117-185
  const double ZETA_OF_2 = 3.14159265358979323846264338327950288 * 3.14159265358979323846264338327950288 / 6.0;
  const double LCB_RATIO = 1.0;
  const double triples_w_gcd = double(triples_w_gcd_), total_triples = double(total_triples_);
  const double prob_per_triple = triples_w_gcd / total_triples;
  const double natural_prob_per_triple = 1.0 / (ZETA_OF_2 * gcd * gcd);
  const double stdev = std::sqrt(natural_prob_per_triple * (1.0 - natural_prob_per_triple) / total_triples);
  const double z_score = (prob_per_triple - natural_prob_per_triple) / stdev;
  if (z_score < 3.0) return false;
  const double triples_w_gcd_lcb = triples_w_gcd - LCB_RATIO * std::sqrt(triples_w_gcd);
  if (triples_w_gcd_lcb <= 0.0) return false;
  const double congruence_prob_per_triple_lcb = std::fmin(ZETA_OF_2 * triples_w_gcd_lcb / total_triples, 1.0);
  const double gcd_m1 = gcd - 1.0;
  const double gcd_m1_inv_sq = 1.0 / (gcd_m1 * gcd_m1);
  auto cube = [](double x) { return x * x * x; };  // powi(3)
  auto f = [&](double p) { return cube(p) + cube(1.0 - p) * gcd_m1_inv_sq - congruence_prob_per_triple_lcb; };
  const double lb = 1.0 / gcd;
  const double ub = std::cbrt(congruence_prob_per_triple_lcb) + 2.220446049250313e-16;  // f64::EPSILON
  double concentrated_p;
  if (!solve_root_by_false_position(f, lb, ub, &concentrated_p)) return false;
  const double worst_case_entropy_mod_gcd = worst_case_categorical_entropy(concentrated_p, gcd_m1);
  const double worst_case_bits_saved = std::log2(gcd) - worst_case_entropy_mod_gcd;
  if (worst_case_bits_saved < MULT_REQUIRED_BITS_SAVED_PER_NUM) return false;
  *score = worst_case_bits_saved;
  return true;
}

// int_mult.rs:206-214 choose_candidate_base + :187-204 most_prominent_gcd.  `sample` = ordered latents.
template <typename L>
inline bool choose_candidate_base(const std::vector<L>& sample, L* base, double* bits_saved) {
  std::vector<L> triple_gcds;
  for (size_t i = 0; i + 3 <= sample.size(); i += 3) {
    L g = calc_triple_gcd<L>(&sample[i]);
    if (g > 1) triple_gcds.push_back(g);
  }
  const size_t total_triples = sample.size() / 3;
  std::sort(triple_gcds.begin(), triple_gcds.end());
  bool found = false;
  for (size_t i = 0; i < triple_gcds.size();) {
    size_t j = i;
    while (j < triple_gcds.size() && triple_gcds[j] == triple_gcds[i]) j++;
    // min(gcd, L::from_u64(u64::MAX)).to_u64() as f64: no-op for <= 64-bit latents
    double score;
    if (filter_score_triple_gcd(double(uint64_t(triple_gcds[i])), j - i, total_triples, &score)) {
      // scores that pass are > 0, where f64::to_latent_ordered is monotone: compare the doubles directly; >= keeps the last max
      if (!found || score >= *bits_saved) {
        found = true;
        *base = triple_gcds[i];
        *bits_saved = score;
      }
    }
    i = j;
  }
  return found;
}

// sampling.rs:105-141 est_bits_saved_per_num specialised to int mult's closure (primary = x / candidate, the same
// bits_saved for every element): each group's savings are `bits_saved` added count times, as the reference accumulates.
template <typename L>
inline double est_bits_saved_per_num_int_mult(const std::vector<L>& sample, L candidate, double bits_saved) {
  std::vector<L> primaries(sample.size());
  for (size_t i = 0; i < sample.size(); i++) primaries[i] = L(sample[i] / candidate);
  std::sort(primaries.begin(), primaries.end());
  const double CLASSIC_MEMORIZABLE_BINS = double(1u << 8);  // constants.rs:50
  const size_t infrequent_cutoff = std::max<size_t>(1, size_t(double(sample.size()) / CLASSIC_MEMORIZABLE_BINS));
  double sample_bits_saved = 0.0;
  for (size_t i = 0; i < primaries.size();) {
    size_t j = i;
    double group = 0.0;
    while (j < primaries.size() && primaries[j] == primaries[i]) {
      group += bits_saved;
      j++;
    }
    if (j - i <= infrequent_cutoff) sample_bits_saved += group;
    i = j;
  }
  return sample_bits_saved / double(sample.size());
}

// int_mult.rs:216-230 choose_base over the ordered latents of the chunk's numbers
template <typename L>
inline bool int_mult_choose_base(const L* ordered_latents, size_t n, L* base) {
  std::vector<size_t> idx;
  if (!choose_mode_sample_indices(n, &idx)) return false;  // every int passes the filter, so the sample has >= MIN_SAMPLE entries
  std::vector<L> sample(idx.size());
  for (size_t i = 0; i < idx.size(); i++) sample[i] = ordered_latents[idx[i]];
  L candidate;
  double bits_saved_per_adj;
  if (!choose_candidate_base<L>(sample, &candidate, &bits_saved_per_adj)) return false;
  if (est_bits_saved_per_num_int_mult<L>(sample, candidate, bits_saved_per_adj) > MULT_REQUIRED_BITS_SAVED_PER_NUM) {
    *base = candidate;
    return true;
  }
  return false;
}


// ----- ModeSpec::Auto for floats (data_types/float.rs:70-98): classic, FloatMult and FloatQuant bid; the best estimate wins ----
// One generic search over the float type.  f16 follows the half crate (2.7.1, Cargo.lock:1353-1356, not under /root/reference): every
// arithmetic operator widens to f32 and rounds the result back, from_f64 rounds once from the double, round / abs / comparisons as in
// data_types/float.rs:254-366.
inline uint16_t f64_to_f16_bits(double d) {  // round-to-nearest-even in one step (finite values; the search never converts NaN)
  const uint16_t sign = std::signbit(d) ? 0x8000 : 0;
  const double a = std::fabs(d);
  if (std::isinf(a)) return uint16_t(sign | 0x7c00);
  if (a == 0.0) return sign;
  int ex;
  std::frexp(a, &ex);
  int e = ex - 1;  // a in [2^e, 2^(e+1))
  if (e < -14) return uint16_t(sign | uint16_t(std::nearbyint(std::ldexp(a, 24))));  // subnormal grid of 2^-24; 1024 is the first normal
  double r = std::nearbyint(std::ldexp(a, 10 - e));                                  // 11 significant bits
  if (r == 2048.0) { r = 1024.0; e += 1; }
  if (e > 15) return uint16_t(sign | 0x7c00);
  return uint16_t(sign | uint16_t((e + 15) << 10) | uint16_t(uint32_t(r) - 1024));
}
inline F16 FloatOps<uint16_t>::from_f64(double x) { return F16{f64_to_f16_bits(x)}; }
inline float f16_f32(F16 x) { return f16_bits_to_f32(x.bits); }
inline F16 f16_from(float x) { return F16{f32_to_f16_bits(x)}; }
inline F16 operator+(F16 a, F16 b) { return f16_from(f16_f32(a) + f16_f32(b)); }
inline F16 operator-(F16 a, F16 b) { return f16_from(f16_f32(a) - f16_f32(b)); }
inline F16 operator*(F16 a, F16 b) { return f16_from(f16_f32(a) * f16_f32(b)); }
inline F16 operator/(F16 a, F16 b) { return f16_from(f16_f32(a) / f16_f32(b)); }
inline F16& operator+=(F16& a, F16 b) { return a = a + b; }
inline bool operator<(F16 a, F16 b) { return f16_f32(a) < f16_f32(b); }
inline bool operator<=(F16 a, F16 b) { return f16_f32(a) <= f16_f32(b); }
inline bool operator>(F16 a, F16 b) { return f16_f32(a) > f16_f32(b); }
inline bool operator>=(F16 a, F16 b) { return f16_f32(a) >= f16_f32(b); }
inline bool operator==(F16 a, F16 b) { return f16_f32(a) == f16_f32(b); }
inline bool operator!=(F16 a, F16 b) { return f16_f32(a) != f16_f32(b); }

template <typename F> struct NativeFloat;
template <> struct NativeFloat<float> {
  using L = uint32_t;
  static constexpr Bitlen PRECISION_BITS = 23, BITS = 32;
  static constexpr int32_t EXP_OFFSET = 127;
  static float max_for_sampling() { return std::numeric_limits<float>::max() * 0.5f; }  // float.rs:141
  static float from_f64(double x) { return float(x); }
  static double to_f64(float x) { return double(x); }
  static float from_latent_numerical(uint32_t l) { return float(l); }
  static float round_(float x) { return std::round(x); }
  static float abs_(float x) { return std::fabs(x); }
  static float max_(float a, float b) { return std::fmax(a, b); }
  static float min_(float a, float b) { return std::fmin(a, b); }
  static bool is_normal(float x) { return std::isnormal(x); }
};
template <> struct NativeFloat<double> {
  using L = uint64_t;
  static constexpr Bitlen PRECISION_BITS = 52, BITS = 64;
  static constexpr int32_t EXP_OFFSET = 1023;
  static double max_for_sampling() { return std::numeric_limits<double>::max() * 0.5; }
  static double from_f64(double x) { return x; }
  static double to_f64(double x) { return x; }
  static double from_latent_numerical(uint64_t l) { return double(l); }
  static double round_(double x) { return std::round(x); }
  static double abs_(double x) { return std::fabs(x); }
  static double max_(double a, double b) { return std::fmax(a, b); }
  static double min_(double a, double b) { return std::fmin(a, b); }
  static bool is_normal(double x) { return std::isnormal(x); }
};
template <> struct NativeFloat<F16> {  // data_types/float.rs:254-366
  using L = uint16_t;
  static constexpr Bitlen PRECISION_BITS = 10, BITS = 16;
  static constexpr int32_t EXP_OFFSET = 15;
  static F16 max_for_sampling() { return F16{30719}; }
  static F16 from_f64(double x) { return F16{f64_to_f16_bits(x)}; }
  static double to_f64(F16 x) { return double(f16_f32(x)); }
  static F16 from_latent_numerical(uint16_t l) { return f16_from(float(l)); }
  static F16 round_(F16 x) { return f16_from(std::round(f16_f32(x))); }
  static F16 abs_(F16 x) { return F16{uint16_t(x.bits & 0x7fff)}; }
  static F16 max_(F16 a, F16 b) { return f16_from(std::fmax(f16_f32(a), f16_f32(b))); }
  static F16 min_(F16 a, F16 b) { return f16_from(std::fmin(f16_f32(a), f16_f32(b))); }
  static bool is_normal(F16 x) { const uint16_t e = x.bits & 0x7c00; return e != 0 && e != 0x7c00; }
};
template <typename F> inline typename NativeFloat<F>::L fl_bits(F x) { typename NativeFloat<F>::L b; std::memcpy(&b, &x, sizeof b); return b; }
template <typename F> inline F fl_from_bits(typename NativeFloat<F>::L b) { F x; std::memcpy(&x, &b, sizeof x); return x; }
template <typename F> inline F fl_exp2(int32_t power) {  // float.rs:158-160 (only meant for a small range; same wrap-around outside it)
  using L = typename NativeFloat<F>::L;
  return fl_from_bits<F>(L(L(int64_t(NativeFloat<F>::EXP_OFFSET + power)) << NativeFloat<F>::PRECISION_BITS));
}
template <typename F> inline int32_t fl_exponent(F x) {  // float.rs:183-185
  return int32_t(fl_bits<F>(NativeFloat<F>::abs_(x)) >> NativeFloat<F>::PRECISION_BITS) - NativeFloat<F>::EXP_OFFSET;
}
template <typename F> inline uint32_t fl_trailing_zeros(F x) {  // float.rs:188-190
  auto b = fl_bits<F>(x);
  if (b == 0) return NativeFloat<F>::BITS;
  return sizeof(b) == 8 ? uint32_t(__builtin_ctzll(uint64_t(b))) : uint32_t(__builtin_ctz(uint32_t(b)));  // b != 0, so narrower types are fine
}
template <typename L> inline uint32_t lat_leading_zeros(L x) {
  if (x == 0) return 8 * sizeof(L);
  return sizeof(L) == 8 ? uint32_t(__builtin_clzll(uint64_t(x))) : uint32_t(__builtin_clz(uint32_t(x))) - uint32_t(32 - 8 * sizeof(L));
}
template <typename F> inline typename NativeFloat<F>::L fl_ordered(F x) { return to_latent_ordered_bits<typename NativeFloat<F>::L>(fl_bits<F>(x), true, false); }

// sampling.rs:105-141 for any closure: (primary, bits_saved) per sample element in sample order.  A group's savings add up in
// sample order as in the reference; the groups are summed in ascending primary order (HashMap order in the reference).
template <typename L>
inline double est_bits_saved_per_num(std::vector<std::pair<L, double>> items) {
  const size_t n = items.size();
  std::stable_sort(items.begin(), items.end(), [](const std::pair<L, double>& a, const std::pair<L, double>& b) { return a.first < b.first; });
  const size_t infrequent_cutoff = std::max<size_t>(1, size_t(double(n) / 256.0));  // CLASSIC_MEMORIZABLE_BINS
  double total = 0.0;
  for (size_t i = 0; i < n;) {
    size_t j = i;
    double group = 0.0;
    while (j < n && items[j].first == items[i].first) group += items[j++].second;
    if (j - i <= infrequent_cutoff) total += group;
    i = j;
  }
  return total / double(n);
}

template <typename F>
struct FloatMultConfig {  // float_mult.rs:318-336
  F base, inv_base;
  static FloatMultConfig from_base(F base) { return {base, NativeFloat<F>::from_f64(1.0) / base}; }
  static FloatMultConfig from_inv_base(F inv_base) { return {NativeFloat<F>::from_f64(1.0) / inv_base, inv_base}; }
};

const Bitlen FM_REQUIRED_PRECISION_BITS = 6;  // float_mult.rs:78-83
template <typename F> inline F insignificant_float_to(F x) {  // :85-88
  const Bitlen P = NativeFloat<F>::PRECISION_BITS;
  const int32_t spare = int32_t(P > FM_REQUIRED_PRECISION_BITS ? P - FM_REQUIRED_PRECISION_BITS : 0);
  return x * fl_exp2<F>(-spare);
}
template <typename F> inline bool is_approx_zero(F small, F big) { return small <= insignificant_float_to<F>(big); }          // :90-92
template <typename F> inline bool is_small_remainder(F remainder, F original) { return remainder <= original * fl_exp2<F>(-16); }  // :94-96
template <typename F> inline bool is_imprecise(F value, F err) { return value <= err * fl_exp2<F>(int32_t(FM_REQUIRED_PRECISION_BITS)); }  // :98-100

template <typename F>
inline bool approx_pair_gcd(F greater, F lesser, F* out) {  // float_mult.rs:102-142
  if (is_approx_zero<F>(lesser, greater) || lesser == greater) return false;
  struct PairMult { F value, err; };
  const F machine_eps = fl_exp2<F>(-int32_t(NativeFloat<F>::PRECISION_BITS));
  auto rem_assign = [&](PairMult& lhs, const PairMult& rhs) {
    const F ratio = NativeFloat<F>::round_(lhs.value / rhs.value);
    lhs.err = lhs.err + (ratio * rhs.err + lhs.value * machine_eps);
    lhs.value = NativeFloat<F>::abs_(lhs.value - ratio * rhs.value);
  };
  PairMult p_greater{greater, NativeFloat<F>::from_f64(0.0)}, p_lesser{lesser, NativeFloat<F>::from_f64(0.0)};
  for (;;) {
    const F prev = p_greater.value;
    rem_assign(p_greater, p_lesser);
    if (is_small_remainder<F>(p_greater.value, prev) || p_greater.value <= p_greater.err) {
      *out = p_lesser.value;
      return true;
    }
    if (is_approx_zero<F>(p_greater.value, greater) || is_imprecise<F>(p_greater.value, p_greater.err)) return false;
    std::swap(p_greater, p_lesser);
  }
}

template <typename F>
inline bool choose_config_by_trailing_zeros(const std::vector<F>& sample, FloatMultConfig<F>* out) {  // float_mult.rs:145-194
  using L = typename NativeFloat<F>::L;
  const Bitlen P = NativeFloat<F>::PRECISION_BITS, BITS = NativeFloat<F>::BITS;
  auto calc_power_of_2_divisor = [&](int32_t exponent, uint32_t tz) { return exponent - int32_t(P > tz ? P - tz : 0); };
  int32_t k = std::numeric_limits<int32_t>::max();
  size_t count = 0;
  for (F x : sample) {
    const uint32_t tz = fl_trailing_zeros<F>(x);
    if (x != NativeFloat<F>::from_f64(0.0) && tz >= 5) {  // INTERESTING_TRAILING_ZEROS
      count++;
      k = std::min(k, calc_power_of_2_divisor(fl_exponent<F>(x), tz));
    }
  }
  const size_t required_samples = std::max<size_t>(size_t(std::ceil(double(sample.size()) * 0.5)), 10);  // REQUIRED_TRAILING_ZEROS_FREQUENCY, MIN_SAMPLE
  if (count < required_samples) return false;
  std::vector<L> int_sample;
  const Bitlen lshift = BITS - P - 1;
  for (F x : sample) {
    const int32_t exponent = fl_exponent<F>(x);
    const int32_t k_prime = calc_power_of_2_divisor(exponent, fl_trailing_zeros<F>(x));
    if (k_prime >= k && exponent < k + int32_t(BITS)) {
      const uint32_t rshift = BITS - 1 - uint32_t(exponent - k);
      const L lshifted_w_explicit_mantissa = L(L(fl_bits<F>(x) << lshift) | LatentTraits<L>::MID);
      int_sample.push_back(L(lshifted_w_explicit_mantissa >> rshift));
    }
  }
  if (int_sample.size() < required_samples) return false;
  L int_base;
  double unused;
  if (!choose_candidate_base<L>(int_sample, &int_base, &unused)) int_base = 1;
  *out = FloatMultConfig<F>::from_base(NativeFloat<F>::from_latent_numerical(int_base) * fl_exp2<F>(k));
  return true;
}

template <typename F>
inline bool approx_sample_gcd_euclidean(const std::vector<F>& sample, F* out) {  // float_mult.rs:197-229
  std::vector<F> gcds;
  for (size_t i = 0; i + 1 < sample.size(); i += 2) {
    F g;
    if (approx_pair_gcd<F>(NativeFloat<F>::max_(sample[i], sample[i + 1]), NativeFloat<F>::min_(sample[i], sample[i + 1]), &g)) gcds.push_back(g);
  }
  const size_t required_pairs_with_common_gcd = 1 + size_t(std::ceil(double(sample.size()) * 0.001));  // REQUIRED_GCD_PAIR_FREQUENCY
  if (gcds.size() < required_pairs_with_common_gcd) return false;
  std::sort(gcds.begin(), gcds.end());
  for (double percentile : {0.1, 0.3, 0.5}) {
    const F candidate = gcds[size_t(percentile * double(gcds.size()))];
    size_t similar = 0;
    for (F g : gcds) similar += NativeFloat<F>::abs_(g - candidate) < NativeFloat<F>::from_f64(0.01) * candidate;
    if (similar >= required_pairs_with_common_gcd) {
      *out = candidate;
      return true;
    }
  }
  return false;
}

template <typename F>
inline F center_sample_base(F base, const std::vector<F>& sample) {  // float_mult.rs:239-259
  const Bitlen P = NativeFloat<F>::PRECISION_BITS;
  const F inv_base = NativeFloat<F>::from_f64(1.0) / base;
  F tweak_sum = NativeFloat<F>::from_f64(0.0), tweak_weight = NativeFloat<F>::from_f64(0.0);
  for (F x : sample) {
    const F mult = NativeFloat<F>::round_(x * inv_base);
    const Bitlen mult_exponent = Bitlen(fl_exponent<F>(mult));  // `as Bitlen`: a negative exponent wraps to a huge value
    if (mult_exponent < P && mult != NativeFloat<F>::from_f64(0.0)) {
      const F overshoot = (mult * base) - x;
      const F weight = NativeFloat<F>::from_f64(double(P - mult_exponent));
      tweak_sum += weight * (overshoot / mult);
      tweak_weight += weight;
    }
  }
  return base - tweak_sum / tweak_weight;
}

template <typename F>
inline FloatMultConfig<F> snap_to_int_reciprocal(F base) {  // float_mult.rs:261-275
  using NF = NativeFloat<F>;
  const F inv_base = NF::from_f64(1.0) / base;
  const F round_inv_base = NF::round_(inv_base);
  const F decimal_inv_base = NF::from_f64(std::pow(10.0, std::round(std::log10(NF::to_f64(inv_base)))));
  if (NF::abs_(inv_base - round_inv_base) < NF::from_f64(0.02)) return FloatMultConfig<F>::from_inv_base(round_inv_base);                 // SNAP_THRESHOLD_ABSOLUTE
  if (NF::abs_(inv_base - decimal_inv_base) / inv_base < NF::from_f64(0.01)) return FloatMultConfig<F>::from_inv_base(decimal_inv_base);  // SNAP_THRESHOLD_DECIMAL_RELATIVE
  return FloatMultConfig<F>::from_base(base);
}

template <typename F>
inline bool choose_config_by_euclidean(const std::vector<F>& sample, FloatMultConfig<F>* out) {  // float_mult.rs:231-236
  F base;
  if (!approx_sample_gcd_euclidean<F>(sample, &base)) return false;
  *out = snap_to_int_reciprocal<F>(center_sample_base<F>(base, sample));
  return true;
}

template <typename F>
inline bool bits_saved_per_num_over_classic(const FloatMultConfig<F>& config, const std::vector<F>& sample, double* out) {  // float_mult.rs:277-315
  using L = typename NativeFloat<F>::L;
  const Bitlen P = NativeFloat<F>::PRECISION_BITS;
  std::vector<std::pair<L, double>> items;
  items.reserve(sample.size());
  for (F x : sample) {
    const F mult = NativeFloat<F>::round_(x * config.inv_base);
    const L primary = int_float_to_latent<L>(mult);
    const Bitlen mult_exponent = Bitlen(fl_exponent<F>(mult));
    const Bitlen inter_base_bits = P > mult_exponent ? P - mult_exponent : 0;
    const L approx_unsigned = fl_ordered<F>(mult * config.base), x_as_unsigned = fl_ordered<F>(x);
    const L abs_adj = L(std::max(x_as_unsigned, approx_unsigned) - std::min(x_as_unsigned, approx_unsigned));
    const Bitlen adj_bits = 1 + 2 * (NativeFloat<F>::BITS - lat_leading_zeros<L>(abs_adj));
    items.emplace_back(primary, double(inter_base_bits) - double(adj_bits));
  }
  const double bits_saved_per_num = est_bits_saved_per_num<L>(std::move(items));
  if (bits_saved_per_num >= MULT_REQUIRED_BITS_SAVED_PER_NUM) {
    *out = bits_saved_per_num;
    return true;
  }
  return false;
}

// f64::total_cmp as an integer key
inline uint64_t f64_total_order_key(double x) { uint64_t b; std::memcpy(&b, &x, 8); return to_latent_ordered_bits<uint64_t>(b, true, false); }

template <typename F>
inline bool float_mult_compute_bid(const std::vector<F>& sample, FloatMultConfig<F>* config, double* bits_saved_per_num) {  // float_mult.rs:338-358
  bool found = false;
  for (int which = 0; which < 2; which++) {
    FloatMultConfig<F> c{NativeFloat<F>::from_f64(0.0), NativeFloat<F>::from_f64(0.0)};
    double saved = 0.0;
    if (!(which == 0 ? choose_config_by_trailing_zeros<F>(sample, &c) : choose_config_by_euclidean<F>(sample, &c))) continue;
    if (!bits_saved_per_num_over_classic<F>(c, sample, &saved)) continue;
    if (!found || f64_total_order_key(saved) >= f64_total_order_key(*bits_saved_per_num)) {  // max_by keeps the last maximum
      found = true;
      *config = c;
      *bits_saved_per_num = saved;
    }
  }
  return found;
}

template <typename F>
inline std::pair<Bitlen, double> float_quant_estimate_best_k_and_bits_saved(const std::vector<F>& sample) {  // float_quant.rs:93-151
  const Bitlen P = NativeFloat<F>::PRECISION_BITS;
  std::vector<uint32_t> hist(P + 1, 0);
  for (F x : sample) hist[std::min<uint32_t>(P, fl_trailing_zeros<F>(x))]++;
  uint32_t rev_csum = 0;
  for (size_t i = hist.size(); i-- > 0;) {
    rev_csum += hist[i];
    hist[i] = rev_csum;
  }
  const double sample_len = double(sample.size());
  Bitlen best_k = 0;
  double best_bits_saved = 0.0;
  for (size_t k = 1; k < hist.size(); k++) {
    if (hist[k] == 0) continue;
    const double freq = double(hist[k]) / sample_len;
    const uint64_t n_categories = (uint64_t(1) << k) - 1;
    const double saved = double(k) - worst_case_categorical_entropy(freq, double(n_categories));
    if (saved > best_bits_saved) {
      best_k = Bitlen(k);
      best_bits_saved = saved;
    } else {
      break;
    }
  }
  return {best_k, best_bits_saved};
}

const double QUANT_REQUIRED_BITS_SAVED_PER_NUM = 1.5;  // constants.rs:49
template <typename F>
inline bool float_quant_compute_bid(const std::vector<F>& sample, Bitlen* k_out, double* bits_saved_per_num) {  // float_quant.rs:73-91
  using L = typename NativeFloat<F>::L;
  auto kb = float_quant_estimate_best_k_and_bits_saved<F>(sample);
  std::vector<std::pair<L, double>> items;
  items.reserve(sample.size());
  for (F x : sample) items.emplace_back(L(fl_bits<F>(x) >> kb.first), kb.second);
  const double saved = est_bits_saved_per_num<L>(std::move(items));
  if (saved > QUANT_REQUIRED_BITS_SAVED_PER_NUM) {
    *k_out = kb.first;
    *bits_saved_per_num = saved;
    return true;
  }
  return false;
}

// data_types/float.rs:70-80 filter_sample over sampling.rs:62-103's draw
template <typename F>
inline bool choose_float_mode_sample(const typename NativeFloat<F>::L* num_bits, size_t n, std::vector<F>* sample) {
  std::vector<size_t> idx;
  if (!choose_mode_sample_indices(n, &idx)) return false;
  sample->clear();
  for (size_t i : idx) {
    const F x = fl_from_bits<F>(num_bits[i]);
    if (NativeFloat<F>::is_normal(x)) {
      const F a = NativeFloat<F>::abs_(x);
      if (a <= NativeFloat<F>::max_for_sampling()) sample->push_back(a);
    }
  }
  return sample->size() >= 10;  // MIN_SAMPLE
}

struct FloatModeChoice {
  ModeKind kind = ModeKind::Classic;
  double base = 0, inv_base = 0;  // FloatMult (exact in a double for f32 too)
  Bitlen k = 0;                   // FloatQuant
  double bits_saved_per_num = 0.0;
};
// data_types/float.rs:82-98 + compression_intermediates.rs:79-84: bids in the order classic, float mult, float quant; the last maximum wins
template <typename F>
inline FloatModeChoice choose_float_mode_from_sample(const std::vector<F>& sample) {
  FloatModeChoice best;
  FloatMultConfig<F> c{NativeFloat<F>::from_f64(0.0), NativeFloat<F>::from_f64(0.0)};
  double saved = 0.0;
  if (float_mult_compute_bid<F>(sample, &c, &saved) && f64_total_order_key(saved) >= f64_total_order_key(best.bits_saved_per_num)) {
    best.kind = ModeKind::FloatMult;
    best.base = NativeFloat<F>::to_f64(c.base);
    best.inv_base = NativeFloat<F>::to_f64(c.inv_base);
    best.bits_saved_per_num = saved;
  }
  Bitlen k;
  if (float_quant_compute_bid<F>(sample, &k, &saved) && f64_total_order_key(saved) >= f64_total_order_key(best.bits_saved_per_num)) {
    best.kind = ModeKind::FloatQuant;
    best.k = k;
    best.bits_saved_per_num = saved;
  }
  return best;
}
template <typename F>
inline FloatModeChoice choose_float_mode(const typename NativeFloat<F>::L* num_bits, size_t n) {
  std::vector<F> sample;
  if (!choose_float_mode_sample<F>(num_bits, n, &sample)) return FloatModeChoice();
  return choose_float_mode_from_sample<F>(sample);
}


template <typename L>
struct SplitLatents {
  std::vector<L> primary;
  bool has_secondary = false;
  std::vector<L> secondary;
};

// chunk_compressor.rs:142-217 + :219-308 new_candidate
template <typename L>
inline std::unique_ptr<ChunkCompressor<L>> new_candidate(SplitLatents<L> latents, const std::vector<size_t>& page_ns, const Mode& mode,
                                                         const DeltaEncoding& delta, Bitlen unoptimized_bins_log,
                                                         uint8_t number_type) {
  std::unique_ptr<ChunkCompressor<L>> cc(new ChunkCompressor<L>());
  cc->number_type = number_type;
  cc->page_ns = page_ns;
  cc->meta.number_bits = sizeof(L) * 8;
  cc->meta.mode = mode;
  cc->meta.delta = delta;
  cc->meta.has_secondary = latents.has_secondary;
  cc->meta.has_delta_var = delta.kind == DeltaKind::Lookback;
  size_t n = latents.primary.size();
  std::vector<uint32_t> delta_latents;
  if (cc->meta.has_delta_var) delta_latents.reserve(n);
  size_t start_idx = 0;
  LatentVarDelta enc_primary = delta_for_latent_var(cc->meta.delta, VarKey::Primary);
  LatentVarDelta enc_secondary = delta_for_latent_var(cc->meta.delta, VarKey::Secondary);
  auto encode_var = [&](const LatentVarDelta& enc, const std::vector<DeltaLookback>& page_lookbacks, std::vector<L>& v, size_t s, size_t e) {
    PageInfoVar<L> pi;
    std::vector<L> st;
    switch (enc.kind) {
      case DeltaKind::NoOp: break;
      case DeltaKind::Consecutive: st = consecutive_encode_in_place<L>(enc.enc->order, v.data() + s, e - s); break;
      case DeltaKind::Lookback: st = lookback_encode_in_place<L>(*enc.enc, page_lookbacks.data(), v.data() + s, e - s); break;
      case DeltaKind::Conv1:
        if constexpr (sizeof(L) <= 4) st = conv1_encode_in_place<L>(*enc.enc, v.data() + s, e - s);
        break;
    }
    for (L x : st) pi.delta_state.push_back(uint64_t(x));
    pi.start = std::min(s + enc.n_latents_per_state(), e);
    pi.end = e;
    return pi;
  };
  for (size_t page_n : page_ns) {
    size_t end_idx = start_idx + page_n;
    std::vector<DeltaLookback> page_lookbacks;
    if (cc->meta.has_delta_var) page_lookbacks = choose_lookbacks<L>(cc->meta.delta, latents.primary.data() + start_idx, page_n);
    cc->pi_primary.push_back(encode_var(enc_primary, page_lookbacks, latents.primary, start_idx, end_idx));
    if (latents.has_secondary) cc->pi_secondary.push_back(encode_var(enc_secondary, page_lookbacks, latents.secondary, start_idx, end_idx));
    if (cc->meta.has_delta_var) {
      PageInfoVar<L> pi;
      pi.start = delta_latents.size();
      pi.end = delta_latents.size() + page_lookbacks.size();
      cc->pi_delta.push_back(pi);
      delta_latents.insert(delta_latents.end(), page_lookbacks.begin(), page_lookbacks.end());
    }
    start_idx = end_idx;
  }
  // train bins per var, in file order
  auto train = [&](auto tag, const auto& var_latents, const auto& page_infos, Bitlen bins_log, LatentVarMeta& vm,
                   std::vector<Weight>& counts) {
    using VL = decltype(tag);
    std::vector<VL> contiguous;
    contiguous.reserve(var_latents.size());
    for (const auto& pi : page_infos) contiguous.insert(contiguous.end(), var_latents.begin() + pi.start, var_latents.begin() + pi.end);
    TrainedBins<VL> trained = train_infos<VL>(std::move(contiguous), bins_log);
    vm.latent_bits = sizeof(VL) * 8;
    vm.ans_size_log = trained.ans_size_log;
    vm.bins.clear();
    for (auto& info : trained.infos) vm.bins.push_back(Bin{info.weight, uint64_t(info.lower), info.offset_bits});
    counts = trained.counts;
    return trained;
  };
  if (cc->meta.has_delta_var) {
    auto trained = train(uint32_t(0), delta_latents, cc->pi_delta, unoptimized_bins_log, cc->meta.delta_var, cc->counts_delta);
    cc->vc_delta.reset(new VarCompressor<uint32_t>(trained, cc->meta.delta_var, std::move(delta_latents)));
  }
  {
    auto trained = train(L(0), latents.primary, cc->pi_primary, unoptimized_bins_log, cc->meta.primary, cc->counts_primary);
    cc->vc_primary.reset(new VarCompressor<L>(trained, cc->meta.primary, std::move(latents.primary)));
  }
  if (latents.has_secondary) {
    auto trained = train(L(0), latents.secondary, cc->pi_secondary, std::min(unoptimized_bins_log, LIMITED_UNOPTIMIZED_BINS_LOG),
                         cc->meta.secondary, cc->counts_secondary);
    cc->vc_secondary.reset(new VarCompressor<L>(trained, cc->meta.secondary, std::move(latents.secondary)));
  }
  validate_chunk_meta(cc->meta);
  return cc;
}

// chunk_compressor.rs:310-360 + :373-394
template <typename L>
inline DeltaEncoding choose_delta_encoding(const SplitLatents<L>& latents, const ChunkConfig& config, Bitlen unoptimized_bins_log,
                                           uint8_t number_type) {
  DeltaEncoding noop;
  size_t n = latents.primary.size();
  switch (config.delta_kind) {
    case DeltaSpecKind::NoOp: return noop;
    case DeltaSpecKind::TryConsecutive: {
      if (config.delta_order == 0) return noop;
      DeltaEncoding d;
      d.kind = DeltaKind::Consecutive;
      d.order = config.delta_order;
      return d;
    }
    case DeltaSpecKind::TryLookback: return new_lookback(n);
    case DeltaSpecKind::TryConv1:
      if (config.delta_order == 0) return noop;
      if constexpr (sizeof(L) <= 4) {  // delta/mod.rs:50-70 (64-bit latents were refused by validate_config)
        DeltaEncoding d;
        return conv1_choose_config<L>(config.delta_order, latents.primary.data(), n, &d) ? d : noop;
      }
      invalid_argument("Conv1 delta encoding cannot be used with 64-bit latents");
    case DeltaSpecKind::Auto: break;
  }
  // choose_auto_delta_encoding
  std::vector<L> sample;
  if (!choose_delta_sample<L>(latents.primary, &sample)) return noop;
  size_t sample_n = sample.size();
  auto cost_of = [&](const DeltaEncoding& enc) -> float {
    SplitLatents<L> s;
    s.primary = sample;
    Mode classic;
    auto cc = new_candidate<L>(std::move(s), {sample_n}, classic, enc, unoptimized_bins_log, number_type);
    return float(cc->meta_size_hint() + cc->page_size_hint_inner(0, 1.0));
  };
  DeltaEncoding best = noop;
  float best_cost = cost_of(noop);
  float lookback_penalty = 0.25f * float(sample_n);
  if (best_cost > lookback_penalty) {
    float lookback_cost = cost_of(new_lookback(sample_n)) + lookback_penalty;
    if (lookback_cost < best_cost) {
      best = new_lookback(n);
      best_cost = lookback_cost;
    }
  }
  for (size_t order = 1; order <= MAX_CONSECUTIVE_DELTA_ORDER; order++) {
    DeltaEncoding enc;
    enc.kind = DeltaKind::Consecutive;
    enc.order = order;
    float cost = cost_of(enc);
    if (cost < best_cost) { best = enc; best_cost = cost; } else break;
  }
  return best;
}

// Mode split (mode/classic.rs:6-12, float_mult.rs:38-60, int_mult.rs:20-36, float_quant.rs:41-73)
template <typename L>
inline SplitLatents<L> split_latents(const L* nums, size_t n, uint8_t number_type, const ChunkConfig& config, Mode* mode_out) {
  bool isf = number_type_is_float(number_type), iss = number_type_is_signed(number_type);
  SplitLatents<L> out;
  Mode mode;
  ModeSpecKind kind = config.mode_kind;
  L auto_base = 0;
  FloatModeChoice auto_float;
  if (kind == ModeSpecKind::Auto && isf) {
    // data_types/float.rs:82-98
    if constexpr (sizeof(L) == 4) auto_float = choose_float_mode<float>(nums, n);
    else if constexpr (sizeof(L) == 8) auto_float = choose_float_mode<double>(nums, n);
    else if constexpr (sizeof(L) == 2) auto_float = choose_float_mode<F16>(nums, n);
    kind = auto_float.kind == ModeKind::FloatMult ? ModeSpecKind::TryFloatMult : auto_float.kind == ModeKind::FloatQuant ? ModeSpecKind::TryFloatQuant : ModeSpecKind::Classic;
  } else if (kind == ModeSpecKind::Auto) {
    // data_types/unsigned.rs:28-35 (signed.rs:41-43 forwards to it)
    std::vector<L> ordered(n);
    for (size_t i = 0; i < n; i++) ordered[i] = to_latent_ordered_bits<L>(nums[i], isf, iss);
    kind = int_mult_choose_base<L>(ordered.data(), n, &auto_base) ? ModeSpecKind::TryIntMult : ModeSpecKind::Classic;
  }
  const bool is_auto = config.mode_kind == ModeSpecKind::Auto;
  if (kind == ModeSpecKind::TryDict) invalid_argument("oracle: Dict mode is encoded by simple_compress (its latents are u32 indices); the wrapped handle does not carry it");
  if (isf && kind == ModeSpecKind::TryIntMult) invalid_argument("unable to use int mult mode on floats");
  if (!isf && (kind == ModeSpecKind::TryFloatMult || kind == ModeSpecKind::TryFloatQuant)) invalid_argument("unable to use float mode for ints");
  out.primary.resize(n);
  switch (kind) {
    case ModeSpecKind::Classic:
      for (size_t i = 0; i < n; i++) out.primary[i] = to_latent_ordered_bits<L>(nums[i], isf, iss);
      break;
    case ModeSpecKind::TryIntMult: {
      mode.kind = ModeKind::IntMult;
      L base = config.mode_kind == ModeSpecKind::Auto ? auto_base : L(config.int_mult_base);
      mode.base_latent = base;
      if (!mode_is_valid(mode, number_type)) invalid_argument("The chosen mode was invalid for the number type");
      out.has_secondary = true;
      out.secondary.resize(n);
      for (size_t i = 0; i < n; i++) {
        L u = to_latent_ordered_bits<L>(nums[i], isf, iss);
        out.primary[i] = L(u / base);
        out.secondary[i] = L(u % base);
      }
      break;
    }
    case ModeSpecKind::TryFloatQuant: {
      mode.kind = ModeKind::FloatQuant;
      mode.k = is_auto ? auto_float.k : config.float_quant_k;
      if (!mode_is_valid(mode, number_type)) invalid_argument("The chosen mode was invalid for the number type");
      out.has_secondary = true;
      out.secondary.resize(n);
      Bitlen k = mode.k;
      L lowest_k_bits_max = L(L(L(1) << k) - 1);
      for (size_t i = 0; i < n; i++) {
        L num_ = to_latent_ordered_bits<L>(nums[i], true, false);
        out.primary[i] = L(num_ >> k);
        L lowest = L(num_ & lowest_k_bits_max);
        bool sign_positive = (nums[i] & LatentTraits<L>::MID) == 0;
        out.secondary[i] = sign_positive ? lowest : L(lowest_k_bits_max - lowest);
      }
      break;
    }
    case ModeSpecKind::TryFloatMult: {
      if constexpr (sizeof(L) == 2 || sizeof(L) == 4 || sizeof(L) == 8) {
        using FO = FloatOps<L>;
        mode.kind = ModeKind::FloatMult;
        // Auto carries its own (base, inv_base) pair: snap_to_int_reciprocal may give inv_base = 100 with base = 1/100, where 1/base != 100
        auto base = FO::from_f64(is_auto ? auto_float.base : config.float_mult_base);
        auto inv_base = is_auto ? FO::from_f64(auto_float.inv_base) : FO::inv(base);
        mode.base_latent = to_latent_ordered_bits<L>(FO::to_bits(base), true, false);
        if (!mode_is_valid(mode, number_type)) invalid_argument("The chosen mode was invalid for the number type");
        out.has_secondary = true;
        out.secondary.resize(n);
        for (size_t i = 0; i < n; i++) {
          auto num = FO::from_bits(nums[i]);
          auto mult = FO::round_(FO::mul(num, inv_base));
          out.primary[i] = int_float_to_latent<L>(mult);
          L a = to_latent_ordered_bits<L>(nums[i], true, false);
          L b = to_latent_ordered_bits<L>(FO::to_bits(FO::mul(mult, base)), true, false);
          out.secondary[i] = L(L(a - b) + LatentTraits<L>::MID);
        }
      } else {
        invalid_argument("unable to use float mode for ints");
      }
      break;
    }
    default: break;
  }
  *mode_out = mode;
  return out;
}

// chunk_compressor.rs:396-500 ChunkCompressor::new (+ fallback_chunk_compressor)
// chunk_compressor.rs:400-436 fallback_chunk_compressor: Classic, NoOp, one bin {weight 1, lower 0, offset_bits L::BITS}
template <typename L>
inline std::unique_ptr<ChunkCompressor<L>> fallback_chunk_compressor(const L* nums, size_t n, uint8_t number_type, const ChunkConfig& config,
                                                                     const std::vector<size_t>& page_ns) {
  ChunkConfig cfg = config;
  cfg.mode_kind = ModeSpecKind::Classic;
  Mode classic;
  SplitLatents<L> split = split_latents<L>(nums, n, number_type, cfg, &classic);
  std::unique_ptr<ChunkCompressor<L>> cc(new ChunkCompressor<L>());
  cc->number_type = number_type;
  cc->page_ns = page_ns;
  cc->meta.number_bits = sizeof(L) * 8;
  cc->meta.primary.latent_bits = sizeof(L) * 8;
  cc->meta.primary.ans_size_log = 0;
  cc->meta.primary.bins = {Bin{1, 0, Bitlen(sizeof(L) * 8)}};
  size_t s = 0;
  for (size_t page_n : page_ns) {
    PageInfoVar<L> pi;
    pi.start = s;
    pi.end = s + page_n;
    cc->pi_primary.push_back(pi);
    s += page_n;
  }
  TrainedBins<L> trained;
  trained.infos = {BinCompressionInfo<L>{1, 0, LatentTraits<L>::MAX, Bitlen(sizeof(L) * 8), 0}};
  trained.ans_size_log = 0;
  trained.counts = {Weight(n)};
  cc->counts_primary = trained.counts;
  cc->vc_primary.reset(new VarCompressor<L>(trained, cc->meta.primary, std::move(split.primary)));
  return cc;
}

template <typename L>
inline std::unique_ptr<ChunkCompressor<L>> new_chunk_compressor(const L* nums, size_t n, uint8_t number_type, const ChunkConfig& config) {
  validate_config(config, sizeof(L) * 8);
  if (n == 0) invalid_argument("cannot compress empty chunk");
  if (n > MAX_ENTRIES) invalid_argument("count may not exceed 16777216 per chunk");
  Mode mode;
  SplitLatents<L> latents = split_latents<L>(nums, n, number_type, config, &mode);
  Bitlen unoptimized_bins_log = choose_unoptimized_bins_log(config.compression_level, n);
  DeltaEncoding delta = choose_delta_encoding<L>(latents, config, unoptimized_bins_log, number_type);
  std::vector<size_t> page_ns = n_per_page(config, n);
  auto candidate = new_candidate<L>(std::move(latents), page_ns, mode, delta, unoptimized_bins_log, number_type);
  if (candidate->should_fallback(n)) return fallback_chunk_compressor<L>(nums, n, number_type, config, page_ns);
  return candidate;
}

// ===========================================================================
// Standalone (pco/src/standalone/{compressor,decompressor,simple}.rs)
// ===========================================================================
// standalone/compressor.rs:191-203
template <typename L>
inline void write_standalone_chunk(ChunkCompressor<L>& cc, std::vector<uint8_t>& dst) {
  BitWriter w(dst);
  w.write_aligned_bytes(&cc.number_type, 1);
  w.write_uint(cc.page_ns[0] - 1, BITS_TO_ENCODE_N_ENTRIES);
  w.finish();
  cc.write_meta(dst);
  cc.write_page(0, dst);
}

// ModeSpec::TryDict (mode/dict.rs:10-68): the distinct ordered latents by descending count form the dictionary (chunk meta), their u32
// indices are the primary latents; then everything runs as for any other u32 latent var.  Equal counts come out in HashMap order in
// the reference (unspecified); here ascending by value, unless a test names the order (dict_tie_order, used to match a golden asset).
inline std::vector<uint64_t>& dict_tie_order() { static std::vector<uint64_t> order; return order; }
template <typename L>
inline void write_standalone_dict_chunk(const L* nums, size_t n, uint8_t number_type, const ChunkConfig& config, std::vector<uint8_t>& dst) {
  validate_config(config, sizeof(L) * 8);
  if (n == 0) invalid_argument("cannot compress empty chunk");
  if (n > MAX_ENTRIES) invalid_argument("count may not exceed 16777216 per chunk");
  const bool isf = number_type_is_float(number_type), iss = number_type_is_signed(number_type);
  std::vector<L> ordered(n);
  for (size_t i = 0; i < n; i++) ordered[i] = to_latent_ordered_bits<L>(nums[i], isf, iss);
  std::vector<L> uniq = ordered;
  std::sort(uniq.begin(), uniq.end());
  std::vector<std::pair<L, uint32_t>> counts;
  for (size_t i = 0; i < uniq.size();) {
    size_t j = i;
    while (j < uniq.size() && uniq[j] == uniq[i]) j++;
    counts.emplace_back(uniq[i], uint32_t(j - i));
    i = j;
  }
  const std::vector<uint64_t>& pref = dict_tie_order();
  auto rank = [&](L v) { auto it = std::find(pref.begin(), pref.end(), uint64_t(v)); return size_t(it - pref.begin()); };
  std::stable_sort(counts.begin(), counts.end(), [&](const std::pair<L, uint32_t>& a, const std::pair<L, uint32_t>& b) {
    if (a.second != b.second) return a.second > b.second;
    return rank(a.first) < rank(b.first);  // equal ranks (no preference) keep ascending value order
  });
  Mode mode;
  mode.kind = ModeKind::Dict;
  for (auto& c : counts) mode.dict.push_back(uint64_t(c.first));
  if (!mode_is_valid(mode, number_type)) invalid_argument("The chosen mode was invalid for the number type");
  SplitLatents<uint32_t> split;
  split.primary.resize(n);
  std::vector<std::pair<L, uint32_t>> index_of;  // value -> position in the dictionary
  for (size_t i = 0; i < counts.size(); i++) index_of.emplace_back(counts[i].first, uint32_t(i));
  std::sort(index_of.begin(), index_of.end());
  for (size_t i = 0; i < n; i++)
    split.primary[i] = std::lower_bound(index_of.begin(), index_of.end(), std::make_pair(ordered[i], uint32_t(0)))->second;
  const Bitlen unoptimized_bins_log = choose_unoptimized_bins_log(config.compression_level, n);
  const DeltaEncoding delta = choose_delta_encoding<uint32_t>(split, config, unoptimized_bins_log, number_type);
  const std::vector<size_t> page_ns = n_per_page(config, n);
  auto cand = new_candidate<uint32_t>(std::move(split), page_ns, mode, delta, unoptimized_bins_log, number_type);
  cand->meta.number_bits = sizeof(L) * 8;  // the dictionary entries and the size baseline are in the NUMBER's width
  if (cand->should_fallback(n)) {
    auto cc = fallback_chunk_compressor<L>(nums, n, number_type, config, page_ns);
    write_standalone_chunk<L>(*cc, dst);
  } else {
    write_standalone_chunk<uint32_t>(*cand, dst);
  }
}

// standalone/simple.rs:22-91; `uniform_type` selects the _into flavour (header byte 5)
template <typename L>
inline void simple_compress(const L* nums, size_t n, uint8_t number_type, const ChunkConfig& config, bool uniform_type,
                            std::vector<uint8_t>& dst) {
  fallback_margins().clear();
  write_standalone_header(dst, n, uniform_type ? number_type : 0);
  std::vector<size_t> chunks = n_per_page(config, n);
  size_t start = 0;
  ChunkConfig this_cfg = config;
  for (size_t page_n : chunks) {
    this_cfg.paging_kind = PagingKind::Exact;
    this_cfg.exact_pages = {page_n};
    if (config.mode_kind == ModeSpecKind::TryDict) {
      write_standalone_dict_chunk<L>(nums + start, page_n, number_type, this_cfg, dst);
    } else {
      auto cc = new_chunk_compressor<L>(nums + start, page_n, number_type, this_cfg);
      write_standalone_chunk<L>(*cc, dst);
    }
    start += page_n;
  }
  dst.push_back(MAGIC_TERMINATION_BYTE);
}

// A standalone file reader over a padded copy of the source
struct PaddedSrc {
  std::vector<uint8_t> buf;
  size_t len;
  PaddedSrc(const uint8_t* src, size_t n) : buf(n + READ_PADDING, 0), len(n) {
    if (n) std::memcpy(buf.data(), src, n);
  }
};

// standalone/decompressor.rs:190-258: returns false at the terminator
template <typename L>
inline bool read_chunk_preamble(BitReader& r, const StandaloneHeader& h, uint8_t expected_type, size_t* n_out) {
  uint8_t b = r.read_aligned_bytes(1)[0];
  r.check_in_bounds();
  if (b == MAGIC_TERMINATION_BYTE) return false;
  if (h.uniform_type != 0 && h.uniform_type != b) corruption("chunk's number type does not match file's uniform number type");
  if (b != expected_type) corruption("requested chunk decompression does not match chunk's number type");
  *n_out = size_t(r.read_uint(BITS_TO_ENCODE_N_ENTRIES)) + 1;
  r.check_in_bounds();
  return true;
}

// standalone/decompressor.rs:265-275 simple_decompress
template <typename L>
inline void simple_decompress(const uint8_t* src, size_t src_len, uint8_t number_type, std::vector<L>& out) {
  PaddedSrc ps(src, src_len);
  BitReader r(ps.buf.data(), ps.len);
  StandaloneHeader h = read_standalone_header(r);
  size_t n;
  while (read_chunk_preamble<L>(r, h, number_type, &n)) {
    ChunkMeta cm = read_chunk_meta(r, h.format, sizeof(L) * 8);
    ChunkDecoder cd(std::move(cm), number_type);
    PageDecoder<L> pd(cd, r, n);
    size_t old = out.size();
    out.resize(old + n);
    pd.read(out.data() + old, n);
  }
}

// standalone/simple.rs:100-143 simple_decompress_into
template <typename L>
inline Progress simple_decompress_into(const uint8_t* src, size_t src_len, uint8_t number_type, L* dst, size_t dst_len) {
  PaddedSrc ps(src, src_len);
  BitReader r(ps.buf.data(), ps.len);
  StandaloneHeader h = read_standalone_header(r);
  std::vector<L> incomplete(FULL_BATCH_N);
  Progress progress;
  for (;;) {
    size_t n;
    if (!read_chunk_preamble<L>(r, h, number_type, &n)) { progress.finished = true; break; }
    ChunkMeta cm = read_chunk_meta(r, h.format, sizeof(L) * 8);
    ChunkDecoder cd(std::move(cm), number_type);
    PageDecoder<L> pd(cd, r, n);
    size_t limit;
    bool is_limited;
    if (dst_len < n) { limit = dst_len / FULL_BATCH_N * FULL_BATCH_N; is_limited = true; } else { limit = dst_len; is_limited = false; }
    Progress p = pd.read(dst, limit);
    dst += p.n_processed;
    dst_len -= p.n_processed;
    progress.n_processed += p.n_processed;
    if (dst_len != 0) {
      Progress p2 = pd.read(incomplete.data(), FULL_BATCH_N);
      size_t np = std::min(dst_len, p2.n_processed);
      std::memcpy(dst, incomplete.data(), np * sizeof(L));
      dst += np;
      dst_len -= np;
      progress.n_processed += np;
    }
    if (dst_len == 0 && is_limited) break;
  }
  return progress;
}

// standalone/guarantee.rs:11-38 + wrapped/guarantee.rs:35-37
inline size_t standalone_header_size() { return 4 + 1 + (BITS_TO_ENCODE_VARINT_POWER + 64 + BITS_TO_ENCODE_STANDALONE_VERSION + 7) / 8 + 2; }
inline size_t wrapped_chunk_size(Bitlen latent_bits, size_t n) {
  ChunkMeta base;
  base.number_bits = latent_bits;
  base.primary.latent_bits = latent_bits;
  base.primary.bins = {Bin{1, 0, latent_bits}};
  return base.max_size() + (n * size_t(latent_bits) + 7) / 8;
}
inline size_t standalone_chunk_size(Bitlen latent_bits, size_t n) { return 1 + 3 + wrapped_chunk_size(latent_bits, n); }
inline size_t standalone_file_size(Bitlen latent_bits, size_t n, const ChunkConfig& paging) {
  size_t res = standalone_header_size();
  for (size_t c : n_per_page(paging, n)) res += standalone_chunk_size(latent_bits, c);
  return res + 1;
}

}  // namespace pco_oracle
