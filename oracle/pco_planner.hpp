// ORACLE — TEST INFRASTRUCTURE ONLY (see pco_core.hpp header).
// Chunk planner: equal-count histogram (partial quicksort), bin optimisation DP,
// tANS weight quantisation.  Bit-exactness of "same bins" rests on this file.
#pragma once
#include <atomic>

#include "pco_format.hpp"

namespace pco_oracle {

// ---------------------------------------------------------------------------
// pco/src/sort_utils.rs
// ---------------------------------------------------------------------------
// sort_utils.rs:5-56
template <typename L>
inline L choose_pivot(const L* v, size_t len) {
  constexpr size_t SHORTEST_MEDIAN_OF_MEDIANS = 50;
  size_t a = len / 4, b = len / 2, c = (len * 3) / 4;
  if (len >= 8) {
    auto sort2 = [&](size_t& x, size_t& y) { if (v[y] < v[x]) std::swap(x, y); };
    auto sort3 = [&](size_t& x, size_t& y, size_t& z) { sort2(x, y); sort2(y, z); sort2(x, y); };
    if (len >= SHORTEST_MEDIAN_OF_MEDIANS) {
      auto sort_adjacent = [&](size_t& x) {
        size_t lo = x - 1, hi = x + 1;
        sort3(lo, x, hi);
      };
      sort_adjacent(a);
      sort_adjacent(b);
      sort_adjacent(c);
    }
    sort3(a, b, c);
  }
  return v[b];
}

// sort_utils.rs:61-105 (64-bit usize branch)
template <typename L>
inline void break_patterns(L* v, size_t len) {
  if (len >= 8) {
    uint64_t seed = len;
    auto gen = [&]() {
      uint64_t r = seed;
      r ^= r << 13;
      r ^= r >> 7;
      r ^= r << 17;
      seed = r;
      return seed;
    };
    uint64_t modulus = 1;
    while (modulus < len) modulus <<= 1;  // next_power_of_two
    size_t pos = len / 4 * 2;
    for (size_t i = 0; i < 3; i++) {
      uint64_t other = gen() & (modulus - 1);
      if (other >= len) other -= len;
      std::swap(v[pos - 1 + i], v[other]);
    }
  }
}

// sort_utils.rs:109-126 (Lomuto partition)
template <typename L>
inline std::pair<size_t, bool> partition_lt(L* v, size_t len, L pivot) {
  size_t left_idx = 0;
  for (size_t pos = 0; pos < len; pos++) {
    L value = v[pos];
    bool lt = value < pivot;
    v[pos] = v[left_idx];
    v[left_idx] = value;
    left_idx += lt ? 1 : 0;
  }
  bool was_bad = 1 + std::min(left_idx, len - left_idx) < len / 8;
  return {left_idx, was_bad};
}

// sort_utils.rs:130-169
template <typename L>
inline void heapsort(L* x, size_t len) {
  auto sift_down = [&](size_t n, size_t node) {
    for (;;) {
      size_t child = 2 * node + 1;
      if (child >= n) break;
      if (child + 1 < n) child += (x[child] < x[child + 1]) ? 1 : 0;
      if (x[node] >= x[child]) break;
      std::swap(x[node], x[child]);
      node = child;
    }
  };
  for (size_t i = len / 2; i-- > 0;) sift_down(len, i);
  for (size_t i = len; i-- > 1;) {
    std::swap(x[0], x[i]);
    sift_down(i, 0);
  }
}

// ---------------------------------------------------------------------------
// pco/src/histograms.rs
// ---------------------------------------------------------------------------
// How often apply_quicksort_recurse ran out of good pivots and took the heapsort + apply_sorted fallback (:250-258), over the
// process.  Test infrastructure: the GPU planner does not reproduce that fallback, so the tests that compare it with the oracle
// check that their inputs never reach it.
inline std::atomic<uint64_t>& heapsort_fallbacks() {
  static std::atomic<uint64_t> count{0};
  return count;
}

template <typename L>
struct HistogramBin {
  size_t count;
  L lower, upper;
};

template <typename L>
struct HistogramBuilder {
  struct Bound { bool tight; L x; };
  uint64_t n, n_bins;
  Bitlen n_bins_log;
  size_t n_applied = 0, next_avail_bin_idx = 0;
  bool has_incomplete = false;
  HistogramBin<L> incomplete{};
  std::vector<HistogramBin<L>> dst;

  HistogramBuilder(size_t n_, Bitlen log) : n(n_), n_bins(uint64_t(1) << log), n_bins_log(log) {}

  // histograms.rs:87-115
  void apply_incomplete(const L* v, size_t len, Bound lower, Bound upper) {
    if (len == 0) return;
    auto smin = [&]() { L m = LatentTraits<L>::MAX; for (size_t i = 0; i < len; i++) m = std::min(m, v[i]); return m; };
    auto smax = [&]() { L m = 0; for (size_t i = 0; i < len; i++) m = std::max(m, v[i]); return m; };
    if (has_incomplete) {
      incomplete.upper = upper.tight ? upper.x : smax();
      incomplete.count += len;
    } else {
      L lb = lower.tight ? lower.x : smin();
      L ub = upper.tight ? upper.x : smax();
      incomplete = HistogramBin<L>{len, lb, ub};
      has_incomplete = true;
    }
    n_applied += len;
  }
  // histograms.rs:118-130
  bool complete_bin(size_t bin_idx) {
    if (!has_incomplete) return false;
    next_avail_bin_idx = bin_idx + 1;
    dst.push_back(incomplete);
    has_incomplete = false;
    return true;
  }
  // histograms.rs:132-140
  size_t bin_idx(size_t c_count) const { return size_t((uint64_t(c_count) << n_bins_log) / n); }
  size_t c_count(size_t bin_idx) const { return size_t((uint64_t(bin_idx + 1) * n + n_bins - 1) >> n_bins_log); }

  // histograms.rs:142-161
  void apply_constant_run(const L* v, size_t len) {
    size_t start = n_applied;
    size_t mid = start + len / 2;
    size_t end = start + len;
    size_t b = bin_idx(mid);
    if (b > next_avail_bin_idx) {
      size_t spare = b - 1;
      if (!complete_bin(spare)) b = spare;
    }
    Bound cb{true, v[0]};
    apply_incomplete(v, len, cb, cb);
    if (end >= c_count(b)) complete_bin(b);
  }

  // histograms.rs:163-206
  void apply_sorted(const L* v, size_t len) {
    while (len > 0) {
      size_t target_bin_idx = bin_idx(n_applied);
      size_t target_c_count = c_count(target_bin_idx);
      size_t target_i = target_c_count - n_applied;
      if (target_i >= len) {
        apply_incomplete(v, len, Bound{true, v[0]}, Bound{true, v[len - 1]});
        if (target_i == len) complete_bin(target_bin_idx);
        break;
      }
      size_t l = target_i - 1, r = target_i;
      L target_x = v[l];
      while (l > 0 && v[l - 1] == target_x) l--;
      while (r < len && v[r] == target_x) r++;
      if (l > 0) apply_incomplete(v, l, Bound{true, v[0]}, Bound{true, v[l - 1]});
      apply_constant_run(v + l, r - l);
      v += r;
      len -= r;
    }
  }

  // histograms.rs:208-281
  void apply_quicksort_recurse(L* v, size_t len, Bound lb, Bound ub, uint32_t bad_pivot_limit) {
    if (len == 0) return;
    size_t target_bin_idx = bin_idx(n_applied);
    size_t target_c_count = c_count(target_bin_idx);
    size_t end = n_applied + len;
    if (end <= target_c_count) {
      apply_incomplete(v, len, lb, ub);
      if (end == target_c_count) complete_bin(target_bin_idx);
      return;
    }
    L loose_lb = lb.x;
    if (loose_lb == ub.x || len == 1) {
      apply_constant_run(v, len);
      return;
    }
    L tentative = choose_pivot(v, len);
    L pivot;
    Bound lhs_ub, rhs_lb;
    if (tentative > loose_lb) {
      pivot = tentative;
      lhs_ub = Bound{false, L(tentative - 1)};
      rhs_lb = Bound{true, tentative};
    } else {
      pivot = L(tentative + 1);
      lhs_ub = Bound{true, tentative};
      rhs_lb = Bound{false, L(tentative + 1)};
    }
    auto pr = partition_lt(v, len, pivot);
    size_t lhs_count = pr.first;
    if (pr.second) {
      bad_pivot_limit -= 1;
      if (bad_pivot_limit == 0) {
        heapsort_fallbacks().fetch_add(1, std::memory_order_relaxed);
        heapsort(v, lhs_count);
        heapsort(v + lhs_count, len - lhs_count);
        apply_sorted(v, len);
        return;
      }
      break_patterns(v, lhs_count);
      break_patterns(v + lhs_count, len - lhs_count);
    }
    apply_quicksort_recurse(v, lhs_count, lb, lhs_ub, bad_pivot_limit);
    apply_quicksort_recurse(v + lhs_count, len - lhs_count, rhs_lb, ub, bad_pivot_limit);
  }
};

// histograms.rs:294-298 (+ RecurseArgs::new :30-36)
template <typename L>
inline std::vector<HistogramBin<L>> histogram(L* latents, size_t n, Bitlen n_bins_log) {
  HistogramBuilder<L> st(n, n_bins_log);
  using Bound = typename HistogramBuilder<L>::Bound;
  uint32_t bad_pivot_limit = 1 + ilog2_u64(uint64_t(n) + 1);
  st.apply_quicksort_recurse(latents, n, Bound{false, 0}, Bound{false, LatentTraits<L>::MAX}, bad_pivot_limit);
  return std::move(st.dst);
}

// ---------------------------------------------------------------------------
// pco/src/bin_optimization.rs
// ---------------------------------------------------------------------------
inline uint32_t f32_bits(float x) { uint32_t b; std::memcpy(&b, &x, 4); return b; }
inline float f32_from_bits(uint32_t b) { float x; std::memcpy(&x, &b, 4); return x; }

// bin_optimization.rs:19-43
inline float log2_approx(float x) {
  const float Z = 0.674f;
  const uint32_t SIGNIF_MASK = 0x7FFFFF;
  const uint32_t Z_SIGNIF = f32_bits(Z) & SIGNIF_MASK;
  const float B = 2.0f / Z;
  const float C = -B / (6.0f * Z);
  const float A = -B - C;
  uint32_t bits = f32_bits(x);
  uint32_t exp = bits >> 23;
  uint32_t signif = bits & SIGNIF_MASK;
  uint32_t high_bit = signif > Z_SIGNIF ? 1 : 0;
  uint32_t log_int = exp + high_bit - 127;
  uint32_t exp2 = 0x7F ^ high_bit;
  float normalized = f32_from_bits((exp2 << 23) | signif);
  // log_int as f32 + A + normalized * (B + C * normalized), left-to-right, no FMA
  float t0 = float(log_int) + A;
  float t1 = C * normalized;
  float t2 = B + t1;
  float t3 = normalized * t2;
  return t0 + t3;
}

template <typename L>
struct BinCompressionInfo {
  Weight weight;
  L lower, upper;
  Bitlen offset_bits;
  Symbol symbol;
};

// bin_optimization.rs:46-57
template <typename L>
inline float bin_cost(float bin_meta_cost, L lower, L upper, Weight count, float total_count_log2) {
  float countf = float(count);
  float ans_cost = total_count_log2 - log2_approx(countf);
  float offset_cost = float(bits_to_encode_offset<L>(L(upper - lower)));
  float s = ans_cost + offset_cost;
  float p = s * countf;
  return bin_meta_cost + p;
}

// bin_optimization.rs:104-178
template <typename L>
inline std::vector<std::pair<size_t, size_t>> choose_optimized_partitioning(const std::vector<HistogramBin<L>>& bins,
                                                                             Bitlen ans_size_log) {
  const float SINGLE_BIN_SPEEDUP_WORTH = 0.1f, TRIVIAL_OFFSET_SPEEDUP_WORTH = 0.1f;
  size_t nb = bins.size();
  std::vector<uint32_t> c_counts(nb + 1);
  std::vector<float> best_costs(nb + 1);
  uint32_t c = 0;
  c_counts[0] = 0;
  best_costs[0] = 0.0f;
  for (size_t i = 0; i < nb; i++) {
    c += uint32_t(bins[i].count);
    c_counts[i + 1] = c;
    best_costs[i + 1] = std::numeric_limits<float>::quiet_NaN();
  }
  uint32_t total_count = c;
  float total_count_log2 = log2_approx(float(c));
  std::vector<size_t> best_js(nb);
  Bitlen l_bits = sizeof(L) * 8;
  float bin_meta_cost = float(ans_size_log + l_bits + bits_to_encode_offset_bits(l_bits));
  for (size_t i = 0; i < nb; i++) {
    float best_cost = std::numeric_limits<float>::max();
    size_t best_j = SIZE_MAX;
    L upper = bins[i].upper;
    uint32_t c_count_i = c_counts[i + 1];
    for (size_t j = i + 1; j-- > 0;) {
      L lower = bins[j].lower;
      float cost = best_costs[j] + bin_cost<L>(bin_meta_cost, lower, upper, c_count_i - c_counts[j], total_count_log2);
      if (cost < best_cost) {
        best_cost = cost;
        best_j = j;
      }
    }
    best_costs[i + 1] = best_cost;
    best_js[i] = best_j;
  }
  float best_cost = best_costs[nb];
  float single_bin_cost = bin_cost<L>(bin_meta_cost, bins[0].lower, bins[nb - 1].upper, total_count, total_count_log2);
  {
    float slack = SINGLE_BIN_SPEEDUP_WORTH * float(total_count);
    if (single_bin_cost < best_cost + slack) return {{0, nb - 1}};
  }
  bool all_trivial = true;
  for (auto& b : bins) if (b.lower != b.upper) { all_trivial = false; break; }
  if (all_trivial) {
    float cost = 0.0f;  // Iterator::sum for f32 (left-to-right)
    for (auto& b : bins) cost = cost + bin_cost<L>(bin_meta_cost, b.lower, b.upper, Weight(b.count), total_count_log2);
    float slack = TRIVIAL_OFFSET_SPEEDUP_WORTH * float(total_count);
    if (cost < best_cost + slack) {
      std::vector<std::pair<size_t, size_t>> p(nb);
      for (size_t i = 0; i < nb; i++) p[i] = {i, i};
      return p;
    }
  }
  // rewind (bin_optimization.rs:85-98)
  std::vector<std::pair<size_t, size_t>> part;
  size_t i = nb - 1;
  for (;;) {
    size_t j = best_js[i];
    part.push_back({j, i});
    if (j > 0) i = j - 1; else break;
  }
  std::reverse(part.begin(), part.end());
  return part;
}

// bin_optimization.rs:180-198
template <typename L>
inline std::vector<BinCompressionInfo<L>> optimize_bins(const std::vector<HistogramBin<L>>& bins, Bitlen ans_size_log) {
  auto part = choose_optimized_partitioning(bins, ans_size_log);
  std::vector<BinCompressionInfo<L>> res;
  res.reserve(part.size());
  for (size_t symbol = 0; symbol < part.size(); symbol++) {
    size_t j = part[symbol].first, i = part[symbol].second;
    size_t count = 0;
    for (size_t t = j; t <= i; t++) count += bins[t].count;
    res.push_back(BinCompressionInfo<L>{Weight(count), bins[j].lower, bins[i].upper,
                                        bits_to_encode_offset<L>(L(bins[i].upper - bins[j].lower)), Symbol(symbol)});
  }
  return res;
}

// ---------------------------------------------------------------------------
// pco/src/wrapped/chunk_compressor.rs:38-99 train_infos
// ---------------------------------------------------------------------------
template <typename L>
struct TrainedBins {
  std::vector<BinCompressionInfo<L>> infos;
  Bitlen ans_size_log = 0;
  std::vector<Weight> counts;
};

template <typename L>
inline TrainedBins<L> train_infos(std::vector<L> latents, Bitlen unoptimized_bins_log) {
  TrainedBins<L> out;
  if (latents.empty()) return out;
  size_t n_latents = latents.size();
  auto unoptimized = histogram<L>(latents.data(), n_latents, unoptimized_bins_log);
  Bitlen n_log_ceil = n_latents <= 1 ? 0 : ilog2_u64(n_latents - 1) + 1;
  Bitlen estimated_ans_size_log = std::min(std::min(unoptimized_bins_log + 2, Bitlen(MAX_COMPRESSION_LEVEL)), n_log_ceil);
  out.infos = optimize_bins<L>(unoptimized, estimated_ans_size_log);
  out.counts.reserve(out.infos.size());
  for (auto& info : out.infos) out.counts.push_back(info.weight);
  auto q = quantize_weights(out.counts, n_latents, estimated_ans_size_log);
  out.ans_size_log = q.first;
  for (size_t i = 0; i < out.infos.size(); i++) out.infos[i].weight = q.second[i];
  return out;
}

// chunk_compressor.rs:362-371
inline Bitlen choose_unoptimized_bins_log(size_t compression_level, size_t n) {
  Bitlen level = Bitlen(compression_level);
  Bitlen log_n = Bitlen(std::floor(std::log2(double(n))));
  Bitlen fast = log_n >= 4 ? log_n - 4 : 0;
  if (level <= fast) return level;
  return fast + (level - fast) / 2;
}

}  // namespace pco_oracle
