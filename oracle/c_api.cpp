// ORACLE — TEST INFRASTRUCTURE ONLY (see pco_core.hpp header).
// extern "C" surface used by tests/ (ctypes), __graft_entry__.smoke() and
// bench.py's cpu_baseline / --impl reference legs.  Never linked by the product.
#include <malloc.h>

#include <atomic>
#include <chrono>
#include <sstream>
#include <thread>

#include "pco_codec.hpp"

using namespace pco_oracle;

extern "C" {

// Same layout as PcoB200ChunkConfig in include/pco_b200.h (mirrors
// pco::ChunkConfig, pco/src/chunk_config.rs:193-224).
struct pco_oracle_config {
  uint32_t compression_level;
  uint32_t mode_spec;
  double float_mult_base;
  uint64_t int_mult_base;
  uint32_t float_quant_k;
  uint32_t delta_spec;
  uint32_t delta_order;
  uint32_t paging_spec;
  uint64_t max_page_n;
  const uint64_t* exact_page_ns;
  uint64_t n_exact_pages;
  uint32_t enable_8_bit;
  uint32_t reserved;
};

// One latent variable of a chunk written by pco_oracle_write_explicit_file: the bins as the chunk meta lists them, and the stored
// latents as (bin index, offset) pairs.  `moments` holds the delta state (`delta_order` latents) when the var uses the delta.
struct pco_oracle_explicit_var {
  uint32_t ans_size_log;
  uint32_t n_bins;
  const uint32_t* weights;
  const uint64_t* lowers;
  const uint32_t* offset_bits;
  uint64_t n_stored;
  const uint32_t* symbols;
  const uint64_t* offsets;
  const uint64_t* moments;
};

// One chunk: mode (ModeKind: 0 Classic, 1 IntMult, 2 FloatMult, 3 FloatQuant) with its parameter (IntMult base, FloatMult base as
// latent-ordered bits, FloatQuant k), consecutive delta of `delta_order` (0 = NoOp), and the primary and secondary vars.
struct pco_oracle_explicit_chunk {
  uint64_t n;
  uint32_t mode;
  uint32_t float_quant_k;
  uint64_t mode_base_latent;
  uint32_t delta_order;
  uint32_t secondary_uses_delta;
  pco_oracle_explicit_var vars[2];
};

}  // extern "C"

static thread_local std::string g_last_error;
static thread_local int g_last_kind = 0;

static ChunkConfig to_config(const pco_oracle_config* c) {
  ChunkConfig cfg;
  if (!c) {
    // pco_c/src/lib.rs:34-55 default: level 8, Auto/Auto, enable_8_bit
    cfg.enable_8_bit = true;
    return cfg;
  }
  cfg.compression_level = c->compression_level;
  cfg.mode_kind = ModeSpecKind(c->mode_spec);
  cfg.float_mult_base = c->float_mult_base;
  cfg.int_mult_base = c->int_mult_base;
  cfg.float_quant_k = c->float_quant_k;
  cfg.delta_kind = DeltaSpecKind(c->delta_spec);
  cfg.delta_order = c->delta_order;
  cfg.paging_kind = PagingKind(c->paging_spec);
  cfg.max_page_n = c->max_page_n == 0 ? DEFAULT_MAX_PAGE_N : size_t(c->max_page_n);
  if (c->paging_spec == 1) cfg.exact_pages.assign(c->exact_page_ns, c->exact_page_ns + c->n_exact_pages);
  cfg.enable_8_bit = c->enable_8_bit != 0;
  return cfg;
}

template <typename Fn>
static int guarded(Fn&& fn) {
  try {
    fn();
    g_last_kind = 0;
    return 0;
  } catch (const PcoError& e) {
    g_last_error = e.msg;
    g_last_kind = int(e.kind);
    return int(e.kind);
  } catch (const std::exception& e) {
    g_last_error = e.what();
    g_last_kind = 99;
    return 99;
  }
}

template <typename Fn>
static void dispatch_bits(uint8_t dtype, Fn&& fn) {
  if (!number_type_valid(dtype)) invalid_argument("unknown number type byte");
  switch (number_type_bits(dtype)) {
    case 8: fn(uint8_t(0)); break;
    case 16: fn(uint16_t(0)); break;
    case 32: fn(uint32_t(0)); break;
    default: fn(uint64_t(0)); break;
  }
}

static uint8_t* dup_bytes(const std::vector<uint8_t>& v, size_t* len) {
  uint8_t* p = static_cast<uint8_t*>(std::malloc(v.size() ? v.size() : 1));
  if (v.size()) std::memcpy(p, v.data(), v.size());
  *len = v.size();
  return p;
}

struct OracleChunkCompressor {
  Bitlen bits;
  std::unique_ptr<ChunkCompressor<uint8_t>> c8;
  std::unique_ptr<ChunkCompressor<uint16_t>> c16;
  std::unique_ptr<ChunkCompressor<uint32_t>> c32;
  std::unique_ptr<ChunkCompressor<uint64_t>> c64;
};

template <typename Fn>
static void with_cc(void* handle, Fn&& fn) {
  auto* h = static_cast<OracleChunkCompressor*>(handle);
  switch (h->bits) {
    case 8: fn(*h->c8); break;
    case 16: fn(*h->c16); break;
    case 32: fn(*h->c32); break;
    default: fn(*h->c64); break;
  }
}

// ----- explicit streams: a chunk built from given bins and (bin, offset) pairs ----------------------------------------------------
// The chunk meta of an explicit chunk, checked against everything the format's reader requires (metadata/chunk_latent_var.rs:102-157,
// mode validity, delta order); anything else is a valid stream, so whatever passes decodes.
static ChunkMeta explicit_chunk_meta(uint8_t dtype, const pco_oracle_explicit_chunk& c) {
  if (!number_type_valid(dtype)) invalid_argument("unknown number type byte");
  const Bitlen bits = number_type_bits(dtype);
  if (c.n == 0 || c.n > MAX_ENTRIES) invalid_argument("chunk count must be in 1..2^24");
  if (c.mode > uint32_t(ModeKind::FloatQuant)) invalid_argument("mode must be Classic, IntMult, FloatMult or FloatQuant");
  if (c.delta_order > MAX_CONSECUTIVE_DELTA_ORDER) invalid_argument("consecutive delta order exceeds 7");
  ChunkMeta m;
  m.number_bits = bits;
  m.mode.kind = ModeKind(c.mode);
  m.mode.base_latent = bits == 64 ? c.mode_base_latent : c.mode_base_latent & ((uint64_t(1) << bits) - 1);
  if (c.mode_base_latent != m.mode.base_latent) invalid_argument("mode base exceeds the number type");
  m.mode.k = c.float_quant_k;
  if (!mode_is_valid(m.mode, dtype)) invalid_argument("mode or mode parameter invalid for the number type");
  if (c.delta_order) {
    m.delta.kind = DeltaKind::Consecutive;
    m.delta.order = c.delta_order;
    m.delta.secondary_uses_delta = c.secondary_uses_delta != 0;
  } else if (c.secondary_uses_delta) {
    invalid_argument("secondary_uses_delta without a delta encoding");
  }
  m.has_secondary = mode_has_secondary(m.mode);
  for (int v = 0; v < (m.has_secondary ? 2 : 1); v++) {
    const pco_oracle_explicit_var& s = c.vars[v];
    LatentVarMeta& vm = v == 0 ? m.primary : m.secondary;
    vm.latent_bits = bits;
    vm.ans_size_log = s.ans_size_log;
    if (s.ans_size_log > MAX_ANS_BITS) invalid_argument("ans_size_log exceeds 14");
    if (s.n_bins > (uint64_t(1) << s.ans_size_log)) invalid_argument("more bins than tANS states");
    if (s.n_bins == 1 && s.ans_size_log > 0) invalid_argument("one bin with ans_size_log > 0");
    uint64_t total = 0;
    for (uint32_t i = 0; i < s.n_bins; i++) {
      if (s.weights[i] == 0) invalid_argument("bin weight 0");
      if (s.offset_bits[i] > bits) invalid_argument("offset_bits exceeds the latent type");
      if (bits < 64 && s.lowers[i] >> bits) invalid_argument("bin lower exceeds the latent type");
      total += s.weights[i];
      vm.bins.push_back(Bin{s.weights[i], s.lowers[i], s.offset_bits[i]});
    }
    if (s.n_bins > 0 && total != (uint64_t(1) << s.ans_size_log)) invalid_argument("weights do not sum to 2^ans_size_log");
    const size_t n_state = delta_for_latent_var(m.delta, v == 0 ? VarKey::Primary : VarKey::Secondary).n_latents_per_state();
    if (s.n_stored != (c.n > n_state ? c.n - n_state : 0)) invalid_argument("stored count must be n minus the var's delta order");
    if (s.n_stored > 0 && s.n_bins == 0) invalid_argument("stored latents without bins");
    for (uint64_t i = 0; i < s.n_stored; i++) {
      if (s.symbols[i] >= s.n_bins) invalid_argument("symbol is not a bin");
      if (s.offset_bits[s.symbols[i]] < 64 && s.offsets[i] >> s.offset_bits[s.symbols[i]]) invalid_argument("offset does not fit its bin's offset_bits");
    }
    for (size_t i = 0; i < n_state; i++)
      if (bits < 64 && s.moments[i] >> bits) invalid_argument("moment exceeds the latent type");
  }
  return m;
}

// The page of an explicit chunk (chunk_compressor.rs:624-705): the interleaved tANS states come from encoding each var's symbols in
// reverse, batch by batch, as the compressor does; the page meta holds the moments and the final states.
static void write_explicit_page(const ChunkMeta& m, const pco_oracle_explicit_chunk& c, std::vector<uint8_t>& dst) {
  struct Var {
    const pco_oracle_explicit_var* s;
    Bitlen size_log;
    std::vector<AnsState> vals;
    std::vector<Bitlen> nbits;
    AnsState finals[ANS_INTERLEAVING];
  };
  std::vector<Var> vars;
  for (int v = 0; v < (m.has_secondary ? 2 : 1); v++) {
    const pco_oracle_explicit_var& s = c.vars[v];
    Var x{&s, s.ans_size_log, std::vector<AnsState>(s.n_stored), std::vector<Bitlen>(s.n_stored, 0), {}};
    const AnsState table = AnsState(1) << s.ans_size_log;
    for (size_t j = 0; j < ANS_INTERLEAVING; j++) x.finals[j] = table;
    if (s.n_bins > 1) {
      AnsEncoder enc(ans_spec_from_weights(s.ans_size_log, std::vector<Weight>(s.weights, s.weights + s.n_bins)));
      const size_t n_batches = (s.n_stored + FULL_BATCH_N - 1) / FULL_BATCH_N;
      for (size_t b = n_batches; b-- > 0;) {
        const size_t start = b * FULL_BATCH_N, end = std::min<size_t>(start + FULL_BATCH_N, s.n_stored);
        for (size_t i = end; i-- > start;) {
          AnsState& st = x.finals[(i - start) % ANS_INTERLEAVING];
          Bitlen nb;
          const AnsState ns = enc.encode(st, s.symbols[i], &nb);
          x.vals[i] = AnsState(lowest_bits_u64(st, nb));
          x.nbits[i] = nb;
          st = ns;
        }
      }
    }
    vars.push_back(std::move(x));
  }
  BitWriter w(dst);
  for (size_t v = 0; v < vars.size(); v++) {
    const LatentVarMeta& vm = v == 0 ? m.primary : m.secondary;
    const size_t n_state = delta_for_latent_var(m.delta, v == 0 ? VarKey::Primary : VarKey::Secondary).n_latents_per_state();
    for (size_t i = 0; i < n_state; i++) w.write_uint(vars[v].s->moments[i], vm.latent_bits);
    for (size_t j = 0; j < ANS_INTERLEAVING; j++) w.write_uint(vars[v].finals[j] - (AnsState(1) << vars[v].size_log), vm.ans_size_log);
  }
  w.finish_byte();
  for (uint64_t start = 0; start < c.n; start += FULL_BATCH_N) {
    for (const Var& x : vars) {
      const pco_oracle_explicit_var& s = *x.s;
      const uint64_t end = std::min<uint64_t>(start + FULL_BATCH_N, s.n_stored);
      if (s.n_bins > 1)
        for (uint64_t i = start; i < end; i++) w.write_uint(x.vals[i], x.nbits[i]);
      for (uint64_t i = start; i < end; i++) w.write_uint(s.offsets[i], s.offset_bits[s.symbols[i]]);
    }
  }
  w.finish();
}

extern "C" {

// A standalone file (header, each chunk's type byte, count, meta and page, terminator) of chunks with explicit bins and stored latents.
// `metas` / `pages`, when not null, receive each chunk's wrapped meta and page bytes back to back, with their lengths in
// meta_lens / page_lens (n_chunks entries each).  An invalid spec is InvalidArgument.
int pco_oracle_write_explicit_file(uint8_t dtype, const pco_oracle_explicit_chunk* chunks, size_t n_chunks, uint8_t** out, size_t* out_len,
                                   uint8_t** metas, size_t* meta_lens, uint8_t** pages, size_t* page_lens) {
  return guarded([&] {
    uint64_t total = 0;
    std::vector<ChunkMeta> cms;
    for (size_t i = 0; i < n_chunks; i++) {
      cms.push_back(explicit_chunk_meta(dtype, chunks[i]));
      total += chunks[i].n;
    }
    std::vector<uint8_t> dst, all_metas, all_pages;
    write_standalone_header(dst, total, 0);
    for (size_t i = 0; i < n_chunks; i++) {
      BitWriter w(dst);
      w.write_aligned_bytes(&dtype, 1);
      w.write_uint(chunks[i].n - 1, BITS_TO_ENCODE_N_ENTRIES);
      w.finish();
      std::vector<uint8_t> meta, page;
      write_chunk_meta(cms[i], meta);
      write_explicit_page(cms[i], chunks[i], page);
      dst.insert(dst.end(), meta.begin(), meta.end());
      dst.insert(dst.end(), page.begin(), page.end());
      all_metas.insert(all_metas.end(), meta.begin(), meta.end());
      all_pages.insert(all_pages.end(), page.begin(), page.end());
      if (meta_lens) meta_lens[i] = meta.size();
      if (page_lens) page_lens[i] = page.size();
    }
    dst.push_back(MAGIC_TERMINATION_BYTE);
    size_t unused;
    if (metas) *metas = dup_bytes(all_metas, &unused);
    if (pages) *pages = dup_bytes(all_pages, &unused);
    *out = dup_bytes(dst, out_len);
  });
}

const char* pco_oracle_last_error() { return g_last_error.c_str(); }
void pco_oracle_free(void* p) { std::free(p); }

// pco::standalone::simple_compress (uniform_type=0) / simple_compress_into (uniform_type=1)
int pco_oracle_simple_compress(const void* nums, size_t n, uint8_t dtype, const pco_oracle_config* config, int uniform_type,
                               uint8_t** out, size_t* out_len) {
  return guarded([&] {
    ChunkConfig cfg = to_config(config);
    std::vector<uint8_t> dst;
    dispatch_bits(dtype, [&](auto tag) {
      using L = decltype(tag);
      simple_compress<L>(static_cast<const L*>(nums), n, dtype, cfg, uniform_type != 0, dst);
    });
    *out = dup_bytes(dst, out_len);
  });
}

// pco::standalone::simple_decompress
int pco_oracle_simple_decompress(const uint8_t* src, size_t src_len, uint8_t dtype, void** out, size_t* n_out) {
  return guarded([&] {
    dispatch_bits(dtype, [&](auto tag) {
      using L = decltype(tag);
      std::vector<L> v;
      simple_decompress<L>(src, src_len, dtype, v);
      L* p = static_cast<L*>(std::malloc(v.size() ? v.size() * sizeof(L) : 1));
      if (!v.empty()) std::memcpy(p, v.data(), v.size() * sizeof(L));
      *out = p;
      *n_out = v.size();
    });
  });
}

// pco::standalone::simple_decompress_into
int pco_oracle_simple_decompress_into(const uint8_t* src, size_t src_len, uint8_t dtype, void* dst, size_t dst_len,
                                      size_t* n_processed, int* finished) {
  return guarded([&] {
    dispatch_bits(dtype, [&](auto tag) {
      using L = decltype(tag);
      Progress p = simple_decompress_into<L>(src, src_len, dtype, static_cast<L*>(dst), dst_len);
      *n_processed = p.n_processed;
      *finished = p.finished ? 1 : 0;
    });
  });
}

// bench.py's CPU arm: compress, then decompress, `n_chunks` independent chunks of `chunk_n` numbers with `threads` native
// threads (one chunk per task; pco_cli/src/bench/mod.rs times its codecs the same way, per-thread), verifying the round
// trip.  Native threads because the Python harness's per-call buffer copies hold the GIL and throttle 100+ threads.
int pco_oracle_bench_roundtrip(const void* nums, size_t n_chunks, size_t chunk_n, uint8_t dtype, const pco_oracle_config* config, int threads,
                               double* compress_s, double* decompress_s, uint64_t* compressed_bytes) {
  return guarded([&] {
    ChunkConfig cfg = to_config(config);
    // the port allocates its MiB-sized scratch vectors per chunk; with glibc's default each is an mmap / munmap and the
    // threads serialise in the kernel (8 threads: 1.6x one thread).  Keep them in the per-thread arenas instead.
    mallopt(M_MMAP_THRESHOLD, 1 << 30);
    mallopt(M_TRIM_THRESHOLD, 1 << 30);
    dispatch_bits(dtype, [&](auto tag) {
      using L = decltype(tag);
      const L* base = static_cast<const L*>(nums);
      std::vector<std::vector<uint8_t>> comp(n_chunks);
      std::vector<std::string> errors(size_t(std::max(threads, 1)));
      auto run = [&](auto&& body) -> double {
        std::atomic<size_t> next{0};
        std::vector<std::thread> pool;
        auto t0 = std::chrono::steady_clock::now();
        for (int t = 0; t < std::max(threads, 1); t++)
          pool.emplace_back([&, t] {
            try {
              for (size_t c = next.fetch_add(1); c < n_chunks; c = next.fetch_add(1)) body(c);
            } catch (const std::exception& e) { errors[size_t(t)] = e.what(); }
          });
        for (auto& th : pool) th.join();
        return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
      };
      *compress_s = run([&](size_t c) { simple_compress<L>(base + c * chunk_n, chunk_n, dtype, cfg, false, comp[c]); });
      std::atomic<size_t> bad{0};
      *decompress_s = run([&](size_t c) {
        std::vector<L> v;
        simple_decompress<L>(comp[c].data(), comp[c].size(), dtype, v);
        if (v.size() != chunk_n || std::memcmp(v.data(), base + c * chunk_n, chunk_n * sizeof(L)) != 0) bad.fetch_add(1);
      });
      for (const auto& e : errors)
        if (!e.empty()) throw PcoError(ErrorKind::Io, "bench worker: " + e);
      if (bad.load()) throw PcoError(ErrorKind::Corruption, "bench round trip mismatch");
      uint64_t total = 0;
      for (const auto& v : comp) total += v.size();
      *compressed_bytes = total;
    });
  });
}

size_t pco_oracle_file_size_guarantee(size_t n, uint8_t dtype) {
  if (!number_type_valid(dtype)) return 0;
  ChunkConfig cfg;
  try {
    return standalone_file_size(number_type_bits(dtype), n, cfg);
  } catch (...) {
    return 0;
  }
}

// ----- wrapped API ----------------------------------------------------------

int pco_oracle_chunk_compressor_new(const void* nums, size_t n, uint8_t dtype, const pco_oracle_config* config, void** handle) {
  return guarded([&] {
    ChunkConfig cfg = to_config(config);
    fallback_margins().clear();
    auto* h = new OracleChunkCompressor();
    h->bits = number_type_valid(dtype) ? number_type_bits(dtype) : 0;
    try {
      dispatch_bits(dtype, [&](auto tag) {
        using L = decltype(tag);
        auto cc = new_chunk_compressor<L>(static_cast<const L*>(nums), n, dtype, cfg);
        if constexpr (sizeof(L) == 1) h->c8 = std::move(cc);
        else if constexpr (sizeof(L) == 2) h->c16 = std::move(cc);
        else if constexpr (sizeof(L) == 4) h->c32 = std::move(cc);
        else h->c64 = std::move(cc);
      });
    } catch (...) {
      delete h;
      throw;
    }
    *handle = h;
  });
}
void pco_oracle_chunk_compressor_free(void* handle) { delete static_cast<OracleChunkCompressor*>(handle); }

size_t pco_oracle_chunk_compressor_n_pages(void* handle) {
  size_t r = 0;
  with_cc(handle, [&](auto& cc) { r = cc.n_pages(); });
  return r;
}
size_t pco_oracle_chunk_compressor_page_n(void* handle, size_t i) {
  size_t r = 0;
  with_cc(handle, [&](auto& cc) { r = cc.page_ns[i]; });
  return r;
}
int pco_oracle_chunk_compressor_write_meta(void* handle, uint8_t** out, size_t* out_len) {
  return guarded([&] {
    std::vector<uint8_t> dst;
    with_cc(handle, [&](auto& cc) { cc.write_meta(dst); });
    *out = dup_bytes(dst, out_len);
  });
}
int pco_oracle_chunk_compressor_write_page(void* handle, size_t page_idx, uint8_t** out, size_t* out_len) {
  return guarded([&] {
    std::vector<uint8_t> dst;
    with_cc(handle, [&](auto& cc) { cc.write_page(page_idx, dst); });
    *out = dup_bytes(dst, out_len);
  });
}

// wrapped decode of one page: `meta` = wrapped chunk meta bytes, `page` = page bytes (format 4.1)
int pco_oracle_wrapped_decompress_page(const uint8_t* meta, size_t meta_len, const uint8_t* page, size_t page_len, uint8_t dtype,
                                       size_t page_n, void* dst, size_t* meta_consumed, size_t* page_consumed) {
  return guarded([&] {
    dispatch_bits(dtype, [&](auto tag) {
      using L = decltype(tag);
      PaddedSrc pm(meta, meta_len);
      BitReader rm(pm.buf.data(), pm.len);
      FormatVersion fv;
      ChunkMeta cm = read_chunk_meta(rm, fv, sizeof(L) * 8);
      *meta_consumed = rm.byte_idx();
      ChunkDecoder cd(std::move(cm), dtype);
      PaddedSrc pp(page, page_len);
      BitReader rp(pp.buf.data(), pp.len);
      PageDecoder<L> pd(cd, rp, page_n);
      pd.read(static_cast<L*>(dst), page_n);
      *page_consumed = rp.byte_idx();
    });
  });
}

// ----- inspection: JSON description of every chunk in a standalone file -----
// Also reports, per chunk, byte offsets of meta/page so tests can slice streams.
int pco_oracle_inspect(const uint8_t* src, size_t src_len, uint8_t dtype, char** json_out) {
  return guarded([&] {
    std::ostringstream os;
    dispatch_bits(dtype, [&](auto tag) {
      using L = decltype(tag);
      PaddedSrc ps(src, src_len);
      BitReader r(ps.buf.data(), ps.len);
      StandaloneHeader h = read_standalone_header(r);
      os << "{\"standalone_version\":" << h.standalone_version << ",\"uniform_type\":" << int(h.uniform_type)
         << ",\"n_hint\":" << h.n_hint << ",\"format\":[" << int(h.format.major) << "," << int(h.format.minor) << "],\"chunks\":[";
      size_t n;
      bool first = true;
      for (;;) {
        size_t chunk_start = r.byte_idx();
        if (!read_chunk_preamble<L>(r, h, dtype, &n)) break;
        size_t meta_start = r.byte_idx();
        ChunkMeta cm = read_chunk_meta(r, h.format, sizeof(L) * 8);
        size_t page_start = r.byte_idx();
        if (!first) os << ",";
        first = false;
        os << "{\"n\":" << n << ",\"chunk_start\":" << chunk_start << ",\"meta_start\":" << meta_start << ",\"page_start\":" << page_start
           << ",\"mode\":" << int(cm.mode.kind) << ",\"mode_base_latent\":" << cm.mode.base_latent << ",\"mode_k\":" << cm.mode.k
           << ",\"dict_len\":" << cm.mode.dict.size() << ",\"delta\":" << int(cm.delta.kind) << ",\"delta_order\":" << cm.delta.order
           << ",\"vars\":[";
        bool fv = true;
        for (auto& kv : cm.vars()) {
          if (!fv) os << ",";
          fv = false;
          os << "{\"key\":" << int(kv.first) << ",\"latent_bits\":" << kv.second->latent_bits << ",\"ans_size_log\":" << kv.second->ans_size_log
             << ",\"bins\":[";
          for (size_t i = 0; i < kv.second->bins.size(); i++) {
            const Bin& b = kv.second->bins[i];
            if (i) os << ",";
            os << "[" << b.weight << "," << b.lower << "," << b.offset_bits << "]";
          }
          os << "]}";
        }
        os << "]";
        ChunkDecoder cd(cm, dtype);
        PageDecoder<L> pd(cd, r, n);
        std::vector<L> tmp(n);
        pd.read(tmp.data(), n);
        os << ",\"chunk_end\":" << r.byte_idx() << "}";
      }
      os << "],\"end\":" << r.byte_idx() << "}";
    });
    std::string s = os.str();
    char* p = static_cast<char*>(std::malloc(s.size() + 1));
    std::memcpy(p, s.c_str(), s.size() + 1);
    *json_out = p;
  });
}

// ----- primitive-level known-answer-test hooks ------------------------------
// pco/src/ans/spec.rs:37 spread_state_symbols
int pco_oracle_kat_spread(uint32_t size_log, const uint32_t* weights, size_t n, uint32_t* out_state_symbols) {
  return guarded([&] {
    AnsSpec s = ans_spec_from_weights(size_log, std::vector<Weight>(weights, weights + n));
    for (size_t i = 0; i < s.state_symbols.size(); i++) out_state_symbols[i] = s.state_symbols[i];
  });
}
// pco/src/ans/encoding.rs:95 / :156
int pco_oracle_kat_quantize_weights_to(const uint32_t* counts, size_t n, size_t total, uint32_t size_log, uint32_t* out) {
  return guarded([&] {
    auto w = quantize_weights_to(std::vector<Weight>(counts, counts + n), total, size_log);
    for (size_t i = 0; i < w.size(); i++) out[i] = w[i];
  });
}
int pco_oracle_kat_quantize_weights(const uint32_t* counts, size_t n, size_t total, uint32_t max_size_log, uint32_t* out_size_log,
                                    uint32_t* out) {
  return guarded([&] {
    auto q = quantize_weights(std::vector<Weight>(counts, counts + n), total, max_size_log);
    *out_size_log = q.first;
    for (size_t i = 0; i < q.second.size(); i++) out[i] = q.second[i];
  });
}
float pco_oracle_kat_log2_approx(float x) { return log2_approx(x); }
// pco/src/histograms.rs:294 (u32); out = [count, lower, upper] triples; returns #bins via *n_out
int pco_oracle_kat_histogram_u32(const uint32_t* latents, size_t n, uint32_t n_bins_log, uint64_t* out, size_t* n_out) {
  return guarded([&] {
    std::vector<uint32_t> v(latents, latents + n);
    auto bins = histogram<uint32_t>(v.data(), n, n_bins_log);
    for (size_t i = 0; i < bins.size(); i++) {
      out[3 * i] = bins[i].count;
      out[3 * i + 1] = bins[i].lower;
      out[3 * i + 2] = bins[i].upper;
    }
    *n_out = bins.size();
  });
}
int pco_oracle_kat_histogram_u64(const uint64_t* latents, size_t n, uint32_t n_bins_log, uint64_t* out, size_t* n_out) {
  return guarded([&] {
    std::vector<uint64_t> v(latents, latents + n);
    auto bins = histogram<uint64_t>(v.data(), n, n_bins_log);
    for (size_t i = 0; i < bins.size(); i++) {
      out[3 * i] = bins[i].count;
      out[3 * i + 1] = bins[i].lower;
      out[3 * i + 2] = bins[i].upper;
    }
    *n_out = bins.size();
  });
}
// histograms.rs:250-258: heapsort fallbacks taken by every histogram built in this process so far
uint64_t pco_oracle_heapsort_fallbacks(void) { return heapsort_fallbacks().load(std::memory_order_relaxed); }

// chunk_compressor.rs:502-541: worst_case_size and baseline (bytes) of each chunk of this thread's last compress (a standalone
// file from pco_oracle_simple_compress, or one wrapped chunk from pco_oracle_chunk_compressor_new), in chunk order; the chunk
// fell back where worst > baseline.  Returns the chunk count, writes up to `cap`.
size_t pco_oracle_last_fallback_margins(uint64_t* worst, uint64_t* baseline, size_t cap) {
  const auto& m = fallback_margins();
  for (size_t i = 0; i < m.size() && i < cap; i++) {
    worst[i] = m[i].first;
    baseline[i] = m[i].second;
  }
  return m.size();
}
// histograms.rs apply_sorted over several pre-sorted slices (tests :375-386)
int pco_oracle_kat_histogram_sorted_u32(const uint32_t* latents, const size_t* slice_lens, size_t n_slices, size_t n, uint32_t n_bins_log,
                                        uint64_t* out, size_t* n_out, uint64_t* incomplete_out, int* has_incomplete) {
  return guarded([&] {
    HistogramBuilder<uint32_t> st(n, n_bins_log);
    size_t off = 0;
    for (size_t s = 0; s < n_slices; s++) {
      st.apply_sorted(latents + off, slice_lens[s]);
      off += slice_lens[s];
    }
    for (size_t i = 0; i < st.dst.size(); i++) {
      out[3 * i] = st.dst[i].count;
      out[3 * i + 1] = st.dst[i].lower;
      out[3 * i + 2] = st.dst[i].upper;
    }
    *n_out = st.dst.size();
    *has_incomplete = st.has_incomplete ? 1 : 0;
    if (st.has_incomplete) {
      incomplete_out[0] = st.incomplete.count;
      incomplete_out[1] = st.incomplete.lower;
      incomplete_out[2] = st.incomplete.upper;
    }
  });
}
// pco/src/bin_optimization.rs:180 (u32); in = [count, lower, upper] triples; out = [weight, lower, upper, offset_bits, symbol]
int pco_oracle_kat_optimize_bins_u32(const uint64_t* in, size_t n, uint32_t ans_size_log, uint64_t* out, size_t* n_out) {
  return guarded([&] {
    std::vector<HistogramBin<uint32_t>> bins;
    for (size_t i = 0; i < n; i++) bins.push_back({size_t(in[3 * i]), uint32_t(in[3 * i + 1]), uint32_t(in[3 * i + 2])});
    auto res = optimize_bins<uint32_t>(bins, ans_size_log);
    for (size_t i = 0; i < res.size(); i++) {
      out[5 * i] = res[i].weight;
      out[5 * i + 1] = res[i].lower;
      out[5 * i + 2] = res[i].upper;
      out[5 * i + 3] = res[i].offset_bits;
      out[5 * i + 4] = res[i].symbol;
    }
    *n_out = res.size();
  });
}
// pco/src/bit_writer.rs:176-203: sequence of (value, nbits) writes -> bytes
int pco_oracle_kat_bit_writer(const uint64_t* vals, const uint32_t* nbits, size_t n, uint8_t** out, size_t* out_len) {
  return guarded([&] {
    std::vector<uint8_t> dst;
    BitWriter w(dst);
    for (size_t i = 0; i < n; i++) w.write_uint(vals[i], nbits[i]);
    w.finish();
    *out = dup_bytes(dst, out_len);
  });
}
// pco/src/ans/mod.rs:26-64 assert_recovers: encode symbols in reverse with a given spec, return byte length and
// decode them back; returns 0 on success and writes the compressed length
int pco_oracle_kat_ans_roundtrip(uint32_t size_log, const uint32_t* state_symbols, size_t table_size, const uint32_t* weights,
                                 size_t n_weights, const uint32_t* symbols, size_t n, size_t* byte_len) {
  return guarded([&] {
    AnsSpec spec;
    spec.size_log = size_log;
    spec.state_symbols.assign(state_symbols, state_symbols + table_size);
    spec.symbol_weights.assign(weights, weights + n_weights);
    AnsEncoder enc(spec);
    AnsState state = enc.default_state();
    std::vector<std::pair<AnsState, Bitlen>> to_write;
    for (size_t i = n; i-- > 0;) {
      Bitlen bl;
      AnsState ns = enc.encode(state, symbols[i], &bl);
      to_write.push_back({state, bl});
      state = ns;
    }
    std::vector<uint8_t> dst;
    BitWriter w(dst);
    for (size_t i = to_write.size(); i-- > 0;) w.write_uint(lowest_bits_u64(to_write[i].first, to_write[i].second), to_write[i].second);
    w.finish();
    *byte_len = dst.size();
    PaddedSrc ps(dst.data(), dst.size());
    BitReader r(ps.buf.data(), ps.len);
    auto nodes = ans_decoder_nodes(spec, {});
    AnsState idx = state - AnsState(spec.table_size());
    for (size_t i = 0; i < n; i++) {
      if (spec.state_symbols[idx] != symbols[i]) corruption("ans roundtrip mismatch");
      const AnsNode& nd = nodes[idx];
      idx = AnsState(nd.next_state_idx_base) + AnsState(r.read_uint(nd.bits_to_read));
    }
  });
}
// pco/src/delta/consecutive.rs:57-78 (u32)
// choose_mode_sample's index draw (sampling.rs:73-95); returns -1 when n < MIN_SAMPLE
int pco_oracle_kat_mode_sample_indices(size_t n, uint64_t* out, size_t* n_out) {
  return guarded([&] {
    std::vector<size_t> idx;
    if (!choose_mode_sample_indices(n, &idx)) { *n_out = 0; return; }
    for (size_t i = 0; i < idx.size(); i++) out[i] = idx[i];
    *n_out = idx.size();
  });
}

// pco/src/mode/int_mult.rs unit tests (:238-320): calc_gcd, calc_triple_gcd, solve_root_by_false_position (case 0: x*x-1 on
// [-0.9,2], 1: x*x, 2: the zero function on [0,1]; returns 0 when there is no root), choose_candidate_base, and choose_base
// over a whole chunk of ordered u32/u64 latents (returns 1 and *base when int mult is bid, 0 for classic)
uint32_t pco_oracle_kat_calc_gcd_u32(uint32_t x, uint32_t y) { return calc_gcd<uint32_t>(x, y); }
uint32_t pco_oracle_kat_calc_triple_gcd_u32(const uint32_t* triple) { return calc_triple_gcd<uint32_t>(triple); }
int pco_oracle_kat_false_position(int which, double* root) {
  switch (which) {
    case 0: return solve_root_by_false_position([](double x) { return x * x - 1.0; }, -0.9, 2.0, root) ? 1 : 0;
    case 1: return solve_root_by_false_position([](double x) { return x * x; }, -0.9, 2.0, root) ? 1 : 0;
    default: return solve_root_by_false_position([](double) { return 0.0; }, 0.0, 1.0, root) ? 1 : 0;
  }
}
int pco_oracle_kat_choose_candidate_base_u32(const uint32_t* sample, size_t n, uint32_t* base, double* bits_saved) {
  std::vector<uint32_t> v(sample, sample + n);
  return choose_candidate_base<uint32_t>(v, base, bits_saved) ? 1 : 0;
}
int pco_oracle_kat_int_mult_choose_base_u32(const uint32_t* latents, size_t n, uint32_t* base) { return int_mult_choose_base<uint32_t>(latents, n, base) ? 1 : 0; }
int pco_oracle_kat_int_mult_choose_base_u64(const uint64_t* latents, size_t n, uint64_t* base) { return int_mult_choose_base<uint64_t>(latents, n, base) ? 1 : 0; }

// pco/src/mode/float_mult.rs :403-653 and float_quant.rs :155-289 unit tests, data_types/float.rs :453-520 (f32 = 0, f64 = 1 where both exist)
float pco_oracle_kat_insignificant_float_to_f32(float x) { return insignificant_float_to<float>(x); }
double pco_oracle_kat_insignificant_float_to_f64(double x) { return insignificant_float_to<double>(x); }
int pco_oracle_kat_approx_pair_gcd_f32(float greater, float lesser, float* out) { return approx_pair_gcd<float>(greater, lesser, out) ? 1 : 0; }
int pco_oracle_kat_approx_pair_gcd_f64(double greater, double lesser, double* out) { return approx_pair_gcd<double>(greater, lesser, out) ? 1 : 0; }
int pco_oracle_kat_config_by_trailing_zeros_f32(const float* sample, size_t n, float* base, float* inv_base) {
  FloatMultConfig<float> c;
  if (!choose_config_by_trailing_zeros<float>(std::vector<float>(sample, sample + n), &c)) return 0;
  *base = c.base;
  *inv_base = c.inv_base;
  return 1;
}
int pco_oracle_kat_config_by_euclidean_f32(const float* sample, size_t n, float* base, float* inv_base) {
  FloatMultConfig<float> c;
  if (!choose_config_by_euclidean<float>(std::vector<float>(sample, sample + n), &c)) return 0;
  *base = c.base;
  *inv_base = c.inv_base;
  return 1;
}
int pco_oracle_kat_sample_gcd_euclidean_f32(const float* sample, size_t n, float* out) {
  return approx_sample_gcd_euclidean<float>(std::vector<float>(sample, sample + n), out) ? 1 : 0;
}
float pco_oracle_kat_center_sample_base_f32(float base, const float* sample, size_t n) { return center_sample_base<float>(base, std::vector<float>(sample, sample + n)); }
void pco_oracle_kat_snap_to_int_reciprocal_f32(float base, float* out_base, float* out_inv_base) {
  auto c = snap_to_int_reciprocal<float>(base);
  *out_base = c.base;
  *out_inv_base = c.inv_base;
}
// bits_saved_per_num_over_classic with FloatMultConfig::from_inv_base(inv_base); returns 0 when below the required savings
int pco_oracle_kat_float_mult_bits_saved_f32(float inv_base, const float* sample, size_t n, double* out) {
  return bits_saved_per_num_over_classic<float>(FloatMultConfig<float>::from_inv_base(inv_base), std::vector<float>(sample, sample + n), out) ? 1 : 0;
}
int pco_oracle_kat_float_mult_compute_bid_f32(const float* sample, size_t n, float* base, double* bits_saved) {
  FloatMultConfig<float> c;
  if (!float_mult_compute_bid<float>(std::vector<float>(sample, sample + n), &c, bits_saved)) return 0;
  *base = c.base;
  return 1;
}
void pco_oracle_kat_float_quant_best_k_f32(const float* sample, size_t n, uint32_t* k, double* bits_saved) {
  auto r = float_quant_estimate_best_k_and_bits_saved<float>(std::vector<float>(sample, sample + n));
  *k = r.first;
  *bits_saved = r.second;
}
void pco_oracle_kat_float_quant_best_k_f64(const double* sample, size_t n, uint32_t* k, double* bits_saved) {
  auto r = float_quant_estimate_best_k_and_bits_saved<double>(std::vector<double>(sample, sample + n));
  *k = r.first;
  *bits_saved = r.second;
}
int pco_oracle_kat_float_quant_compute_bid_f32(const float* sample, size_t n, uint32_t* k, double* bits_saved) {
  return float_quant_compute_bid<float>(std::vector<float>(sample, sample + n), k, bits_saved) ? 1 : 0;
}
// choose_mode over whole chunks (data_types/float.rs:453-457): kind (ModeKind), base as f64, k
void pco_oracle_kat_choose_float_mode_f32(const float* nums, size_t n, int* kind, double* base, uint32_t* k) {
  auto c = choose_float_mode<float>(reinterpret_cast<const uint32_t*>(nums), n);
  *kind = int(c.kind);
  *base = c.base;
  *k = c.k;
}
void pco_oracle_kat_choose_float_mode_f64(const double* nums, size_t n, int* kind, double* base, uint32_t* k) {
  auto c = choose_float_mode<double>(reinterpret_cast<const uint64_t*>(nums), n);
  *kind = int(c.kind);
  *base = c.base;
  *k = c.k;
}
uint16_t pco_oracle_kat_f64_to_f16_bits(double x) { return f64_to_f16_bits(x); }
void pco_oracle_kat_choose_float_mode_f16(const uint16_t* nums, size_t n, int* kind, double* base, uint32_t* k) {
  auto c = choose_float_mode<F16>(nums, n);
  *kind = int(c.kind);
  *base = c.base;
  *k = c.k;
}
int32_t pco_oracle_kat_float_exponent_f32(float x) { return fl_exponent<float>(x); }
float pco_oracle_kat_float_exp2_f32(int32_t p) { return fl_exp2<float>(p); }

void pco_oracle_kat_dict_tie_order(const uint64_t* values, size_t n) { dict_tie_order().assign(values, values + n); }
void pco_oracle_kat_conv1_v1_0_0_parameters(int on) { conv1_v1_0_0_parameters() = on != 0; }
// pco/src/delta/conv1.rs unit tests (:503-583): matrices are row-major here (h x w), column-major inside
void pco_oracle_kat_conv_autocov_mats(const double* v, size_t n, size_t order, double regularization, double* xtx_colmajor, double* xty) {
  ConvMatrix xtx(0.0, 0, 0), y(0.0, 0, 0);
  conv_autocov_mats(std::vector<double>(v, v + n), order, regularization, &xtx, &y);
  for (size_t i = 0; i < xtx.data.size(); i++) xtx_colmajor[i] = xtx.data[i];
  for (size_t i = 0; i < y.data.size(); i++) xty[i] = y.data[i];
}
static ConvMatrix conv_from_rows(const double* rows, size_t h, size_t w) {
  ConvMatrix m(0.0, h, w);
  for (size_t i = 0; i < h; i++) for (size_t j = 0; j < w; j++) m.at(i, j) = rows[i * w + j];
  return m;
}
void pco_oracle_kat_conv_cholesky(const double* rows, size_t h, double* out_colmajor) {
  ConvMatrix c = conv_cholesky(conv_from_rows(rows, h, h));
  for (size_t i = 0; i < c.data.size(); i++) out_colmajor[i] = c.data[i];
}
void pco_oracle_kat_conv_sub(int transposed_backward, const double* l_rows, size_t h, const double* y, double* out) {
  ConvMatrix l = conv_from_rows(l_rows, h, h), yy = conv_from_rows(y, h, 1);
  ConvMatrix x = transposed_backward ? conv_transposed_backward_sub(l, std::move(yy)) : conv_forward_sub(l, std::move(yy));
  for (size_t i = 0; i < h; i++) out[i] = x.data[i];
}

int pco_oracle_kat_consecutive_encode_u32(uint32_t* latents, size_t n, size_t order, uint32_t* moments_out) {
  return guarded([&] {
    auto m = consecutive_encode_in_place<uint32_t>(order, latents, n);
    for (size_t i = 0; i < m.size(); i++) moments_out[i] = m[i];
  });
}
int pco_oracle_kat_consecutive_decode_u32(uint32_t* moments, size_t order, uint32_t* latents, size_t n) {
  return guarded([&] {
    std::vector<uint32_t> m(moments, moments + order);
    consecutive_decode_in_place<uint32_t>(m, latents, n);
    for (size_t i = 0; i < order; i++) moments[i] = m[i];
  });
}

}  // extern "C"
