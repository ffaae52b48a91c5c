// libcpcodec.so — C-ABI entry points (include/cpcodec.h, include/pco_b200.h) over the sm_90a kernels.
// There is no CPU implementation of the hot path in this library: without a CUDA device every
// compute entry point fails with PCO_B200_CUDA.
#include <algorithm>
#include <functional>
#include <initializer_list>

#include "async_compress.cuh"
#include "async_compress_files.cuh"
#include "async_compress_wrapped.cuh"
#include "async_aggregate_kernels.cuh"
#include "async_filter_files_kernels.cuh"
#include "async_filter_kernels.cuh"
#include "async_files_kernels.cuh"
#include "async_index_kernels.cuh"
#include "async_kernels.cuh"
#include "async_pages_kernels.cuh"
#include "async_pages_to_file_kernels.cuh"
#include "async_ranges_kernels.cuh"
#include "async_take_kernels.cuh"
#include "compress_host.cuh"
#include "decode_kernels.cuh"
#include "decode_fused.cuh"
#include "gather_kernels.cuh"
#include "decode_cold.cuh"
#include "files_kernels.cuh"
#include "host_common.hpp"
#include "ranges_kernels.cuh"
#include "wrapped_kernels.cuh"

namespace pcob200 {

// Every device scratch buffer of a context, listed once: Context declares them and reset_context frees them all.
#define PCOB_CONTEXT_BUFFERS(X)                                                                                   \
  X(src) X(out) X(index) X(statuses) X(misc) X(dec_syms) X(dec_offs) X(gather) X(cold) X(cold_res) X(spec)        \
  /* pco_b200_decompress_pages / pco_b200_compress_wrapped */                                                     \
  X(wrap_metas) X(wrap_frames) X(wrap_tab) X(wrap_res) X(wrap_file) X(wrap_index) X(wrap_out)                     \
  /* pco_b200_compress_files / pco_b200_decompress_files */                                                       \
  X(files_tab) X(files_res) X(files_out) X(files_idx) X(files_arena) X(files_cold)                                \
  /* pco_b200_decompress_ranges */                                                                                \
  X(rng_tab) X(rng_stage) X(rng_cold) X(rng_copies)

// One Context per host thread (thread_local): its scratch buffers, events and the last call's profile belong to the calling
// thread, so calls from different threads run concurrently (e.g. compress of chunk group g + 1 while group g decompresses, each
// on its own stream) and the entry points are thread-safe the way the reference documents its own (pco_c/src/lib.rs:57-70).
// The context follows the thread's current device: a cudaSetDevice between calls drops the scratch of the previous device.
struct Context {
  int device = -1;
  bool attrs_set[5] = {false, false, false, false, false};  // set_decode_attrs<WIN, FILT, AGG, TAKE> has run (index WIN + 2 FILT + AGG + 2 TAKE)
  bool initialized = false;
  bool device_ok = false;
  std::string device_err;
#define PCOB_DECLARE_BUFFER(name) DevBuf name;
  PCOB_CONTEXT_BUFFERS(PCOB_DECLARE_BUFFER)
#undef PCOB_DECLARE_BUFFER
  CompressScratch enc;
  Binoms* d_binoms = nullptr;
  int sm_count = 0;
  uint32_t last_decode_chunks = 0;  // chunks of the last decode launch (their class bytes are still at d_cls)
  uint8_t* d_cls = nullptr;         // class bytes of the last decode launch (they live behind the status words in `statuses`)
  void* pinned_res = nullptr;       // page-locked landing buffer for the statuses + class bytes of a decode launch
  size_t pinned_cap = 0;
  uint32_t* gather_err = nullptr;   // error word of the last page gather (inside `gather`)
};

static Context& ctx() {
  static thread_local Context c;
  return c;
}

// Frees the context's device memory and marks it uninitialised, so that the next call on this thread sets the device up again.  That
// includes the binomial table ensure_device builds once per context: a context left initialised without it sent the next decode that
// reached decode_kernel to a null table (an illegal address).
static void reset_context(Context& c) {
#define PCOB_RELEASE_BUFFER(name) c.name.release();
  PCOB_CONTEXT_BUFFERS(PCOB_RELEASE_BUFFER)
#undef PCOB_RELEASE_BUFFER
  c.enc.release();
  c.gather_err = nullptr;
  c.d_cls = nullptr;
  if (c.pinned_res) cudaFreeHost(c.pinned_res);
  c.pinned_res = nullptr;
  c.pinned_cap = 0;
  if (c.d_binoms) cudaFree(c.d_binoms);
  c.d_binoms = nullptr;
  c.initialized = false;
  c.device_ok = false;
  for (bool& a : c.attrs_set) a = false;
}

static PcoB200Error ensure_device(Context& c) {
  if (c.initialized && c.device_ok) {
    int cur = -1;
    if (cudaGetDevice(&cur) == cudaSuccess && cur != c.device) {  // the thread moved to another device: start over there
      cudaSetDevice(c.device);
      reset_context(c);
      cudaSetDevice(cur);
    }
  }
  // Only permanent outcomes are cached (set up, no device, not sm_90).  A set-up step that fails - a cudaMalloc refused on a GPU that
  // is short of memory, or while another thread captures a CUDA graph in global mode - frees what it made and leaves the context
  // uninitialised, so the thread's next call tries again.
  if (!c.initialized) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
      c.initialized = true;
      c.device_err = e != cudaSuccess ? cudaGetErrorString(e) : "no CUDA device";
      cudaGetLastError();
    } else {
      cudaDeviceProp prop;
      int dev = 0;
      PCOB_CUDA_TRY(cudaGetDevice(&dev));
      PCOB_CUDA_TRY(cudaGetDeviceProperties(&prop, dev));
      c.device = dev;
      if (prop.major != 9 || prop.minor != 0) {
        c.initialized = true;
        c.device_err = std::string("device ") + prop.name + " is not sm_90 (the kernels are built for sm_90a only)";
      } else {
        c.sm_count = prop.multiProcessorCount;
        // binomials mod 2^64 by Pascal additions
        Binoms hb;
        std::vector<std::vector<uint64_t>> C(257, std::vector<uint64_t>(MAX_ORDER, 0));
        for (int nn = 0; nn <= 256; nn++) {
          C[nn][0] = 1;
          for (int j = 1; j < MAX_ORDER; j++) C[nn][j] = nn == 0 ? 0 : C[nn - 1][j - 1] + C[nn - 1][j];
        }
        for (int l = 0; l < 32; l++)
          for (int j = 0; j < MAX_ORDER; j++) hb.lane8[l][j] = C[8 * l][j];
        for (int j = 0; j < MAX_ORDER; j++) hb.full[j] = C[256][j];
        if (!c.d_binoms) e = cudaMalloc(&c.d_binoms, sizeof(Binoms));
        if (e == cudaSuccess) e = cudaMemcpy(c.d_binoms, &hb, sizeof(Binoms), cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(walk_kernel<12>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(WalkSmem<12>));
        if (e == cudaSuccess) e = cudaFuncSetAttribute(walk_kernel<SMALL_MAX_SIZE_LOG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(WalkSmem<SMALL_MAX_SIZE_LOG>));
        if (e != cudaSuccess) {
          // a free that is refused as well (the same global capture) keeps the table for the next try; reset_context frees it
          if (c.d_binoms && cudaFree(c.d_binoms) == cudaSuccess) c.d_binoms = nullptr;
          return cuda_fail(e, "CUDA device set-up (binomial table, walk kernel attributes)");
        }
        c.initialized = true;
        c.device_ok = true;
      }
    }
  }
  if (!c.device_ok)
    return fail(PCO_B200_CUDA, "CUDA device unavailable (" + c.device_err + "); libcpcodec has no CPU fallback");
  return PCO_B200_OK;
}

template <typename Fn>
static auto dispatch_latent(uint32_t dtype, Fn&& fn) {
  switch (nt_bits(dtype)) {
    case 8: return fn(uint8_t(0));
    case 16: return fn(uint16_t(0));
    case 32: return fn(uint32_t(0));
    default: return fn(uint64_t(0));
  }
}

struct DecodeOutcome {
  uint64_t n_total = 0;   // numbers in the chunks seen
  bool terminated = false;
};

// Shared-memory attributes of the decode kernels (the window-mode instantiations when WIN, the filter-mode ones when FILT, the
// aggregate-mode ones when AGG too, the take-mode ones when TAKE too), set once per context before their first launch.
template <bool WIN, bool FILT = false, bool AGG = false, bool TAKE = false>
static PcoB200Error set_decode_attrs(Context& c) {
  static_assert(!(WIN && FILT) && (FILT || !AGG) && (FILT || !TAKE) && !(AGG && TAKE),
                "no instantiation is both window and filter mode; aggregate and take mode are filter modes, and exclusive");
  if (c.attrs_set[WIN + 2 * FILT + AGG + 2 * TAKE]) return PCO_B200_OK;
  auto max_shared = [](auto* kernel, size_t smem) {
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
    return e != cudaSuccess ? e : cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, int(cudaSharedmemCarveoutMaxShared));
  };
  PCOB_CUDA_TRY(max_shared(symwalk_kernel<WIN>, sizeof(SymWalkSmem)));
  PCOB_CUDA_TRY(max_shared(fused_narrow_kernel<uint64_t, WIN, FILT, AGG, TAKE>, sizeof(FusedSmem)));
  PCOB_CUDA_TRY(max_shared(fused_narrow_kernel<uint32_t, WIN, FILT, AGG, TAKE>, sizeof(FusedSmem)));
  PCOB_CUDA_TRY(max_shared(fused_narrow_kernel<uint16_t, WIN, FILT, AGG, TAKE>, sizeof(FusedSmem)));
  PCOB_CUDA_TRY(max_shared(fused_narrow_kernel<uint8_t, WIN, FILT, AGG, TAKE>, sizeof(FusedSmem)));
  c.attrs_set[WIN + 2 * FILT + AGG + 2 * TAKE] = true;  // only once every attribute is set: a failed call leaves them to the next
  return PCO_B200_OK;
}

// Launch the decode over `n_chunks` IndexChunk records that live on the device.
//   1. fused_narrow_kernel (decode_fused.cuh): parses and classifies every chunk and fully decodes the narrow class;
//   2. only if some chunk is of another class: symwalk_kernel + decode_kernel<L, 1 / 2> for those.
// A failing chunk fails the launch ("... chunk k"); `bad_chunk`, when given, receives its position k among the launch's records.
static PcoB200Error launch_decode(Context& c, const FileParams& fp, const uint8_t* d_index, uint64_t index_len, uint64_t chunks_offset, uint32_t n_chunks,
                                  void* d_out, uint64_t out_len, cudaStream_t stream, uint32_t* bad_chunk = nullptr) {
  if (n_chunks == 0) return PCO_B200_OK;
  // status words and class bytes side by side: one copy brings both back
  const size_t res_bytes = size_t(n_chunks) * (sizeof(uint32_t) + 1);
  PCOB_CUDA_TRY(c.statuses.reserve(res_bytes + 64));
  uint32_t* d_st = c.statuses.as<uint32_t>();
  uint8_t* d_cls = reinterpret_cast<uint8_t*>(d_st + n_chunks);
  c.d_cls = d_cls;
  if (c.pinned_cap < res_bytes) {
    if (c.pinned_res) cudaFreeHost(c.pinned_res);
    c.pinned_res = nullptr;
    c.pinned_cap = 0;
    PCOB_CUDA_TRY(cudaHostAlloc(&c.pinned_res, res_bytes + (res_bytes >> 1) + 4096, cudaHostAllocDefault));
    c.pinned_cap = res_bytes + (res_bytes >> 1) + 4096;
  }
  const IndexChunk* d_chunks = reinterpret_cast<const IndexChunk*>(d_index + chunks_offset);
  if (PcoB200Error e = set_decode_attrs<false>(c)) return e;
  c.last_decode_chunks = n_chunks;
  const uint32_t* st = static_cast<const uint32_t*>(c.pinned_res);
  auto chunk_fail = [&](uint32_t i) {
    if (bad_chunk) *bad_chunk = i;
    return status_to_error(st[i], ("chunk " + std::to_string(i)).c_str());
  };
  profiler().begin("fused_narrow_kernel", stream);
  dispatch_latent(fp.dtype, [&](auto tag) {
    using L = decltype(tag);
    fused_narrow_kernel<L><<<n_chunks, FZ_THREADS, sizeof(FusedSmem), stream>>>(fp, d_chunks, d_index, index_len, d_st, d_cls, static_cast<L*>(d_out), out_len);
    return 0;
  });
  profiler().end(stream);
  PCOB_CUDA_TRY(cudaGetLastError());
  // statuses and class bytes come back in one round trip; the general kernels only run if some chunk still needs them
  PCOB_CUDA_TRY(readback_small_sync(c.pinned_res, d_st, (res_bytes + 3) & ~size_t(3), stream));  // the buffers hold res_bytes + 64
  const uint8_t* cls = reinterpret_cast<const uint8_t*>(st + n_chunks);
  bool pending = false;
  for (uint32_t i = 0; i < n_chunks; i++) {
    if (!(cls[i] & CLS_DONE)) { pending = true; continue; }
    if (st[i] != ST_OK) return chunk_fail(i);
  }
  if (!pending) return PCO_B200_OK;
  // scratch between the two kernels: one symbol byte per latent the destination can take, one section start per batch
  const uint64_t rows = scratch_rows_total(out_len, n_chunks);
  PCOB_CUDA_TRY(c.dec_syms.reserve(rows * BATCH_N + 64));
  PCOB_CUDA_TRY(c.dec_offs.reserve(rows * sizeof(uint32_t) + 64));
  profiler().begin("symwalk_kernel", stream);
  symwalk_kernel<<<n_chunks, SW_THREADS, sizeof(SymWalkSmem), stream>>>(fp, d_chunks, d_index, index_len, out_len, c.dec_syms.as<uint8_t>(), c.dec_offs.as<uint32_t>(),
                                                                        d_cls);
  profiler().end(stream);
  profiler().begin("decode_kernel", stream);  // the span covers every decode instantiation (a chunk runs in exactly one)
  dispatch_latent(fp.dtype, [&](auto tag) {
    using L = decltype(tag);
    decode_kernel<L, 1><<<n_chunks, DEC_THREADS, sizeof(DecodeSmem), stream>>>(fp, d_chunks, d_st, d_index, index_len, static_cast<L*>(d_out), out_len, c.d_binoms,
                                                                                c.dec_syms.as<uint8_t>(), c.dec_offs.as<uint32_t>(), d_cls);
    decode_kernel<L, 2><<<n_chunks, DEC_THREADS, sizeof(DecodeSmem), stream>>>(fp, d_chunks, d_st, d_index, index_len, static_cast<L*>(d_out), out_len, c.d_binoms,
                                                                                c.dec_syms.as<uint8_t>(), c.dec_offs.as<uint32_t>(), d_cls);
    return 0;
  });
  profiler().end(stream);
  PCOB_CUDA_TRY(cudaGetLastError());
  PCOB_CUDA_TRY(readback_small_sync(c.pinned_res, d_st, size_t(n_chunks) * sizeof(uint32_t), stream));
  for (uint32_t i = 0; i < n_chunks; i++)
    if (st[i] != ST_OK) return chunk_fail(i);
  return PCO_B200_OK;
}

// The file's first bytes (at most 32) and, when `ih` is given, the side index header (zeros when `index` holds none), from host or
// device memory - one synchronisation for both - and the standalone header parsed from those bytes.
static PcoB200Error read_heads(const void* src, size_t src_len, bool src_dev, const void* index, size_t index_len, bool idx_dev, IndexHeader* ih,
                               StandaloneHeader* hdr, cudaStream_t stream) {
  uint8_t head[32] = {0};
  const size_t avail = std::min<size_t>(src_len, sizeof(head));
  bool need_sync = false;
  if (avail) {
    if (src_dev) { PCOB_CUDA_TRY(cudaMemcpyAsync(head, src, avail, cudaMemcpyDeviceToHost, stream)); need_sync = true; }
    else std::memcpy(head, src, avail);
  }
  if (ih) {
    std::memset(ih, 0, sizeof(*ih));
    if (index && index_len >= sizeof(IndexHeader)) {
      if (idx_dev) { PCOB_CUDA_TRY(cudaMemcpyAsync(ih, index, sizeof(*ih), cudaMemcpyDeviceToHost, stream)); need_sync = true; }
      else std::memcpy(ih, index, sizeof(*ih));
    }
  }
  if (need_sync) PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
  return parse_standalone_header(head, avail, src_len, hdr);
}

// A caller's buffer in HBM: the buffer itself when it is on the device, else its bytes copied into `buf`.
static PcoB200Error stage_in(DevBuf& buf, const void* p, size_t len, bool on_device, cudaStream_t stream, const uint8_t** d_p) {
  *d_p = static_cast<const uint8_t*>(p);
  if (on_device) return PCO_B200_OK;
  PCOB_CUDA_TRY(buf.reserve(len + 16));
  if (len) PCOB_CUDA_TRY(copy_sliced(buf.p, p, len, cudaMemcpyHostToDevice, stream));
  *d_p = buf.as<uint8_t>();
  return PCO_B200_OK;
}

// Where the kernels write the output: the caller's device buffer, or `c.out` (at least `bytes`) for a host one.
static PcoB200Error out_buffer(Context& c, void* dst, bool dst_dev, uint64_t bytes, void** d_out) {
  *d_out = dst;
  if (dst_dev) return PCO_B200_OK;
  PCOB_CUDA_TRY(c.out.reserve(bytes + 64));
  *d_out = c.out.p;
  return PCO_B200_OK;
}

// Placeholder records for a walk: from `begin` on, each record gets the entries of MAX_VARS vars of its `n` numbers.  Returns where the entries end.
static uint64_t lay_out_entries(IndexChunk* recs, size_t n_recs, uint64_t begin) {
  for (size_t k = 0; k < n_recs; k++) {
    recs[k].entries_offset = begin;
    begin += entries_bytes(MAX_VARS, recs[k].n);
  }
  return begin;
}

// One catch-all decode: the chunks of `fp` from byte `first_byte` on, into `out`, which takes `cap` numbers.
struct ColdJob {
  FileParams fp;
  uint64_t first_byte;
  void* out;
  uint64_t cap;
};

// cold_decode_kernel over every job (one single-thread launch each), the results read back into `res`.  Lookback windows beyond 2^16
// numbers get the large scratch on a second pass, which takes the jobs whose result `retry` accepts.
template <typename Retry>
static PcoB200Error cold_decode_jobs(Context& c, uint32_t dtype, const std::vector<ColdJob>& jobs, Retry retry, std::vector<ColdResult>* res,
                                     cudaStream_t stream) {
  const size_t nj = jobs.size();
  res->assign(nj, ColdResult{});
  PCOB_CUDA_TRY(c.cold_res.reserve(nj * sizeof(ColdResult) + 64));
  ColdResult* d_res = c.cold_res.as<ColdResult>();
  std::vector<size_t> todo(nj);
  for (size_t k = 0; k < nj; k++) todo[k] = k;
  for (uint32_t window_cap : {16u, COLD_MAX_WINDOW_LOG}) {
    if (todo.empty()) break;
    PCOB_CUDA_TRY(c.cold.reserve(cold_scratch_bytes(window_cap)));
    profiler().begin("cold_decode_kernel", stream);
    for (size_t k : todo) {
      const ColdJob& j = jobs[k];
      dispatch_latent(dtype, [&](auto tag) {
        using L = decltype(tag);
        cold_decode_kernel<L><<<1, 32, 0, stream>>>(j.fp, j.first_byte, static_cast<L*>(j.out), j.cap, c.cold.as<uint8_t>(), window_cap, d_res + k);
        return 0;
      });
    }
    profiler().end(stream);
    PCOB_CUDA_TRY(cudaGetLastError());
    PCOB_CUDA_TRY(readback_small_sync(res->data(), d_res, nj * sizeof(ColdResult), stream));
    std::vector<size_t> again;
    for (size_t k : todo)
      if (retry((*res)[k])) again.push_back(k);
    todo.swap(again);
  }
  return PCO_B200_OK;
}
// A whole file is decoded again with the large window on any such refusal; a page or a range's chunk only if no chunk of it finished.
static bool cold_retry_file(const ColdResult& r) { return r.status == ST_UNSUPPORTED; }
static bool cold_retry_chunk(const ColdResult& r) { return r.n_chunks == 0 && r.status == ST_UNSUPPORTED; }

// Bytes at many positions of `base`, a buffer in host memory or, when `on_device`, in device memory (one readback):
// out[k * width + j] = base[offs[k] + j] for j < min(width, lens[k]), 0 behind that.
static PcoB200Error peek(Context& c, const void* base, bool on_device, const std::vector<uint64_t>& offs, const std::vector<uint64_t>& lens, uint32_t width,
                         std::vector<uint8_t>* out, cudaStream_t stream) {
  const size_t m = offs.size();
  out->assign(m * width, 0);
  if (m == 0) return PCO_B200_OK;
  if (!on_device) {
    for (size_t k = 0; k < m; k++) std::memcpy(out->data() + k * width, static_cast<const uint8_t*>(base) + offs[k], std::min<uint64_t>(lens[k], width));
    return PCO_B200_OK;
  }
  if (m == 1) {  // a one-file walk: a plain copy costs less than uploading the table
    PCOB_CUDA_TRY(cudaMemcpyAsync(out->data(), static_cast<const uint8_t*>(base) + offs[0], std::min<uint64_t>(lens[0], width), cudaMemcpyDeviceToHost, stream));
    PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
    return PCO_B200_OK;
  }
  PCOB_CUDA_TRY(c.files_tab.reserve(m * 16 + 64));
  PCOB_CUDA_TRY(c.files_res.reserve(m * width + 64));
  uint64_t* d_offs = c.files_tab.as<uint64_t>();
  PCOB_CUDA_TRY(cudaMemcpyAsync(d_offs, offs.data(), m * 8, cudaMemcpyHostToDevice, stream));
  PCOB_CUDA_TRY(cudaMemcpyAsync(d_offs + m, lens.data(), m * 8, cudaMemcpyHostToDevice, stream));
  peek_bytes_kernel<<<uint32_t((m + 7) / 8), 256, 0, stream>>>(static_cast<const uint8_t*>(base), d_offs, d_offs + m, uint32_t(m), width, c.files_res.as<uint8_t>());
  PCOB_CUDA_TRY(cudaGetLastError());
  PCOB_CUDA_TRY(readback_small_sync(out->data(), c.files_res.p, (m * width + 3) & ~size_t(3), stream));
  return PCO_B200_OK;
}

// How the walk of an index-free file ended.  COLD: a chunk the fast kernels decline, or one beyond the index scratch (the catch-all
// decoder still reads such a file); FAILED: any other error.  Both leave the error's kind and message.  OPEN: not walked to an end,
// because a file in front of it failed.
enum class WalkEnd { OPEN, TERMINATED, DST_FULL, COLD, FAILED };

// An index-free file for walk_index_free: its bytes src[begin, end), its header, the walk cursor and a cap on its numbers.  The walk
// stops behind the chunk that takes the count past `cap` (DST_FULL: simple_decompress_into's short destination).  `expect` is the
// count the serial walker's scratch is sized for: the destination's room for one file, the header's count hint in a batch.  The walk
// appends the file's chunk records - chunk_offset in src, entries_offset in the arena, out_offset from the file's first number - and
// counts their numbers.
struct WalkFile {
  StandaloneHeader hdr;
  uint64_t begin = 0, end = 0;
  uint64_t pos = 0;
  uint64_t cap = ~uint64_t(0);
  uint64_t expect = 0;
  uint64_t count = 0;
  std::vector<IndexChunk> recs;
  WalkEnd how = WalkEnd::OPEN;
  PcoB200Error err = PCO_B200_OK;
  std::string msg;
};

// Index-free files, the parallel part (the reference's decompressor walks chunk after chunk, standalone/decompressor.rs:150-215; so does
// the serial walk_kernel<<<1>>>, at one GPU thread's speed).  Chunk lengths are not in a file, but its chunks nearly always start with
// the same 4 bytes - the type byte and count - 1 (docs/format.md:186-192).  So in each round, from every file's first unread chunk:
//   1. find_file_starts_kernel lists every position behind it, inside its file, that carries the same 4 bytes (the real chunk starts
//      of that size plus, once per ~4 GB of compressed bytes, a coincidence), for all files in one launch;
//   2. walk_kernel walks ALL of them at once, one CTA each, as if each were a chunk start: index entries, status, end position;
//   3. the host follows each file's chain from its first chunk: the chunk at p is real, it ends at e(p), and if e(p) is on the list
//      the chunk there is real too (a coincidence is never reached: no verified chunk ends on it).
// The rounds repeat from where the chains stopped (chunks of another size - typically a file's last one - start a new pattern).  A
// file leaves them at its terminator, at a chunk past its cap, with too many candidates, or once a round verifies nothing for it:
// walk_index_free finishes it.  A round lays out its candidates' entries, then their records, from *arena_end on, and moves *arena_end
// behind the entries of the last chunk a chain took: the next round reuses the rest.
static PcoB200Error speculative_walk_rounds(Context& c, const uint8_t* src, bool src_dev, const uint8_t* d_src, size_t src_len, uint32_t dtype,
                                            const std::vector<WalkFile*>& files, DevBuf& arena, uint64_t* arena_end, cudaStream_t stream) {
  constexpr uint64_t FILE_CAND_CAP = 1u << 16;             // a file with more candidates is not worth speculating on
  constexpr uint64_t INDEX_BUDGET = uint64_t(768) << 20;   // bytes of walked records and entries per round
  const uint32_t n = uint32_t(files.size());
  const uint32_t cand_cap = uint32_t(std::min<uint64_t>(uint64_t(1) << 22, n * FILE_CAND_CAP));  // candidates listed per round, all files together
  std::vector<uint8_t> tail(n, 0);                         // 1: the file has left the rounds
  for (uint32_t i = 0; i < n; i++)
    if (files[i]->hdr.uniform_type != 0 && files[i]->hdr.uniform_type != dtype) tail[i] = 1;  // no chunk can pass
  for (int round = 0; round < 4096; round++) {
    std::vector<uint32_t> act;
    std::vector<uint64_t> offs, lens;
    for (uint32_t i = 0; i < n; i++)
      if (!tail[i]) {
        if (files[i]->pos + 4 > files[i]->end) { tail[i] = 1; continue; }
        act.push_back(i);
        offs.push_back(files[i]->pos);
        lens.push_back(4);
      }
    if (act.empty()) break;
    std::vector<uint8_t> h4;
    if (PcoB200Error e = peek(c, src, src_dev, offs, lens, 4, &h4, stream)) return e;
    std::vector<FileScan> scans;
    std::vector<uint32_t> scan_file;
    uint64_t blocks = 0;
    const uint64_t per_block = uint64_t(FIND_THREADS) * FIND_PER_THREAD;
    for (size_t k = 0; k < act.size(); k++) {
      const uint32_t i = act[k];
      const uint8_t* b = h4.data() + k * 4;
      // the terminator, or a type byte the serial walker reports; or a chunk past the cap, whose semantics the serial walker owns
      if (b[0] != dtype || files[i]->count + ((uint32_t(b[1]) | (uint32_t(b[2]) << 8) | (uint32_t(b[3]) << 16)) + 1) > files[i]->cap) {
        tail[i] = 1;
        continue;
      }
      FileScan s;
      s.begin = files[i]->pos;
      s.end = files[i]->end - 3;  // last position + 1 whose 4 bytes lie inside the file
      s.pattern = uint32_t(b[0]) | (uint32_t(b[1]) << 8) | (uint32_t(b[2]) << 16) | (uint32_t(b[3]) << 24);
      s.block0 = uint32_t(blocks);
      blocks += (s.end - s.begin + per_block - 1) / per_block;
      scans.push_back(s);
      scan_file.push_back(i);
    }
    if (scans.empty()) break;
    if (blocks > 0x7fffffffull) { for (uint32_t i : scan_file) tail[i] = 1; break; }
    // scratch: count | candidate positions | their files | statuses | chunk ends
    PCOB_CUDA_TRY(c.spec.reserve(64 + size_t(cand_cap) * (8 + 4)));
    PCOB_CUDA_TRY(c.files_tab.reserve(scans.size() * sizeof(FileScan) + 64));
    uint32_t* d_count = c.spec.as<uint32_t>();
    uint64_t* d_cand = reinterpret_cast<uint64_t*>(c.spec.as<uint8_t>() + 64);
    uint32_t* d_cfile = reinterpret_cast<uint32_t*>(d_cand + cand_cap);
    PCOB_CUDA_TRY(cudaMemcpyAsync(c.files_tab.p, scans.data(), scans.size() * sizeof(FileScan), cudaMemcpyHostToDevice, stream));
    PCOB_CUDA_TRY(cudaMemsetAsync(d_count, 0, 4, stream));
    profiler().begin("find_file_starts_kernel", stream);
    find_file_starts_kernel<<<uint32_t(blocks), FIND_THREADS, 0, stream>>>(d_src, c.files_tab.as<FileScan>(), uint32_t(scans.size()), d_cand, d_cfile, cand_cap, d_count);
    profiler().end(stream);
    PCOB_CUDA_TRY(cudaGetLastError());
    uint32_t count = 0;
    PCOB_CUDA_TRY(readback_small_sync(&count, d_count, 4, stream));
    if (count > cand_cap) { for (uint32_t i : scan_file) tail[i] = 1; break; }
    std::vector<uint64_t> cpos(count);
    std::vector<uint32_t> cfile(count);
    PCOB_CUDA_TRY(cudaMemcpyAsync(cpos.data(), d_cand, size_t(count) * 8, cudaMemcpyDeviceToHost, stream));
    PCOB_CUDA_TRY(cudaMemcpyAsync(cfile.data(), d_cfile, size_t(count) * 4, cudaMemcpyDeviceToHost, stream));
    PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
    std::vector<std::vector<uint64_t>> cand(scans.size());
    for (uint32_t k = 0; k < count; k++) cand[cfile[k]].push_back(cpos[k]);
    // the round's walk: every file's candidates (as many as its budget share and its cap allow), one CTA each.  FileParams carries one
    // uniform type and format version per launch, so the records are laid out flavour by flavour and each flavour present is one launch.
    auto flavour = [&](uint32_t i) { return (files[i]->hdr.uniform_type << 8) | files[i]->hdr.format_major; };
    std::vector<uint32_t> scan_order(scans.size());
    for (size_t s = 0; s < scans.size(); s++) scan_order[s] = uint32_t(s);
    std::stable_sort(scan_order.begin(), scan_order.end(), [&](uint32_t a, uint32_t b) { return flavour(scan_file[a]) < flavour(scan_file[b]); });
    std::vector<IndexChunk> recs;
    std::vector<uint32_t> walked;           // scan index of each file walked this round
    std::vector<size_t> first_rec;          // its first record
    uint64_t budget = INDEX_BUDGET;
    for (uint32_t s : scan_order) {
      const uint32_t i = scan_file[s];
      const WalkFile& f = *files[i];
      std::vector<uint64_t>& cs = cand[s];
      std::sort(cs.begin(), cs.end());
      if (cs.empty() || cs.size() > FILE_CAND_CAP || cs[0] != f.pos) { tail[i] = 1; continue; }
      const uint32_t n0 = ((scans[s].pattern >> 8) & 0xffffffu) + 1;
      const uint64_t stride = entries_bytes(MAX_VARS, n0);
      const uint64_t fit = std::min((f.cap - f.count) / n0, FILE_CAND_CAP);  // chunks of this size the cap still takes (>= 1)
      // a few more candidates than fit: coincidences may lie in front of the last chunk that does
      uint64_t m = std::min<uint64_t>({cs.size(), std::max<uint64_t>(1, INDEX_BUDGET / (stride + sizeof(IndexChunk))), fit + 8});
      if (!walked.empty() && m * (stride + sizeof(IndexChunk)) > budget) continue;  // waits for the next round
      budget -= std::min(budget, m * (stride + sizeof(IndexChunk)));
      cs.resize(m);
      walked.push_back(uint32_t(s));
      first_rec.push_back(recs.size());
      for (uint64_t k = 0; k < m; k++) {
        IndexChunk ic;
        ic.chunk_offset = cs[k];
        ic.n = n0;
        ic.n_vars = 0;
        ic.out_offset = 0;
        recs.push_back(ic);
      }
    }
    if (recs.empty()) break;
    const uint32_t mt = uint32_t(recs.size());
    const uint64_t chunks_at = lay_out_entries(recs.data(), mt, (*arena_end + 15) & ~uint64_t(15));  // the records behind the entries
    PCOB_CUDA_TRY(arena.grow_preserve(chunks_at + uint64_t(mt) * sizeof(IndexChunk) + 64, *arena_end, stream));
    PCOB_CUDA_TRY(c.spec.reserve(64 + size_t(cand_cap) * (8 + 4) + size_t(mt) * (4 + 8) + 64));
    uint32_t* d_stat = reinterpret_cast<uint32_t*>(c.spec.as<uint8_t>() + 64 + size_t(cand_cap) * 12);
    uint64_t* d_ends = reinterpret_cast<uint64_t*>(c.spec.as<uint8_t>() + 64 + size_t(cand_cap) * 12 + ((size_t(mt) * 4 + 15) & ~size_t(15)));
    PCOB_CUDA_TRY(cudaMemcpyAsync(arena.as<uint8_t>() + chunks_at, recs.data(), size_t(mt) * sizeof(IndexChunk), cudaMemcpyHostToDevice, stream));
    PCOB_CUDA_TRY(cudaMemsetAsync(d_stat, 0xff, size_t(mt) * 4, stream));
    PCOB_CUDA_TRY(cudaMemsetAsync(d_ends, 0, size_t(mt) * 8, stream));
    PCOB_CUDA_TRY(c.misc.reserve(sizeof(WalkResult)));
    for (size_t w0 = 0; w0 < walked.size();) {  // one launch per flavour: its walked files' records are consecutive
      const uint32_t fl = flavour(scan_file[walked[w0]]);
      size_t w1 = w0 + 1;
      while (w1 < walked.size() && flavour(scan_file[walked[w1]]) == fl) w1++;
      const size_t r_lo = first_rec[w0], r_hi = w1 < walked.size() ? first_rec[w1] : recs.size();
      const FileParams fp{d_src, src_len, dtype, fl >> 8, fl & 0xff};
      profiler().begin("walk_kernel", stream);
      walk_kernel<SMALL_MAX_SIZE_LOG><<<uint32_t(r_hi - r_lo), WALK_THREADS, sizeof(WalkSmem<SMALL_MAX_SIZE_LOG>), stream>>>(
          fp, arena.as<uint8_t>(), chunks_at + r_lo * sizeof(IndexChunk), uint32_t(r_hi - r_lo), 0, chunks_at, 0, 0, ~uint64_t(0), d_stat + r_lo,
          c.misc.as<WalkResult>(), 0, d_ends + r_lo);
      profiler().end(stream);
      PCOB_CUDA_TRY(cudaGetLastError());
      w0 = w1;
    }
    std::vector<uint32_t> st(mt);
    std::vector<uint64_t> ends(mt);
    PCOB_CUDA_TRY(cudaMemcpyAsync(st.data(), d_stat, size_t(mt) * 4, cudaMemcpyDeviceToHost, stream));
    PCOB_CUDA_TRY(cudaMemcpyAsync(ends.data(), d_ends, size_t(mt) * 8, cudaMemcpyDeviceToHost, stream));
    PCOB_CUDA_TRY(cudaMemcpyAsync(recs.data(), arena.as<uint8_t>() + chunks_at, size_t(mt) * sizeof(IndexChunk), cudaMemcpyDeviceToHost, stream));  // n_vars as walked
    PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
    bool progress = false;
    uint64_t kept_end = *arena_end;
    for (size_t w = 0; w < walked.size(); w++) {
      const uint32_t s = walked[w], i = scan_file[s];
      WalkFile& f = *files[i];
      const size_t r0 = first_rec[w];
      const uint32_t m = uint32_t(cand[s].size());
      const uint32_t n0 = recs[r0].n;
      uint64_t p = f.pos;
      const std::vector<uint32_t> chain = follow_chunk_chain(cand[s].data(), st.data() + r0, ends.data() + r0, m, f.pos, n0, f.count, f.cap, f.end, &p);
      if (chain.empty()) { tail[i] = 1; continue; }
      for (uint32_t k : chain) {
        IndexChunk ic = recs[r0 + k];
        ic.out_offset = f.count;
        f.count += n0;
        f.recs.push_back(ic);
        kept_end = std::max(kept_end, ic.entries_offset + entries_bytes(MAX_VARS, n0));
      }
      f.pos = p;
      progress = true;
    }
    *arena_end = kept_end;
    if (!progress) break;
  }
  return PCO_B200_OK;
}

// Walks index-free files to their end: the speculative rounds (PCOB200_SPECULATIVE_WALK=0 skips them), then a peek at every file's
// next byte - a file the rounds walked to its terminator is done - and the serial walker, one file at a time, for every other file.
// So the terminator, a chunk past the cap, a corrupt or truncated chunk and every other special case keep the serial walker's semantics
// and error reporting.  The serial walks go in list order and stop at the first file that fails: a caller that reports the lowest
// failing file needs nothing behind it, and those files stay OPEN.  `src` is the caller's buffer (in device memory when src_dev),
// `d_src` its bytes in HBM; the walked chunks' entries go into `arena` from *arena_end on, which moves behind them.
static PcoB200Error walk_index_free(Context& c, const uint8_t* src, bool src_dev, const uint8_t* d_src, size_t src_len, uint32_t dtype,
                                    const std::vector<WalkFile*>& files, DevBuf& arena, uint64_t* arena_end, cudaStream_t stream) {
  *arena_end = std::max<uint64_t>(*arena_end, 16);  // entries_offset 0 means "no entries" to the decode kernels
  const char* spec = std::getenv("PCOB200_SPECULATIVE_WALK");  // read per call: tests of the serial walk switch it off in-process
  if (!(spec && spec[0] == '0'))
    if (PcoB200Error e = speculative_walk_rounds(c, src, src_dev, d_src, src_len, dtype, files, arena, arena_end, stream)) return e;
  std::vector<uint8_t> done(files.size(), 0);
  {
    std::vector<size_t> at;
    std::vector<uint64_t> offs, lens;
    for (size_t k = 0; k < files.size(); k++)
      if (files[k]->pos < files[k]->end) {
        at.push_back(k);
        offs.push_back(files[k]->pos);
        lens.push_back(1);
      }
    std::vector<uint8_t> b;
    if (PcoB200Error e = peek(c, src, src_dev, offs, lens, 4, &b, stream)) return e;
    for (size_t j = 0; j < at.size(); j++)
      if (b[j * 4] == 0) done[at[j]] = 1;
  }
  PCOB_CUDA_TRY(c.misc.reserve(sizeof(WalkResult)));
  for (size_t k = 0; k < files.size(); k++) {
    WalkFile& f = *files[k];
    f.how = WalkEnd::TERMINATED;
    if (done[k]) continue;
    const FileParams fpf{d_src + f.begin, f.end - f.begin, dtype, f.hdr.uniform_type, f.hdr.format_major};
    const uint32_t max_chunks = uint32_t(std::min<uint64_t>((f.end - f.begin) / 5 + 2, 1u << 16));
    uint64_t next = f.pos - f.begin;
    for (;;) {
      // entries for the batches still to come (by `expect`) plus 2 per chunk, for 2 vars; then room for the records, which the next
      // round reuses
      const uint64_t entries_begin = (*arena_end + 15) & ~uint64_t(15);
      uint64_t want_batches = (f.expect > f.count ? (f.expect - f.count) / BATCH_N : 0) + 2ull * max_chunks + 2;
      want_batches = std::min<uint64_t>(want_batches, uint64_t(1) << 23);
      const uint64_t entries_end = entries_begin + want_batches * MAX_VARS * sizeof(BatchEntry) + 16ull * max_chunks + 64;
      const uint64_t chunks_at = (entries_end + 15) & ~uint64_t(15);
      PCOB_CUDA_TRY(arena.grow_preserve(chunks_at + uint64_t(max_chunks) * sizeof(IndexChunk) + 64, *arena_end, stream));
      profiler().begin("walk_kernel", stream);
      walk_kernel<12><<<1, WALK_THREADS, sizeof(WalkSmem<12>), stream>>>(fpf, arena.as<uint8_t>(), chunks_at, max_chunks, entries_begin, entries_end, next, f.count,
                                                                        f.cap, nullptr, c.misc.as<WalkResult>(), 1);
      profiler().end(stream);
      PCOB_CUDA_TRY(cudaGetLastError());
      WalkResult res;
      PCOB_CUDA_TRY(readback_small_sync(&res, c.misc.p, sizeof(res), stream));
      if (res.n_chunks > 0) {
        std::vector<IndexChunk> got(res.n_chunks);
        PCOB_CUDA_TRY(cudaMemcpyAsync(got.data(), arena.as<uint8_t>() + chunks_at, got.size() * sizeof(IndexChunk), cudaMemcpyDeviceToHost, stream));
        PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
        for (IndexChunk& ic : got) {
          ic.chunk_offset += f.begin;
          f.recs.push_back(ic);
        }
        *arena_end = res.entries_end;
      }
      f.count += res.n_total;
      next = res.next_byte;
      if (res.status == ST_TERMINATOR) break;
      if (res.status == ST_DST_FULL) { f.how = WalkEnd::DST_FULL; break; }
      if (res.status == ST_INDEX_FULL && res.n_chunks > 0) continue;
      f.how = res.status == ST_UNSUPPORTED || res.status == ST_INDEX_FULL ? WalkEnd::COLD : WalkEnd::FAILED;
      f.err = res.status == ST_INDEX_FULL ? fail(PCO_B200_UNSUPPORTED, "a single chunk exceeds the device index scratch")
                                          : status_to_error(res.status, ("chunk " + std::to_string(res.n_chunks) + " of this walk round").c_str());
      f.msg = last_error_ref();
      break;
    }
    if (f.how == WalkEnd::FAILED) break;
  }
  return PCO_B200_OK;
}


// The fast kernels behind every decompress entry point.  The walk goes on while the numbers seen fit the destination - an exact fit still
// has to find the terminator (a truncated file is an error for both of the reference's semantics) - and stops with `terminated = false`
// and n_total > dst_len at the first chunk that does not fit: pco_standalone_simple_decompress_into turns that into its "exceeds dst_cap"
// error (pco_c/src/lib.rs:98-120), pco_b200_decompress_ex into Progress{finished = false} (standalone/simple.rs:115-140).
static PcoB200Error decompress_fast(const void* compressed, size_t compressed_len, uint32_t dtype, void* dst, size_t dst_len,
                                    const void* index, size_t index_len, uint32_t flags, void* cuda_stream, DecodeOutcome* outcome) {
  if (!nt_valid(dtype)) return fail(PCO_B200_INVALID_TYPE, "unknown number type byte: " + std::to_string(dtype));
  Context& c = ctx();
  if (PcoB200Error e = ensure_device(c)) return e;
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  const bool src_dev = flags & PCO_B200_SRC_ON_DEVICE, dst_dev = flags & PCO_B200_DST_ON_DEVICE;
  const size_t elem = nt_bits(dtype) / 8;

  // 1. standalone header (host parse of the first bytes); the side index header comes back in the same round trip
  const bool have_index = index != nullptr && index_len >= sizeof(IndexHeader);
  const bool idx_dev = flags & PCO_B200_INDEX_ON_DEVICE;
  IndexHeader ih;
  StandaloneHeader hdr;
  if (PcoB200Error e = read_heads(compressed, compressed_len, src_dev, index, index_len, idx_dev, &ih, &hdr, stream)) return e;

  // 2. the file in HBM
  const uint8_t* d_src;
  call_trace().mark("d.begin");
  if (PcoB200Error e = stage_in(c.src, compressed, compressed_len, src_dev, stream, &d_src)) return e;
  call_trace().mark("d.h2d_submitted");
  const FileParams fp{d_src, compressed_len, dtype, hdr.uniform_type, hdr.format_major};

  // 3a. caller-supplied side index
  if (have_index) {
    if (!index_header_ok(ih, compressed_len, index_len)) return fail(PCO_B200_INVALID_ARGUMENT, "side index does not belong to this file");
    const uint8_t* d_idx;
    if (PcoB200Error e = stage_in(c.index, index, index_len, idx_dev, stream, &d_idx)) return e;
    uint64_t n_emit = std::min<uint64_t>(ih.n_total, dst_len);
    // a page-locked destination is written in place by the decode kernels (every number is stored once, in 32-byte pieces that a
    // warp lays down as 1 KiB runs): no staging buffer, no copy behind the kernel (host_common.hpp, zero copy)
    void* d_out = !dst_dev && (zero_copy_mask().load(std::memory_order_relaxed) & 2) ? mapped_host_ptr(dst) : nullptr;
    const bool dst_in_place = d_out != nullptr;
    if (!dst_in_place)
      if (PcoB200Error e = out_buffer(c, dst, dst_dev, n_emit * elem, &d_out)) return e;
    if (ih.n_chunks > 0xffffffffull) return fail(PCO_B200_INVALID_ARGUMENT, "too many chunks");
    // a host destination holds (or is staged in c.out, which holds) n_emit numbers: that is the kernels' bound, whatever the index claims
    if (PcoB200Error e = launch_decode(c, fp, d_idx, index_len, ih.chunks_offset, uint32_t(ih.n_chunks), d_out, dst_dev ? uint64_t(dst_len) : n_emit, stream)) return e;
    call_trace().mark("d.decoded");
    if (dst_in_place) {
      PCOB_CUDA_TRY(cudaStreamSynchronize(stream));  // launch_decode has read the statuses back already: the stores are in host memory
    } else if (!dst_dev && n_emit) {
      PCOB_CUDA_TRY(copy_sliced(dst, d_out, n_emit * elem, cudaMemcpyDeviceToHost, stream));
      call_trace().mark("d.d2h_submitted");
      PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
    }
    call_trace().mark("d.end");
    call_trace().flush("decompress");
    outcome->n_total = ih.n_total;
    outcome->terminated = ih.end_byte != 0;
    return PCO_B200_OK;
  }

  // 3b. no index: walk the file (walk_index_free), then decode every chunk walked in one launch.  The kernels write no number past dst_len:
  // a destination that ends inside a chunk gets that chunk's first numbers.
  WalkFile f;
  f.hdr = hdr;
  f.end = compressed_len;
  f.pos = hdr.first_chunk_byte;
  f.cap = f.expect = dst_len;
  uint64_t arena_end = 0;
  if (PcoB200Error e = walk_index_free(c, static_cast<const uint8_t*>(compressed), src_dev, d_src, compressed_len, dtype, {&f}, c.index, &arena_end, stream)) return e;
  const uint64_t n_emit = std::min<uint64_t>(f.count, dst_len);
  void* d_out;
  if (PcoB200Error e = out_buffer(c, dst, dst_dev, n_emit * elem, &d_out)) return e;
  const uint64_t list_at = (arena_end + 15) & ~uint64_t(15), list_end = list_at + f.recs.size() * sizeof(IndexChunk);
  PCOB_CUDA_TRY(c.index.grow_preserve(list_end + 64, arena_end, stream));
  if (!f.recs.empty())
    PCOB_CUDA_TRY(cudaMemcpyAsync(c.index.as<uint8_t>() + list_at, f.recs.data(), f.recs.size() * sizeof(IndexChunk), cudaMemcpyHostToDevice, stream));
  // the chunks in front of a failing one are decoded too, as the reference emits them; a failing decode is the error that wins
  if (PcoB200Error e = launch_decode(c, fp, c.index.as<uint8_t>(), list_end, list_at, uint32_t(f.recs.size()), d_out, dst_dev ? uint64_t(dst_len) : n_emit, stream))
    return e;
  if (f.how == WalkEnd::COLD || f.how == WalkEnd::FAILED) return fail(f.err, f.msg);  // decompress_core takes a cold file to the catch-all decoder
  outcome->n_total = f.count;
  outcome->terminated = f.how == WalkEnd::TERMINATED;
  if (!dst_dev && n_emit) {
    PCOB_CUDA_TRY(copy_sliced(dst, d_out, n_emit * elem, cudaMemcpyDeviceToHost, stream));
    PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
  }
  return PCO_B200_OK;
}

// The catch-all behind the fast kernels: the whole file through cold_decode_kernel (decode_cold.cuh) - one GPU thread, any valid pco.
static PcoB200Error decompress_cold(const void* compressed, size_t compressed_len, uint32_t dtype, void* dst, size_t dst_len, uint32_t flags, void* cuda_stream,
                                    DecodeOutcome* outcome) {
  Context& c = ctx();
  if (PcoB200Error e = ensure_device(c)) return e;
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  const bool src_dev = flags & PCO_B200_SRC_ON_DEVICE, dst_dev = flags & PCO_B200_DST_ON_DEVICE;
  const size_t elem = nt_bits(dtype) / 8;
  StandaloneHeader hdr;
  if (PcoB200Error e = read_heads(compressed, compressed_len, src_dev, nullptr, 0, false, nullptr, &hdr, stream)) return e;
  const uint8_t* d_src;
  if (PcoB200Error e = stage_in(c.src, compressed, compressed_len, src_dev, stream, &d_src)) return e;
  void* d_out;
  if (PcoB200Error e = out_buffer(c, dst, dst_dev, uint64_t(dst_len) * elem, &d_out)) return e;
  const FileParams fp{d_src, compressed_len, dtype, hdr.uniform_type, hdr.format_major};
  std::vector<ColdResult> cres;
  if (PcoB200Error e = cold_decode_jobs(c, dtype, {ColdJob{fp, hdr.first_chunk_byte, d_out, uint64_t(dst_len)}}, cold_retry_file, &cres, stream)) return e;
  const ColdResult& res = cres[0];
  // like the walk path: the chunks before a failing one have been emitted (the reference's decoder stops where the error is)
  const uint64_t n_emit = std::min<uint64_t>(res.n_total, dst_len);
  if (!dst_dev && n_emit) {
    PCOB_CUDA_TRY(copy_sliced(dst, d_out, n_emit * elem, cudaMemcpyDeviceToHost, stream));
    PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
  }
  if (res.status != ST_TERMINATOR && res.status != ST_DST_FULL) return status_to_error(res.status, ("chunk " + std::to_string(res.n_chunks)).c_str());
  outcome->n_total = res.n_total;
  outcome->terminated = res.status == ST_TERMINATOR;
  return PCO_B200_OK;
}

// Core of every decompress entry point: the fast kernels, and for streams they decline (valid pco with Dict mode, Lookback / Conv1
// deltas, tANS tables beyond 2^10 states or 256 bins, ...) the single-thread device decoder.  PCOB200_COLD_DECODE=0 keeps the refusal.
static PcoB200Error decompress_core(const void* compressed, size_t compressed_len, uint32_t dtype, void* dst, size_t dst_len,
                                    const void* index, size_t index_len, uint32_t flags, void* cuda_stream, DecodeOutcome* outcome) {
  PcoB200Error e = decompress_fast(compressed, compressed_len, dtype, dst, dst_len, index, index_len, flags, cuda_stream, outcome);
  static const bool cold_ok = [] { const char* v = std::getenv("PCOB200_COLD_DECODE"); return !(v && v[0] == '0'); }();
  if (e == PCO_B200_UNSUPPORTED && cold_ok) {
    *outcome = DecodeOutcome();
    e = decompress_cold(compressed, compressed_len, dtype, dst, dst_len, flags, cuda_stream, outcome);
  }
  return e;
}

// ---- the asynchronous calls' shared host steps.  Each call enqueues a fixed sequence of launches on the caller's stream (AsyncLaunch,
// host_common.hpp) and makes no host decision between them; its plan does the one-time device set-up, here and not in a call (which may
// be inside a capture).

// Every kernel in `kernels` loaded now (with lazy module loading a kernel is otherwise loaded at its first launch).
static PcoB200Error load_kernels(std::initializer_list<const void*> kernels) {
  cudaFuncAttributes fa;
  for (const void* k : kernels) PCOB_CUDA_TRY(cudaFuncGetAttributes(&fa, k));
  return PCO_B200_OK;
}

// The PcoB200Error of an asynchronous call's status kind, as its *_result function returns it (a kind no call writes reads as Corruption)
static PcoB200Error async_result_kind(uint32_t kind) { return kind <= PCO_B200_UNSUPPORTED ? PcoB200Error(kind) : PCO_B200_CORRUPTION; }

// The set-up of an asynchronous decompress plan: the device, the decode kernels' attributes (the window-mode instantiations when WIN, the
// filter-mode ones when FILT, the aggregate-mode ones when AGG too, the take-mode ones when TAKE too), and loaded: the decode stage's
// kernels for dtype, the call's catch-all kernel (cold(tag) for a latent type tag) and the call's `kernels`.
template <bool WIN, bool FILT = false, bool AGG = false, bool TAKE = false, typename Cold>
static PcoB200Error async_decode_setup(unsigned char dtype, Cold cold, std::initializer_list<const void*> kernels) {
  Context& c = ctx();
  if (PcoB200Error e = ensure_device(c)) return e;
  if (PcoB200Error e = set_decode_attrs<WIN, FILT, AGG, TAKE>(c)) return e;
  if (PcoB200Error e = load_kernels(kernels)) return e;
  return dispatch_latent(dtype, [&](auto tag) -> PcoB200Error {
    using L = decltype(tag);
    return load_kernels({(const void*)fused_narrow_kernel<L, WIN, FILT, AGG, TAKE>, (const void*)symwalk_kernel<WIN>,
                         (const void*)decode_kernel<L, 1, WIN, FILT, AGG, TAKE>, (const void*)decode_kernel<L, 2, WIN, FILT, AGG, TAKE>, cold(tag)});
  });
}

// The plan fields an explicit ModeSpec and DeltaSpec fix (P: any of the three asynchronous compress plans)
template <typename P>
static void fill_explicit_spec(P* plan, const ConfigCheck& ck) {
  plan->mode = ck.explicit_mode.mode;
  plan->order = ck.explicit_order;
  plan->n_vars = ck.explicit_mode.mode == MODE_CLASSIC ? 1 : 2;
  plan->mode_k = ck.explicit_mode.mode_k;
  plan->mode_base = ck.explicit_mode.mode_base;
  plan->base_bits = ck.explicit_mode.base_bits;
  plan->inv_base_bits = ck.explicit_mode.inv_base_bits;
}

// The one-time device set-up of an asynchronous compress plan, here and not in a call (which may be inside a capture): the device, the
// attributes plan_front sets on first use (set_encode_attrs), and loaded: the encode stage's kernels for dtype (split_count_kernel and the planner
// kernels in their CHUNK_BINS instantiations when CHUNK_BINS) and the call's `extra` kernels.
template <bool CHUNK_BINS>
static PcoB200Error async_encode_setup(unsigned char dtype, std::initializer_list<const void*> extra) {
  Context& c = ctx();
  if (PcoB200Error e = ensure_device(c)) return e;
  if (PcoB200Error e = load_kernels(extra)) return e;
  if (PcoB200Error e = load_kernels({(const void*)acomp_two_gate_kernel, (const void*)acomp_var_gate_kernel, (const void*)acomp_pack_gate_kernel,
                                     (const void*)segment_offsets_kernel, (const void*)fallback_kernel<false>, (const void*)ans_encode_kernel<false>,
                                     (const void*)layout_kernel<false>})) return e;
  return dispatch_latent(dtype, [&](auto tag) -> PcoB200Error {
    using L = decltype(tag);
    PCOB_CUDA_TRY((set_encode_attrs<L, false, CHUNK_BINS>()));
    return load_kernels({(const void*)split_count_kernel<L, CHUNK_BINS>, (const void*)split_delta_kernel<L, MODE_CLASSIC>, (const void*)split_delta_kernel<L, MODE_INT_MULT>,
                         (const void*)split_delta_kernel<L, MODE_FLOAT_QUANT>, (const void*)split_delta_kernel<L, MODE_FLOAT_MULT>,
                         (const void*)plan_probe_kernel<L, false, false, CHUNK_BINS>, (const void*)sort_keys_kernel<L>, (const void*)plan_solve_kernel<L, CHUNK_BINS>,
                         (const void*)bin_kernel<L, false>});
  });
}

// The checks of a plan that takes the first bytes of a file: dtype, the buffers (`plan` is the caller's output), the standalone header
// in head, and its uniform type against dtype.
static PcoB200Error check_async_head(const void* head, size_t head_len, unsigned char dtype, const void* plan, StandaloneHeader* hdr) {
  if (!nt_valid(dtype)) return fail(PCO_B200_INVALID_TYPE, "unknown number type byte: " + std::to_string(dtype));
  if (!plan || (!head && head_len)) return fail(PCO_B200_INVALID_ARGUMENT, "null buffer");
  if (PcoB200Error e = parse_standalone_header(static_cast<const uint8_t*>(head), std::min<size_t>(head_len, 32), head_len, hdr)) return e;
  if (hdr->uniform_type != 0 && hdr->uniform_type != dtype)
    return fail(PCO_B200_INVALID_ARGUMENT, "the header's uniform type " + std::to_string(hdr->uniform_type) + " is not dtype " + std::to_string(dtype));
  return PCO_B200_OK;
}

// The decode stage of an asynchronous decompress: fused_narrow_kernel, symwalk_kernel and decode_kernel<L, 1 / 2> over the `slots`
// records of `table`, one CTA each, in window mode when WIN (wins says which numbers of each task are wanted, and dst is unused).
struct DecodeStage {
  FileParams fp;
  const IndexChunk* table;
  const uint8_t* index;
  uint64_t index_len;
  uint32_t slots;
  uint32_t* st;
  uint8_t* cls;
  uint8_t* syms;
  uint32_t* offs;
  const Binoms* binoms;
  void* dst;
  uint64_t dst_cap;
  const WinTask* wins;
  FiltStage filt;  // FILT: dst is the value staging (decode_kernels.cuh, filt_store8); AGG: dst is null (agg_store8); TAKE: likewise (take_store8)
};
template <bool WIN, bool FILT = false, bool AGG = false, bool TAKE = false>
static void enqueue_decode_stage(const AsyncLaunch& ln, const DecodeStage& d) {
  const cudaStream_t stream = ln.stream;
  ln.begin("fused_narrow_kernel");
  dispatch_latent(d.fp.dtype, [&](auto tag) {
    using L = decltype(tag);
    fused_narrow_kernel<L, WIN, FILT, AGG, TAKE><<<d.slots, FZ_THREADS, sizeof(FusedSmem), stream>>>(d.fp, d.table, d.index, d.index_len, d.st, d.cls,
                                                                                         static_cast<L*>(d.dst), d.dst_cap, d.wins, d.filt);
    return 0;
  });
  ln.end();
  ln.begin("symwalk_kernel");
  symwalk_kernel<WIN><<<d.slots, SW_THREADS, sizeof(SymWalkSmem), stream>>>(d.fp, d.table, d.index, d.index_len, d.dst_cap, d.syms, d.offs, d.cls, d.wins);
  ln.end();
  ln.begin("decode_kernel");
  dispatch_latent(d.fp.dtype, [&](auto tag) {
    using L = decltype(tag);
    decode_kernel<L, 1, WIN, FILT, AGG, TAKE><<<d.slots, DEC_THREADS, sizeof(DecodeSmem), stream>>>(d.fp, d.table, d.st, d.index, d.index_len, static_cast<L*>(d.dst),
                                                                                        d.dst_cap, d.binoms, d.syms, d.offs, d.cls, d.wins, d.filt);
    decode_kernel<L, 2, WIN, FILT, AGG, TAKE><<<d.slots, DEC_THREADS, sizeof(DecodeSmem), stream>>>(d.fp, d.table, d.st, d.index, d.index_len, static_cast<L*>(d.dst),
                                                                                        d.dst_cap, d.binoms, d.syms, d.offs, d.cls, d.wins, d.filt);
    return 0;
  });
  ln.end();
}

// The message of a standalone-header refusal of a decompress call (the file's own words: pco_b200_decompress_files_async names the file
// in front), or nullptr for any other status.
static const char* async_header_refusal(uint32_t device_status) {
  switch (device_status) {
    case PCO_B200_ASYNC_HEADER_CORRUPT: return "corrupt standalone header (magic, version, type byte or size hint)";
    case PCO_B200_ASYNC_HEADER_SHORT: return "insufficient data: the file ends inside its standalone header";
    case PCO_B200_ASYNC_HEADER_MISMATCH: return "the file's uniform type or format version differs from the plan's";
    default: return nullptr;
  }
}

}  // namespace pcob200

using namespace pcob200;

extern "C" {

const char* pco_b200_last_error_message(void) { return last_error_ref().c_str(); }

int pco_b200_device_available(void) {
  Context& c = ctx();
  return ensure_device(c) == PCO_B200_OK ? 1 : 0;
}

// pco_c/src/lib.rs:127-139
size_t pco_standalone_guarantee_file_size(size_t n, unsigned char dtype) {
  if (!nt_valid(dtype)) return 0;
  // PagingSpec::default() = EqualPagesUpTo(2^18) (pco/src/chunk_config.rs:127-132, :134-183)
  const EqualPages ep = equal_pages(n, 0);
  size_t res = standalone_header_size();
  if (n > 0) res += ep.rem * standalone_chunk_size_guarantee(nt_bits(dtype), ep.low + 1) + (ep.n_chunks - ep.rem) * standalone_chunk_size_guarantee(nt_bits(dtype), ep.low);
  return res + 1;
}

// pco_c/src/lib.rs:98-120,178-195: full simple_decompress, then fail if it does not fit.
enum PcoError pco_standalone_simple_decompress_into(const void* compressed, size_t compressed_len, unsigned char dtype, void* dst,
                                                    size_t dst_cap, size_t* n_written) {
  if (!nt_valid(dtype)) return PcoInvalidType;
  DecodeOutcome oc;
  PcoB200Error e = decompress_core(compressed, compressed_len, dtype, dst, dst_cap, nullptr, 0, 0, nullptr, &oc);
  if (e != PCO_B200_OK) return PcoDecompressionError;
  if (oc.n_total > dst_cap) {
    fail(PCO_B200_IO, "decompressed count exceeds dst_cap");
    return PcoDecompressionError;
  }
  if (n_written) *n_written = size_t(oc.n_total);
  return PcoSuccess;
}

PcoB200Error pco_b200_decompress_ex(const void* compressed, size_t compressed_len, unsigned char dtype, void* dst, size_t dst_len,
                                    PcoB200Progress* progress, const void* index, size_t index_len, uint32_t flags, void* cuda_stream) {
  DecodeOutcome oc;
  PcoB200Error e = decompress_core(compressed, compressed_len, dtype, dst, dst_len, index, index_len, flags, cuda_stream, &oc);
  profiler().resolve();
  if (e != PCO_B200_OK) return e;
  if (progress) {
    progress->n_processed = size_t(std::min<uint64_t>(oc.n_total, dst_len));
    progress->finished = (oc.terminated && oc.n_total <= dst_len) ? 1 : 0;
  }
  return PCO_B200_OK;
}

PcoB200Error pco_b200_simple_decompress_into(const void* compressed, size_t compressed_len, unsigned char dtype, void* dst, size_t dst_len,
                                             PcoB200Progress* progress) {
  return pco_b200_decompress_ex(compressed, compressed_len, dtype, dst, dst_len, progress, nullptr, 0, 0, nullptr);
}

// The config a call runs: *config, or pco::ChunkConfig::default() (level 8, Auto, Auto, EqualPagesUpTo(2^18)) when config is null
static PcoB200ChunkConfig default_chunk_config(const PcoB200ChunkConfig* config) {
  if (config) return *config;
  PcoB200ChunkConfig cfg;
  std::memset(&cfg, 0, sizeof(cfg));
  cfg.compression_level = 8;
  return cfg;
}

static PcoB200Error compress_dispatch(const void* nums, size_t n, unsigned char dtype, const PcoB200ChunkConfig* config, bool uniform, void* dst,
                                      size_t dst_cap, size_t* n_written, void* index, size_t index_cap, size_t* index_len, uint32_t flags,
                                      void* cuda_stream) {
  if (!nt_valid(dtype)) return fail(PCO_B200_INVALID_TYPE, "unknown number type byte: " + std::to_string(dtype));
  const PcoB200ChunkConfig cfg = default_chunk_config(config);
  Context& c = ctx();
  if (PcoB200Error e = ensure_device(c)) return e;
  CompressResult res;
  PcoB200Error e = dispatch_latent(dtype, [&](auto tag) {
    using L = decltype(tag);
    return compress_typed<L>(c.enc, nums, n, dtype, cfg, uniform, dst, dst_cap, index, index_cap, flags, static_cast<cudaStream_t>(cuda_stream), &res);
  });
  profiler().resolve();
  if (e != PCO_B200_OK) return e;
  if (n_written) *n_written = size_t(res.total_bytes);
  if (index_len) *index_len = size_t(res.index_bytes);
  return PCO_B200_OK;
}

PcoB200Error pco_b200_compress_ex(const void* nums, size_t n, unsigned char dtype, const PcoB200ChunkConfig* config, int uniform_type_header,
                                  void* dst, size_t dst_cap, size_t* n_written, void* index, size_t index_cap, size_t* index_len, uint32_t flags,
                                  void* cuda_stream) {
  return compress_dispatch(nums, n, dtype, config, uniform_type_header != 0, dst, dst_cap, n_written, index, index_cap, index_len, flags, cuda_stream);
}
PcoB200Error pco_b200_simple_compress(const void* nums, size_t n, unsigned char dtype, const PcoB200ChunkConfig* config, void* dst, size_t dst_cap,
                                      size_t* n_written) {
  return compress_dispatch(nums, n, dtype, config, false, dst, dst_cap, n_written, nullptr, 0, nullptr, 0, nullptr);
}
PcoB200Error pco_b200_simple_compress_into(const void* nums, size_t n, unsigned char dtype, const PcoB200ChunkConfig* config, void* dst,
                                           size_t dst_cap, size_t* n_written) {
  return compress_dispatch(nums, n, dtype, config, true, dst, dst_cap, n_written, nullptr, 0, nullptr, 0, nullptr);
}

// pco_c/src/lib.rs:76-96,146-169: Auto mode / Auto delta, enable_8_bit, uniform-type header
enum PcoError pco_standalone_simple_compress_into(const void* nums, size_t n, unsigned char dtype, const struct PcoChunkConfig* config, void* dst,
                                                  size_t dst_cap, size_t* n_written) {
  if (!nt_valid(dtype)) return PcoInvalidType;
  PcoB200ChunkConfig cfg;
  std::memset(&cfg, 0, sizeof(cfg));
  cfg.compression_level = config ? config->compression_level : 8;
  cfg.max_page_n = config ? config->max_page_n : 0;
  cfg.mode_spec = PCO_B200_MODE_AUTO;
  cfg.delta_spec = PCO_B200_DELTA_AUTO;
  cfg.enable_8_bit = 1;
  PcoB200Error e = compress_dispatch(nums, n, dtype, &cfg, true, dst, dst_cap, n_written, nullptr, 0, nullptr, 0, nullptr);
  return e == PCO_B200_OK ? PcoSuccess : PcoCompressionError;
}

// ---------------------------------------------------------------------------
// Wrapped format (pco/src/wrapped/): one page per chunk.  A wrapped chunk = chunk meta bytes + page bytes, i.e. a
// standalone chunk without its 4-byte preamble, so the compressor handle holds one CHUNKS_ONLY chunk and the page
// decoder re-frames meta + page as a one-chunk standalone file for the same kernels.
// ---------------------------------------------------------------------------
struct PcoB200ChunkCompressor {
  // one emission per page, back to back: [type byte][page_n - 1 (24 bits)][chunk meta][page]; the pages of a chunk share
  // their bins, so every emission carries the same chunk meta
  std::vector<uint8_t> bytes;
  size_t meta_len = 0;
  size_t n = 0;
  std::vector<size_t> page_off, page_n;  // byte offset of each emission (+ one past the last), numbers per page
};

PcoB200Error pco_b200_file_compressor_write_header(void* dst, size_t dst_cap, size_t* n_written) {
  if (dst_cap < 2) return fail(PCO_B200_IO, "failed to write whole buffer");
  static_cast<uint8_t*>(dst)[0] = 4;  // FormatVersion { major: 4, minor: 1 } (metadata/format_version.rs:30-34,87-91)
  static_cast<uint8_t*>(dst)[1] = 1;
  if (n_written) *n_written = 2;
  return PCO_B200_OK;
}

PcoB200Error pco_b200_file_decompressor_read_header(const void* src, size_t src_len, size_t* n_read) {
  const uint8_t* b = static_cast<const uint8_t*>(src);
  if (src_len < 1) return fail(PCO_B200_INSUFFICIENT_DATA, "empty wrapped header");
  const uint8_t major = b[0];
  if (major > 4) return fail(PCO_B200_CORRUPTION, "file's format version exceeds the max supported version");  // format_version.rs:60-72
  size_t used = 1;
  if (major >= 4) {  // the minor version byte exists from 4.0 on
    if (src_len < 2) return fail(PCO_B200_INSUFFICIENT_DATA, "wrapped header is cut short");
    used = 2;
  }
  if (major < 4) return fail(PCO_B200_UNSUPPORTED, "wrapped files older than format 4 are outside the GPU hot path");
  if (n_read) *n_read = used;
  return PCO_B200_OK;
}

PcoB200Error pco_b200_chunk_compressor_new(const void* nums, size_t n, unsigned char dtype, const PcoB200ChunkConfig* config,
                                           PcoB200ChunkCompressor** out) {
  if (!out) return fail(PCO_B200_INVALID_ARGUMENT, "null output handle");
  *out = nullptr;
  if (!nt_valid(dtype)) return fail(PCO_B200_INVALID_TYPE, "unknown number type byte: " + std::to_string(dtype));
  if (n == 0) return fail(PCO_B200_INVALID_ARGUMENT, "cannot compress empty chunk");  // chunk_compressor.rs:113-127
  const PcoB200ChunkConfig cfg = default_chunk_config(config);
  std::vector<uint64_t> pages;
  if (PcoB200Error e = n_per_page(cfg, n, &pages)) return e;
  auto cc = std::make_unique<PcoB200ChunkCompressor>();
  cc->n = n;
  const ChunksScratch cs = chunks_only_scratch(nt_bits(dtype), n, pages);
  cc->bytes.resize(cs.bytes);
  size_t written = 0, ilen = 0;
  std::vector<uint8_t> index(cs.index);
  // several pages: the pipeline runs them as the call's chunks with ONE set of bins trained on all of them
  const uint32_t flags = PCO_B200_CHUNKS_ONLY | (pages.size() > 1 ? PCO_B200_INTERNAL_SHARED_BINS : 0u);
  if (PcoB200Error e = compress_dispatch(nums, n, dtype, &cfg, false, cc->bytes.data(), cc->bytes.size(), &written, index.data(), index.size(), &ilen, flags,
                                         nullptr))
    return e;
  cc->bytes.resize(written);
  if (written < 4 || ilen < sizeof(IndexHeader)) return fail(PCO_B200_CUDA, "compressor returned a truncated chunk");
  IndexHeader ih;
  std::memcpy(&ih, index.data(), sizeof(ih));
  if (ih.n_chunks != pages.size() || ih.chunks_offset + ih.n_chunks * sizeof(IndexChunk) > ilen) return fail(PCO_B200_CUDA, "compressor returned an inconsistent page table");
  for (size_t p = 0; p < pages.size(); p++) {
    IndexChunk ic;
    std::memcpy(&ic, index.data() + ih.chunks_offset + p * sizeof(IndexChunk), sizeof(ic));
    cc->page_off.push_back(size_t(ic.chunk_offset));
    cc->page_n.push_back(size_t(pages[p]));
  }
  cc->page_off.push_back(written);
  if (PcoB200Error e = pco_b200_chunk_meta_size(cc->bytes.data() + 4, cc->page_off[1] - 4, dtype, &cc->meta_len)) return e;
  for (size_t p = 1; p < pages.size(); p++)  // shared bins: every page's emission repeats the chunk meta
    if (cc->page_off[p + 1] - cc->page_off[p] < 4 + cc->meta_len ||
        std::memcmp(cc->bytes.data() + 4, cc->bytes.data() + cc->page_off[p] + 4, cc->meta_len) != 0)
      return fail(PCO_B200_CUDA, "pages of one chunk came back with different chunk metas");
  *out = cc.release();
  return PCO_B200_OK;
}
void pco_b200_chunk_compressor_free(PcoB200ChunkCompressor* cc) { delete cc; }
size_t pco_b200_chunk_compressor_n_pages(const PcoB200ChunkCompressor* cc) { return cc ? cc->page_n.size() : 0; }
size_t pco_b200_chunk_compressor_page_n(const PcoB200ChunkCompressor* cc, size_t page_idx) {
  return (cc && page_idx < cc->page_n.size()) ? cc->page_n[page_idx] : 0;
}
size_t pco_b200_chunk_compressor_meta_size(const PcoB200ChunkCompressor* cc) { return cc ? cc->meta_len : 0; }
size_t pco_b200_chunk_compressor_page_size(const PcoB200ChunkCompressor* cc, size_t page_idx) {
  return (cc && page_idx < cc->page_n.size()) ? cc->page_off[page_idx + 1] - cc->page_off[page_idx] - 4 - cc->meta_len : 0;
}
PcoB200Error pco_b200_chunk_compressor_write_meta(const PcoB200ChunkCompressor* cc, void* dst, size_t dst_cap, size_t* n_written) {
  if (!cc) return fail(PCO_B200_INVALID_ARGUMENT, "null chunk compressor");
  if (dst_cap < cc->meta_len) return fail(PCO_B200_IO, "failed to write whole buffer");
  std::memcpy(dst, cc->bytes.data() + 4, cc->meta_len);
  if (n_written) *n_written = cc->meta_len;
  return PCO_B200_OK;
}
PcoB200Error pco_b200_chunk_compressor_write_page(const PcoB200ChunkCompressor* cc, size_t page_idx, void* dst, size_t dst_cap, size_t* n_written) {
  if (!cc) return fail(PCO_B200_INVALID_ARGUMENT, "null chunk compressor");
  if (page_idx >= cc->page_n.size())  // chunk_compressor.rs:661-666
    return fail(PCO_B200_INVALID_ARGUMENT, "page idx exceeds num pages (" + std::to_string(page_idx) + " >= " + std::to_string(cc->page_n.size()) + ")");
  const size_t begin = cc->page_off[page_idx] + 4 + cc->meta_len, len = cc->page_off[page_idx + 1] - begin;
  if (dst_cap < len) return fail(PCO_B200_IO, "failed to write whole buffer");
  std::memcpy(dst, cc->bytes.data() + begin, len);
  if (n_written) *n_written = len;
  return PCO_B200_OK;
}

// Only what the GPU path writes and reads is accepted: Classic / IntMult / FloatMult / FloatQuant, delta None / Consecutive.
PcoB200Error pco_b200_chunk_meta_size(const void* src, size_t src_len, unsigned char dtype, size_t* meta_len) {
  if (!nt_valid(dtype)) return fail(PCO_B200_INVALID_TYPE, "unknown number type byte: " + std::to_string(dtype));
  uint64_t len = 0;
  bool cold = false;
  uint32_t mode = 0, variant = 0;
  wrapped_meta_len(static_cast<const uint8_t*>(src), src_len, dtype, &len, &cold, &mode, &variant);
  if (mode > MODE_FLOAT_QUANT) return fail(PCO_B200_UNSUPPORTED, "wrapped chunk meta: mode outside the GPU hot path");
  if (variant > DELTA_CONSECUTIVE) return fail(PCO_B200_UNSUPPORTED, "wrapped chunk meta: delta encoding outside the GPU hot path");
  if (len > src_len) return fail(PCO_B200_INSUFFICIENT_DATA, "chunk meta is cut short");
  if (meta_len) *meta_len = size_t(len);
  return PCO_B200_OK;
}

PcoB200Error pco_b200_page_decompress(const void* chunk_meta, size_t meta_len, const void* page, size_t page_len, size_t page_n,
                                      unsigned char dtype, void* dst, size_t dst_len, PcoB200Progress* progress, size_t* bytes_read) {
  if (!nt_valid(dtype)) return fail(PCO_B200_INVALID_TYPE, "unknown number type byte: " + std::to_string(dtype));
  if (page_n == 0 || page_n > (size_t(1) << 24)) return fail(PCO_B200_INVALID_ARGUMENT, "page n out of range");
  // PageDecompressor::read: dst must take whole batches or the rest of the page (page_decompressor.rs:200-206)
  if (dst_len % BATCH_N != 0 && dst_len < page_n)
    return fail(PCO_B200_INVALID_ARGUMENT, "num_dst's length must either be a multiple of 256 or be at least the count of numbers remaining");
  // one-chunk standalone file around the same bytes: header | type byte | n - 1 | meta | page | terminator
  std::vector<uint8_t> file = make_standalone_header(page_n, 0);
  file.push_back(dtype);
  const uint32_t nm1 = uint32_t(page_n - 1);
  file.push_back(uint8_t(nm1)); file.push_back(uint8_t(nm1 >> 8)); file.push_back(uint8_t(nm1 >> 16));
  const uint8_t* m = static_cast<const uint8_t*>(chunk_meta);
  const uint8_t* p = static_cast<const uint8_t*>(page);
  file.insert(file.end(), m, m + meta_len);
  file.insert(file.end(), p, p + page_len);
  file.push_back(0);
  PcoB200Progress prog{0, 0};
  if (PcoB200Error e = pco_b200_decompress_ex(file.data(), file.size(), dtype, dst, dst_len, &prog, nullptr, 0, 0, nullptr)) return e;
  prog.finished = prog.n_processed >= page_n ? 1 : 0;
  if (progress) *progress = prog;
  if (bytes_read) *bytes_read = page_len;
  return PCO_B200_OK;
}

#ifdef PCOB_DEC_TIMING
// experiment builds only: read and reset the decode kernel's region timers
int pco_b200_debug_dec_timing(unsigned long long* out16) {
  cudaDeviceSynchronize();
  cudaMemcpyFromSymbol(out16, g_dec_timing, sizeof(unsigned long long) * 16);
  unsigned long long z[16] = {0};
  cudaMemcpyToSymbol(g_dec_timing, z, sizeof(z));
  return 0;
}
#endif

#ifdef PCOB_ENC_TIMING
int pco_b200_debug_enc_timing(unsigned long long* out32) {
  cudaDeviceSynchronize();
  cudaMemcpyFromSymbol(out32, g_enc_timing, sizeof(unsigned long long) * 32);
  unsigned long long z[32] = {0};
  cudaMemcpyToSymbol(g_enc_timing, z, sizeof(z));
  return 0;
}
#endif

// ModeSpec::Auto for one chunk in host memory (mode_search.hpp); no device involved
PcoB200Error pco_b200_choose_mode(const void* nums, size_t n, unsigned char dtype, PcoB200ModeChoice* out) {
  if (!out || (!nums && n)) return fail(PCO_B200_INVALID_ARGUMENT, "null argument");
  if (!nt_valid(dtype)) return fail(PCO_B200_INVALID_ARGUMENT, "unknown number type byte");
  if (n > (size_t(1) << 24)) return fail(PCO_B200_INVALID_ARGUMENT, "count may not exceed 16777216 per chunk");
  std::memset(out, 0, sizeof(*out));
  mode_search::Choice c;
  const bool is_float = nt_is_float(dtype), is_signed = nt_is_signed(dtype);
  switch (nt_bits(dtype)) {
    case 64: c = is_float ? mode_search::choose_float<double>(static_cast<const uint64_t*>(nums), n) : mode_search::choose_int<uint64_t>(static_cast<const uint64_t*>(nums), n, is_signed); break;
    case 32: c = is_float ? mode_search::choose_float<float>(static_cast<const uint32_t*>(nums), n) : mode_search::choose_int<uint32_t>(static_cast<const uint32_t*>(nums), n, is_signed); break;
    case 16: c = is_float ? mode_search::choose_float<mode_search::Half>(static_cast<const uint16_t*>(nums), n) : mode_search::choose_int<uint16_t>(static_cast<const uint16_t*>(nums), n, is_signed); break;
    default: c = mode_search::choose_int<uint8_t>(static_cast<const uint8_t*>(nums), n, is_signed); break;
  }
  out->mode_spec = c.kind == 1 ? PCO_B200_MODE_TRY_INT_MULT : c.kind == 2 ? PCO_B200_MODE_TRY_FLOAT_MULT : c.kind == 3 ? PCO_B200_MODE_TRY_FLOAT_QUANT : PCO_B200_MODE_CLASSIC;
  out->float_quant_k = c.k;
  out->float_mult_base = c.base;
  out->float_mult_inv_base = c.inv_base;
  out->int_mult_base = c.int_base;
  out->bits_saved_per_num = c.bits_saved_per_num;
  return PCO_B200_OK;
}

void pco_b200_profile_enable(int on) { profiler_enabled().store(on != 0); }
// Test hook for the host logic of the speculative index-free walk (no device involved): follow_chunk_chain over caller-made tables.
// Returns the number of verified chunks; their candidate indices go to `verified` (room for m), the position behind the last one to *next_pos.
size_t pco_b200_debug_follow_chain(const uint64_t* cand, const uint32_t* statuses, const uint64_t* ends, uint32_t m, uint64_t pos, uint64_t n0, uint64_t out_off,
                                   uint64_t dst_len, uint64_t src_len, uint32_t* verified, uint64_t* next_pos) {
  uint64_t p = pos;
  const std::vector<uint32_t> chain = follow_chunk_chain(cand, statuses, ends, m, pos, n0, out_off, dst_len, src_len, &p);
  for (size_t i = 0; i < chain.size(); i++) verified[i] = chain[i];
  if (next_pos) *next_pos = p;
  return chain.size();
}
int pco_b200_zero_copy(int mask) { return mask < 0 ? zero_copy_mask().load() : zero_copy_mask().exchange(mask & 7); }
// Frees the calling thread's device scratch (a worker thread calls this before it exits; the buffers are otherwise kept for the
// thread's next call).
void pco_b200_thread_release(void) {
  Context& c = ctx();
  if (c.initialized || c.d_binoms) reset_context(c);  // also a context whose set-up failed (it may hold the binomial table)
  readback_bounce().release();
}
// Which decode instantiation served the chunks of the last decode launch: counts[k] = chunks of class k
// (1, 2: decode_kernel<L, 1 / 2>; 3, 4, 5: fused_narrow_kernel, delta order 0 / 1 / 2..7).  Returns the number of chunks.
int pco_b200_profile_chunk_classes(unsigned* counts8) {
  Context& c = ctx();
  for (int i = 0; i < 8; i++) counts8[i] = 0;
  if (!c.device_ok || c.last_decode_chunks == 0 || !c.d_cls) return 0;
  std::vector<uint8_t> cls(c.last_decode_chunks);
  if (cudaMemcpy(cls.data(), c.d_cls, cls.size(), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  for (uint8_t k : cls) counts8[(k & 0x7f) < 8 ? (k & 0x7f) : 0]++;
  return int(cls.size());
}
// How ans_encode_kernel resolved the tANS rounds of the last compress pass on this thread, when it ran with profiling on: counts[k] =
// (chunk, var, round) triples resolved by k (0: speculation held, 1: fix-up converged, 2: transfer functions, 3: in-order pass),
// counts[4 + k] = those among them that were not a page's first round.  Returns the number of rounds counted (0 and all zeros without a
// profiled compress).
int pco_b200_profile_ans_paths(unsigned* counts8) {
  Context& c = ctx();
  for (int i = 0; i < 8; i++) counts8[i] = 0;
  if (!c.device_ok || !c.enc.ans_paths_valid) return 0;
  if (cudaMemcpy(counts8, c.enc.ans_paths.p, ANS_PATH_SLOTS * sizeof(uint32_t), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  return int(counts8[ANS_PATH_SPECULATION] + counts8[ANS_PATH_FIXUP] + counts8[ANS_PATH_TRANSFER] + counts8[ANS_PATH_IN_ORDER]);
}
// Copies "name=ms;name=ms;..." of the last finished call into buf; returns the number of spans.
int pco_b200_profile_last(char* buf, size_t cap) {
  if (!profiler().spans.empty()) profiler().resolve();  // an asynchronous call leaves its spans pending: wait for them here
  std::string s;
  for (auto& kv : profiler().last) s += kv.first + "=" + std::to_string(kv.second) + ";";
  if (cap) {
    size_t n = std::min(cap - 1, s.size());
    std::memcpy(buf, s.data(), n);
    buf[n] = 0;
  }
  return int(profiler().last.size());
}

size_t pco_b200_index_size_bound(size_t n, size_t n_chunks_hint) {
  size_t chunks = n_chunks_hint + 2;
  size_t batches = n / BATCH_N + 2 * chunks;
  return sizeof(IndexHeader) + chunks * sizeof(IndexChunk) + batches * MAX_VARS * sizeof(BatchEntry) + 16 * chunks + 64;
}

// Batched decompress of chunks whose byte offsets the caller knows (SURVEY.md 8b "decompress_chunks"): a container that
// keeps chunk / page offsets beside the bytes - pco's wrapped use case, a sharded writer's offset table - needs no side
// index.  The per-batch index is built on the device by one tANS walk per chunk, ALL CHUNKS IN PARALLEL (the standalone
// format's single serial cursor only exists because chunk lengths are not in the stream), then the ordinary decode runs.
PcoB200Error pco_b200_decompress_chunks(const void* compressed, size_t compressed_len, unsigned char dtype, const uint64_t* chunk_offsets,
                                        const uint32_t* chunk_ns, size_t n_chunks, void* dst, size_t dst_len, size_t* n_written, uint32_t flags,
                                        void* cuda_stream) {
  if (!nt_valid(dtype)) return fail(PCO_B200_INVALID_TYPE, "unknown number type byte: " + std::to_string(dtype));
  if (n_written) *n_written = 0;
  if (n_chunks == 0) return PCO_B200_OK;
  if (!chunk_offsets || !chunk_ns) return fail(PCO_B200_INVALID_ARGUMENT, "chunk_offsets and chunk_ns are required");
  if (n_chunks > 0x7fffffffull) return fail(PCO_B200_INVALID_ARGUMENT, "too many chunks");
  Context& c = ctx();
  if (PcoB200Error e = ensure_device(c)) return e;
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  const bool src_dev = flags & PCO_B200_SRC_ON_DEVICE, dst_dev = flags & PCO_B200_DST_ON_DEVICE;
  const size_t elem = nt_bits(dtype) / 8;
  // a standalone file (magic present) carries the format version and the uniform type; bare chunks are format 4.1
  uint32_t format_major = 4, uniform_type = 0;
  {
    uint8_t head[32] = {0};
    const size_t avail = std::min<size_t>(compressed_len, sizeof(head));
    if (avail) {
      if (src_dev) { PCOB_CUDA_TRY(cudaMemcpyAsync(head, compressed, avail, cudaMemcpyDeviceToHost, stream)); PCOB_CUDA_TRY(cudaStreamSynchronize(stream)); }
      else std::memcpy(head, compressed, avail);
    }
    static const uint8_t MAGIC[4] = {112, 99, 111, 33};
    if (avail >= 4 && std::memcmp(head, MAGIC, 4) == 0 && chunk_offsets[0] >= 4) {
      StandaloneHeader hdr;
      if (PcoB200Error e = parse_standalone_header(head, avail, compressed_len, &hdr)) return e;
      format_major = hdr.format_major;
      uniform_type = hdr.uniform_type;
    }
  }
  // index skeleton: chunk records from the caller's table, room for 2 vars of entries per chunk
  const uint64_t chunks_offset = sizeof(IndexHeader);
  std::vector<IndexChunk> recs(n_chunks);
  uint64_t out_off = 0;
  for (size_t i = 0; i < n_chunks; i++) {
    if (chunk_offsets[i] >= compressed_len) return fail(PCO_B200_INVALID_ARGUMENT, "chunk offset " + std::to_string(i) + " lies outside the buffer");
    if (chunk_ns[i] == 0 || chunk_ns[i] > (1u << 24)) return fail(PCO_B200_INVALID_ARGUMENT, "chunk " + std::to_string(i) + ": count must be 1..2^24");
    recs[i].chunk_offset = chunk_offsets[i];
    recs[i].n = chunk_ns[i];
    recs[i].n_vars = 0;
    recs[i].out_offset = out_off;
    out_off += chunk_ns[i];
  }
  const uint64_t off = lay_out_entries(recs.data(), n_chunks, (chunks_offset + uint64_t(n_chunks) * sizeof(IndexChunk) + 15) & ~uint64_t(15));
  const uint64_t n_total = out_off;
  if (n_total > dst_len) return fail(PCO_B200_INVALID_ARGUMENT, "dst holds " + std::to_string(dst_len) + " numbers, the chunks " + std::to_string(n_total));
  const uint8_t* d_src;
  if (PcoB200Error e = stage_in(c.src, compressed, compressed_len, src_dev, stream, &d_src)) return e;
  const FileParams fp{d_src, compressed_len, dtype, uniform_type, format_major};
  PCOB_CUDA_TRY(c.index.reserve(off + 64));
  uint8_t* d_index = c.index.as<uint8_t>();
  PCOB_CUDA_TRY(cudaMemcpyAsync(d_index + chunks_offset, recs.data(), n_chunks * sizeof(IndexChunk), cudaMemcpyHostToDevice, stream));
  PCOB_CUDA_TRY(c.statuses.reserve((n_chunks + 1) * sizeof(uint32_t)));
  PCOB_CUDA_TRY(c.misc.reserve(sizeof(WalkResult)));
  PCOB_CUDA_TRY(cudaMemsetAsync(c.statuses.p, 0xff, n_chunks * sizeof(uint32_t), stream));
  profiler().begin("walk_kernel", stream);
  walk_kernel<SMALL_MAX_SIZE_LOG><<<uint32_t(n_chunks), WALK_THREADS, sizeof(WalkSmem<SMALL_MAX_SIZE_LOG>), stream>>>(
      fp, d_index, chunks_offset, uint32_t(n_chunks), 0, off, 0, 0, ~uint64_t(0), c.statuses.as<uint32_t>(), c.misc.as<WalkResult>(), 0);
  profiler().end(stream);
  PCOB_CUDA_TRY(cudaGetLastError());
  {
    std::vector<uint32_t> st(n_chunks);
    PCOB_CUDA_TRY(cudaMemcpyAsync(st.data(), c.statuses.p, n_chunks * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
    PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
    for (size_t i = 0; i < n_chunks; i++)
      if (st[i] != ST_OK) { profiler().resolve(); return status_to_error(st[i], ("chunk " + std::to_string(i)).c_str()); }
  }
  void* d_out;
  if (PcoB200Error e = out_buffer(c, dst, dst_dev, n_total * elem, &d_out)) return e;
  PcoB200Error e = launch_decode(c, fp, d_index, off, chunks_offset, uint32_t(n_chunks), d_out, dst_dev ? uint64_t(dst_len) : n_total, stream);
  profiler().resolve();
  if (e != PCO_B200_OK) return e;
  if (!dst_dev && n_total) {
    PCOB_CUDA_TRY(copy_sliced(dst, d_out, n_total * elem, cudaMemcpyDeviceToHost, stream));
    PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
  }
  if (n_written) *n_written = size_t(n_total);
  return PCO_B200_OK;
}

// ---------------------------------------------------------------------------
// Batched wrapped pages (wrapped_kernels.cuh).  Decode: every page is framed as a standalone chunk in scratch, all of them are walked
// at once and the ordinary decode kernels take the pages they serve; the pages they decline go through cold_decode_kernel, one launch
// per page.  Encode: the CHUNKS_ONLY pipeline, then every chunk's meta and page are split into the caller's two buffers.
// ---------------------------------------------------------------------------
static PcoB200Error page_fail(PcoB200Error kind, size_t page, const std::string& what) {
  return fail(kind, "page " + std::to_string(page) + ": " + what);
}
static PcoB200Error page_status_fail(uint32_t st, size_t page) {
  const PcoB200Error e = status_to_error(st, "the page");
  return page_fail(e, page, last_error_ref());
}

static PcoB200Error decompress_pages_impl(const void* metas, size_t metas_len, const void* pages, size_t pages_len, uint32_t dtype,
                                          const PcoB200PageRef* refs, size_t n_pages, void* dst, size_t dst_len, size_t* n_written, uint32_t flags,
                                          cudaStream_t stream) {
  // ---- argument checks: host only, before any device work
  if (!nt_valid(dtype)) return fail(PCO_B200_INVALID_TYPE, "unknown number type byte: " + std::to_string(dtype));
  if (n_written) *n_written = 0;
  if (n_pages == 0) return PCO_B200_OK;
  if (!refs) return fail(PCO_B200_INVALID_ARGUMENT, "refs are required");
  if (n_pages > 0x7ffffffeull) return fail(PCO_B200_INVALID_ARGUMENT, "too many pages");
  if ((!metas && metas_len) || (!pages && pages_len) || !dst) return fail(PCO_B200_INVALID_ARGUMENT, "null buffer");
  // page table, and the index skeleton: one IndexChunk per page plus a spare one (a failing page walked on its own)
  const uint64_t chunks_offset = sizeof(IndexHeader);
  std::vector<WrappedPage> tab(n_pages);
  std::vector<IndexChunk> recs(n_pages + 1);
  uint64_t frames_len = 0, n_total = 0;
  for (size_t i = 0; i < n_pages; i++) {
    const PcoB200PageRef& r = refs[i];
    if (r.meta_len > metas_len || r.meta_offset > metas_len - r.meta_len) return page_fail(PCO_B200_INVALID_ARGUMENT, i, "chunk meta lies outside metas");
    if (r.page_len > pages_len || r.page_offset > pages_len - r.page_len) return page_fail(PCO_B200_INVALID_ARGUMENT, i, "page lies outside pages");
    if (r.page_n == 0 || r.page_n > (uint64_t(1) << 24)) return page_fail(PCO_B200_INVALID_ARGUMENT, i, "page n must be 1..2^24");
    WrappedPage& w = tab[i];
    w.meta_off = r.meta_offset; w.meta_len = r.meta_len; w.page_off = r.page_offset; w.page_len = r.page_len;
    w.frame_off = frames_len; w.page_n = uint32_t(r.page_n); w.pad = 0;
    recs[i].chunk_offset = frames_len;
    recs[i].n = uint32_t(r.page_n);
    recs[i].n_vars = 0;
    recs[i].out_offset = n_total;
    frames_len += (4 + r.meta_len + r.page_len + 15) & ~uint64_t(15);  // 16-byte aligned chunk starts for the kernels' block reads
    n_total += r.page_n;
  }
  if (n_total > dst_len) return fail(PCO_B200_INVALID_ARGUMENT, "dst holds " + std::to_string(dst_len) + " numbers, the pages " + std::to_string(n_total));
  const uint64_t entries = lay_out_entries(recs.data(), n_pages, (chunks_offset + (uint64_t(n_pages) + 1) * sizeof(IndexChunk) + 15) & ~uint64_t(15));

  Context& c = ctx();
  if (PcoB200Error e = ensure_device(c)) return e;
  const bool src_dev = flags & PCO_B200_SRC_ON_DEVICE, dst_dev = flags & PCO_B200_DST_ON_DEVICE;
  const size_t elem = nt_bits(dtype) / 8;
  const uint32_t n = uint32_t(n_pages);
  const uint8_t *d_metas, *d_pages;
  if (PcoB200Error e = stage_in(c.wrap_metas, metas, metas_len, src_dev, stream, &d_metas)) return e;
  if (PcoB200Error e = stage_in(c.src, pages, pages_len, src_dev, stream, &d_pages)) return e;
  PCOB_CUDA_TRY(c.wrap_tab.reserve(n_pages * sizeof(WrappedPage)));
  PCOB_CUDA_TRY(cudaMemcpyAsync(c.wrap_tab.p, tab.data(), n_pages * sizeof(WrappedPage), cudaMemcpyHostToDevice, stream));
  PCOB_CUDA_TRY(c.index.reserve(entries + 64));
  uint8_t* d_index = c.index.as<uint8_t>();
  PCOB_CUDA_TRY(cudaMemcpyAsync(d_index + chunks_offset, recs.data(), n_pages * sizeof(IndexChunk), cudaMemcpyHostToDevice, stream));
  PCOB_CUDA_TRY(c.wrap_frames.reserve(frames_len + 64));
  uint8_t* d_frames = c.wrap_frames.as<uint8_t>();
  // results: frame_pages_kernel's route per page | walk status per page | walk end per page | the spare walk's status
  const size_t res_words = 2 * size_t(n) + 2 * size_t(n) + 2;
  PCOB_CUDA_TRY(c.wrap_res.reserve(res_words * 4 + 64));
  uint32_t* d_pstat = c.wrap_res.as<uint32_t>();
  uint32_t* d_wst = d_pstat + n;
  uint64_t* d_ends = reinterpret_cast<uint64_t*>(d_pstat + 2 * size_t(n));  // 8-byte aligned: 2n words behind the buffer's start
  uint32_t* d_spare_st = reinterpret_cast<uint32_t*>(d_ends + n);
  PCOB_CUDA_TRY(cudaMemsetAsync(d_wst, 0xff, size_t(n) * 4, stream));
  PCOB_CUDA_TRY(c.misc.reserve(sizeof(WalkResult)));
  profiler().begin("frame_pages_kernel", stream);
  frame_pages_kernel<<<n, WRAP_THREADS, 0, stream>>>(d_metas, metas_len, d_pages, dtype, c.wrap_tab.as<WrappedPage>(), d_frames, d_pstat);
  profiler().end(stream);
  PCOB_CUDA_TRY(cudaGetLastError());
  const FileParams fp{d_frames, frames_len, dtype, 0, 4};  // wrapped format 4.x; a page carries no uniform type
  profiler().begin("walk_kernel", stream);
  walk_kernel<SMALL_MAX_SIZE_LOG><<<n, WALK_THREADS, sizeof(WalkSmem<SMALL_MAX_SIZE_LOG>), stream>>>(
      fp, d_index, chunks_offset, n, 0, entries, 0, 0, ~uint64_t(0), d_wst, c.misc.as<WalkResult>(), 0, d_ends);
  profiler().end(stream);
  PCOB_CUDA_TRY(cudaGetLastError());
  std::vector<uint32_t> res(4 * size_t(n));
  PCOB_CUDA_TRY(readback_small_sync(res.data(), d_pstat, res.size() * 4, stream));
  const uint32_t* pstat = res.data();
  const uint32_t* wst = pstat + n;
  const uint64_t* ends = reinterpret_cast<const uint64_t*>(pstat + 2 * size_t(n));

  // ---- routes: fast kernels, catch-all decoder, or the first failing page (nothing behind it needs decoding)
  std::vector<uint32_t> fast, cold;
  size_t fail_page = n_pages;
  uint32_t fail_st = ST_OK;                   // the failure's device status, unless
  PcoB200Error decode_kind = PCO_B200_OK;     // the decode kernels reported it (kind and message)
  std::string decode_msg;
  for (uint32_t i = 0; i < n; i++) {
    const uint64_t frame_end = tab[i].frame_off + 4 + tab[i].meta_len + tab[i].page_len;
    uint32_t st = pstat[i];
    bool rewalk = false;
    if (st == ST_OK) {
      st = wst[i];
      if (st == ST_UNSUPPORTED) st = WP_COLD;
      else if (st == ST_OK && ends[i] > frame_end) st = ST_INSUFFICIENT_DATA;  // the walk ran past the page into the next frame
      else rewalk = st != ST_OK;
    }
    if (st == ST_OK) { fast.push_back(i); continue; }
    if (st == WP_COLD) { cold.push_back(i); continue; }
    fail_page = i;
    fail_st = st;
    if (rewalk) {
      // a walk that leaves its page reads the next frame, not the zeros pco_b200_page_decompress would see there: walk the page once
      // more over its own frame alone for the kind that call reports
      IndexChunk one = recs[i];
      one.chunk_offset = 0;
      PCOB_CUDA_TRY(cudaMemcpyAsync(d_index + chunks_offset + uint64_t(n) * sizeof(IndexChunk), &one, sizeof(one), cudaMemcpyHostToDevice, stream));
      PCOB_CUDA_TRY(cudaMemsetAsync(d_spare_st, 0xff, 4, stream));
      const FileParams fp1{d_frames + tab[i].frame_off, frame_end - tab[i].frame_off, dtype, 0, 4};
      walk_kernel<SMALL_MAX_SIZE_LOG><<<1, WALK_THREADS, sizeof(WalkSmem<SMALL_MAX_SIZE_LOG>), stream>>>(
          fp1, d_index, chunks_offset + uint64_t(n) * sizeof(IndexChunk), 1, 0, entries, 0, 0, ~uint64_t(0), d_spare_st, c.misc.as<WalkResult>(), 0);
      PCOB_CUDA_TRY(cudaGetLastError());
      uint32_t st1 = ST_OK;
      PCOB_CUDA_TRY(readback_small_sync(&st1, d_spare_st, 4, stream));
      if (st1 != ST_OK) fail_st = st1;
    }
    break;
  }

  void* d_out;
  if (PcoB200Error e = out_buffer(c, dst, dst_dev, n_total * elem, &d_out)) return e;
  const uint64_t out_len = dst_dev ? uint64_t(dst_len) : n_total;
  // ---- fast pages: the ordinary decode over their walked index records
  if (!fast.empty()) {
    if (fast.size() != n_pages) {  // some pages take another route: keep the records of the fast ones, in page order
      std::vector<IndexChunk> walked(n_pages), sel;
      PCOB_CUDA_TRY(cudaMemcpyAsync(walked.data(), d_index + chunks_offset, n_pages * sizeof(IndexChunk), cudaMemcpyDeviceToHost, stream));
      PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
      sel.reserve(fast.size());
      for (uint32_t i : fast) sel.push_back(walked[i]);
      PCOB_CUDA_TRY(cudaMemcpyAsync(d_index + chunks_offset, sel.data(), sel.size() * sizeof(IndexChunk), cudaMemcpyHostToDevice, stream));
    }
    uint32_t bad = 0;  // the first failing chunk of the launch: the bad-th fast page
    if (PcoB200Error e = launch_decode(c, fp, d_index, entries, chunks_offset, uint32_t(fast.size()), d_out, out_len, stream, &bad)) {
      if (e == PCO_B200_CUDA) return e;
      if (fast[bad] < fail_page) {
        fail_page = fast[bad];
        decode_kind = e;
        decode_msg = last_error_ref();
      }
    }
  }
  while (!cold.empty() && cold.back() > fail_page) cold.pop_back();  // pages behind a failing one need no decoding
  // ---- pages only the catch-all decoder takes: one single-thread launch per page, straight into the page's slot of the output.
  // One launch per page rather than one over a file of all of them: a page may be followed by bytes it does not use, and the catch-all
  // decoder would read those as the next chunk.
  if (!cold.empty()) {
    const size_t nc = cold.size();
    std::vector<ColdJob> jobs;
    for (uint32_t i : cold) {
      const WrappedPage& w = tab[i];
      jobs.push_back(ColdJob{FileParams{d_frames + w.frame_off, 4 + w.meta_len + w.page_len, dtype, 0, 4}, 0,
                             static_cast<uint8_t*>(d_out) + recs[i].out_offset * elem, w.page_n});
    }
    std::vector<ColdResult> cres;
    if (PcoB200Error e = cold_decode_jobs(c, dtype, jobs, cold_retry_chunk, &cres, stream)) return e;
    // the page is decoded once its chunk is (what the decoder reads behind it is not the page's)
    for (size_t k = 0; k < nc; k++)
      if (cres[k].n_chunks == 0) {
        if (cold[k] < fail_page) { fail_page = cold[k]; fail_st = cres[k].status; decode_kind = PCO_B200_OK; }
        break;
      }
  }
  if (fail_page < n_pages) return decode_kind != PCO_B200_OK ? page_fail(decode_kind, fail_page, decode_msg) : page_status_fail(fail_st, fail_page);
  if (!dst_dev) {
    PCOB_CUDA_TRY(copy_sliced(dst, d_out, n_total * elem, cudaMemcpyDeviceToHost, stream));
  }
  PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
  if (n_written) *n_written = size_t(n_total);
  return PCO_B200_OK;
}

PcoB200Error pco_b200_decompress_pages(const void* metas, size_t metas_len, const void* pages, size_t pages_len, unsigned char dtype,
                                       const PcoB200PageRef* refs, size_t n_pages, void* dst, size_t dst_len, size_t* n_written, uint32_t flags,
                                       void* cuda_stream) {
  const PcoB200Error e = decompress_pages_impl(metas, metas_len, pages, pages_len, dtype, refs, n_pages, dst, dst_len, n_written, flags,
                                               static_cast<cudaStream_t>(cuda_stream));
  profiler().resolve();
  return e;
}

static PcoB200Error compress_wrapped_impl(const void* nums, size_t n, uint32_t dtype, const PcoB200ChunkConfig* config, void* metas, size_t metas_cap,
                                          size_t* metas_len, void* pages, size_t pages_cap, size_t* pages_len, PcoB200PageRef* refs, size_t refs_cap,
                                          size_t* n_chunks_out, uint32_t flags, cudaStream_t stream) {
  if (!nt_valid(dtype)) return fail(PCO_B200_INVALID_TYPE, "unknown number type byte: " + std::to_string(dtype));
  if ((!metas && metas_cap) || (!pages && pages_cap) || (!refs && refs_cap)) return fail(PCO_B200_INVALID_ARGUMENT, "null buffer");
  if (metas_len) *metas_len = 0;
  if (pages_len) *pages_len = 0;
  if (n_chunks_out) *n_chunks_out = 0;
  const PcoB200ChunkConfig cfg = default_chunk_config(config);
  Context& c = ctx();
  if (PcoB200Error e = ensure_device(c)) return e;
  // the chunks simple_compress would write; a paging spec that does not fit is reported by the pipeline, with its other checks
  std::vector<uint64_t> chunk_ns;
  if (n_per_page(cfg, n, &chunk_ns) != PCO_B200_OK) chunk_ns.clear();
  const ChunksScratch cs = chunks_only_scratch(nt_bits(dtype), n, chunk_ns);
  const size_t cap = cs.bytes, icap = cs.index;
  PCOB_CUDA_TRY(c.wrap_file.reserve(cap + 32));
  PCOB_CUDA_TRY(c.wrap_index.reserve(icap));
  uint8_t* d_file = c.wrap_file.as<uint8_t>();
  uint8_t* d_idx = c.wrap_index.as<uint8_t>();
  CompressResult cr;
  // an empty array is compressed (the config still checked) with host buffers: no chunk, nothing on the device to split
  const bool empty = n == 0;
  IndexHeader empty_ih;
  uint8_t empty_dst[8];
  const uint32_t cflags = (flags & PCO_B200_SRC_ON_DEVICE) | PCO_B200_CHUNKS_ONLY | (empty ? 0u : (PCO_B200_DST_ON_DEVICE | PCO_B200_INDEX_ON_DEVICE));
  PcoB200Error e = dispatch_latent(dtype, [&](auto tag) {
    using L = decltype(tag);
    return compress_typed<L>(c.enc, nums, n, dtype, cfg, false, empty ? static_cast<void*>(empty_dst) : d_file, empty ? sizeof(empty_dst) : cap,
                             empty ? static_cast<void*>(&empty_ih) : d_idx, empty ? sizeof(empty_ih) : icap, cflags, stream, &cr);
  });
  if (e != PCO_B200_OK || empty) return e;
  const uint32_t nc = uint32_t(chunk_ns.size());
  // scratch: sizes | refs | totals | error word
  PCOB_CUDA_TRY(c.wrap_res.reserve(size_t(nc) * (8 + sizeof(PcoB200PageRef)) + 64));
  uint64_t* d_sizes = c.wrap_res.as<uint64_t>();
  PcoB200PageRef* d_refs = reinterpret_cast<PcoB200PageRef*>(d_sizes + nc);
  uint64_t* d_tot = reinterpret_cast<uint64_t*>(d_refs + nc);
  uint32_t* d_err = reinterpret_cast<uint32_t*>(d_tot + 2);
  PCOB_CUDA_TRY(cudaMemsetAsync(d_err, 0, 4, stream));
  profiler().begin("chunk_refs_kernel", stream);
  chunk_sizes_kernel<<<std::min<uint32_t>((nc + 255) / 256, 1024), 256, 0, stream>>>(d_idx, cr.index_bytes, d_sizes, nc, d_err);
  // compress_typed writes the IndexChunk records right behind the header
  chunk_refs_kernel<<<1, 1024, 0, stream>>>(d_file, reinterpret_cast<const IndexChunk*>(d_idx + sizeof(IndexHeader)), d_sizes, nc, dtype, d_refs, d_tot, d_err);
  profiler().end(stream);
  PCOB_CUDA_TRY(cudaGetLastError());
  const bool dst_dev = flags & PCO_B200_DST_ON_DEVICE;
  const IndexChunk* d_chunks = reinterpret_cast<const IndexChunk*>(d_idx + sizeof(IndexHeader));
  if (dst_dev) {
    // device buffers: the split goes out right behind the scan and checks the totals against the capacities itself, so that one
    // readback serves the whole call
    profiler().begin("split_chunks_kernel", stream);
    split_chunks_kernel<<<nc, WRAP_THREADS, 0, stream>>>(d_file, d_chunks, d_refs, d_tot, d_err, metas_cap, pages_cap, nc <= refs_cap ? 1u : 0u,
                                                         static_cast<uint8_t*>(metas), static_cast<uint8_t*>(pages));
    profiler().end(stream);
    PCOB_CUDA_TRY(cudaGetLastError());
  }
  std::vector<PcoB200PageRef> h_refs(nc);
  struct { uint64_t tot[2]; uint32_t err, pad; } tail;
  static_assert(sizeof(PcoB200PageRef) == 40, "ref layout");
  std::vector<uint32_t> back((size_t(nc) * sizeof(PcoB200PageRef) + 20) / 4);
  PCOB_CUDA_TRY(readback_small_sync(back.data(), d_refs, back.size() * 4, stream));
  std::memcpy(h_refs.data(), back.data(), size_t(nc) * sizeof(PcoB200PageRef));
  std::memcpy(&tail, reinterpret_cast<const uint8_t*>(back.data()) + size_t(nc) * sizeof(PcoB200PageRef), 20);
  if (tail.err != 0) return fail(PCO_B200_CUDA, "compressor returned chunks that do not split into meta and page");
  if (metas_len) *metas_len = size_t(tail.tot[0]);
  if (pages_len) *pages_len = size_t(tail.tot[1]);
  if (n_chunks_out) *n_chunks_out = nc;
  if (tail.tot[0] > metas_cap || tail.tot[1] > pages_cap || nc > refs_cap)
    return fail(PCO_B200_IO, "failed to write whole buffer (need " + std::to_string(tail.tot[0]) + " meta bytes, " + std::to_string(tail.tot[1]) +
                                 " page bytes and " + std::to_string(nc) + " refs)");
  if (!dst_dev) {  // host buffers: split into scratch, then two copies down
    const uint64_t pages_at = (tail.tot[0] + 15) & ~uint64_t(15);
    PCOB_CUDA_TRY(c.wrap_out.reserve(pages_at + tail.tot[1] + 32));
    uint8_t* d_metas = c.wrap_out.as<uint8_t>();
    uint8_t* d_pages = d_metas + pages_at;
    profiler().begin("split_chunks_kernel", stream);
    split_chunks_kernel<<<nc, WRAP_THREADS, 0, stream>>>(d_file, d_chunks, d_refs, d_tot, d_err, ~uint64_t(0), ~uint64_t(0), 1u, d_metas, d_pages);
    profiler().end(stream);
    PCOB_CUDA_TRY(cudaGetLastError());
    if (tail.tot[0]) PCOB_CUDA_TRY(copy_sliced(metas, d_metas, tail.tot[0], cudaMemcpyDeviceToHost, stream));
    if (tail.tot[1]) PCOB_CUDA_TRY(copy_sliced(pages, d_pages, tail.tot[1], cudaMemcpyDeviceToHost, stream));
    PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
  }
  std::memcpy(refs, h_refs.data(), size_t(nc) * sizeof(PcoB200PageRef));
  return PCO_B200_OK;
}

PcoB200Error pco_b200_compress_wrapped(const void* nums, size_t n, unsigned char dtype, const PcoB200ChunkConfig* config, void* metas, size_t metas_cap,
                                       size_t* metas_len, void* pages, size_t pages_cap, size_t* pages_len, PcoB200PageRef* refs, size_t refs_cap,
                                       size_t* n_chunks, uint32_t flags, void* cuda_stream) {
  const PcoB200Error e = compress_wrapped_impl(nums, n, dtype, config, metas, metas_cap, metas_len, pages, pages_cap, pages_len, refs, refs_cap, n_chunks,
                                               flags, static_cast<cudaStream_t>(cuda_stream));
  profiler().resolve();
  return e;
}

// ---------------------------------------------------------------------------
// Batches of standalone files (files_kernels.cuh).  Compress: the files' chunks run through the CHUNKS_ONLY pipeline as the chunks of
// one call (Exact paging over every file's pages), then frame_files_kernel writes each file and its side index.  Under Auto the
// pipeline takes one unoptimized_bins_log per call, so files are grouped by theirs and each group is one pass.
// ---------------------------------------------------------------------------
static PcoB200Error file_fail(PcoB200Error kind, size_t file, const std::string& what) {
  return fail(kind, "file " + std::to_string(file) + ": " + what);
}

// Lowest file among [0, n_files) that pco_b200_compress_ex refuses on the device (the Auto searches' refusals), one file at a time.
static PcoB200Error compress_files_find_refusal(Context& c, const void* nums, const uint64_t* file_ns, size_t n_files, uint32_t dtype,
                                                const PcoB200ChunkConfig& cfg, bool uniform, uint32_t flags, cudaStream_t stream, size_t* refused) {
  const size_t elem = nt_bits(dtype) / 8;
  uint64_t at = 0;
  for (size_t i = 0; i < n_files; i++) {
    const size_t n = size_t(file_ns[i]);
    std::vector<uint64_t> pages;
    n_per_page(cfg, n, &pages);
    const ChunksScratch cs = chunks_only_scratch(nt_bits(dtype), n, pages);
    const size_t cap = cs.bytes, icap = cs.index;
    PCOB_CUDA_TRY(c.wrap_file.reserve(cap + 32));
    PCOB_CUDA_TRY(c.wrap_index.reserve(icap));
    CompressResult cr;
    const PcoB200Error e = dispatch_latent(dtype, [&](auto tag) {
      using L = decltype(tag);
      return compress_typed<L>(c.enc, static_cast<const uint8_t*>(nums) + at * elem, n, dtype, cfg, uniform, c.wrap_file.p, cap, c.wrap_index.p, icap,
                               (flags & PCO_B200_SRC_ON_DEVICE) | PCO_B200_CHUNKS_ONLY | PCO_B200_DST_ON_DEVICE | PCO_B200_INDEX_ON_DEVICE, stream, &cr);
    });
    if (e == PCO_B200_CUDA) return e;
    if (e != PCO_B200_OK) { *refused = i; return e; }
    at += n;
  }
  *refused = n_files;
  return PCO_B200_OK;
}

static PcoB200Error compress_files_impl(const void* nums, const uint64_t* file_ns, size_t n_files, uint32_t dtype, const PcoB200ChunkConfig* config, bool uniform,
                                        void* dst, size_t dst_cap, void* index, size_t index_cap, PcoB200FileRef* files, uint32_t flags, cudaStream_t stream) {
  if (!nt_valid(dtype)) return fail(PCO_B200_INVALID_TYPE, "unknown number type byte: " + std::to_string(dtype));
  if (flags & PCO_B200_CHUNKS_ONLY) return fail(PCO_B200_INVALID_ARGUMENT, "PCO_B200_CHUNKS_ONLY does not apply to whole files");
  if (n_files == 0) return PCO_B200_OK;
  if (!file_ns || !files) return fail(PCO_B200_INVALID_ARGUMENT, "file_ns and files are required");
  if ((!dst && dst_cap) || (!index && index_cap)) return fail(PCO_B200_INVALID_ARGUMENT, "null buffer");
  const PcoB200ChunkConfig cfg = default_chunk_config(config);
  // ---- every file's config check, on the host and in file order
  const uint32_t lbits = nt_bits(dtype);
  size_t first_bad = n_files;
  PcoB200Error bad_kind = PCO_B200_OK;
  std::string bad_msg;
  bool auto_any = false;
  std::vector<std::vector<uint64_t>> pages(n_files);
  std::vector<uint32_t> bins(n_files, 0);
  for (size_t i = 0; i < n_files; i++) {
    ConfigCheck ck;
    PcoB200Error e = check_config(cfg, dtype, size_t(file_ns[i]), &ck);
    if (e == PCO_B200_OK && !ck.pages.empty()) {
      bins[i] = unoptimized_bins_log(cfg.compression_level, ck.pages[0], 0);
      bool uniform_bins = true;
      for (uint64_t p : ck.pages) uniform_bins = uniform_bins && unoptimized_bins_log(cfg.compression_level, p, 0) == bins[i];
      if (!uniform_bins && (ck.auto_mode || ck.auto_delta))  // compress_typed's refusal for one array
        e = fail(PCO_B200_UNSUPPORTED, "ModeSpec::Auto / DeltaSpec::Auto over chunks whose sizes imply different unoptimized_bins_log in one call");
    }
    if (e != PCO_B200_OK) {
      first_bad = i;
      bad_kind = e;
      bad_msg = last_error_ref();
      break;
    }
    auto_any = ck.auto_mode || ck.auto_delta;
    pages[i] = std::move(ck.pages);
  }
  // explicit specs: the pipeline refuses nothing the checks passed, so a refusal is final here; under Auto a file in front of it may
  // still be refused by the device searches
  if (first_bad == 0 || (first_bad < n_files && !auto_any)) return file_fail(bad_kind, first_bad, bad_msg);

  Context& c = ctx();
  if (PcoB200Error e = ensure_device(c)) return e;
  const bool src_dev = flags & PCO_B200_SRC_ON_DEVICE, dst_dev = flags & PCO_B200_DST_ON_DEVICE, idx_dev = flags & PCO_B200_INDEX_ON_DEVICE;
  const size_t elem = lbits / 8;
  std::vector<uint64_t> num_at(first_bad + 1, 0);
  for (size_t i = 0; i < first_bad; i++) num_at[i + 1] = num_at[i] + file_ns[i];
  // ---- groups: one pipeline pass per unoptimized_bins_log.  Auto needs it; explicit specs gain from it: the pipeline splits a pass into
  // runs wherever consecutive chunks change the value, and every run waits for the host, so files of mixed sizes in file order would
  // make hundreds of runs.
  std::map<uint32_t, std::vector<uint32_t>> groups;
  for (size_t i = 0; i < first_bad; i++)
    if (file_ns[i] > 0) groups[bins[i]].push_back(uint32_t(i));
  struct Group { uint64_t out_at, out_cap, idx_at, idx_cap, total, index_bytes; std::vector<IndexChunk> recs; std::vector<uint64_t> exact; };
  std::vector<Group> gs;
  std::vector<uint32_t> file_group(first_bad, 0), file_c0(first_bad, 0);
  uint64_t out_scratch = 0, idx_scratch = 0;
  for (auto& kv : groups) {
    Group g{};
    uint64_t n = 0;
    for (uint32_t f : kv.second) {
      file_group[f] = uint32_t(gs.size());
      file_c0[f] = uint32_t(g.exact.size());
      g.exact.insert(g.exact.end(), pages[f].begin(), pages[f].end());
      n += file_ns[f];
    }
    const ChunksScratch cs = chunks_only_scratch(lbits, n, g.exact);
    g.out_at = out_scratch;
    g.out_cap = cs.bytes;
    g.idx_at = idx_scratch;
    g.idx_cap = cs.index;
    out_scratch += (g.out_cap + 15) & ~uint64_t(15);
    idx_scratch += (g.idx_cap + 15) & ~uint64_t(15);
    gs.push_back(std::move(g));
  }
  PCOB_CUDA_TRY(c.wrap_file.reserve(out_scratch + 64));
  PCOB_CUDA_TRY(c.wrap_index.reserve(idx_scratch + 64));
  uint8_t* d_chunks = c.wrap_file.as<uint8_t>();
  uint8_t* d_pidx = c.wrap_index.as<uint8_t>();
  size_t gi = 0;
  for (auto& kv : groups) {
    Group& g = gs[gi++];
    const std::vector<uint32_t>& fl = kv.second;
    const std::vector<uint64_t>& exact = g.exact;
    PcoB200ChunkConfig cg = cfg;
    cg.paging_spec = PCO_B200_PAGING_EXACT;
    cg.exact_page_ns = exact.data();
    cg.n_exact_pages = exact.size();
    // the group's numbers back to back: the array itself when the files of the group are consecutive, else gathered
    const uint8_t* g_nums = static_cast<const uint8_t*>(nums) + num_at[fl.front()] * elem;
    uint64_t g_n = 0;
    for (uint32_t f : fl) g_n += file_ns[f];
    std::vector<uint8_t> h_gather;
    if (num_at[fl.back() + 1] - num_at[fl.front()] != g_n) {
      if (src_dev) {
        PCOB_CUDA_TRY(c.wrap_out.reserve(g_n * elem + 64));
        uint64_t at = 0;
        for (uint32_t f : fl) {
          PCOB_CUDA_TRY(cudaMemcpyAsync(c.wrap_out.as<uint8_t>() + at * elem, static_cast<const uint8_t*>(nums) + num_at[f] * elem, file_ns[f] * elem,
                                        cudaMemcpyDeviceToDevice, stream));
          at += file_ns[f];
        }
        g_nums = c.wrap_out.as<uint8_t>();
      } else {
        h_gather.resize(g_n * elem);
        uint64_t at = 0;
        for (uint32_t f : fl) {
          std::memcpy(h_gather.data() + at * elem, static_cast<const uint8_t*>(nums) + num_at[f] * elem, file_ns[f] * elem);
          at += file_ns[f];
        }
        g_nums = h_gather.data();
      }
    }
    CompressResult cr;
    const PcoB200Error e = dispatch_latent(dtype, [&](auto tag) {
      using L = decltype(tag);
      return compress_typed<L>(c.enc, g_nums, size_t(g_n), dtype, cg, uniform, d_chunks + g.out_at, g.out_cap, d_pidx + g.idx_at, g.idx_cap,
                               (src_dev ? PCO_B200_SRC_ON_DEVICE : 0u) | PCO_B200_CHUNKS_ONLY | PCO_B200_DST_ON_DEVICE | PCO_B200_INDEX_ON_DEVICE, stream, &cr);
    });
    if (e == PCO_B200_CUDA) return e;
    if (e != PCO_B200_OK) {  // an Auto search refused a chunk: find the lowest file compress_ex refuses
      size_t refused = first_bad;
      const PcoB200Error e2 = compress_files_find_refusal(c, nums, file_ns, first_bad, dtype, cfg, uniform, flags, stream, &refused);
      if (refused < first_bad) return file_fail(e2, refused, last_error_ref());
      if (e2 != PCO_B200_OK) return e2;
      if (first_bad < n_files) return file_fail(bad_kind, first_bad, bad_msg);
      return fail(PCO_B200_CUDA, "a batch was refused that no file of it is refused alone");
    }
    g.total = cr.total_bytes;
    g.index_bytes = cr.index_bytes;
    g.recs.resize(exact.size());
    PCOB_CUDA_TRY(cudaMemcpyAsync(g.recs.data(), d_pidx + g.idx_at + sizeof(IndexHeader), exact.size() * sizeof(IndexChunk), cudaMemcpyDeviceToHost, stream));
    PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
  }
  if (first_bad < n_files) return file_fail(bad_kind, first_bad, bad_msg);

  // ---- the files' layout in dst and index
  std::vector<FileFrame> tab(n_files);
  uint64_t dst_total = 0, idx_total = 0;
  for (size_t i = 0; i < n_files; i++) {
    FileFrame& f = tab[i];
    std::memset(&f, 0, sizeof(f));
    const std::vector<uint8_t> hdr = make_standalone_header(file_ns[i], uint8_t(uniform ? dtype : 0));
    f.hdr_len = uint32_t(hdr.size());
    std::memcpy(f.hdr, hdr.data(), hdr.size());
    f.n = file_ns[i];
    f.n_chunks = uint32_t(pages[i].size());
    if (f.n_chunks) {
      const Group& g = gs[file_group[i]];
      const uint32_t c0 = file_c0[i], c1 = c0 + f.n_chunks;
      const uint64_t end = c1 < g.recs.size() ? g.recs[c1].chunk_offset : g.total;
      const uint64_t eend = c1 < g.recs.size() ? g.recs[c1].entries_offset : g.index_bytes;
      f.chunks_src = g.out_at + g.recs[c0].chunk_offset;
      f.chunks_len = end - g.recs[c0].chunk_offset;
      f.recs_src = g.idx_at + sizeof(IndexHeader) + uint64_t(c0) * sizeof(IndexChunk);
      f.entries_src = g.idx_at + g.recs[c0].entries_offset;
      f.entries_len = eend - g.recs[c0].entries_offset;
    }
    f.dst_off = dst_total;
    f.index_off = idx_total;
    const uint64_t flen = f.hdr_len + f.chunks_len + 1;
    const uint64_t ilen = sizeof(IndexHeader) + uint64_t(f.n_chunks) * sizeof(IndexChunk) + f.entries_len;
    files[i].offset = dst_total;
    files[i].len = flen;
    files[i].index_offset = index ? idx_total : 0;
    files[i].index_len = index ? ilen : 0;
    dst_total += flen;
    if (index) idx_total += (ilen + 15) & ~uint64_t(15);
  }
  if (dst_total > dst_cap || (index && idx_total > index_cap))
    return fail(PCO_B200_IO, "failed to write whole buffer (need " + std::to_string(dst_total) + " file bytes and " + std::to_string(idx_total) + " index bytes)");

  // ---- framing: the files straight into a device dst (byte-granular stores, any alignment) or into scratch for a host one; the
  // indexes always into scratch, whose base is aligned for the kernel's 8-byte record stores, then one copy into the caller's buffer,
  // which may start at any byte (as compress_ex's index may)
  PCOB_CUDA_TRY(c.files_tab.reserve(n_files * sizeof(FileFrame)));
  PCOB_CUDA_TRY(cudaMemcpyAsync(c.files_tab.p, tab.data(), n_files * sizeof(FileFrame), cudaMemcpyHostToDevice, stream));
  uint8_t* d_dst = static_cast<uint8_t*>(dst);
  uint8_t* d_index = nullptr;
  if (!dst_dev) {
    PCOB_CUDA_TRY(c.files_out.reserve(dst_total + 64));
    d_dst = c.files_out.as<uint8_t>();
  }
  if (index) {
    PCOB_CUDA_TRY(c.files_idx.reserve(idx_total + 64));
    d_index = c.files_idx.as<uint8_t>();
  }
  profiler().begin("frame_files_kernel", stream);
  frame_files_kernel<<<uint32_t(n_files), FILES_THREADS, 0, stream>>>(d_chunks, d_pidx, c.files_tab.as<FileFrame>(), d_dst, d_index);
  profiler().end(stream);
  PCOB_CUDA_TRY(cudaGetLastError());
  if (!dst_dev) PCOB_CUDA_TRY(copy_sliced(dst, d_dst, dst_total, cudaMemcpyDeviceToHost, stream));
  if (index) PCOB_CUDA_TRY(copy_sliced(index, d_index, idx_total, idx_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, stream));
  PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
  return PCO_B200_OK;
}

PcoB200Error pco_b200_compress_files(const void* nums, const uint64_t* file_ns, size_t n_files, unsigned char dtype, const PcoB200ChunkConfig* config,
                                     int uniform_type_header, void* dst, size_t dst_cap, void* index, size_t index_cap, PcoB200FileRef* files, uint32_t flags,
                                     void* cuda_stream) {
  const PcoB200Error e = compress_files_impl(nums, file_ns, n_files, dtype, config, uniform_type_header != 0, dst, dst_cap, index, index_cap, files, flags,
                                             static_cast<cudaStream_t>(cuda_stream));
  profiler().resolve();
  return e;
}

// Decompress.  Every file's count is known before anything is decoded - from its side index, or from walking it - so the numbers land
// in place and the whole batch is ONE chunk list for the ordinary decode kernels (one launch_decode per header flavour and format
// version, which FileParams carries per launch):
//   1. the files' heads (and index headers) come back in one readback and are parsed on the host;
//   2. index-free files are walked together (walk_index_free): speculative rounds over all of them, then the serial walker for each
//      file the rounds did not take to its terminator.  The walked records stay in an arena beside the staged indexes; a file whose
//      walk meets a chunk the fast kernels decline is cold;
//   3. check_index_kernel tests every indexed file's records against its own file (a file that fails decodes on its own, through
//      decompress_core) and marks cold files; then
//      merge_index_kernel writes the indexed files' records, rebased, into the list beside the walked ones; launch_decode runs over
//      it.  A failing chunk names its file: a chunk the fast kernels decline makes that file cold and the list is decoded again
//      without it; any other failure drops the files from it on and the rest is decoded again, so that the lowest failure is found;
//   4. cold files go through cold_decode_kernel, one launch per file.
// A file of the batch.  An indexed file uses hdr, begin, end and count (from its index) of WalkFile; an index-free one all of it.
struct BatchFile : WalkFile {
  bool indexed = false, walk = false, cold = false, staged = false;
  bool alone = false;            // indexed, with a record outside its own file: decoded by itself, as decompress_ex decodes it
  uint64_t idx_recs = 0;         // indexed: byte offset of its IndexChunk[0] in the arena
  uint64_t idx_base = 0;         // indexed: byte offset of its index in the arena
  uint64_t n_idx_chunks = 0;
  uint64_t out_base = 0;
  uint64_t staged_at = 0;        // cold without index: element offset of its numbers in files_cold
};

static PcoB200Error decompress_files_impl(const void* src, size_t src_len, const void* index, size_t index_len, uint32_t dtype, const PcoB200FileRef* files,
                                          size_t n_files, void* dst, size_t dst_len, uint64_t* file_ns, size_t* n_written, uint32_t flags,
                                          cudaStream_t stream) {
  // ---- argument checks: host only, before any device work
  if (!nt_valid(dtype)) return fail(PCO_B200_INVALID_TYPE, "unknown number type byte: " + std::to_string(dtype));
  if (n_written) *n_written = 0;
  if (n_files == 0) return PCO_B200_OK;
  if (!files) return fail(PCO_B200_INVALID_ARGUMENT, "files are required");
  if (n_files > 0x7fffffffull) return fail(PCO_B200_INVALID_ARGUMENT, "too many files");
  if ((!src && src_len) || (!index && index_len) || (!dst && dst_len)) return fail(PCO_B200_INVALID_ARGUMENT, "null buffer");
  bool any_index = false;
  for (size_t i = 0; i < n_files; i++) {
    const PcoB200FileRef& r = files[i];
    if (r.len > src_len || r.offset > src_len - r.len) return file_fail(PCO_B200_INVALID_ARGUMENT, i, "file lies outside src");
    if (r.index_len) {
      if (r.index_offset % 16) return file_fail(PCO_B200_INVALID_ARGUMENT, i, "index offset is not a multiple of 16");
      if (r.index_len > index_len || r.index_offset > index_len - r.index_len) return file_fail(PCO_B200_INVALID_ARGUMENT, i, "side index lies outside index");
      any_index = any_index || r.index_len >= sizeof(IndexHeader);
    }
  }
  Context& c = ctx();
  if (PcoB200Error e = ensure_device(c)) return e;
  static const bool cold_ok = [] { const char* v = std::getenv("PCOB200_COLD_DECODE"); return !(v && v[0] == '0'); }();
  const bool src_dev = flags & PCO_B200_SRC_ON_DEVICE, dst_dev = flags & PCO_B200_DST_ON_DEVICE, idx_dev = flags & PCO_B200_INDEX_ON_DEVICE;
  const size_t elem = nt_bits(dtype) / 8;
  const uint32_t n = uint32_t(n_files);
  // the lowest failing file so far: files from it on need no work
  size_t limit = n_files;
  PcoB200Error fkind = PCO_B200_OK;
  std::string fmsg;
  auto fail_at = [&](size_t i, PcoB200Error k, const std::string& m) {
    if (i < limit) { limit = i; fkind = k; fmsg = m; }
  };

  // ---- the bytes in HBM: src, and the arena = [the caller's index | walked records and entries | the merged chunk list]
  const uint8_t* d_src;
  if (PcoB200Error e = stage_in(c.src, src, src_len, src_dev, stream, &d_src)) return e;
  uint64_t arena_end = any_index ? (uint64_t(index_len) + 15) & ~uint64_t(15) : 0;
  PCOB_CUDA_TRY(c.files_arena.reserve(arena_end + 64));
  if (any_index) PCOB_CUDA_TRY(copy_sliced(c.files_arena.p, index, index_len, idx_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, stream));
  auto arena = [&]() { return c.files_arena.as<uint8_t>(); };

  // ---- 1. heads and index headers
  std::vector<BatchFile> bf(n_files);
  {
    std::vector<uint64_t> offs(n), lens(n), ioffs, ilens;
    std::vector<uint32_t> with_index;
    for (uint32_t i = 0; i < n; i++) {
      offs[i] = files[i].offset;
      lens[i] = std::min<uint64_t>(files[i].len, 32);
      if (files[i].index_len >= sizeof(IndexHeader)) {
        with_index.push_back(i);
        ioffs.push_back(files[i].index_offset);
        ilens.push_back(sizeof(IndexHeader));
      }
    }
    std::vector<uint8_t> heads, iheads;
    if (PcoB200Error e = peek(c, src, src_dev, offs, lens, 32, &heads, stream)) return e;
    if (PcoB200Error e = peek(c, index, idx_dev, ioffs, ilens, sizeof(IndexHeader), &iheads, stream)) return e;
    size_t wi = 0;
    for (uint32_t i = 0; i < n; i++) {
      BatchFile& f = bf[i];
      const PcoB200FileRef& r = files[i];
      f.begin = r.offset;
      f.end = r.offset + r.len;
      if (PcoB200Error e = parse_standalone_header(heads.data() + size_t(i) * 32, size_t(lens[i]), size_t(r.len), &f.hdr)) {
        fail_at(i, e, last_error_ref());
        break;
      }
      if (wi < with_index.size() && with_index[wi] == i) {
        IndexHeader ih;
        std::memcpy(&ih, iheads.data() + wi * sizeof(IndexHeader), sizeof(ih));
        wi++;
        // as decompress_ex checks it; the chunk table must also be 8-byte aligned for the kernels' loads
        if (!index_header_ok(ih, r.len, r.index_len) || ih.chunks_offset % 8 != 0) {
          fail_at(i, PCO_B200_INVALID_ARGUMENT, "side index does not belong to this file");
          break;
        }
        f.indexed = true;
        f.count = ih.n_total;
        f.n_idx_chunks = ih.n_chunks;
        f.idx_base = r.index_offset;
        f.idx_recs = r.index_offset + ih.chunks_offset;
      } else {
        f.walk = true;
        f.pos = r.offset + f.hdr.first_chunk_byte;
        f.expect = f.hdr.n_hint;
      }
    }
  }

  // ---- 2. index-free files, walked together; a cold one goes to the catch-all decoder, as in decompress_ex
  {
    std::vector<WalkFile*> walks;
    for (uint32_t i = 0; i < n && i < limit; i++)
      if (bf[i].walk) walks.push_back(&bf[i]);
    if (PcoB200Error e = walk_index_free(c, static_cast<const uint8_t*>(src), src_dev, d_src, src_len, dtype, walks, c.files_arena, &arena_end, stream)) return e;
    for (uint32_t i = 0; i < n && i < limit; i++) {
      BatchFile& f = bf[i];
      if (!f.walk || f.how == WalkEnd::TERMINATED) continue;
      if (f.how == WalkEnd::COLD && cold_ok) f.cold = f.staged = true;
      else fail_at(i, f.err, f.msg);
    }
  }

  // ---- indexed files: every record checked against its own file before anything is decoded.  A file whose records stay inside it joins
  // the merged list; one with a record outside it decodes on its own with its own bounds (decompress_core, as decompress_ex), one whose
  // chunk metas route it to the catch-all decoder is cold - both into scratch, since their count is only known once decoded
  {
    std::vector<uint32_t> ids;
    std::vector<FileCheck> chk;
    for (uint32_t i = 0; i < n && i < limit; i++)
      if (bf[i].indexed && bf[i].n_idx_chunks > 0) {
        ids.push_back(i);
        chk.push_back(FileCheck{bf[i].idx_recs, bf[i].n_idx_chunks, bf[i].begin, bf[i].end - bf[i].begin, bf[i].idx_base, files[i].index_len, bf[i].count,
                                bf[i].hdr.format_major, 0});
      }
    if (!ids.empty()) {
      PCOB_CUDA_TRY(c.files_tab.reserve(chk.size() * sizeof(FileCheck) + 64));
      PCOB_CUDA_TRY(c.files_res.reserve(chk.size() * 4 + 64));
      PCOB_CUDA_TRY(cudaMemcpyAsync(c.files_tab.p, chk.data(), chk.size() * sizeof(FileCheck), cudaMemcpyHostToDevice, stream));
      profiler().begin("check_index_kernel", stream);
      check_index_kernel<<<uint32_t(ids.size()), 256, 0, stream>>>(d_src, arena(), dtype, c.files_tab.as<FileCheck>(), c.files_res.as<uint32_t>());
      profiler().end(stream);
      PCOB_CUDA_TRY(cudaGetLastError());
      std::vector<uint32_t> verdict(ids.size());
      PCOB_CUDA_TRY(readback_small_sync(verdict.data(), c.files_res.p, ids.size() * 4, stream));
      for (size_t k = 0; k < ids.size(); k++) {
        BatchFile& f = bf[ids[k]];
        if (verdict[k] == IDX_MISALIGNED) fail_at(ids[k], PCO_B200_INVALID_ARGUMENT, "side index does not belong to this file (misaligned entries)");
        else if (verdict[k] == IDX_OUTSIDE) f.alone = f.staged = true;
        else if (verdict[k] == IDX_COLD && cold_ok) f.cold = f.staged = true;
      }
    }
  }

  // ---- cold files, and indexed files that decode on their own: their count is only known once decoded, so they decode into scratch first
  auto cold_decode = [&](const BatchFile& f, void* out, uint64_t cap, ColdResult* res) -> PcoB200Error {
    const FileParams fpf{d_src + f.begin, f.end - f.begin, dtype, f.hdr.uniform_type, f.hdr.format_major};
    std::vector<ColdResult> cres;
    if (PcoB200Error e = cold_decode_jobs(c, dtype, {ColdJob{fpf, f.hdr.first_chunk_byte, out, cap}}, cold_retry_file, &cres, stream)) return e;
    *res = cres[0];
    return PCO_B200_OK;
  };
  uint64_t staged_end = 0;
  for (uint32_t i = 0; i < n && i < limit; i++) {
    BatchFile& f = bf[i];
    if (!f.staged) continue;
    if (f.alone) {
      // decompress_ex's own path over this file and its index: the kernels' bounds are the file, the index and the count.  A count beyond
      // dst is left to the placement below (IO).
      if (f.count > dst_len) continue;
      for (uint64_t cap = std::max<uint64_t>(f.count, 1);;) {
        PCOB_CUDA_TRY(c.files_cold.grow_preserve((staged_end + cap) * elem + 64, staged_end * elem, stream));
        DecodeOutcome oc;
        const PcoB200Error e = decompress_core(d_src + f.begin, size_t(f.end - f.begin), dtype, c.files_cold.as<uint8_t>() + staged_end * elem, size_t(cap),
                                               arena() + f.idx_base, size_t(files[i].index_len),
                                               PCO_B200_SRC_ON_DEVICE | PCO_B200_DST_ON_DEVICE | PCO_B200_INDEX_ON_DEVICE, stream, &oc);
        if (e == PCO_B200_CUDA) return e;
        if (e != PCO_B200_OK) { fail_at(i, e, last_error_ref()); break; }
        if (oc.n_total > cap && cap < dst_len) { cap = std::min<uint64_t>(oc.n_total, dst_len); continue; }  // the catch-all decoder found more
        f.count = oc.n_total;
        f.staged_at = staged_end;
        staged_end += std::min<uint64_t>(oc.n_total, cap);
        break;
      }
      continue;
    }
    uint64_t cap = std::max<uint64_t>(std::min<uint64_t>(f.hdr.n_hint, uint64_t(1) << 24), uint64_t(1) << 16);  // the hint is untrusted
    for (;;) {
      PCOB_CUDA_TRY(c.files_cold.grow_preserve((staged_end + cap) * elem + 64, staged_end * elem, stream));
      ColdResult res;
      if (PcoB200Error e = cold_decode(f, c.files_cold.as<uint8_t>() + staged_end * elem, cap, &res)) return e;
      if (res.status == ST_DST_FULL) { cap = std::max<uint64_t>(2 * cap, res.n_total + (uint64_t(1) << 16)); continue; }
      if (res.status != ST_TERMINATOR) fail_at(i, status_to_error(res.status, ("chunk " + std::to_string(res.n_chunks)).c_str()), last_error_ref());
      f.count = res.n_total;
      f.staged_at = staged_end;
      f.recs.clear();
      staged_end += res.n_total;
      break;
    }
  }

  // ---- placement
  uint64_t total = 0;
  for (uint32_t i = 0; i < n && i < limit; i++) {
    if (bf[i].count > dst_len - std::min<uint64_t>(total, dst_len)) {
      fail_at(i, PCO_B200_IO, "dst holds " + std::to_string(dst_len) + " numbers, the files up to this one " + std::to_string(total + bf[i].count));
      break;
    }
    bf[i].out_base = total;
    total += bf[i].count;
  }
  void* d_out;
  if (PcoB200Error e = out_buffer(c, dst, dst_dev, total * elem, &d_out)) return e;
  const uint64_t out_len = dst_dev ? uint64_t(dst_len) : total;

  // ---- 3. one chunk list for the fast kernels, grouped by (uniform type, format major)
  std::map<uint32_t, std::vector<uint32_t>> flavours;
  for (uint32_t i = 0; i < n && i < limit; i++)
    if (!bf[i].cold && !bf[i].staged && (bf[i].indexed ? bf[i].n_idx_chunks : bf[i].recs.size()) > 0) flavours[(bf[i].hdr.uniform_type << 8) | bf[i].hdr.format_major].push_back(i);
  struct Slot { uint32_t file; uint64_t at, n; };
  std::vector<Slot> slots;
  std::vector<FileMerge> merges;
  uint64_t list_n = 0;
  for (auto& kv : flavours)
    for (uint32_t i : kv.second) {
      const uint64_t k = bf[i].indexed ? bf[i].n_idx_chunks : bf[i].recs.size();
      slots.push_back(Slot{i, list_n, k});
      if (bf[i].indexed) merges.push_back(FileMerge{bf[i].idx_recs, list_n, files[i].offset, bf[i].idx_base, bf[i].out_base, k});
      list_n += k;
    }
  if (list_n > 0xffffffffull) return fail(PCO_B200_UNSUPPORTED, "more than 2^32 chunks in one call");
  const uint64_t list_at = (arena_end + 15) & ~uint64_t(15);
  PCOB_CUDA_TRY(c.files_arena.grow_preserve(list_at + list_n * sizeof(IndexChunk) + 64, arena_end, stream));
  if (list_n) {
    std::vector<IndexChunk> list(list_n);
    for (const Slot& s : slots)
      if (!bf[s.file].indexed)
        for (uint64_t k = 0; k < s.n; k++) {
          list[s.at + k] = bf[s.file].recs[k];
          list[s.at + k].out_offset += bf[s.file].out_base;
        }
    PCOB_CUDA_TRY(cudaMemcpyAsync(arena() + list_at, list.data(), list_n * sizeof(IndexChunk), cudaMemcpyHostToDevice, stream));
    if (!merges.empty()) {
      PCOB_CUDA_TRY(c.files_tab.reserve(merges.size() * sizeof(FileMerge) + 64));
      PCOB_CUDA_TRY(cudaMemcpyAsync(c.files_tab.p, merges.data(), merges.size() * sizeof(FileMerge), cudaMemcpyHostToDevice, stream));
      profiler().begin("merge_index_kernel", stream);
      merge_index_kernel<<<uint32_t(merges.size()), 256, 0, stream>>>(arena(), c.files_tab.as<FileMerge>(), reinterpret_cast<IndexChunk*>(arena() + list_at));
      profiler().end(stream);
      PCOB_CUDA_TRY(cudaGetLastError());
    }
  }
  const uint64_t arena_len = list_at + list_n * sizeof(IndexChunk);
  {
    size_t si = 0;
    for (auto& kv : flavours) {
      const BatchFile& f0 = bf[kv.second.front()];
      const FileParams fp{d_src, src_len, dtype, f0.hdr.uniform_type, f0.hdr.format_major};
      const size_t s_lo = si, s_hi = si + kv.second.size();  // this flavour's slots
      si = s_hi;
      std::vector<std::pair<size_t, size_t>> work{{s_lo, s_hi}};  // ranges of slots still to decode
      while (!work.empty()) {
        const auto [a, b] = work.back();
        work.pop_back();
        size_t hi = a;
        while (hi < b && slots[hi].file < limit) hi++;  // files from the lowest failure on need no decoding
        if (hi == a) continue;
        const uint64_t first = slots[a].at, cnt = slots[hi - 1].at + slots[hi - 1].n - first;
        uint32_t bad = 0;
        const PcoB200Error e = launch_decode(c, fp, arena(), arena_len, list_at + first * sizeof(IndexChunk), uint32_t(cnt), d_out, out_len, stream, &bad);
        if (e == PCO_B200_OK) continue;
        if (e == PCO_B200_CUDA) return e;
        // the first failing chunk of the launch: find its file
        const std::string msg = last_error_ref();
        const uint64_t k = first + bad;
        size_t s = a;
        while (s + 1 < hi && slots[s + 1].at <= k) s++;
        const uint32_t fi = slots[s].file;
        if (e == PCO_B200_UNSUPPORTED && cold_ok) {
          bf[fi].cold = true;
          if (s + 1 < hi) work.push_back({s + 1, hi});
        } else {
          fail_at(fi, e, msg);
        }
        if (s > a) work.push_back({a, s});
      }
    }
  }

  // ---- 4. staged numbers moved into their slot; cold files found by the merged decode (an older format, whose chunk metas the check
  // does not parse) through the catch-all decoder into their slot, sized by their index's count
  for (uint32_t i = 0; i < n && i < limit; i++) {
    BatchFile& f = bf[i];
    uint8_t* slot = static_cast<uint8_t*>(d_out) + f.out_base * elem;
    if (f.staged) {
      if (f.count) PCOB_CUDA_TRY(cudaMemcpyAsync(slot, c.files_cold.as<uint8_t>() + f.staged_at * elem, f.count * elem, cudaMemcpyDeviceToDevice, stream));
      continue;
    }
    if (!f.cold) continue;
    ColdResult res;
    if (PcoB200Error e = cold_decode(f, slot, f.count, &res)) return e;
    if (res.status == ST_DST_FULL)  // the file holds more numbers than its index counts: refused rather than cut short
      fail_at(i, PCO_B200_INVALID_ARGUMENT, "side index does not belong to this file (it counts " + std::to_string(f.count) + " numbers, the file holds more)");
    else if (res.status != ST_TERMINATOR) fail_at(i, status_to_error(res.status, ("chunk " + std::to_string(res.n_chunks)).c_str()), last_error_ref());
  }
  if (limit < n_files) return file_fail(fkind, limit, fmsg);
  if (!dst_dev && total) PCOB_CUDA_TRY(copy_sliced(dst, d_out, total * elem, cudaMemcpyDeviceToHost, stream));
  PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
  if (file_ns)
    for (uint32_t i = 0; i < n; i++) file_ns[i] = bf[i].count;
  if (n_written) *n_written = size_t(total);
  return PCO_B200_OK;
}

PcoB200Error pco_b200_decompress_files(const void* src, size_t src_len, const void* index, size_t index_len, unsigned char dtype, const PcoB200FileRef* files,
                                       size_t n_files, void* dst, size_t dst_len, uint64_t* file_ns, size_t* n_written, uint32_t flags, void* cuda_stream) {
  const PcoB200Error e = decompress_files_impl(src, src_len, index, index_len, dtype, files, n_files, dst, dst_len, file_ns, n_written, flags,
                                               static_cast<cudaStream_t>(cuda_stream));
  profiler().resolve();
  return e;
}

// ---- ranges of an indexed standalone file (pco_b200_decompress_ranges)
// A piece is the part of one range that lies in one chunk.  A task decodes one touched chunk, once, however many pieces it has: a
// direct task (one piece) straight into the piece's place in the destination, a staged task (several pieces) as the window
// [min lo, max hi) into a scratch slot, from which gather_ranges_kernel copies every piece to its place.
struct RangePiece {
  uint32_t chunk, task;
  uint32_t lo, hi;    // chunk-relative numbers
  uint64_t dst_off;   // element offset of number lo in dst
  uint64_t range;     // the range it belongs to
};
struct RangeTask {
  uint32_t chunk;
  uint32_t lo, hi;          // the window: min lo and max hi of its pieces
  uint32_t piece0, n_pieces;  // its pieces: pieces[by_chunk[piece0 .. piece0 + n_pieces)]
  uint64_t first_range;     // the lowest-index range with numbers in the chunk
};

static PcoB200Error range_fail(PcoB200Error kind, uint64_t range, const std::string& what) {
  return fail(kind, "range " + std::to_string(range) + ": " + what);
}

// Splits the ranges at chunk boundaries (a binary search over out_offset) and groups the pieces by chunk.  That search needs chunk
// records that tile [0, n_total) in order, out_offset[k] = n[0] + ... + n[k - 1] with every n >= 1; an index is untrusted input, so
// that is checked first.  Pieces come in range order, tasks in chunk order; *total = the sum of the counts.
static PcoB200Error plan_ranges(const IndexChunk* recs, uint64_t n_chunks, uint64_t n_total, const PcoB200Range* ranges, size_t n_ranges,
                                std::vector<RangePiece>& pieces, std::vector<RangeTask>& tasks, std::vector<uint32_t>& by_chunk, uint64_t* total) {
  pieces.clear();
  tasks.clear();
  by_chunk.clear();
  uint64_t sum = 0;
  for (uint64_t k = 0; k < n_chunks; k++) {
    if (recs[k].n == 0 || recs[k].out_offset != sum)
      return fail(PCO_B200_INVALID_ARGUMENT, "side index: chunk " + std::to_string(k) + " does not start where the chunks before it end");
    sum += recs[k].n;
  }
  if (sum != n_total)
    return fail(PCO_B200_INVALID_ARGUMENT, "side index: its chunks hold " + std::to_string(sum) + " numbers, its header " + std::to_string(n_total));
  uint64_t tot = 0;
  for (size_t i = 0; i < n_ranges; i++) {
    const uint64_t s = ranges[i].start, cnt = ranges[i].count;
    if (cnt > n_total || s > n_total - cnt)
      return range_fail(PCO_B200_INVALID_ARGUMENT, i, "start " + std::to_string(s) + " + count " + std::to_string(cnt) + " lies past the file's " +
                                                          std::to_string(n_total) + " numbers");
    if (cnt > ~uint64_t(0) - tot) return range_fail(PCO_B200_INVALID_ARGUMENT, i, "the counts add up to more than 2^64 numbers");
    tot += cnt;
  }
  *total = tot;
  uint64_t off = 0;
  for (size_t i = 0; i < n_ranges; i++) {
    uint64_t s = ranges[i].start, left = ranges[i].count;
    while (left) {
      uint64_t a = 0, b = n_chunks;  // the last chunk whose out_offset <= s
      while (b - a > 1) {
        const uint64_t m = a + (b - a) / 2;
        if (recs[m].out_offset <= s) a = m;
        else b = m;
      }
      const uint32_t lo = uint32_t(s - recs[a].out_offset);
      const uint32_t take = uint32_t(std::min<uint64_t>(left, recs[a].n - lo));
      pieces.push_back(RangePiece{uint32_t(a), 0, lo, lo + take, off, uint64_t(i)});
      s += take;
      left -= take;
      off += take;
    }
  }
  by_chunk.resize(pieces.size());
  for (size_t p = 0; p < pieces.size(); p++) by_chunk[p] = uint32_t(p);
  std::stable_sort(by_chunk.begin(), by_chunk.end(), [&](uint32_t x, uint32_t y) { return pieces[x].chunk < pieces[y].chunk; });
  for (size_t p = 0; p < by_chunk.size();) {
    RangeTask t{pieces[by_chunk[p]].chunk, ~0u, 0u, uint32_t(p), 0u, pieces[by_chunk[p]].range};  // stable: the first piece has the lowest range
    size_t q = p;
    for (; q < by_chunk.size() && pieces[by_chunk[q]].chunk == t.chunk; q++) {
      RangePiece& pc = pieces[by_chunk[q]];
      t.lo = std::min(t.lo, pc.lo);
      t.hi = std::max(t.hi, pc.hi);
      pc.task = uint32_t(tasks.size());
    }
    t.n_pieces = uint32_t(q - p);
    tasks.push_back(t);
    p = q;
  }
  return PCO_B200_OK;
}

static PcoB200Error decompress_ranges_impl(const void* compressed, size_t compressed_len, uint32_t dtype, const void* index, size_t index_len,
                                           const PcoB200Range* ranges, size_t n_ranges, void* dst, size_t dst_len, size_t* n_written, uint32_t flags,
                                           cudaStream_t stream) {
  // ---- argument checks: host only, before any device work (headers in device memory are read back first)
  if (!nt_valid(dtype)) return fail(PCO_B200_INVALID_TYPE, "unknown number type byte: " + std::to_string(dtype));
  if (n_written) *n_written = 0;
  if (!index || index_len == 0) return fail(PCO_B200_INVALID_ARGUMENT, "a side index is required (pco_b200_build_index makes one)");
  if (!ranges && n_ranges) return fail(PCO_B200_INVALID_ARGUMENT, "ranges are required");
  if (n_ranges == 0) return PCO_B200_OK;
  if (!compressed && compressed_len) return fail(PCO_B200_INVALID_ARGUMENT, "null buffer");
  const bool src_dev = flags & PCO_B200_SRC_ON_DEVICE, dst_dev = flags & PCO_B200_DST_ON_DEVICE, idx_dev = flags & PCO_B200_INDEX_ON_DEVICE;
  const size_t elem = nt_bits(dtype) / 8;
  Context& c = ctx();
  if (src_dev || idx_dev)
    if (PcoB200Error e = ensure_device(c)) return e;
  // the file header and the index header: host copies, or one readback
  IndexHeader ih;
  StandaloneHeader hdr;
  if (PcoB200Error e = read_heads(compressed, compressed_len, src_dev, index, index_len, idx_dev, &ih, &hdr, stream)) return e;
  // the same check as the side-index path of pco_b200_decompress_ex
  if (!index_header_ok(ih, compressed_len, index_len)) return fail(PCO_B200_INVALID_ARGUMENT, "side index does not belong to this file");
  if (ih.n_chunks > 0x7fffffffull) return fail(PCO_B200_INVALID_ARGUMENT, "too many chunks");
  // the chunk table: a host copy, or a second readback
  std::vector<IndexChunk> recs(ih.n_chunks);
  if (ih.n_chunks) {
    const uint8_t* at = static_cast<const uint8_t*>(index) + ih.chunks_offset;
    if (idx_dev) {
      PCOB_CUDA_TRY(cudaMemcpyAsync(recs.data(), at, recs.size() * sizeof(IndexChunk), cudaMemcpyDeviceToHost, stream));
      PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
    } else {
      std::memcpy(recs.data(), at, recs.size() * sizeof(IndexChunk));
    }
  }
  std::vector<RangePiece> pieces;
  std::vector<RangeTask> tasks;
  std::vector<uint32_t> by_chunk;
  uint64_t total = 0;
  if (PcoB200Error e = plan_ranges(recs.data(), recs.size(), ih.n_total, ranges, n_ranges, pieces, tasks, by_chunk, &total)) return e;
  if (total > dst_len) return fail(PCO_B200_INVALID_ARGUMENT, "dst holds " + std::to_string(dst_len) + " numbers, the ranges " + std::to_string(total));
  if (total == 0) return PCO_B200_OK;
  if (!dst) return fail(PCO_B200_INVALID_ARGUMENT, "null buffer");
  if (pieces.size() > 0x7fffffffull) return fail(PCO_B200_INVALID_ARGUMENT, "the ranges make too many pieces");

  // ---- the file, the index and the destination in HBM
  if (PcoB200Error e = ensure_device(c)) return e;
  const uint8_t *d_src, *d_idx;
  if (PcoB200Error e = stage_in(c.src, compressed, compressed_len, src_dev, stream, &d_src)) return e;
  if (PcoB200Error e = stage_in(c.index, index, index_len, idx_dev, stream, &d_idx)) return e;
  void* d_out_v;
  if (PcoB200Error e = out_buffer(c, dst, dst_dev, total * elem, &d_out_v)) return e;
  uint8_t* d_out = static_cast<uint8_t*>(d_out_v);
  const FileParams fp{d_src, compressed_len, dtype, hdr.uniform_type, hdr.format_major};
  const uint32_t T = uint32_t(tasks.size());
  auto align16 = [](uint64_t x) { return (x + 15) & ~uint64_t(15); };
  // scratch slots of the staged tasks
  std::vector<uint64_t> slot(T, 0);
  uint64_t stage_bytes = 0;
  for (uint32_t t = 0; t < T; t++)
    if (tasks[t].n_pieces > 1) {
      slot[t] = stage_bytes;
      stage_bytes += align16(uint64_t(tasks[t].hi - tasks[t].lo) * elem);
    }
  PCOB_CUDA_TRY(c.rng_stage.reserve(stage_bytes + 64));
  uint8_t* d_stage = c.rng_stage.as<uint8_t>();
  // task table: IndexChunk[T] (the chunks' own records) | WinTask[T]
  const uint64_t wins_at = align16(uint64_t(T) * sizeof(IndexChunk));
  PCOB_CUDA_TRY(c.rng_tab.reserve(wins_at + uint64_t(T) * sizeof(WinTask) + 64));
  const IndexChunk* d_tasks = c.rng_tab.as<IndexChunk>();
  WinTask* d_wins = reinterpret_cast<WinTask*>(c.rng_tab.as<uint8_t>() + wins_at);
  std::vector<IndexChunk> trec(T);
  std::vector<WinTask> wins(T);
  for (uint32_t t = 0; t < T; t++) {
    const RangeTask& k = tasks[t];
    trec[t] = recs[k.chunk];
    const uint8_t* at = k.n_pieces > 1 ? d_stage + slot[t] : d_out + pieces[by_chunk[k.piece0]].dst_off * elem;
    wins[t] = WinTask{k.lo, k.hi, uint64_t(reinterpret_cast<uintptr_t>(at)), 0};
  }
  PCOB_CUDA_TRY(cudaMemcpyAsync(c.rng_tab.p, trec.data(), size_t(T) * sizeof(IndexChunk), cudaMemcpyHostToDevice, stream));
  PCOB_CUDA_TRY(cudaMemcpyAsync(d_wins, wins.data(), size_t(T) * sizeof(WinTask), cudaMemcpyHostToDevice, stream));
  // statuses and class bytes side by side: one readback brings both
  const size_t res_bytes = (size_t(T) * (sizeof(uint32_t) + 1) + 3) & ~size_t(3);
  PCOB_CUDA_TRY(c.statuses.reserve(res_bytes + 64));
  uint32_t* d_st = c.statuses.as<uint32_t>();
  uint8_t* d_cls = reinterpret_cast<uint8_t*>(d_st + T);
  if (PcoB200Error e = set_decode_attrs<true>(c)) return e;

  // ---- 1. fused_narrow_kernel decodes the narrow chunks' windows and classifies the rest
  profiler().begin("fused_narrow_kernel", stream);
  dispatch_latent(dtype, [&](auto tag) {
    using L = decltype(tag);
    fused_narrow_kernel<L, true><<<T, FZ_THREADS, sizeof(FusedSmem), stream>>>(fp, d_tasks, d_idx, index_len, d_st, d_cls, nullptr, 0, d_wins);
    return 0;
  });
  profiler().end(stream);
  PCOB_CUDA_TRY(cudaGetLastError());
  std::vector<uint32_t> res(res_bytes / 4);
  PCOB_CUDA_TRY(readback_small_sync(res.data(), d_st, res_bytes, stream));
  const uint8_t* cls = reinterpret_cast<const uint8_t*>(res.data() + T);
  std::vector<uint32_t> st(T, ST_OK);
  std::vector<uint32_t> general, cold;
  uint64_t rows = 0;
  for (uint32_t t = 0; t < T; t++) {
    if (cls[t] & CLS_DONE) {
      if (res[t] == ST_UNSUPPORTED) cold.push_back(t);
      else st[t] = res[t];
      continue;
    }
    // the general pair: the status word holds the task's first batch; it needs a row per var and batch from there on
    general.push_back(t);
    wins[t].row0 = rows;
    rows += uint64_t(cls[t] == 2 ? 2 : 1) * (n_batches_of(tasks[t].hi) - std::min(res[t], n_batches_of(tasks[t].hi)));
  }

  // ---- 2. symwalk_kernel + decode_kernel for the others
  if (!general.empty()) {
    PCOB_CUDA_TRY(c.dec_syms.reserve(rows * BATCH_N + 64));
    PCOB_CUDA_TRY(c.dec_offs.reserve(rows * sizeof(uint32_t) + 64));
    PCOB_CUDA_TRY(cudaMemcpyAsync(d_wins, wins.data(), size_t(T) * sizeof(WinTask), cudaMemcpyHostToDevice, stream));
    profiler().begin("symwalk_kernel", stream);
    symwalk_kernel<true><<<T, SW_THREADS, sizeof(SymWalkSmem), stream>>>(fp, d_tasks, d_idx, index_len, 0, c.dec_syms.as<uint8_t>(), c.dec_offs.as<uint32_t>(),
                                                                          d_cls, d_wins);
    profiler().end(stream);
    profiler().begin("decode_kernel", stream);
    dispatch_latent(dtype, [&](auto tag) {
      using L = decltype(tag);
      decode_kernel<L, 1, true><<<T, DEC_THREADS, sizeof(DecodeSmem), stream>>>(fp, d_tasks, d_st, d_idx, index_len, nullptr, 0, c.d_binoms,
                                                                                c.dec_syms.as<uint8_t>(), c.dec_offs.as<uint32_t>(), d_cls, d_wins);
      decode_kernel<L, 2, true><<<T, DEC_THREADS, sizeof(DecodeSmem), stream>>>(fp, d_tasks, d_st, d_idx, index_len, nullptr, 0, c.d_binoms,
                                                                                c.dec_syms.as<uint8_t>(), c.dec_offs.as<uint32_t>(), d_cls, d_wins);
      return 0;
    });
    profiler().end(stream);
    PCOB_CUDA_TRY(cudaGetLastError());
    PCOB_CUDA_TRY(readback_small_sync(res.data(), d_st, size_t(T) * sizeof(uint32_t), stream));
    for (uint32_t t : general) {
      if (res[t] == ST_UNSUPPORTED) cold.push_back(t);
      else st[t] = res[t];
    }
  }

  // ---- 3. chunks only the catch-all decoder takes: one single-thread launch per chunk, from the chunk's start to max hi, into a slot
  // of its own.  It stops there (ST_DST_FULL) or, when the window reaches the chunk's end, behind the chunk: the chunk is decoded once
  // the decoder has counted it.
  std::vector<uint64_t> cold_slot(T, 0);
  uint8_t* d_cold = nullptr;
  if (!cold.empty()) {
    std::sort(cold.begin(), cold.end());
    uint64_t cold_bytes = 0;
    for (uint32_t t : cold) {
      cold_slot[t] = cold_bytes;
      cold_bytes += align16(uint64_t(tasks[t].hi) * elem);
    }
    PCOB_CUDA_TRY(c.rng_cold.reserve(cold_bytes + 64));
    d_cold = c.rng_cold.as<uint8_t>();
    const size_t nc = cold.size();
    std::vector<ColdJob> jobs;
    for (uint32_t t : cold) jobs.push_back(ColdJob{fp, trec[t].chunk_offset, d_cold + cold_slot[t], tasks[t].hi});
    std::vector<ColdResult> cres;
    if (PcoB200Error e = cold_decode_jobs(c, dtype, jobs, cold_retry_chunk, &cres, stream)) return e;
    for (size_t k = 0; k < nc; k++) {
      const uint32_t s = cres[k].status;
      st[cold[k]] = cres[k].n_chunks > 0 ? ST_OK : (s == ST_OK || s == ST_TERMINATOR || s == ST_DST_FULL) ? ST_CORRUPTION : s;
    }
  }

  // ---- a failing chunk fails the call, named by the lowest-index range with numbers in it
  {
    uint32_t worst = T;
    for (uint32_t t = 0; t < T; t++)
      if (st[t] != ST_OK && (worst == T || tasks[t].first_range < tasks[worst].first_range)) worst = t;
    if (worst < T) {
      const PcoB200Error e = status_to_error(st[worst], ("chunk " + std::to_string(tasks[worst].chunk)).c_str());
      return range_fail(e, tasks[worst].first_range, last_error_ref());
    }
  }

  // ---- 4. pieces of staged and catch-all tasks: slot -> destination
  std::vector<RangeCopy> copies;
  for (uint32_t t = 0; t < T; t++) {
    const RangeTask& k = tasks[t];
    const bool is_cold = d_cold && std::binary_search(cold.begin(), cold.end(), t);
    if (k.n_pieces == 1 && !is_cold) continue;
    const uint8_t* base = is_cold ? d_cold + cold_slot[t] : d_stage + slot[t];
    const uint32_t wlo = is_cold ? 0u : k.lo;
    for (uint32_t q = 0; q < k.n_pieces; q++) {
      const RangePiece& p = pieces[by_chunk[k.piece0 + q]];
      copies.push_back(RangeCopy{uint64_t(reinterpret_cast<uintptr_t>(base + uint64_t(p.lo - wlo) * elem)),
                                 uint64_t(reinterpret_cast<uintptr_t>(d_out + p.dst_off * elem)), uint64_t(p.hi - p.lo) * elem});
    }
  }
  if (!copies.empty()) {
    PCOB_CUDA_TRY(c.rng_copies.reserve(copies.size() * sizeof(RangeCopy) + 64));
    PCOB_CUDA_TRY(cudaMemcpyAsync(c.rng_copies.p, copies.data(), copies.size() * sizeof(RangeCopy), cudaMemcpyHostToDevice, stream));
    profiler().begin("gather_ranges_kernel", stream);
    gather_ranges_kernel<<<uint32_t(copies.size()), RANGES_THREADS, 0, stream>>>(c.rng_copies.as<RangeCopy>());
    profiler().end(stream);
    PCOB_CUDA_TRY(cudaGetLastError());
  }
  if (!dst_dev) PCOB_CUDA_TRY(copy_sliced(dst, d_out, total * elem, cudaMemcpyDeviceToHost, stream));
  PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
  if (n_written) *n_written = size_t(total);
  return PCO_B200_OK;
}

PcoB200Error pco_b200_decompress_ranges(const void* compressed, size_t compressed_len, unsigned char dtype, const void* index, size_t index_len,
                                        const PcoB200Range* ranges, size_t n_ranges, void* dst, size_t dst_len, size_t* n_written, uint32_t flags,
                                        void* cuda_stream) {
  const PcoB200Error e = decompress_ranges_impl(compressed, compressed_len, dtype, index, index_len, ranges, n_ranges, dst, dst_len, n_written, flags,
                                                static_cast<cudaStream_t>(cuda_stream));
  profiler().resolve();
  return e;
}

PcoB200Error pco_b200_debug_plan_ranges(const void* chunk_table, size_t n_chunks, uint64_t n_total, const PcoB200Range* ranges, size_t n_ranges,
                                        uint64_t* pieces_out, size_t pieces_cap, size_t* n_pieces, uint64_t* tasks_out, size_t tasks_cap, size_t* n_tasks) {
  if ((!chunk_table && n_chunks) || (!ranges && n_ranges)) return fail(PCO_B200_INVALID_ARGUMENT, "null table");
  std::vector<IndexChunk> recs(n_chunks);
  if (n_chunks) std::memcpy(recs.data(), chunk_table, n_chunks * sizeof(IndexChunk));
  std::vector<RangePiece> pieces;
  std::vector<RangeTask> tasks;
  std::vector<uint32_t> by_chunk;
  uint64_t total = 0;
  if (PcoB200Error e = plan_ranges(recs.data(), n_chunks, n_total, ranges, n_ranges, pieces, tasks, by_chunk, &total)) return e;
  if (n_pieces) *n_pieces = pieces.size();
  if (n_tasks) *n_tasks = tasks.size();
  if (pieces.size() > pieces_cap || tasks.size() > tasks_cap) return fail(PCO_B200_IO, "the tables are too small");
  for (size_t p = 0; p < pieces.size(); p++) {
    const RangePiece& x = pieces[p];
    const uint64_t row[6] = {x.chunk, x.lo, x.hi, x.dst_off, x.range, x.task};
    std::memcpy(pieces_out + 6 * p, row, sizeof(row));
  }
  for (size_t t = 0; t < tasks.size(); t++) {
    const RangeTask& x = tasks[t];
    const uint64_t row[6] = {x.chunk, x.lo, x.hi, x.n_pieces, x.first_range, x.n_pieces > 1 ? 1u : 0u};
    std::memcpy(tasks_out + 6 * t, row, sizeof(row));
  }
  return PCO_B200_OK;
}

unsigned pco_b200_debug_async_kind(unsigned device_status) { return async_kind_of(device_status); }

// ---- asynchronous decompress of an indexed standalone file (pco_b200_decompress_async; kernels in async_kernels.cuh)
// The plan fixes what the launches take by value (FileParams' number type, uniform type and format major) and every grid size (from
// max_chunks); the file's own length, chunk count and n_total are read from its side index on the device.  So a call is a fixed
// sequence of seven launches and nothing else: check, fused, symwalk, decode<1>, decode<2>, cold, finish.  A kernel that has nothing
// to do for a chunk leaves at its first line.

static bool async_plan_ok(const PcoB200AsyncPlan* p) {
  return nt_valid(p->dtype) && p->max_chunks >= 1 && p->max_chunks <= 0xffffffffull && p->dst_cap <= (uint64_t(1) << 56) &&
         p->workspace_bytes == async_layout(p->dst_cap, uint32_t(p->max_chunks)).total;
}

PcoB200Error pco_b200_decompress_async_plan(const void* head, size_t head_len, unsigned char dtype, size_t src_cap, size_t index_cap, size_t dst_cap,
                                            size_t max_chunks, PcoB200AsyncPlan* plan) {
  StandaloneHeader hdr;
  if (PcoB200Error e = check_async_head(head, head_len, dtype, plan, &hdr)) return e;
  if (max_chunks == 0 || uint64_t(max_chunks) > 0xffffffffull) return fail(PCO_B200_INVALID_ARGUMENT, "max_chunks must be 1 .. 2^32 - 1");
  if (uint64_t(dst_cap) > (uint64_t(1) << 56)) return fail(PCO_B200_INVALID_ARGUMENT, "dst_cap above 2^56 numbers");
  std::memset(plan, 0, sizeof(*plan));
  plan->dtype = dtype;
  plan->uniform_type = hdr.uniform_type;
  plan->format_major = hdr.format_major;
  plan->src_cap = src_cap;
  plan->index_cap = index_cap;
  plan->dst_cap = dst_cap;
  plan->max_chunks = max_chunks;
  plan->workspace_bytes = async_layout(dst_cap, uint32_t(max_chunks)).total;
  return async_decode_setup<false>(dtype, [](auto tag) { return (const void*)cold_chunks_kernel<decltype(tag)>; },
                                   {(const void*)async_check_kernel, (const void*)async_finish_kernel});
}

PcoB200Error pco_b200_decompress_async(const PcoB200AsyncPlan* plan, const void* src, const void* index, void* dst, void* workspace,
                                       PcoB200AsyncStatus* status, void* cuda_stream) {
  if (!plan || !src || !index || !workspace || !status || (!dst && plan->dst_cap)) return fail(PCO_B200_INVALID_ARGUMENT, "null buffer");
  if (!async_plan_ok(plan)) return fail(PCO_B200_INVALID_ARGUMENT, "the plan was not made by pco_b200_decompress_async_plan");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail(PCO_B200_INVALID_ARGUMENT, "the workspace is not 256-byte aligned");
  AsyncLaunch ln;
  if (PcoB200Error e = open_async_launch(cuda_stream, &ln)) return e;
  const cudaStream_t stream = ln.stream;

  const uint32_t mc = uint32_t(plan->max_chunks);
  const AsyncLayout lay = async_layout(plan->dst_cap, mc);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  AsyncCheck* chk = reinterpret_cast<AsyncCheck*>(ws);
  IndexChunk* table = reinterpret_cast<IndexChunk*>(ws + lay.table);
  uint32_t* d_st = reinterpret_cast<uint32_t*>(ws + lay.st);
  AsyncArgs a;
  a.fp = FileParams{src, plan->src_cap, plan->dtype, plan->uniform_type, plan->format_major};
  a.index = static_cast<const uint8_t*>(index);
  a.index_cap = plan->index_cap;
  a.dst_cap = plan->dst_cap;
  a.max_chunks = mc;

  ln.begin("async_check_kernel");
  async_check_kernel<<<(mc + ASYNC_CHECK_RECS - 1) / ASYNC_CHECK_RECS, ASYNC_THREADS, 0, stream>>>(a, chk, table);
  ln.end();
  enqueue_decode_stage<false>(ln, DecodeStage{a.fp, table, a.index, a.index_cap, mc, d_st, ws + lay.cls, ws + lay.syms,
                                              reinterpret_cast<uint32_t*>(ws + lay.offs), &chk->binoms, dst, a.dst_cap, nullptr});
  ln.begin("cold_chunks_kernel");
  dispatch_latent(plan->dtype, [&](auto tag) {
    using L = decltype(tag);
    cold_chunks_kernel<L><<<1, ASYNC_THREADS, 0, stream>>>(a.fp, table, chk, d_st, static_cast<L*>(dst), a.dst_cap, ws + lay.cold);
    return 0;
  });
  ln.end();
  ln.begin("async_finish_kernel");
  async_finish_kernel<<<1, 1024, 0, stream>>>(a.dst_cap, chk, d_st, status);
  ln.end();
  PCOB_CUDA_TRY(cudaGetLastError());
  return PCO_B200_OK;  // spans stay pending until pco_b200_profile_last reads them
}

PcoB200Error pco_b200_decompress_async_result(const PcoB200AsyncStatus* s, PcoB200Progress* progress) {
  if (!s) return fail(PCO_B200_INVALID_ARGUMENT, "null status");
  const PcoB200Error kind = async_result_kind(s->kind);
  if (kind == PCO_B200_OK) {
    if (progress) {
      progress->n_processed = size_t(s->n_processed);
      progress->finished = s->finished ? 1 : 0;
    }
    return PCO_B200_OK;
  }
  if (const char* h = async_header_refusal(s->device_status)) return fail(kind, h);
  switch (s->device_status) {
    case PCO_B200_ASYNC_INDEX_FOREIGN: return fail(kind, "side index does not belong to this file (or its file length exceeds src_cap)");
    case PCO_B200_ASYNC_TOO_MANY_CHUNKS:
      return fail(kind, "the side index lists " + std::to_string(s->n_chunks) + " chunks, more than the plan's max_chunks");
    default:
      status_to_error(s->device_status, "this chunk");
      return fail(kind, "chunk " + std::to_string(s->chunk) + ": " + last_error_ref());
  }
}

// ---- asynchronous ranges of an indexed standalone file (pco_b200_decompress_ranges_async; kernels in async_ranges_kernels.cuh)
// The plan fixes every grid size (from max_chunks and max_ranges) and the byte layout of the workspace; the file's length, chunk count and
// n_total come from its side index, and the number of ranges from *n_ranges, on the device.  A call is a fixed sequence of fifteen
// launches: check, chunks, count, scan, mark, window, gate, tasks, fused, symwalk, decode<1>, decode<2>, cold, gather, finish.

static bool ar_plan_ok(const PcoB200AsyncRangesPlan* p) {
  return nt_valid(p->dtype) && p->max_chunks >= 1 && p->max_chunks <= 0xffffffffull && p->max_ranges >= 1 && p->max_ranges <= 0xffffffffull &&
         p->dst_cap <= (uint64_t(1) << 56) && p->window_cap <= (uint64_t(1) << 56) &&
         p->workspace_bytes == ar_layout(p->max_chunks, p->max_ranges, p->window_cap, nt_bits(p->dtype) / 8).total;
}

PcoB200Error pco_b200_decompress_ranges_async_plan(const void* head, size_t head_len, unsigned char dtype, size_t src_cap, size_t index_cap,
                                                   size_t max_chunks, size_t max_ranges, size_t dst_cap, size_t window_cap, PcoB200AsyncRangesPlan* plan) {
  StandaloneHeader hdr;
  if (PcoB200Error e = check_async_head(head, head_len, dtype, plan, &hdr)) return e;
  if (max_chunks == 0 || uint64_t(max_chunks) > 0xffffffffull) return fail(PCO_B200_INVALID_ARGUMENT, "max_chunks must be 1 .. 2^32 - 1");
  if (max_ranges == 0 || uint64_t(max_ranges) > 0xffffffffull) return fail(PCO_B200_INVALID_ARGUMENT, "max_ranges must be 1 .. 2^32 - 1");
  if (uint64_t(dst_cap) > (uint64_t(1) << 56)) return fail(PCO_B200_INVALID_ARGUMENT, "dst_cap above 2^56 numbers");
  if (uint64_t(window_cap) > (uint64_t(1) << 56)) return fail(PCO_B200_INVALID_ARGUMENT, "window_cap above 2^56 numbers");
  std::memset(plan, 0, sizeof(*plan));
  plan->dtype = dtype;
  plan->uniform_type = hdr.uniform_type;
  plan->format_major = hdr.format_major;
  plan->src_cap = src_cap;
  plan->index_cap = index_cap;
  plan->max_chunks = max_chunks;
  plan->max_ranges = max_ranges;
  plan->dst_cap = dst_cap;
  plan->window_cap = window_cap;
  plan->workspace_bytes = ar_layout(max_chunks, max_ranges, window_cap, nt_bits(dtype) / 8).total;
  return async_decode_setup<true>(dtype, [](auto tag) { return (const void*)ar_cold_kernel<decltype(tag)>; },
                                  {(const void*)async_check_kernel, (const void*)ar_chunks_kernel, (const void*)ar_count_kernel, (const void*)ar_scan_kernel,
                                   (const void*)ar_mark_kernel, (const void*)ar_window_kernel, (const void*)ar_gate_kernel, (const void*)ar_tasks_kernel,
                                   (const void*)ar_gather_kernel, (const void*)ar_finish_kernel});
}

PcoB200Error pco_b200_decompress_ranges_async(const PcoB200AsyncRangesPlan* plan, const void* src, const void* index, const PcoB200Range* ranges,
                                              const uint64_t* n_ranges, void* dst, void* workspace, PcoB200AsyncRangesStatus* status, void* cuda_stream) {
  if (!plan || !src || !index || !ranges || !n_ranges || !workspace || !status || (!dst && plan->dst_cap))
    return fail(PCO_B200_INVALID_ARGUMENT, "null buffer");
  if (!ar_plan_ok(plan)) return fail(PCO_B200_INVALID_ARGUMENT, "the plan was not made by pco_b200_decompress_ranges_async_plan");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail(PCO_B200_INVALID_ARGUMENT, "the workspace is not 256-byte aligned");
  AsyncLaunch ln;
  if (PcoB200Error e = open_async_launch(cuda_stream, &ln)) return e;
  const cudaStream_t stream = ln.stream;

  const uint32_t mc = uint32_t(plan->max_chunks), mr = uint32_t(plan->max_ranges), elem = nt_bits(plan->dtype) / 8;
  const ArLayout lay = ar_layout(mc, mr, plan->window_cap, elem);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  AsyncCheck* chk = reinterpret_cast<AsyncCheck*>(ws);
  ArState* state = reinterpret_cast<ArState*>(ws + lay.state);
  IndexChunk* table = reinterpret_cast<IndexChunk*>(ws + lay.table);
  ArMark* marks = reinterpret_cast<ArMark*>(ws + lay.marks);
  ArChunkPart* cparts = reinterpret_cast<ArChunkPart*>(ws + lay.cparts);
  ArRangePart* rparts = reinterpret_cast<ArRangePart*>(ws + lay.rparts);
  uint64_t* roff = reinterpret_cast<uint64_t*>(ws + lay.roff);
  uint2* rspan = reinterpret_cast<uint2*>(ws + lay.rspan);
  IndexChunk* tasks = reinterpret_cast<IndexChunk*>(ws + lay.tasks);
  WinTask* wins = reinterpret_cast<WinTask*>(ws + lay.wins);
  ArTask* tinfo = reinterpret_cast<ArTask*>(ws + lay.tinfo);
  uint32_t* d_st = reinterpret_cast<uint32_t*>(ws + lay.st);
  uint8_t* d_stage = ws + lay.stage;
  ArArgs g;
  g.a.fp = FileParams{src, plan->src_cap, plan->dtype, plan->uniform_type, plan->format_major};
  g.a.index = static_cast<const uint8_t*>(index);
  g.a.index_cap = plan->index_cap;
  g.a.dst_cap = plan->dst_cap;
  g.a.max_chunks = mc;
  g.ranges = ranges;
  g.n_ranges = n_ranges;
  g.window_cap = plan->window_cap;
  g.max_ranges = mr;
  g.elem = elem;
  const uint32_t cb = uint32_t(ctas_of<AR_THREADS>(mc)), rb = uint32_t(ctas_of<AR_THREADS>(mr));

  ln.begin("async_check_kernel");
  async_check_kernel<<<(mc + ASYNC_CHECK_RECS - 1) / ASYNC_CHECK_RECS, ASYNC_THREADS, 0, stream>>>(g.a, chk, table);
  ln.end();
  ln.begin("ar_chunks_kernel");
  ar_chunks_kernel<<<cb, AR_THREADS, 0, stream>>>(chk, table, marks, cparts);
  ln.end();
  ln.begin("ar_count_kernel");
  ar_count_kernel<<<rb, AR_THREADS, 0, stream>>>(g, chk, rparts);
  ln.end();
  ln.begin("ar_scan_kernel");
  ar_scan_kernel<<<1, AR_SCAN_THREADS, 0, stream>>>(g, chk, cparts, rparts, state);
  ln.end();
  ln.begin("ar_mark_kernel");
  ar_mark_kernel<<<rb, AR_THREADS, 0, stream>>>(g, chk, table, rparts, state, marks, roff, rspan);
  ln.end();
  ln.begin("ar_window_kernel");
  ar_window_kernel<<<cb, AR_THREADS, 0, stream>>>(chk, state, marks, cparts);
  ln.end();
  ln.begin("ar_gate_kernel");
  ar_gate_kernel<<<1, AR_SCAN_THREADS, 0, stream>>>(g, cparts, state);
  ln.end();
  ln.begin("ar_tasks_kernel");
  ar_tasks_kernel<<<cb, AR_THREADS, 0, stream>>>(g, chk, state, table, marks, cparts, tasks, wins, tinfo, static_cast<uint8_t*>(dst), d_stage);
  ln.end();
  // window mode: the decode writes to the tasks' destinations or slots (wins), not to a dst of its own
  enqueue_decode_stage<true>(ln, DecodeStage{g.a.fp, tasks, g.a.index, g.a.index_cap, mc, d_st, ws + lay.cls, ws + lay.syms,
                                             reinterpret_cast<uint32_t*>(ws + lay.offs), &chk->binoms, nullptr, 0, wins});
  ln.begin("ar_cold_kernel");
  dispatch_latent(plan->dtype, [&](auto tag) {
    using L = decltype(tag);
    ar_cold_kernel<L><<<1, AR_THREADS, 0, stream>>>(g.a.fp, state, tasks, wins, tinfo, d_st, reinterpret_cast<L*>(d_stage), ws + lay.cold);
    return 0;
  });
  ln.end();
  ln.begin("ar_gather_kernel");
  ar_gather_kernel<<<std::min(mr, AR_GATHER_MAX_CTAS), AR_THREADS, 0, stream>>>(g, state, table, marks, wins, tinfo, d_st, roff, rspan,
                                                                                  static_cast<uint8_t*>(dst), d_stage);
  ln.end();
  ln.begin("ar_finish_kernel");
  ar_finish_kernel<<<1, AR_SCAN_THREADS, 0, stream>>>(state, tinfo, d_st, status);
  ln.end();
  PCOB_CUDA_TRY(cudaGetLastError());
  return PCO_B200_OK;  // spans stay pending until pco_b200_profile_last reads them
}

PcoB200Error pco_b200_decompress_ranges_async_result(const PcoB200AsyncRangesStatus* s, size_t* n_written) {
  if (!s) return fail(PCO_B200_INVALID_ARGUMENT, "null status");
  const PcoB200Error kind = async_result_kind(s->kind);
  if (kind == PCO_B200_OK) {
    if (n_written) *n_written = size_t(s->n_written);
    return PCO_B200_OK;
  }
  if (const char* h = async_header_refusal(s->device_status)) return fail(kind, h);
  switch (s->device_status) {
    case PCO_B200_ASYNC_INDEX_FOREIGN: return fail(kind, "side index does not belong to this file (or its file length exceeds src_cap)");
    case PCO_B200_ASYNC_TOO_MANY_CHUNKS: return fail(kind, "the side index lists more chunks than the plan's max_chunks");
    case PCO_B200_ASYNC_INDEX_TILING:
      return fail(kind, "side index: chunk " + std::to_string(s->chunk) + " does not start where the chunks before it end");
    case PCO_B200_ASYNC_INDEX_TOTAL: return fail(kind, "side index: its chunks do not hold the number of numbers its header states");
    case PCO_B200_ASYNC_TOO_MANY_RANGES: return fail(kind, "*n_ranges is above the plan's max_ranges");
    case PCO_B200_ASYNC_RANGE_PAST: return range_fail(kind, s->range, "start + count lies past the file's numbers");
    case PCO_B200_ASYNC_RANGE_OVERFLOW: return range_fail(kind, s->range, "the counts add up to more than 2^64 numbers");
    case PCO_B200_ASYNC_DST_SHORT: return fail(kind, "dst_cap is below the ranges' " + std::to_string(s->n_written) + " numbers");
    case PCO_B200_ASYNC_WINDOW:
      return fail(kind, "the ranges need a window of " + std::to_string(s->window_needed) + " numbers, more than the plan's window_cap");
    default:
      status_to_error(s->device_status, ("chunk " + std::to_string(s->chunk)).c_str());
      return range_fail(kind, s->range, last_error_ref());
  }
}

// ---- asynchronous batch of indexed standalone files (pco_b200_decompress_files_async; kernels in async_files_kernels.cuh)
// The plan fixes every grid size (from max_files and max_chunks) and the byte layout of the workspace; the refs and their count are read
// on the device.  A call is a fixed sequence of twelve launches: files, check_index, scan, place, table, merge_index, fused, symwalk,
// decode<1>, decode<2>, cold, finish.

static bool af_plan_ok(const PcoB200AsyncFilesPlan* p) {
  return nt_valid(p->dtype) && p->max_files >= 1 && p->max_files <= 0x7fffffffull && p->max_chunks >= 1 && p->max_chunks <= 0xffffffffull &&
         p->dst_cap <= (uint64_t(1) << 56) && p->workspace_bytes == af_layout(p->max_files, p->max_chunks, p->dst_cap).total;
}

PcoB200Error pco_b200_decompress_files_async_plan(const void* head, size_t head_len, unsigned char dtype, size_t src_cap, size_t index_cap,
                                                  size_t max_files, size_t max_chunks, size_t dst_cap, PcoB200AsyncFilesPlan* plan) {
  StandaloneHeader hdr;
  if (PcoB200Error e = check_async_head(head, head_len, dtype, plan, &hdr)) return e;
  if (max_files == 0 || uint64_t(max_files) > 0x7fffffffull) return fail(PCO_B200_INVALID_ARGUMENT, "max_files must be 1 .. 2^31 - 1");
  if (max_chunks == 0 || uint64_t(max_chunks) > 0xffffffffull) return fail(PCO_B200_INVALID_ARGUMENT, "max_chunks must be 1 .. 2^32 - 1");
  if (uint64_t(dst_cap) > (uint64_t(1) << 56)) return fail(PCO_B200_INVALID_ARGUMENT, "dst_cap above 2^56 numbers");
  std::memset(plan, 0, sizeof(*plan));
  plan->dtype = dtype;
  plan->uniform_type = hdr.uniform_type;
  plan->format_major = hdr.format_major;
  plan->src_cap = src_cap;
  plan->index_cap = index_cap;
  plan->max_files = max_files;
  plan->max_chunks = max_chunks;
  plan->dst_cap = dst_cap;
  plan->workspace_bytes = af_layout(max_files, max_chunks, dst_cap).total;
  return async_decode_setup<false>(dtype, [](auto tag) { return (const void*)cold_chunks_kernel<decltype(tag)>; },
                                   {(const void*)af_files_kernel, (const void*)check_index_kernel, (const void*)af_scan_kernel, (const void*)af_place_kernel,
                                    (const void*)af_table_kernel, (const void*)merge_index_kernel, (const void*)af_finish_kernel});
}

// The launches of pco_b200_decompress_files_async over the workspace `ws` laid out by `lay`: the front end, the decode stage, the
// catch-all decoder into dst and af_finish_kernel into *status (and file_ns).  With `filt` the decode stage runs its filter-mode
// instantiations, dst is their value staging, and ff_cold_list_kernel records the cold records in the cold list `cold_list` before the
// catch-all decoder runs (pco_b200_filter_files_async).  With `agg` too, the aggregate-mode instantiations, which store nothing to dst;
// dst is the catch-all decoder's value staging only (pco_b200_aggregate_files_async).  With `take` instead of `agg`, the take-mode
// instantiations, likewise (pco_b200_take_files_async).  `between`, when given, enqueues its launches behind the front end
// (merge_index_kernel) and before the decode stage.
static void enqueue_files(const AsyncLaunch& ln, const AfArgs& g, const AfLayout& lay, uint8_t* ws, void* dst, const FiltStage* filt,
                          uint32_t* cold_list, uint64_t* file_ns, PcoB200AsyncFilesStatus* status, bool agg = false, bool take = false,
                          const std::function<void()>& between = {}) {
  const cudaStream_t stream = ln.stream;
  const uint32_t mf = g.max_files, mc = g.max_chunks;
  AsyncCheck* chk = reinterpret_cast<AsyncCheck*>(ws);
  AfState* state = reinterpret_cast<AfState*>(ws + lay.state);
  uint32_t* fst = reinterpret_cast<uint32_t*>(ws + lay.fst);
  FileCheck* fchk = reinterpret_cast<FileCheck*>(ws + lay.fchk);
  uint32_t* verdict = reinterpret_cast<uint32_t*>(ws + lay.verdict);
  FileMerge* merges = reinterpret_cast<FileMerge*>(ws + lay.merges);
  AfPart* parts = reinterpret_cast<AfPart*>(ws + lay.parts);
  IndexChunk* table = reinterpret_cast<IndexChunk*>(ws + lay.table);
  uint32_t* d_st = reinterpret_cast<uint32_t*>(ws + lay.st);
  const uint8_t* d_idx = g.index;
  const uint32_t fb = uint32_t(ctas_of<AF_THREADS>(mf)), tb = uint32_t(std::max(ctas_of<AF_THREADS>(mf), ctas_of<AF_THREADS>(mc)));

  ln.begin("af_files_kernel");
  af_files_kernel<<<fb, AF_THREADS, 0, stream>>>(g, chk, fst, fchk, merges, parts);
  ln.end();
  ln.begin("check_index_kernel");
  check_index_kernel<<<mf, 256, 0, stream>>>(static_cast<const uint8_t*>(g.fp.src), d_idx, g.fp.dtype, fchk, verdict);
  ln.end();
  ln.begin("af_scan_kernel");
  af_scan_kernel<<<1, AF_SCAN_THREADS, 0, stream>>>(g, parts, state);
  ln.end();
  ln.begin("af_place_kernel");
  af_place_kernel<<<fb, AF_THREADS, 0, stream>>>(g, fst, fchk, verdict, parts, merges, state);
  ln.end();
  ln.begin("af_table_kernel");
  af_table_kernel<<<tb, AF_THREADS, 0, stream>>>(g, state, chk, merges, table);
  ln.end();
  ln.begin("merge_index_kernel");
  merge_index_kernel<<<mf, 256, 0, stream>>>(d_idx, merges, table);
  ln.end();
  if (between) between();
  const DecodeStage d{g.fp, table, d_idx, g.index_cap, mc, d_st, ws + lay.cls, ws + lay.syms, reinterpret_cast<uint32_t*>(ws + lay.offs),
                      &chk->binoms, agg || take ? nullptr : dst, g.dst_cap, nullptr, filt ? *filt : FiltStage{}};
  if (filt) {
    if (agg) enqueue_decode_stage<false, true, true>(ln, d);
    else if (take) enqueue_decode_stage<false, true, false, true>(ln, d);
    else enqueue_decode_stage<false, true>(ln, d);
    ln.begin("ff_cold_list_kernel");
    ff_cold_list_kernel<<<uint32_t(ctas_of<FF_THREADS>(mc)), FF_THREADS, 0, stream>>>(chk, d_st, cold_list);
    ln.end();
  } else {
    enqueue_decode_stage<false>(ln, d);
  }
  ln.begin("cold_chunks_kernel");
  dispatch_latent(g.fp.dtype, [&](auto tag) {
    using L = decltype(tag);
    cold_chunks_kernel<L><<<1, ASYNC_THREADS, 0, stream>>>(g.fp, table, chk, d_st, static_cast<L*>(dst), g.dst_cap, ws + lay.cold);
    return 0;
  });
  ln.end();
  ln.begin("af_finish_kernel");
  af_finish_kernel<<<1, AF_SCAN_THREADS, 0, stream>>>(state, chk, merges, fchk, d_st, file_ns, status);
  ln.end();
}

PcoB200Error pco_b200_decompress_files_async(const PcoB200AsyncFilesPlan* plan, const void* src, const void* index, const PcoB200FileRef* files,
                                             const uint64_t* n_files, void* dst, uint64_t* file_ns, void* workspace, PcoB200AsyncFilesStatus* status,
                                             void* cuda_stream) {
  if (!plan || !src || !index || !files || !n_files || !workspace || !status || (!dst && plan->dst_cap))
    return fail(PCO_B200_INVALID_ARGUMENT, "null buffer");
  if (!af_plan_ok(plan)) return fail(PCO_B200_INVALID_ARGUMENT, "the plan was not made by pco_b200_decompress_files_async_plan");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail(PCO_B200_INVALID_ARGUMENT, "the workspace is not 256-byte aligned");
  AsyncLaunch ln;
  if (PcoB200Error e = open_async_launch(cuda_stream, &ln)) return e;

  const uint32_t mf = uint32_t(plan->max_files), mc = uint32_t(plan->max_chunks);
  const AfArgs g{FileParams{src, plan->src_cap, plan->dtype, plan->uniform_type, plan->format_major}, static_cast<const uint8_t*>(index),
                 plan->index_cap, plan->dst_cap, files, n_files, mf, mc};
  enqueue_files(ln, g, af_layout(mf, mc, plan->dst_cap), static_cast<uint8_t*>(workspace), dst, nullptr, nullptr, file_ns, status);
  PCOB_CUDA_TRY(cudaGetLastError());
  return PCO_B200_OK;  // spans stay pending until pco_b200_profile_last reads them
}

PcoB200Error pco_b200_decompress_files_async_result(const PcoB200AsyncFilesStatus* s, size_t* n_written) {
  if (!s) return fail(PCO_B200_INVALID_ARGUMENT, "null status");
  const PcoB200Error kind = async_result_kind(s->kind);
  if (kind == PCO_B200_OK) {
    if (n_written) *n_written = size_t(s->n_written);
    return PCO_B200_OK;
  }
  const uint64_t f = s->file;
  if (const char* h = async_header_refusal(s->device_status)) return file_fail(kind, f, h);
  switch (s->device_status) {
    case PCO_B200_ASYNC_TOO_MANY_FILES:
      return fail(kind, "*n_files is " + std::to_string(s->n_files) + ", above the plan's max_files");
    case PCO_B200_ASYNC_FILE_OUTSIDE: return file_fail(kind, f, "file lies outside src");
    case PCO_B200_ASYNC_INDEX_OFFSET: return file_fail(kind, f, "index offset is not a multiple of 16");
    case PCO_B200_ASYNC_INDEX_OUTSIDE: return file_fail(kind, f, "side index lies outside index");
    case PCO_B200_ASYNC_NO_INDEX: return file_fail(kind, f, "no side index (files without one are walked, which needs the host)");
    case PCO_B200_ASYNC_INDEX_FOREIGN: return file_fail(kind, f, "side index does not belong to this file");
    case PCO_B200_ASYNC_ENTRIES_MISALIGNED: return file_fail(kind, f, "side index does not belong to this file (misaligned entries)");
    case PCO_B200_ASYNC_RECORDS_OUTSIDE:
      return file_fail(kind, f, "side index does not belong to this file (a record points outside the file, its index or its count)");
    case PCO_B200_ASYNC_FILES_DST: return file_fail(kind, f, "dst holds fewer numbers than the files up to this one");
    case PCO_B200_ASYNC_TOO_MANY_CHUNKS: return file_fail(kind, f, "the files up to this one hold more chunks than the plan's max_chunks");
    default:
      status_to_error(s->device_status, ("chunk " + std::to_string(s->chunk)).c_str());
      return file_fail(kind, f, last_error_ref());
  }
}

// ---- asynchronous filter of indexed standalone files (pco_b200_filter_files_async; kernels in async_filter_files_kernels.cuh).  A memset
// of the slot counts and ff_map_kernel, then the files call's launches (enqueue_files, with the decode stage's filter-mode instantiations,
// ff_cold_list_kernel and rows_cap as dst_cap), then ff_cold, fl_count, ff_finish and fl_gather.

static bool ff_plan_ok(const PcoB200AsyncFilesFilterPlan* p) {
  return nt_valid(p->dtype) && p->max_files >= 1 && p->max_files <= 0x7fffffffull && p->max_chunks >= 1 && p->max_chunks <= 0xffffffffull &&
         p->rows_cap <= (uint64_t(1) << 56) && p->out_cap <= (uint64_t(1) << 56) &&
         p->workspace_bytes == ff_layout(p->max_files, p->max_chunks, p->rows_cap, nt_bits(p->dtype) / 8).ff_total;
}

PcoB200Error pco_b200_filter_files_async_plan(const void* head, size_t head_len, unsigned char dtype, size_t src_cap, size_t index_cap,
                                              size_t max_files, size_t max_chunks, size_t rows_cap, size_t out_cap, PcoB200AsyncFilesFilterPlan* plan) {
  StandaloneHeader hdr;
  if (PcoB200Error e = check_async_head(head, head_len, dtype, plan, &hdr)) return e;
  if (max_files == 0 || uint64_t(max_files) > 0x7fffffffull) return fail(PCO_B200_INVALID_ARGUMENT, "max_files must be 1 .. 2^31 - 1");
  if (max_chunks == 0 || uint64_t(max_chunks) > 0xffffffffull) return fail(PCO_B200_INVALID_ARGUMENT, "max_chunks must be 1 .. 2^32 - 1");
  if (uint64_t(rows_cap) > (uint64_t(1) << 56)) return fail(PCO_B200_INVALID_ARGUMENT, "rows_cap above 2^56 numbers");
  if (uint64_t(out_cap) > (uint64_t(1) << 56)) return fail(PCO_B200_INVALID_ARGUMENT, "out_cap above 2^56 numbers");
  std::memset(plan, 0, sizeof(*plan));
  plan->dtype = dtype;
  plan->uniform_type = hdr.uniform_type;
  plan->format_major = hdr.format_major;
  plan->src_cap = src_cap;
  plan->index_cap = index_cap;
  plan->max_files = max_files;
  plan->max_chunks = max_chunks;
  plan->rows_cap = rows_cap;
  plan->out_cap = out_cap;
  plan->workspace_bytes = ff_layout(max_files, max_chunks, rows_cap, nt_bits(dtype) / 8).ff_total;
  if (PcoB200Error e = async_decode_setup<false, true>(dtype, [](auto tag) { return (const void*)cold_chunks_kernel<decltype(tag)>; },
                                                       {(const void*)af_files_kernel, (const void*)check_index_kernel, (const void*)af_scan_kernel,
                                                        (const void*)af_place_kernel, (const void*)af_table_kernel, (const void*)merge_index_kernel,
                                                        (const void*)af_finish_kernel, (const void*)ff_map_kernel, (const void*)ff_cold_list_kernel,
                                                        (const void*)fl_count_kernel, (const void*)ff_finish_kernel}))
    return e;
  return dispatch_latent(dtype, [&](auto tag) -> PcoB200Error {
    using L = decltype(tag);
    return load_kernels({(const void*)ff_cold_kernel<L>, (const void*)fl_gather_kernel<L>});
  });
}

PcoB200Error pco_b200_filter_files_async(const PcoB200AsyncFilesFilterPlan* plan, const void* src, const void* index, const PcoB200FileRef* files,
                                         const uint64_t* n_files, const PcoB200Interval* interval, void* out_values, uint64_t* out_positions,
                                         uint64_t* n_matches, uint64_t* file_ns, void* workspace, PcoB200AsyncFilesFilterStatus* status,
                                         void* cuda_stream) {
  if (!plan || !src || !index || !files || !n_files || !interval || !n_matches || !workspace || !status ||
      ((!out_values || !out_positions) && plan->out_cap))
    return fail(PCO_B200_INVALID_ARGUMENT, "null buffer");
  if (!ff_plan_ok(plan)) return fail(PCO_B200_INVALID_ARGUMENT, "the plan was not made by pco_b200_filter_files_async_plan");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail(PCO_B200_INVALID_ARGUMENT, "the workspace is not 256-byte aligned");
  AsyncLaunch ln;
  if (PcoB200Error e = open_async_launch(cuda_stream, &ln)) return e;
  const cudaStream_t stream = ln.stream;

  const uint32_t mf = uint32_t(plan->max_files), mc = uint32_t(plan->max_chunks);
  const FfLayout lay = ff_layout(mf, mc, plan->rows_cap, nt_bits(plan->dtype) / 8);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  const uint64_t slots = fl_slots(mc, plan->rows_cap), n_parts = ctas_of<FL_THREADS>(slots);
  const AfArgs g{FileParams{src, plan->src_cap, plan->dtype, plan->uniform_type, plan->format_major}, static_cast<const uint8_t*>(index),
                 plan->index_cap, plan->rows_cap, files, n_files, mf, mc};
  const FiltStage filt{reinterpret_cast<const uint64_t*>(interval), reinterpret_cast<const uint32_t*>(ws + lay.slot_map),
                       reinterpret_cast<uint32_t*>(ws + lay.counts), reinterpret_cast<uint64_t*>(ws + lay.rows), ws + lay.soffs};
  auto* fstatus = reinterpret_cast<PcoB200AsyncFilesStatus*>(ws + lay.fstatus);
  auto* fstate = reinterpret_cast<FlState*>(ws + lay.fstate);
  auto* cparts = reinterpret_cast<uint64_t*>(ws + lay.cparts);
  auto* cold_list = reinterpret_cast<uint32_t*>(ws + lay.cold_list);

  PCOB_CUDA_TRY(cudaMemsetAsync(filt.counts, 0, slots * sizeof(uint32_t), stream));
  ln.begin("ff_map_kernel");
  ff_map_kernel<<<uint32_t(ctas_of<FF_THREADS>(mc)), FF_THREADS, 0, stream>>>(mc, reinterpret_cast<uint32_t*>(ws + lay.slot_map), cold_list);
  ln.end();
  enqueue_files(ln, g, lay, ws, ws + lay.stage, &filt, cold_list, file_ns, fstatus);
  dispatch_latent(plan->dtype, [&](auto tag) {
    using L = decltype(tag);
    ln.begin("ff_cold_kernel");
    ff_cold_kernel<L><<<std::min(mc, uint32_t(FF_COLD_CTAS)), FL_THREADS, 0, stream>>>(cold_list, reinterpret_cast<const IndexChunk*>(ws + lay.table), filt,
                                                                                       plan->dtype, reinterpret_cast<L*>(ws + lay.stage));
    ln.end();
    ln.begin("fl_count_kernel");
    fl_count_kernel<<<uint32_t(n_parts), FL_THREADS, 0, stream>>>(filt.counts, slots, cparts);
    ln.end();
    ln.begin("ff_finish_kernel");
    ff_finish_kernel<<<1, FL_SCAN_THREADS, 0, stream>>>(fstatus, cparts, n_parts, plan->out_cap, fstate, n_matches, status);
    ln.end();
    ln.begin("fl_gather_kernel");
    fl_gather_kernel<L><<<uint32_t(n_parts), FL_THREADS, 0, stream>>>(fstate, filt.counts, filt.rows, cparts, slots, reinterpret_cast<const L*>(ws + lay.stage),
                                                                     ws + lay.soffs, plan->out_cap, static_cast<L*>(out_values), out_positions);
    ln.end();
    return 0;
  });
  PCOB_CUDA_TRY(cudaGetLastError());
  return PCO_B200_OK;  // spans stay pending until pco_b200_profile_last reads them
}

PcoB200Error pco_b200_filter_files_async_result(const PcoB200AsyncFilesFilterStatus* s, size_t* n_matches) {
  if (!s) return fail(PCO_B200_INVALID_ARGUMENT, "null status");
  const PcoB200Error kind = async_result_kind(s->kind);
  if (kind == PCO_B200_OK) {
    if (n_matches) *n_matches = size_t(s->n_matches);
    return PCO_B200_OK;
  }
  switch (s->device_status) {
    case PCO_B200_FILTER_OUT_FULL:
      return fail(kind, "the files hold " + std::to_string(s->matches_needed) + " matches, more than the plan's out_cap");
    case PCO_B200_ASYNC_FILES_DST: return file_fail(kind, size_t(s->file), "the files up to this one hold more numbers than rows_cap");
    default: {  // the files call's outcome, in its words
      const PcoB200AsyncFilesStatus f{s->kind, s->device_status, s->file, s->chunk, s->n_written, s->n_files};
      return pco_b200_decompress_files_async_result(&f, nullptr);
    }
  }
}

// ---- asynchronous batch of wrapped pages (pco_b200_decompress_pages_async; kernels in async_pages_kernels.cuh)
// The plan fixes every grid size (from max_pages) and the byte layout of the workspace; the refs and their count are read on the device.
// A call is a fixed sequence of thirteen launches: pages, scan, place, frame_pages, walk, route, rewalk, fused, symwalk, decode<1>,
// decode<2>, cold, finish.

static bool ap_plan_ok(const PcoB200AsyncPagesPlan* p) {
  return nt_valid(p->dtype) && p->max_pages >= 1 && p->max_pages <= 0x7fffffffull && p->dst_cap <= (uint64_t(1) << 56) &&
         p->frame_cap <= (uint64_t(1) << 56) && p->workspace_bytes == ap_layout(p->max_pages, p->dst_cap, p->frame_cap).total;
}

PcoB200Error pco_b200_decompress_pages_async_plan(unsigned char dtype, size_t metas_cap, size_t pages_cap, size_t max_pages, size_t dst_cap,
                                                  size_t frame_cap, PcoB200AsyncPagesPlan* plan) {
  if (!nt_valid(dtype)) return fail(PCO_B200_INVALID_TYPE, "unknown number type byte: " + std::to_string(dtype));
  if (!plan) return fail(PCO_B200_INVALID_ARGUMENT, "null plan");
  if (max_pages == 0 || uint64_t(max_pages) > 0x7fffffffull) return fail(PCO_B200_INVALID_ARGUMENT, "max_pages must be 1 .. 2^31 - 1");
  if (uint64_t(dst_cap) > (uint64_t(1) << 56)) return fail(PCO_B200_INVALID_ARGUMENT, "dst_cap above 2^56 numbers");
  if (uint64_t(frame_cap) > (uint64_t(1) << 56)) return fail(PCO_B200_INVALID_ARGUMENT, "frame_cap above 2^56 bytes");
  std::memset(plan, 0, sizeof(*plan));
  plan->dtype = dtype;
  plan->metas_cap = metas_cap;
  plan->pages_cap = pages_cap;
  plan->max_pages = max_pages;
  plan->dst_cap = dst_cap;
  plan->frame_cap = frame_cap;
  plan->workspace_bytes = ap_layout(max_pages, dst_cap, frame_cap).total;
  return async_decode_setup<false>(dtype, [](auto tag) { return (const void*)ap_cold_kernel<decltype(tag)>; },
                                   {(const void*)ap_pages_kernel, (const void*)ap_scan_kernel, (const void*)ap_place_kernel, (const void*)frame_pages_kernel,
                                    (const void*)walk_kernel<SMALL_MAX_SIZE_LOG>, (const void*)ap_route_kernel, (const void*)ap_rewalk_kernel,
                                    (const void*)ap_finish_kernel});
}

// The pages front end of pco_b200_decompress_pages_async over the workspace `ws` laid out by `lay`: every page checked, placed, framed
// and walked, and routed, up to the re-walk of the lowest failing page (ap_pages ... ap_rewalk).  enqueue_pages runs it in front of the
// decode stage, pco_b200_pages_to_file_async in front of its writers.
static void enqueue_pages_front(const AsyncLaunch& ln, const ApArgs& g, const ApLayout& lay, uint8_t* ws) {
  const cudaStream_t stream = ln.stream;
  AsyncCheck* chk = reinterpret_cast<AsyncCheck*>(ws);
  ApState* state = reinterpret_cast<ApState*>(ws + lay.state);
  WrappedPage* tab = reinterpret_cast<WrappedPage*>(ws + lay.tab);
  uint8_t* d_idx = ws + lay.index;
  IndexChunk* recs = reinterpret_cast<IndexChunk*>(d_idx);
  uint8_t* d_frames = ws + lay.frames;
  uint32_t* pstat = reinterpret_cast<uint32_t*>(ws + lay.pstat);
  uint32_t* wst = reinterpret_cast<uint32_t*>(ws + lay.wst);
  uint64_t* ends = reinterpret_cast<uint64_t*>(ws + lay.ends);
  ApPart* parts = reinterpret_cast<ApPart*>(ws + lay.parts);
  IndexChunk* table = reinterpret_cast<IndexChunk*>(ws + lay.table);
  uint32_t* fast_page = reinterpret_cast<uint32_t*>(ws + lay.fast_page);
  uint32_t* cold_list = reinterpret_cast<uint32_t*>(ws + lay.cold_list);
  // the frames as one file: every page's frame below frame_cap, the pad frame behind them
  const FileParams fp{d_frames, lay.pad_frame + 64, g.dtype, 0, 4};
  const uint32_t mp = g.max_pages, pb = uint32_t(ctas_of<AP_THREADS>(mp));

  ln.begin("ap_pages_kernel");
  ap_pages_kernel<<<pb, AP_THREADS, 0, stream>>>(g, chk, parts);
  ln.end();
  ln.begin("ap_scan_kernel");
  ap_scan_kernel<<<1, AP_SCAN_THREADS, 0, stream>>>(g, parts, state);
  ln.end();
  ln.begin("ap_place_kernel");
  ap_place_kernel<<<pb, AP_THREADS, 0, stream>>>(g, parts, state, tab, recs, d_frames, lay.pad_frame, (uint64_t(mp) + 1) * sizeof(IndexChunk));
  ln.end();
  ln.begin("frame_pages_kernel");
  frame_pages_kernel<<<mp, WRAP_THREADS, 0, stream>>>(g.metas, g.metas_cap, g.pages, g.dtype, tab, d_frames, pstat);
  ln.end();
  ln.begin("walk_kernel");
  walk_kernel<SMALL_MAX_SIZE_LOG><<<mp, WALK_THREADS, sizeof(WalkSmem<SMALL_MAX_SIZE_LOG>), stream>>>(
      fp, d_idx, 0, mp, 0, lay.index_len, 0, 0, ~uint64_t(0), wst, &state->walk, 0, ends);
  ln.end();
  ln.begin("ap_route_kernel");
  ap_route_kernel<<<1, AP_SCAN_THREADS, 0, stream>>>(g, state, tab, recs, pstat, wst, ends, table, fast_page, cold_list, fp.src_len);
  ln.end();
  ln.begin("ap_rewalk_kernel");
  ap_rewalk_kernel<<<1, WALK_THREADS, sizeof(WalkSmem<SMALL_MAX_SIZE_LOG>), stream>>>(g, state, tab, d_frames, d_idx, lay.index_len);
  ln.end();
}

// The launches of pco_b200_decompress_pages_async over the workspace `ws` laid out by `lay`: the front end, the decode stage, the
// catch-all decoder into dst and ap_finish_kernel into *status.  With `filt` the decode stage runs its filter-mode instantiations and dst
// is their value staging (pco_b200_filter_pages_async).  With `agg` too, the aggregate-mode instantiations, which store nothing to dst;
// dst is the catch-all decoder's value staging only (pco_b200_aggregate_pages_async).  With `take` instead of `agg`, the take-mode
// instantiations, likewise (pco_b200_take_pages_async).  `between`, when given, enqueues its launches behind the front end
// (ap_rewalk_kernel) and before the decode stage.
static void enqueue_pages(const AsyncLaunch& ln, const ApArgs& g, const ApLayout& lay, uint8_t* ws, void* dst, const FiltStage* filt,
                          PcoB200AsyncPagesStatus* status, bool agg = false, bool take = false, const std::function<void()>& between = {}) {
  const cudaStream_t stream = ln.stream;
  AsyncCheck* chk = reinterpret_cast<AsyncCheck*>(ws);
  ApState* state = reinterpret_cast<ApState*>(ws + lay.state);
  WrappedPage* tab = reinterpret_cast<WrappedPage*>(ws + lay.tab);
  uint8_t* d_idx = ws + lay.index;
  IndexChunk* recs = reinterpret_cast<IndexChunk*>(d_idx);
  uint8_t* d_frames = ws + lay.frames;
  IndexChunk* table = reinterpret_cast<IndexChunk*>(ws + lay.table);
  uint32_t* fast_page = reinterpret_cast<uint32_t*>(ws + lay.fast_page);
  uint32_t* cold_list = reinterpret_cast<uint32_t*>(ws + lay.cold_list);
  uint32_t* d_st = reinterpret_cast<uint32_t*>(ws + lay.st);
  const FileParams fp{d_frames, lay.pad_frame + 64, g.dtype, 0, 4};
  const uint32_t mp = g.max_pages;

  enqueue_pages_front(ln, g, lay, ws);
  if (between) between();
  const DecodeStage d{fp, table, d_idx, lay.index_len, mp, d_st, ws + lay.cls, ws + lay.syms, reinterpret_cast<uint32_t*>(ws + lay.offs),
                      &chk->binoms, agg || take ? nullptr : dst, g.dst_cap, nullptr, filt ? *filt : FiltStage{}};
  if (agg) enqueue_decode_stage<false, true, true>(ln, d);
  else if (take) enqueue_decode_stage<false, true, false, true>(ln, d);
  else if (filt) enqueue_decode_stage<false, true>(ln, d);
  else enqueue_decode_stage<false>(ln, d);
  ln.begin("ap_cold_kernel");
  dispatch_latent(g.dtype, [&](auto tag) {
    using L = decltype(tag);
    ap_cold_kernel<L><<<1, ASYNC_THREADS, 0, stream>>>(g, state, tab, recs, d_st, fast_page, cold_list, d_frames, static_cast<L*>(dst), ws + lay.cold);
    return 0;
  });
  ln.end();
  ln.begin("ap_finish_kernel");
  ap_finish_kernel<<<1, 32, 0, stream>>>(state, status);
  ln.end();
}

PcoB200Error pco_b200_decompress_pages_async(const PcoB200AsyncPagesPlan* plan, const void* metas, const void* pages, const PcoB200PageRef* refs,
                                             const uint64_t* n_pages, void* dst, void* workspace, PcoB200AsyncPagesStatus* status, void* cuda_stream) {
  if (!plan || !metas || !pages || !refs || !n_pages || !workspace || !status || (!dst && plan->dst_cap))
    return fail(PCO_B200_INVALID_ARGUMENT, "null buffer");
  if (!ap_plan_ok(plan)) return fail(PCO_B200_INVALID_ARGUMENT, "the plan was not made by pco_b200_decompress_pages_async_plan");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail(PCO_B200_INVALID_ARGUMENT, "the workspace is not 256-byte aligned");
  AsyncLaunch ln;
  if (PcoB200Error e = open_async_launch(cuda_stream, &ln)) return e;

  const uint32_t mp = uint32_t(plan->max_pages);
  const ApLayout lay = ap_layout(mp, plan->dst_cap, plan->frame_cap);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  const ApArgs g{static_cast<const uint8_t*>(metas), static_cast<const uint8_t*>(pages), refs, n_pages, plan->metas_cap, plan->pages_cap, plan->dst_cap,
                 plan->frame_cap, plan->dtype, mp};
  enqueue_pages(ln, g, lay, ws, dst, nullptr, status);
  PCOB_CUDA_TRY(cudaGetLastError());
  return PCO_B200_OK;  // spans stay pending until pco_b200_profile_last reads them
}

PcoB200Error pco_b200_decompress_pages_async_result(const PcoB200AsyncPagesStatus* s, size_t* n_written) {
  if (!s) return fail(PCO_B200_INVALID_ARGUMENT, "null status");
  const PcoB200Error kind = async_result_kind(s->kind);
  if (kind == PCO_B200_OK) {
    if (n_written) *n_written = size_t(s->n_written);
    return PCO_B200_OK;
  }
  const size_t p = size_t(s->page);
  switch (s->device_status) {
    case PCO_B200_ASYNC_TOO_MANY_PAGES: return fail(kind, "*n_pages is " + std::to_string(s->n_pages) + ", above the plan's max_pages");
    case PCO_B200_ASYNC_META_OUTSIDE: return page_fail(kind, p, "chunk meta lies outside metas");
    case PCO_B200_ASYNC_PAGE_OUTSIDE: return page_fail(kind, p, "page lies outside pages");
    case PCO_B200_ASYNC_PAGE_N: return page_fail(kind, p, "page n must be 1..2^24");
    case PCO_B200_ASYNC_PAGES_DST: return page_fail(kind, p, "dst holds fewer numbers than the pages up to this one");
    case PCO_B200_ASYNC_FRAMES:
      return fail(kind, "the framed pages need " + std::to_string(s->frames_needed) + " bytes, more than the plan's frame_cap");
    default:
      status_to_error(s->device_status, "the page");
      return page_fail(kind, p, last_error_ref());
  }
}

// ---- asynchronous filter of wrapped pages (pco_b200_filter_pages_async; kernels in async_filter_kernels.cuh).  The pages call's launches
// (enqueue_pages, with the decode stage's filter-mode instantiations and rows_cap as dst_cap) behind a memset of the slot counts, then
// fl_cold, fl_count, fl_finish and fl_gather.

static bool fl_plan_ok(const PcoB200AsyncFilterPlan* p) {
  return nt_valid(p->dtype) && p->max_pages >= 1 && p->max_pages <= 0x7fffffffull && p->rows_cap <= (uint64_t(1) << 56) &&
         p->frame_cap <= (uint64_t(1) << 56) && p->out_cap <= (uint64_t(1) << 56) &&
         p->workspace_bytes == fl_layout(p->max_pages, p->rows_cap, p->frame_cap, nt_bits(p->dtype) / 8).fl_total;
}

PcoB200Error pco_b200_filter_pages_async_plan(unsigned char dtype, size_t metas_cap, size_t pages_cap, size_t max_pages, size_t rows_cap,
                                              size_t frame_cap, size_t out_cap, PcoB200AsyncFilterPlan* plan) {
  if (!nt_valid(dtype)) return fail(PCO_B200_INVALID_TYPE, "unknown number type byte: " + std::to_string(dtype));
  if (!plan) return fail(PCO_B200_INVALID_ARGUMENT, "null plan");
  if (max_pages == 0 || uint64_t(max_pages) > 0x7fffffffull) return fail(PCO_B200_INVALID_ARGUMENT, "max_pages must be 1 .. 2^31 - 1");
  if (uint64_t(rows_cap) > (uint64_t(1) << 56)) return fail(PCO_B200_INVALID_ARGUMENT, "rows_cap above 2^56 numbers");
  if (uint64_t(frame_cap) > (uint64_t(1) << 56)) return fail(PCO_B200_INVALID_ARGUMENT, "frame_cap above 2^56 bytes");
  if (uint64_t(out_cap) > (uint64_t(1) << 56)) return fail(PCO_B200_INVALID_ARGUMENT, "out_cap above 2^56 numbers");
  std::memset(plan, 0, sizeof(*plan));
  plan->dtype = dtype;
  plan->metas_cap = metas_cap;
  plan->pages_cap = pages_cap;
  plan->max_pages = max_pages;
  plan->rows_cap = rows_cap;
  plan->frame_cap = frame_cap;
  plan->out_cap = out_cap;
  plan->workspace_bytes = fl_layout(max_pages, rows_cap, frame_cap, nt_bits(dtype) / 8).fl_total;
  if (PcoB200Error e = async_decode_setup<false, true>(dtype, [](auto tag) { return (const void*)ap_cold_kernel<decltype(tag)>; },
                                                       {(const void*)ap_pages_kernel, (const void*)ap_scan_kernel, (const void*)ap_place_kernel,
                                                        (const void*)frame_pages_kernel, (const void*)walk_kernel<SMALL_MAX_SIZE_LOG>,
                                                        (const void*)ap_route_kernel, (const void*)ap_rewalk_kernel, (const void*)ap_finish_kernel,
                                                        (const void*)fl_count_kernel, (const void*)fl_finish_kernel}))
    return e;
  return dispatch_latent(dtype, [&](auto tag) -> PcoB200Error {
    using L = decltype(tag);
    return load_kernels({(const void*)fl_cold_kernel<L>, (const void*)fl_gather_kernel<L>});
  });
}

PcoB200Error pco_b200_filter_pages_async(const PcoB200AsyncFilterPlan* plan, const void* metas, const void* pages, const PcoB200PageRef* refs,
                                         const uint64_t* n_pages, const PcoB200Interval* interval, void* out_values, uint64_t* out_positions,
                                         uint64_t* n_matches, void* workspace, PcoB200AsyncFilterStatus* status, void* cuda_stream) {
  if (!plan || !metas || !pages || !refs || !n_pages || !interval || !n_matches || !workspace || !status ||
      ((!out_values || !out_positions) && plan->out_cap))
    return fail(PCO_B200_INVALID_ARGUMENT, "null buffer");
  if (!fl_plan_ok(plan)) return fail(PCO_B200_INVALID_ARGUMENT, "the plan was not made by pco_b200_filter_pages_async_plan");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail(PCO_B200_INVALID_ARGUMENT, "the workspace is not 256-byte aligned");
  AsyncLaunch ln;
  if (PcoB200Error e = open_async_launch(cuda_stream, &ln)) return e;
  const cudaStream_t stream = ln.stream;

  const uint32_t mp = uint32_t(plan->max_pages);
  const FlLayout lay = fl_layout(mp, plan->rows_cap, plan->frame_cap, nt_bits(plan->dtype) / 8);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  const uint64_t slots = fl_slots(mp, plan->rows_cap), n_parts = ctas_of<FL_THREADS>(slots);
  const ApArgs g{static_cast<const uint8_t*>(metas), static_cast<const uint8_t*>(pages), refs, n_pages, plan->metas_cap, plan->pages_cap, plan->rows_cap,
                 plan->frame_cap, plan->dtype, mp};
  const FiltStage filt{reinterpret_cast<const uint64_t*>(interval), reinterpret_cast<const uint32_t*>(ws + lay.fast_page),
                       reinterpret_cast<uint32_t*>(ws + lay.counts), reinterpret_cast<uint64_t*>(ws + lay.rows), ws + lay.soffs};
  auto* pstatus = reinterpret_cast<PcoB200AsyncPagesStatus*>(ws + lay.pstatus);
  auto* fstate = reinterpret_cast<FlState*>(ws + lay.fstate);
  auto* cparts = reinterpret_cast<uint64_t*>(ws + lay.cparts);

  PCOB_CUDA_TRY(cudaMemsetAsync(filt.counts, 0, slots * sizeof(uint32_t), stream));
  enqueue_pages(ln, g, lay, ws, ws + lay.stage, &filt, pstatus);
  dispatch_latent(plan->dtype, [&](auto tag) {
    using L = decltype(tag);
    ln.begin("fl_cold_kernel");
    fl_cold_kernel<L><<<mp, FL_THREADS, 0, stream>>>(reinterpret_cast<const ApState*>(ws + lay.state), reinterpret_cast<const IndexChunk*>(ws + lay.index),
                                                    reinterpret_cast<const uint32_t*>(ws + lay.cold_list), filt, plan->dtype,
                                                    reinterpret_cast<L*>(ws + lay.stage));
    ln.end();
    ln.begin("fl_count_kernel");
    fl_count_kernel<<<uint32_t(n_parts), FL_THREADS, 0, stream>>>(filt.counts, slots, cparts);
    ln.end();
    ln.begin("fl_finish_kernel");
    fl_finish_kernel<<<1, FL_SCAN_THREADS, 0, stream>>>(pstatus, cparts, n_parts, plan->out_cap, fstate, n_matches, status);
    ln.end();
    ln.begin("fl_gather_kernel");
    fl_gather_kernel<L><<<uint32_t(n_parts), FL_THREADS, 0, stream>>>(fstate, filt.counts, filt.rows, cparts, slots, reinterpret_cast<const L*>(ws + lay.stage),
                                                                     ws + lay.soffs, plan->out_cap, static_cast<L*>(out_values), out_positions);
    ln.end();
    return 0;
  });
  PCOB_CUDA_TRY(cudaGetLastError());
  return PCO_B200_OK;  // spans stay pending until pco_b200_profile_last reads them
}

PcoB200Error pco_b200_filter_pages_async_result(const PcoB200AsyncFilterStatus* s, size_t* n_matches) {
  if (!s) return fail(PCO_B200_INVALID_ARGUMENT, "null status");
  const PcoB200Error kind = async_result_kind(s->kind);
  if (kind == PCO_B200_OK) {
    if (n_matches) *n_matches = size_t(s->n_matches);
    return PCO_B200_OK;
  }
  switch (s->device_status) {
    case PCO_B200_FILTER_OUT_FULL:
      return fail(kind, "the pages hold " + std::to_string(s->matches_needed) + " matches, more than the plan's out_cap");
    case PCO_B200_ASYNC_PAGES_DST: return page_fail(kind, size_t(s->page), "the pages up to this one hold more numbers than rows_cap");
    default: {  // the pages call's outcome, in its words
      const PcoB200AsyncPagesStatus p{s->kind, s->device_status, s->page, s->n_written, s->n_pages, s->frames_needed};
      return pco_b200_decompress_pages_async_result(&p, nullptr);
    }
  }
}

// ---- asynchronous aggregates of wrapped pages and of indexed files (pco_b200_aggregate_pages_async, pco_b200_aggregate_files_async;
// kernels in async_aggregate_kernels.cuh).  A memset of the slot counts (and, for files, ff_map_kernel), then the decompress call's
// launches (enqueue_pages / enqueue_files with the decode stage's aggregate-mode instantiations and rows_cap as dst_cap), then the cold
// pass (fl_cold / ff_cold in aggregate mode), the group kernel over (groups, ag_split) CTAs, and the finish.  A second memset clears the
// groups' accumulators.

static bool ag_plan_ok(const PcoB200AsyncAggregatePlan* p) {
  return nt_valid(p->dtype) && p->max_pages >= 1 && p->max_pages <= 0x7fffffffull && p->rows_cap <= (uint64_t(1) << 56) &&
         p->frame_cap <= (uint64_t(1) << 56) && p->workspace_bytes == ag_layout(p->max_pages, p->rows_cap, p->frame_cap, nt_bits(p->dtype) / 8).ag_total;
}

PcoB200Error pco_b200_aggregate_pages_async_plan(unsigned char dtype, size_t metas_cap, size_t pages_cap, size_t max_pages, size_t rows_cap,
                                                 size_t frame_cap, PcoB200AsyncAggregatePlan* plan) {
  if (!nt_valid(dtype)) return fail(PCO_B200_INVALID_TYPE, "unknown number type byte: " + std::to_string(dtype));
  if (!plan) return fail(PCO_B200_INVALID_ARGUMENT, "null plan");
  if (max_pages == 0 || uint64_t(max_pages) > 0x7fffffffull) return fail(PCO_B200_INVALID_ARGUMENT, "max_pages must be 1 .. 2^31 - 1");
  if (uint64_t(rows_cap) > (uint64_t(1) << 56)) return fail(PCO_B200_INVALID_ARGUMENT, "rows_cap above 2^56 numbers");
  if (uint64_t(frame_cap) > (uint64_t(1) << 56)) return fail(PCO_B200_INVALID_ARGUMENT, "frame_cap above 2^56 bytes");
  std::memset(plan, 0, sizeof(*plan));
  plan->dtype = dtype;
  plan->metas_cap = metas_cap;
  plan->pages_cap = pages_cap;
  plan->max_pages = max_pages;
  plan->rows_cap = rows_cap;
  plan->frame_cap = frame_cap;
  plan->workspace_bytes = ag_layout(max_pages, rows_cap, frame_cap, nt_bits(dtype) / 8).ag_total;
  if (PcoB200Error e = async_decode_setup<false, true, true>(dtype, [](auto tag) { return (const void*)ap_cold_kernel<decltype(tag)>; },
                                                             {(const void*)ap_pages_kernel, (const void*)ap_scan_kernel, (const void*)ap_place_kernel,
                                                              (const void*)frame_pages_kernel, (const void*)walk_kernel<SMALL_MAX_SIZE_LOG>,
                                                              (const void*)ap_route_kernel, (const void*)ap_rewalk_kernel, (const void*)ap_finish_kernel}))
    return e;
  return dispatch_latent(dtype, [&](auto tag) -> PcoB200Error {
    using L = decltype(tag);
    return load_kernels({(const void*)fl_cold_kernel<L, true>, (const void*)ag_pages_kernel, (const void*)ag_finish_kernel<L>});
  });
}

PcoB200Error pco_b200_aggregate_pages_async(const PcoB200AsyncAggregatePlan* plan, const void* metas, const void* pages, const PcoB200PageRef* refs,
                                            const uint64_t* n_pages, const PcoB200Interval* interval, PcoB200Aggregate* aggs, PcoB200Aggregate* total,
                                            void* workspace, PcoB200AsyncAggregateStatus* status, void* cuda_stream) {
  if (!plan || !metas || !pages || !refs || !n_pages || !interval || !aggs || !total || !workspace || !status)
    return fail(PCO_B200_INVALID_ARGUMENT, "null buffer");
  if (!ag_plan_ok(plan)) return fail(PCO_B200_INVALID_ARGUMENT, "the plan was not made by pco_b200_aggregate_pages_async_plan");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail(PCO_B200_INVALID_ARGUMENT, "the workspace is not 256-byte aligned");
  AsyncLaunch ln;
  if (PcoB200Error e = open_async_launch(cuda_stream, &ln)) return e;
  const cudaStream_t stream = ln.stream;

  const uint32_t mp = uint32_t(plan->max_pages);
  const AgLayout lay = ag_layout(mp, plan->rows_cap, plan->frame_cap, nt_bits(plan->dtype) / 8);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  const uint64_t slots = fl_slots(mp, plan->rows_cap);
  const ApArgs g{static_cast<const uint8_t*>(metas), static_cast<const uint8_t*>(pages), refs, n_pages, plan->metas_cap, plan->pages_cap, plan->rows_cap,
                 plan->frame_cap, plan->dtype, mp};
  // aggregate mode: the AggSlot array travels in FiltStage's rows pointer (agg_slots)
  const FiltStage filt{reinterpret_cast<const uint64_t*>(interval), reinterpret_cast<const uint32_t*>(ws + lay.fast_page),
                       reinterpret_cast<uint32_t*>(ws + lay.counts), reinterpret_cast<uint64_t*>(ws + lay.aslots), nullptr};
  auto* groups = reinterpret_cast<AgGroup*>(ws + lay.groups);
  auto* pstatus = reinterpret_cast<PcoB200AsyncPagesStatus*>(ws + lay.pstatus);

  PCOB_CUDA_TRY(cudaMemsetAsync(filt.counts, 0, slots * sizeof(uint32_t), stream));
  PCOB_CUDA_TRY(cudaMemsetAsync(groups, 0, uint64_t(mp) * sizeof(AgGroup), stream));
  enqueue_pages(ln, g, lay, ws, ws + lay.stage, &filt, pstatus, true);
  dispatch_latent(plan->dtype, [&](auto tag) {
    using L = decltype(tag);
    ln.begin("fl_cold_kernel");
    fl_cold_kernel<L, true><<<mp, FL_THREADS, 0, stream>>>(reinterpret_cast<const ApState*>(ws + lay.state), reinterpret_cast<const IndexChunk*>(ws + lay.index),
                                                          reinterpret_cast<const uint32_t*>(ws + lay.cold_list), filt, plan->dtype,
                                                          reinterpret_cast<L*>(ws + lay.stage));
    ln.end();
    ln.begin("ag_pages_kernel");
    ag_pages_kernel<<<dim3(mp, ag_split(slots, mp)), AG_THREADS, 0, stream>>>(pstatus, reinterpret_cast<const IndexChunk*>(ws + lay.index), filt.counts,
                                                                            agg_slots(filt), plan->dtype, groups);
    ln.end();
    ln.begin("ag_finish_kernel");
    ag_finish_kernel<L><<<1, AG_THREADS, 0, stream>>>(pstatus, groups, reinterpret_cast<const IndexChunk*>(ws + lay.index), plan->dtype, aggs, total, status);
    ln.end();
    return 0;
  });
  PCOB_CUDA_TRY(cudaGetLastError());
  return PCO_B200_OK;  // spans stay pending until pco_b200_profile_last reads them
}

PcoB200Error pco_b200_aggregate_pages_async_result(const PcoB200AsyncAggregateStatus* s, size_t* n_matches) {
  if (!s) return fail(PCO_B200_INVALID_ARGUMENT, "null status");
  const PcoB200AsyncFilterStatus f{s->kind, s->device_status, s->page, s->n_written, s->n_pages, s->frames_needed, s->n_matches, s->n_matches};
  return pco_b200_filter_pages_async_result(&f, n_matches);  // the pages filter's words: rows_cap in the role of dst_cap
}

static bool agf_plan_ok(const PcoB200AsyncFilesAggregatePlan* p) {
  return nt_valid(p->dtype) && p->max_files >= 1 && p->max_files <= 0x7fffffffull && p->max_chunks >= 1 && p->max_chunks <= 0xffffffffull &&
         p->rows_cap <= (uint64_t(1) << 56) &&
         p->workspace_bytes == agf_layout(p->max_files, p->max_chunks, p->rows_cap, nt_bits(p->dtype) / 8).agf_total;
}

PcoB200Error pco_b200_aggregate_files_async_plan(const void* head, size_t head_len, unsigned char dtype, size_t src_cap, size_t index_cap,
                                                 size_t max_files, size_t max_chunks, size_t rows_cap, PcoB200AsyncFilesAggregatePlan* plan) {
  StandaloneHeader hdr;
  if (PcoB200Error e = check_async_head(head, head_len, dtype, plan, &hdr)) return e;
  if (max_files == 0 || uint64_t(max_files) > 0x7fffffffull) return fail(PCO_B200_INVALID_ARGUMENT, "max_files must be 1 .. 2^31 - 1");
  if (max_chunks == 0 || uint64_t(max_chunks) > 0xffffffffull) return fail(PCO_B200_INVALID_ARGUMENT, "max_chunks must be 1 .. 2^32 - 1");
  if (uint64_t(rows_cap) > (uint64_t(1) << 56)) return fail(PCO_B200_INVALID_ARGUMENT, "rows_cap above 2^56 numbers");
  std::memset(plan, 0, sizeof(*plan));
  plan->dtype = dtype;
  plan->uniform_type = hdr.uniform_type;
  plan->format_major = hdr.format_major;
  plan->src_cap = src_cap;
  plan->index_cap = index_cap;
  plan->max_files = max_files;
  plan->max_chunks = max_chunks;
  plan->rows_cap = rows_cap;
  plan->workspace_bytes = agf_layout(max_files, max_chunks, rows_cap, nt_bits(dtype) / 8).agf_total;
  if (PcoB200Error e = async_decode_setup<false, true, true>(dtype, [](auto tag) { return (const void*)cold_chunks_kernel<decltype(tag)>; },
                                                             {(const void*)af_files_kernel, (const void*)check_index_kernel, (const void*)af_scan_kernel,
                                                              (const void*)af_place_kernel, (const void*)af_table_kernel, (const void*)merge_index_kernel,
                                                              (const void*)af_finish_kernel, (const void*)ff_map_kernel, (const void*)ff_cold_list_kernel}))
    return e;
  return dispatch_latent(dtype, [&](auto tag) -> PcoB200Error {
    using L = decltype(tag);
    return load_kernels({(const void*)ff_cold_kernel<L, true>, (const void*)ag_files_kernel, (const void*)agf_finish_kernel<L>});
  });
}

PcoB200Error pco_b200_aggregate_files_async(const PcoB200AsyncFilesAggregatePlan* plan, const void* src, const void* index, const PcoB200FileRef* files,
                                            const uint64_t* n_files, const PcoB200Interval* interval, PcoB200Aggregate* aggs, PcoB200Aggregate* total,
                                            void* workspace, PcoB200AsyncFilesAggregateStatus* status, void* cuda_stream) {
  if (!plan || !src || !index || !files || !n_files || !interval || !aggs || !total || !workspace || !status)
    return fail(PCO_B200_INVALID_ARGUMENT, "null buffer");
  if (!agf_plan_ok(plan)) return fail(PCO_B200_INVALID_ARGUMENT, "the plan was not made by pco_b200_aggregate_files_async_plan");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail(PCO_B200_INVALID_ARGUMENT, "the workspace is not 256-byte aligned");
  AsyncLaunch ln;
  if (PcoB200Error e = open_async_launch(cuda_stream, &ln)) return e;
  const cudaStream_t stream = ln.stream;

  const uint32_t mf = uint32_t(plan->max_files), mc = uint32_t(plan->max_chunks);
  const AgfLayout lay = agf_layout(mf, mc, plan->rows_cap, nt_bits(plan->dtype) / 8);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  const uint64_t slots = fl_slots(mc, plan->rows_cap);
  const AfArgs g{FileParams{src, plan->src_cap, plan->dtype, plan->uniform_type, plan->format_major}, static_cast<const uint8_t*>(index),
                 plan->index_cap, plan->rows_cap, files, n_files, mf, mc};
  // aggregate mode: the AggSlot array travels in FiltStage's rows pointer (agg_slots)
  const FiltStage filt{reinterpret_cast<const uint64_t*>(interval), reinterpret_cast<const uint32_t*>(ws + lay.slot_map),
                       reinterpret_cast<uint32_t*>(ws + lay.counts), reinterpret_cast<uint64_t*>(ws + lay.aslots), nullptr};
  auto* groups = reinterpret_cast<AgGroup*>(ws + lay.groups);
  auto* fstatus = reinterpret_cast<PcoB200AsyncFilesStatus*>(ws + lay.fstatus);
  auto* cold_list = reinterpret_cast<uint32_t*>(ws + lay.cold_list);

  PCOB_CUDA_TRY(cudaMemsetAsync(filt.counts, 0, slots * sizeof(uint32_t), stream));
  PCOB_CUDA_TRY(cudaMemsetAsync(groups, 0, uint64_t(mf) * sizeof(AgGroup), stream));
  ln.begin("ff_map_kernel");
  ff_map_kernel<<<uint32_t(ctas_of<FF_THREADS>(mc)), FF_THREADS, 0, stream>>>(mc, reinterpret_cast<uint32_t*>(ws + lay.slot_map), cold_list);
  ln.end();
  enqueue_files(ln, g, lay, ws, ws + lay.stage, &filt, cold_list, nullptr, fstatus, true);
  dispatch_latent(plan->dtype, [&](auto tag) {
    using L = decltype(tag);
    ln.begin("ff_cold_kernel");
    ff_cold_kernel<L, true><<<std::min(mc, uint32_t(FF_COLD_CTAS)), FL_THREADS, 0, stream>>>(cold_list, reinterpret_cast<const IndexChunk*>(ws + lay.table),
                                                                                             filt, plan->dtype, reinterpret_cast<L*>(ws + lay.stage));
    ln.end();
    ln.begin("ag_files_kernel");
    ag_files_kernel<<<dim3(mf, ag_split(slots, mf)), AG_THREADS, 0, stream>>>(fstatus, reinterpret_cast<const FileMerge*>(ws + lay.merges),
                                                                            reinterpret_cast<const IndexChunk*>(ws + lay.table), filt.counts,
                                                                            agg_slots(filt), plan->dtype, groups);
    ln.end();
    ln.begin("agf_finish_kernel");
    agf_finish_kernel<L><<<1, AG_THREADS, 0, stream>>>(fstatus, groups, reinterpret_cast<const FileCheck*>(ws + lay.fchk), plan->dtype, aggs, total, status);
    ln.end();
    return 0;
  });
  PCOB_CUDA_TRY(cudaGetLastError());
  return PCO_B200_OK;  // spans stay pending until pco_b200_profile_last reads them
}

PcoB200Error pco_b200_aggregate_files_async_result(const PcoB200AsyncFilesAggregateStatus* s, size_t* n_matches) {
  if (!s) return fail(PCO_B200_INVALID_ARGUMENT, "null status");
  const PcoB200AsyncFilesFilterStatus f{s->kind, s->device_status, s->file, s->chunk, s->n_written, s->n_files, s->n_matches, s->n_matches};
  return pco_b200_filter_files_async_result(&f, n_matches);  // the files filter's words: rows_cap in the role of dst_cap
}

// ---- asynchronous take from wrapped pages and from indexed files (pco_b200_take_pages_async, pco_b200_take_files_async; kernels in
// async_take_kernels.cuh).  The decompress call's launches (enqueue_pages / enqueue_files with the decode stage's take-mode instantiations
// and rows_cap as dst_cap; for files behind ff_map_kernel) with the take's plan between the front end and the decode stage: the front
// kernel, the position checks, the marks (and, for pages, the cold list kept to the touched pages); then the cold take and the finish.

// The take's plan, enqueued between the front end and the decode stage; `front` writes the TkState.
static void enqueue_take_plan(const AsyncLaunch& ln, const std::function<void()>& front, const uint64_t* positions, uint64_t max_positions,
                              const IndexChunk* recs, uint64_t max_records, TkState* ts, uint32_t* touched, TakeRun* runs) {
  const cudaStream_t stream = ln.stream;
  front();
  ln.begin("tk_check_kernel");
  tk_check_kernel<<<uint32_t(std::min(ctas_of<TK_THREADS>(max_positions), TK_MAX_CTAS)), TK_THREADS, 0, stream>>>(positions, max_positions, ts);
  ln.end();
  ln.begin("tk_mark_kernel");
  tk_mark_kernel<<<uint32_t(std::min(max_records, TK_MAX_CTAS)), TK_THREADS, 0, stream>>>(positions, max_positions, recs, ts, touched, runs);
  ln.end();
}

static bool tk_plan_ok(const PcoB200AsyncTakePlan* p) {
  return nt_valid(p->dtype) && p->max_pages >= 1 && p->max_pages <= 0x7fffffffull && p->rows_cap <= (uint64_t(1) << 56) &&
         p->frame_cap <= (uint64_t(1) << 56) && p->max_positions >= 1 && p->max_positions <= (uint64_t(1) << 56) &&
         p->workspace_bytes == tk_layout(p->max_pages, p->rows_cap, p->frame_cap, nt_bits(p->dtype) / 8).tk_total;
}

PcoB200Error pco_b200_take_pages_async_plan(unsigned char dtype, size_t metas_cap, size_t pages_cap, size_t max_pages, size_t rows_cap,
                                            size_t frame_cap, size_t max_positions, PcoB200AsyncTakePlan* plan) {
  if (!nt_valid(dtype)) return fail(PCO_B200_INVALID_TYPE, "unknown number type byte: " + std::to_string(dtype));
  if (!plan) return fail(PCO_B200_INVALID_ARGUMENT, "null plan");
  if (max_pages == 0 || uint64_t(max_pages) > 0x7fffffffull) return fail(PCO_B200_INVALID_ARGUMENT, "max_pages must be 1 .. 2^31 - 1");
  if (uint64_t(rows_cap) > (uint64_t(1) << 56)) return fail(PCO_B200_INVALID_ARGUMENT, "rows_cap above 2^56 numbers");
  if (uint64_t(frame_cap) > (uint64_t(1) << 56)) return fail(PCO_B200_INVALID_ARGUMENT, "frame_cap above 2^56 bytes");
  if (max_positions == 0 || uint64_t(max_positions) > (uint64_t(1) << 56)) return fail(PCO_B200_INVALID_ARGUMENT, "max_positions must be 1 .. 2^56");
  std::memset(plan, 0, sizeof(*plan));
  plan->dtype = dtype;
  plan->metas_cap = metas_cap;
  plan->pages_cap = pages_cap;
  plan->max_pages = max_pages;
  plan->rows_cap = rows_cap;
  plan->frame_cap = frame_cap;
  plan->max_positions = max_positions;
  plan->workspace_bytes = tk_layout(max_pages, rows_cap, frame_cap, nt_bits(dtype) / 8).tk_total;
  if (PcoB200Error e = async_decode_setup<false, true, false, true>(
          dtype, [](auto tag) { return (const void*)ap_cold_kernel<decltype(tag)>; },
          {(const void*)ap_pages_kernel, (const void*)ap_scan_kernel, (const void*)ap_place_kernel, (const void*)frame_pages_kernel,
           (const void*)walk_kernel<SMALL_MAX_SIZE_LOG>, (const void*)ap_route_kernel, (const void*)ap_rewalk_kernel, (const void*)ap_finish_kernel,
           (const void*)tk_front_pages_kernel, (const void*)tk_check_kernel, (const void*)tk_mark_kernel, (const void*)tk_cold_list_kernel,
           (const void*)tk_finish_pages_kernel}))
    return e;
  return dispatch_latent(dtype, [&](auto tag) -> PcoB200Error { return load_kernels({(const void*)tk_cold_pages_kernel<decltype(tag)>}); });
}

PcoB200Error pco_b200_take_pages_async(const PcoB200AsyncTakePlan* plan, const void* metas, const void* pages, const PcoB200PageRef* refs,
                                       const uint64_t* n_pages, const uint64_t* positions, const uint64_t* n_positions, void* out_values,
                                       void* workspace, PcoB200AsyncTakeStatus* status, void* cuda_stream) {
  if (!plan || !metas || !pages || !refs || !n_pages || !positions || !n_positions || !out_values || !workspace || !status)
    return fail(PCO_B200_INVALID_ARGUMENT, "null buffer");
  if (!tk_plan_ok(plan)) return fail(PCO_B200_INVALID_ARGUMENT, "the plan was not made by pco_b200_take_pages_async_plan");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail(PCO_B200_INVALID_ARGUMENT, "the workspace is not 256-byte aligned");
  AsyncLaunch ln;
  if (PcoB200Error e = open_async_launch(cuda_stream, &ln)) return e;
  const cudaStream_t stream = ln.stream;

  const uint32_t mp = uint32_t(plan->max_pages);
  const TkLayout lay = tk_layout(mp, plan->rows_cap, plan->frame_cap, nt_bits(plan->dtype) / 8);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  const ApArgs g{static_cast<const uint8_t*>(metas), static_cast<const uint8_t*>(pages), refs, n_pages, plan->metas_cap, plan->pages_cap, plan->rows_cap,
                 plan->frame_cap, plan->dtype, mp};
  // take mode: the positions travel in FiltStage's interval pointer, the touched flags in counts, the runs in rows, out_values in offs
  const FiltStage filt{positions, reinterpret_cast<const uint32_t*>(ws + lay.fast_page), reinterpret_cast<uint32_t*>(ws + lay.touched),
                       reinterpret_cast<uint64_t*>(ws + lay.runs), static_cast<uint8_t*>(out_values)};
  auto* state = reinterpret_cast<ApState*>(ws + lay.state);
  auto* recs = reinterpret_cast<const IndexChunk*>(ws + lay.index);
  auto* cold_list = reinterpret_cast<uint32_t*>(ws + lay.cold_list);
  auto* pstatus = reinterpret_cast<PcoB200AsyncPagesStatus*>(ws + lay.pstatus);
  auto* ts = reinterpret_cast<TkState*>(ws + lay.tstate);

  enqueue_pages(ln, g, lay, ws, ws + lay.stage, &filt, pstatus, false, true, [&] {
    auto front = [&] {
      ln.begin("tk_front_pages_kernel");
      tk_front_pages_kernel<<<1, 32, 0, stream>>>(state, n_positions, ts);
      ln.end();
    };
    enqueue_take_plan(ln, front, positions, plan->max_positions, recs, mp, ts, filt.counts, take_runs(filt));
    ln.begin("tk_cold_list_kernel");
    tk_cold_list_kernel<<<1, TK_SCAN_THREADS, 0, stream>>>(state, cold_list, filt.counts);
    ln.end();
  });
  dispatch_latent(plan->dtype, [&](auto tag) {
    using L = decltype(tag);
    ln.begin("tk_cold_pages_kernel");
    tk_cold_pages_kernel<L><<<mp, TK_THREADS, 0, stream>>>(state, recs, cold_list, filt, reinterpret_cast<const L*>(ws + lay.stage));
    ln.end();
    return 0;
  });
  ln.begin("tk_finish_pages_kernel");
  tk_finish_pages_kernel<<<1, 32, 0, stream>>>(pstatus, ts, plan->max_positions, status);
  ln.end();
  PCOB_CUDA_TRY(cudaGetLastError());
  return PCO_B200_OK;  // spans stay pending until pco_b200_profile_last reads them
}

// The words of the take's own refusals of a position, or nullptr for any other status.
static const char* tk_refusal(uint32_t device_status) {
  switch (device_status) {
    case PCO_B200_TAKE_ORDER: return "not above the position before it (positions must be strictly ascending)";
    case PCO_B200_TAKE_PAST: return "lies at or past the rows of the concatenation";
    default: return nullptr;
  }
}
static PcoB200Error tk_result(PcoB200Error kind, uint32_t device_status, uint64_t n_positions, uint64_t position, uint64_t rows) {
  if (device_status == PCO_B200_TAKE_TOO_MANY)
    return fail(kind, "*n_positions is " + std::to_string(n_positions) + ", above the plan's max_positions");
  std::string what = "position " + std::to_string(position) + ": " + tk_refusal(device_status);
  if (device_status == PCO_B200_TAKE_PAST) what += " (" + std::to_string(rows) + " rows)";
  return fail(kind, what);
}

PcoB200Error pco_b200_take_pages_async_result(const PcoB200AsyncTakeStatus* s, size_t* n_written) {
  if (!s) return fail(PCO_B200_INVALID_ARGUMENT, "null status");
  const PcoB200Error kind = async_result_kind(s->kind);
  if (kind == PCO_B200_OK) {
    if (n_written) *n_written = size_t(s->n_positions);
    return PCO_B200_OK;
  }
  if (s->device_status == PCO_B200_TAKE_TOO_MANY || tk_refusal(s->device_status))
    return tk_result(kind, s->device_status, s->n_positions, s->position, s->n_written);
  const PcoB200AsyncFilterStatus f{s->kind, s->device_status, s->page, s->n_written, s->n_pages, s->frames_needed, 0, 0};
  return pco_b200_filter_pages_async_result(&f, nullptr);  // the pages filter's words: rows_cap in the role of dst_cap
}

static bool tkf_plan_ok(const PcoB200AsyncFilesTakePlan* p) {
  return nt_valid(p->dtype) && p->max_files >= 1 && p->max_files <= 0x7fffffffull && p->max_chunks >= 1 && p->max_chunks <= 0xffffffffull &&
         p->rows_cap <= (uint64_t(1) << 56) && p->max_positions >= 1 && p->max_positions <= (uint64_t(1) << 56) &&
         p->workspace_bytes == tkf_layout(p->max_files, p->max_chunks, p->rows_cap, nt_bits(p->dtype) / 8).tkf_total;
}

PcoB200Error pco_b200_take_files_async_plan(const void* head, size_t head_len, unsigned char dtype, size_t src_cap, size_t index_cap,
                                            size_t max_files, size_t max_chunks, size_t rows_cap, size_t max_positions, PcoB200AsyncFilesTakePlan* plan) {
  StandaloneHeader hdr;
  if (PcoB200Error e = check_async_head(head, head_len, dtype, plan, &hdr)) return e;
  if (max_files == 0 || uint64_t(max_files) > 0x7fffffffull) return fail(PCO_B200_INVALID_ARGUMENT, "max_files must be 1 .. 2^31 - 1");
  if (max_chunks == 0 || uint64_t(max_chunks) > 0xffffffffull) return fail(PCO_B200_INVALID_ARGUMENT, "max_chunks must be 1 .. 2^32 - 1");
  if (uint64_t(rows_cap) > (uint64_t(1) << 56)) return fail(PCO_B200_INVALID_ARGUMENT, "rows_cap above 2^56 numbers");
  if (max_positions == 0 || uint64_t(max_positions) > (uint64_t(1) << 56)) return fail(PCO_B200_INVALID_ARGUMENT, "max_positions must be 1 .. 2^56");
  std::memset(plan, 0, sizeof(*plan));
  plan->dtype = dtype;
  plan->uniform_type = hdr.uniform_type;
  plan->format_major = hdr.format_major;
  plan->src_cap = src_cap;
  plan->index_cap = index_cap;
  plan->max_files = max_files;
  plan->max_chunks = max_chunks;
  plan->rows_cap = rows_cap;
  plan->max_positions = max_positions;
  plan->workspace_bytes = tkf_layout(max_files, max_chunks, rows_cap, nt_bits(dtype) / 8).tkf_total;
  if (PcoB200Error e = async_decode_setup<false, true, false, true>(
          dtype, [](auto tag) { return (const void*)cold_chunks_kernel<decltype(tag)>; },
          {(const void*)af_files_kernel, (const void*)check_index_kernel, (const void*)af_scan_kernel, (const void*)af_place_kernel,
           (const void*)af_table_kernel, (const void*)merge_index_kernel, (const void*)af_finish_kernel, (const void*)ff_map_kernel,
           (const void*)ff_cold_list_kernel, (const void*)tk_front_files_kernel, (const void*)tk_check_kernel, (const void*)tk_mark_kernel,
           (const void*)tk_finish_files_kernel}))
    return e;
  return dispatch_latent(dtype, [&](auto tag) -> PcoB200Error { return load_kernels({(const void*)tk_cold_files_kernel<decltype(tag)>}); });
}

PcoB200Error pco_b200_take_files_async(const PcoB200AsyncFilesTakePlan* plan, const void* src, const void* index, const PcoB200FileRef* files,
                                       const uint64_t* n_files, const uint64_t* positions, const uint64_t* n_positions, void* out_values,
                                       uint64_t* file_ns, void* workspace, PcoB200AsyncFilesTakeStatus* status, void* cuda_stream) {
  if (!plan || !src || !index || !files || !n_files || !positions || !n_positions || !out_values || !workspace || !status)
    return fail(PCO_B200_INVALID_ARGUMENT, "null buffer");
  if (!tkf_plan_ok(plan)) return fail(PCO_B200_INVALID_ARGUMENT, "the plan was not made by pco_b200_take_files_async_plan");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail(PCO_B200_INVALID_ARGUMENT, "the workspace is not 256-byte aligned");
  AsyncLaunch ln;
  if (PcoB200Error e = open_async_launch(cuda_stream, &ln)) return e;
  const cudaStream_t stream = ln.stream;

  const uint32_t mf = uint32_t(plan->max_files), mc = uint32_t(plan->max_chunks);
  const TkfLayout lay = tkf_layout(mf, mc, plan->rows_cap, nt_bits(plan->dtype) / 8);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  const AfArgs g{FileParams{src, plan->src_cap, plan->dtype, plan->uniform_type, plan->format_major}, static_cast<const uint8_t*>(index),
                 plan->index_cap, plan->rows_cap, files, n_files, mf, mc};
  // take mode: the positions travel in FiltStage's interval pointer, the touched flags in counts, the runs in rows, out_values in offs
  const FiltStage filt{positions, reinterpret_cast<const uint32_t*>(ws + lay.slot_map), reinterpret_cast<uint32_t*>(ws + lay.touched),
                       reinterpret_cast<uint64_t*>(ws + lay.runs), static_cast<uint8_t*>(out_values)};
  auto* fstatus = reinterpret_cast<PcoB200AsyncFilesStatus*>(ws + lay.fstatus);
  auto* ts = reinterpret_cast<TkState*>(ws + lay.tstate);
  auto* cold_list = reinterpret_cast<uint32_t*>(ws + lay.cold_list);
  auto* table = reinterpret_cast<const IndexChunk*>(ws + lay.table);
  auto* afstate = reinterpret_cast<const AfState*>(ws + lay.state);

  ln.begin("ff_map_kernel");
  ff_map_kernel<<<uint32_t(ctas_of<FF_THREADS>(mc)), FF_THREADS, 0, stream>>>(mc, reinterpret_cast<uint32_t*>(ws + lay.slot_map), cold_list);
  ln.end();
  // file_ns: tk_finish_files_kernel writes it, only when the take succeeds
  enqueue_files(ln, g, lay, ws, ws + lay.stage, &filt, cold_list, nullptr, fstatus, false, true, [&] {
    auto front = [&] {
      ln.begin("tk_front_files_kernel");
      tk_front_files_kernel<<<1, 32, 0, stream>>>(afstate, reinterpret_cast<const AsyncCheck*>(ws), n_positions, ts);
      ln.end();
    };
    enqueue_take_plan(ln, front, positions, plan->max_positions, table, mc, ts, filt.counts, take_runs(filt));
  });
  dispatch_latent(plan->dtype, [&](auto tag) {
    using L = decltype(tag);
    ln.begin("tk_cold_files_kernel");
    tk_cold_files_kernel<L><<<std::min(mc, uint32_t(FF_COLD_CTAS)), TK_THREADS, 0, stream>>>(cold_list, table, reinterpret_cast<const uint32_t*>(ws + lay.st),
                                                                                             filt, reinterpret_cast<const L*>(ws + lay.stage));
    ln.end();
    return 0;
  });
  ln.begin("tk_finish_files_kernel");
  tk_finish_files_kernel<<<1, TK_SCAN_THREADS, 0, stream>>>(fstatus, ts, afstate, reinterpret_cast<const FileCheck*>(ws + lay.fchk), plan->max_positions,
                                                            file_ns, status);
  ln.end();
  PCOB_CUDA_TRY(cudaGetLastError());
  return PCO_B200_OK;  // spans stay pending until pco_b200_profile_last reads them
}

PcoB200Error pco_b200_take_files_async_result(const PcoB200AsyncFilesTakeStatus* s, size_t* n_written) {
  if (!s) return fail(PCO_B200_INVALID_ARGUMENT, "null status");
  const PcoB200Error kind = async_result_kind(s->kind);
  if (kind == PCO_B200_OK) {
    if (n_written) *n_written = size_t(s->n_positions);
    return PCO_B200_OK;
  }
  if (s->device_status == PCO_B200_TAKE_TOO_MANY || tk_refusal(s->device_status))
    return tk_result(kind, s->device_status, s->n_positions, s->position, s->n_written);
  const PcoB200AsyncFilesFilterStatus f{s->kind, s->device_status, s->file, s->chunk, s->n_written, s->n_files, 0, 0};
  return pco_b200_filter_files_async_result(&f, nullptr);  // the files filter's words: rows_cap in the role of dst_cap
}

// ---- asynchronous compress (pco_b200_compress_async; gate kernels in async_compress.cuh).  The plan fixes the layout and the config;
// the call is a fixed sequence of launches: init, the encode stage (enqueue_encode_kernels: [split_count], two-kernel gate, split_delta,
// range gate, per var (counting probe, sort keys, segment offsets, radix sort, sorted probe, solve), fallback, per var (bin_lut, bin),
// ans, layout), chunk offsets, pack gate, one pack per choice of keys (enqueue_pack), header, [index], finish.  n == 0 is init and
// finish only.

PcoB200Error pco_b200_compress_async_plan(size_t n, unsigned char dtype, const PcoB200ChunkConfig* config, int uniform_type_header, size_t dst_cap,
                                          size_t index_cap, PcoB200AsyncCompressPlan* plan) {
  if (!nt_valid(dtype)) return fail(PCO_B200_INVALID_TYPE, "unknown number type byte: " + std::to_string(dtype));
  if (!plan) return fail(PCO_B200_INVALID_ARGUMENT, "null plan");
  const PcoB200ChunkConfig cfg = default_chunk_config(config);
  ConfigCheck ck;
  if (PcoB200Error e = check_config(cfg, dtype, n, &ck)) return e;
  if (ck.auto_mode || ck.auto_delta)
    return fail(PCO_B200_UNSUPPORTED, "ModeSpec::Auto and DeltaSpec::Auto search on host threads: the asynchronous compress takes explicit specs only");
  if (cfg.paging_spec == PCO_B200_PAGING_EXACT) return fail(PCO_B200_UNSUPPORTED, "PagingSpec::Exact: the asynchronous compress takes EqualPagesUpTo only");
  const AcompGeom g = acomp_geom(n, cfg.max_page_n);
  uint32_t bins_log = 0;
  if (n > 0) {
    bins_log = unoptimized_bins_log(cfg.compression_level, g.max_n, 0);
    if (bins_log > ENC_NARROW_BINS_LOG)
      return fail(PCO_B200_UNSUPPORTED, "more than 256 unoptimized bins (levels 9-12): the asynchronous compress runs the narrow kernels only");
    if (g.rem != 0 && g.low > 0 && unoptimized_bins_log(cfg.compression_level, g.low, 0) != bins_log)
      return fail(PCO_B200_UNSUPPORTED, "the chunk sizes imply different unoptimized_bins_log (compress_ex encodes them in several runs)");
  }
  std::memset(plan, 0, sizeof(*plan));
  plan->dtype = dtype;
  plan->uniform_type_header = uniform_type_header ? 1 : 0;
  fill_explicit_spec(plan, ck);
  plan->bins_log = bins_log;
  plan->n = n;
  plan->max_page_n = cfg.max_page_n;
  plan->dst_cap = dst_cap;
  plan->index_cap = index_cap;
  plan->index_bytes = equal_pages(n, cfg.max_page_n).index_bytes(plan->n_vars);
  plan->workspace_bytes = acomp_layout(g, nt_bits(dtype) / 8, plan->n_vars).total;
  if (index_cap != 0 && index_cap < plan->index_bytes)
    return fail(PCO_B200_IO, "index buffer too small (need " + std::to_string(plan->index_bytes) + " bytes)");
  return async_encode_setup<false>(dtype, {(const void*)acomp_init_kernel, (const void*)acomp_finish_kernel, (const void*)chunk_offsets_kernel,
                                           (const void*)header_footer_kernel, (const void*)emit_index_kernel});
}

PcoB200Error pco_b200_compress_async(const PcoB200AsyncCompressPlan* plan, const void* nums, void* dst, void* index, void* workspace,
                                     PcoB200AsyncCompressStatus* status, void* cuda_stream) {
  if (!plan || !workspace || !status || (!nums && plan->n) || (!dst && plan->dst_cap)) return fail(PCO_B200_INVALID_ARGUMENT, "null buffer");
  AcompGeom g;
  AcompArgs a;
  std::memset(&a, 0, sizeof(a));
  if (PcoB200Error e = acomp_check_plan(plan, &g, &a.lay)) return e;
  if (index && plan->index_cap == 0) return fail(PCO_B200_INVALID_ARGUMENT, "an index with a plan made without one (index_cap 0)");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail(PCO_B200_INVALID_ARGUMENT, "the workspace is not 256-byte aligned");
  if (reinterpret_cast<uintptr_t>(index) & 15) return fail(PCO_B200_INVALID_ARGUMENT, "the index is not 16-byte aligned");
  AsyncLaunch ln;
  if (PcoB200Error e = open_async_launch(cuda_stream, &ln)) return e;
  a.n = plan->n;
  a.n_chunks = g.n_chunks;
  a.low = g.low;
  a.rem = g.rem;
  a.dst_cap = plan->dst_cap;
  a.index_bytes = index ? plan->index_bytes : 0;
  a.n_vars = plan->n_vars;
  a.ws = static_cast<uint8_t*>(workspace);
  a.dst = static_cast<uint8_t*>(dst);
  a.index = static_cast<uint8_t*>(index);
  a.header_bytes = standalone_header_into(plan->n, uint8_t(plan->uniform_type_header ? plan->dtype : 0), a.header);
  dispatch_latent(plan->dtype, [&](auto tag) {
    acomp_launch<decltype(tag)>(*plan, g, a, nums, status, ln);
    return 0;
  });
  PCOB_CUDA_TRY(cudaGetLastError());
  return PCO_B200_OK;  // spans stay pending until pco_b200_profile_last reads them
}

PcoB200Error pco_b200_compress_async_result(const PcoB200AsyncCompressStatus* s, size_t* n_written, size_t* index_len) {
  if (!s) return fail(PCO_B200_INVALID_ARGUMENT, "null status");
  const PcoB200Error kind = async_result_kind(s->kind);
  if (kind == PCO_B200_OK) {
    if (n_written) *n_written = size_t(s->n_written);
    if (index_len) *index_len = size_t(s->index_bytes);
    return PCO_B200_OK;
  }
  if (s->device_status == PCO_B200_ASYNC_DST_FULL)
    return fail(kind, "failed to write whole buffer (need " + std::to_string(s->file_bytes) + " bytes)");
  return fail(kind, "asynchronous compress failed (device status " + std::to_string(s->device_status) + ")");
}

// ---- asynchronous batch compress (pco_b200_compress_files_async; kernels in async_compress_files.cuh).  The plan fixes the config and the
// grids from the capacities; the call is a fixed sequence of launches: files, scan, place, init, the encode stage of
// pco_b200_compress_async (enqueue_encode_kernels, with split_count and the planner kernels in their CHUNK_BINS instantiations), bytes,
// bytes scan, offsets, pack gate, one pack per choice of keys (enqueue_pack), frame, [index], finish.

// The refusals of the asynchronous batch compress plans, in their order, with `item` naming what the batch holds ("file" or "array"):
// the capacities, PagingSpec::Exact, the config, Auto specs, more than 256 unoptimized bins at the largest chunk, the CTA limit.  Fills
// the config, its check and the chunk slots.
static PcoB200Error acf_plan_checks(unsigned char dtype, const PcoB200ChunkConfig* config, size_t max_items, size_t nums_cap, size_t max_item_n,
                                    const std::string& item, PcoB200ChunkConfig* cfg_out, ConfigCheck* ck_out, uint64_t* max_chunks_out) {
  const PcoB200ChunkConfig cfg = default_chunk_config(config);
  if (max_items == 0 || max_items > 0x7fffffffu) return fail(PCO_B200_INVALID_ARGUMENT, "max_" + item + "s must be in 1 .. 2^31 - 1");
  if (max_item_n == 0) return fail(PCO_B200_INVALID_ARGUMENT, "max_" + item + "_n must be at least 1");
  if (uint64_t(nums_cap) > (uint64_t(1) << 56)) return fail(PCO_B200_INVALID_ARGUMENT, "nums_cap must be at most 2^56");
  // the config as compress_async_plan checks it, at the largest chunk (a file of min(max_page_n, max_file_n, nums_cap) numbers is one chunk)
  // (Exact paging first: its page sizes are checked against a count, and a batch has none)
  if (cfg.paging_spec == PCO_B200_PAGING_EXACT) return fail(PCO_B200_UNSUPPORTED, "PagingSpec::Exact: the asynchronous compress takes EqualPagesUpTo only");
  const uint64_t chunk_n = acf_chunk_n(cfg.max_page_n, max_item_n, nums_cap);
  ConfigCheck ck;
  if (PcoB200Error e = check_config(cfg, dtype, size_t(chunk_n), &ck)) return e;
  if (ck.auto_mode || ck.auto_delta)
    return fail(PCO_B200_UNSUPPORTED, "ModeSpec::Auto and DeltaSpec::Auto search on host threads: the asynchronous compress takes explicit specs only");
  if (unoptimized_bins_log(cfg.compression_level, chunk_n, 0) > ENC_NARROW_BINS_LOG)
    return fail(PCO_B200_UNSUPPORTED, "more than 256 unoptimized bins (levels 9-12): the asynchronous compress runs the narrow kernels only");
  const uint64_t max_chunks = uint64_t(nums_cap) / chunk_n + max_items;
  const uint64_t tiles = (chunk_n + SPLIT_TILE - 1) / SPLIT_TILE, bpc = n_batches_of(uint32_t(chunk_n));
  const uint64_t per_chunk = std::max<uint64_t>({tiles, (bpc + BINL_BATCHES - 1) / BINL_BATCHES, (bpc + 7) / 8, uint64_t(MAX_VARS)});
  if (max_chunks > 0x7fffffffu / per_chunk)
    return fail(PCO_B200_INVALID_ARGUMENT, "the capacities give " + std::to_string(max_chunks) + " chunk slots, more than one launch can cover");
  *cfg_out = cfg;
  *ck_out = ck;
  *max_chunks_out = max_chunks;
  return PCO_B200_OK;
}

PcoB200Error pco_b200_compress_files_async_plan(unsigned char dtype, const PcoB200ChunkConfig* config, int uniform_type_header, size_t max_files,
                                                size_t nums_cap, size_t max_file_n, size_t dst_cap, size_t index_cap,
                                                PcoB200AsyncCompressFilesPlan* plan) {
  if (!nt_valid(dtype)) return fail(PCO_B200_INVALID_TYPE, "unknown number type byte: " + std::to_string(dtype));
  if (!plan) return fail(PCO_B200_INVALID_ARGUMENT, "null plan");
  PcoB200ChunkConfig cfg;
  ConfigCheck ck;
  uint64_t max_chunks = 0;
  if (PcoB200Error e = acf_plan_checks(dtype, config, max_files, nums_cap, max_file_n, "file", &cfg, &ck, &max_chunks)) return e;
  std::memset(plan, 0, sizeof(*plan));
  plan->dtype = dtype;
  plan->uniform_type_header = uniform_type_header ? 1 : 0;
  fill_explicit_spec(plan, ck);
  plan->level = cfg.compression_level;
  plan->max_files = max_files;
  plan->nums_cap = nums_cap;
  plan->max_file_n = max_file_n;
  plan->max_page_n = cfg.max_page_n;
  plan->max_chunks = max_chunks;
  plan->dst_cap = dst_cap;
  plan->index_cap = index_cap;
  const uint64_t lbits = nt_bits(dtype);
  plan->dst_bound = uint64_t(max_files) * (standalone_header_size() + 1) + max_chunks * (5 + baseline_chunk_meta_size(uint32_t(lbits))) +
                    (uint64_t(nums_cap) * lbits + 7) / 8;
  plan->index_bound = uint64_t(max_files) * sizeof(IndexHeader) + max_chunks * (sizeof(IndexChunk) + plan->n_vars * sizeof(BatchEntry) + 15) +
                      plan->n_vars * sizeof(BatchEntry) * ((uint64_t(nums_cap) + BATCH_N - 1) / BATCH_N);
  plan->workspace_bytes = acf_plan_geom(*plan).l.total;
  return async_encode_setup<true>(dtype, {(const void*)acf_files_kernel, (const void*)acf_scan_kernel, (const void*)acf_place_kernel, (const void*)acf_init_kernel,
                                          (const void*)acf_bytes_kernel, (const void*)acf_bytes_scan_kernel, (const void*)acf_offsets_kernel,
                                          (const void*)acf_frame_kernel, (const void*)acf_index_kernel, (const void*)acf_finish_kernel});
}

// What the launches of a batch compress take by value (framed: 1 for standalone files, 0 for bare chunks)
static AcfArgs acf_args(const PcoB200AsyncCompressFilesPlan& p, const AcfPlanGeom& pg, void* workspace, void* dst, void* index, const uint64_t* ns,
                        const uint64_t* n_items, PcoB200FileRef* files, uint32_t framed) {
  AcfArgs fa;
  std::memset(&fa, 0, sizeof(fa));
  fa.a.n_chunks = pg.g.n_chunks;
  fa.a.dst_cap = p.dst_cap;
  fa.a.n_vars = p.n_vars;
  fa.a.ws = static_cast<uint8_t*>(workspace);
  fa.a.dst = static_cast<uint8_t*>(dst);
  fa.a.index = static_cast<uint8_t*>(index);
  fa.a.lay = pg.l.enc;
  fa.l = pg.l;
  fa.file_ns = ns;
  fa.n_files = n_items;
  fa.files = files;
  fa.max_files = p.max_files;
  fa.max_file_n = p.max_file_n;
  fa.nums_cap = p.nums_cap;
  fa.max_page_n = p.max_page_n;
  fa.index_cap = index ? p.index_cap : 0;
  fa.uniform_type = p.uniform_type_header ? p.dtype : 0;
  fa.bpc = pg.g.bpc;
  fa.framed = framed;
  return fa;
}

PcoB200Error pco_b200_compress_files_async(const PcoB200AsyncCompressFilesPlan* plan, const void* nums, const uint64_t* file_ns, const uint64_t* n_files,
                                           void* dst, void* index, PcoB200FileRef* files, void* workspace, PcoB200AsyncCompressFilesStatus* status,
                                           void* cuda_stream) {
  if (!plan || !file_ns || !n_files || !files || !workspace || !status || (!nums && plan->nums_cap) || (!dst && plan->dst_cap))
    return fail(PCO_B200_INVALID_ARGUMENT, "null buffer");
  AcfPlanGeom pg;
  if (PcoB200Error e = acf_check_plan(plan, &pg)) return e;
  if (index && plan->index_cap == 0) return fail(PCO_B200_INVALID_ARGUMENT, "an index with a plan made without one (index_cap 0)");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail(PCO_B200_INVALID_ARGUMENT, "the workspace is not 256-byte aligned");
  if (reinterpret_cast<uintptr_t>(index) & 15) return fail(PCO_B200_INVALID_ARGUMENT, "the index is not 16-byte aligned");
  AsyncLaunch ln;
  if (PcoB200Error e = open_async_launch(cuda_stream, &ln)) return e;
  const AcfArgs fa = acf_args(*plan, pg, workspace, dst, index, file_ns, n_files, files, 1);
  dispatch_latent(plan->dtype, [&](auto tag) {
    acf_launch<decltype(tag)>(*plan, pg.g, fa, nums, status, ln);
    return 0;
  });
  PCOB_CUDA_TRY(cudaGetLastError());
  return PCO_B200_OK;
}

size_t pco_b200_debug_standalone_header(uint64_t n_hint, unsigned char uniform_type, unsigned char* out) {
  return standalone_header_into(n_hint, uniform_type, out);
}

PcoB200Error pco_b200_compress_files_async_result(const PcoB200AsyncCompressFilesStatus* s, size_t* dst_len, size_t* index_len) {
  if (!s) return fail(PCO_B200_INVALID_ARGUMENT, "null status");
  const PcoB200Error kind = async_result_kind(s->kind);
  if (kind == PCO_B200_OK) {
    if (dst_len) *dst_len = size_t(s->dst_written);
    if (index_len) *index_len = size_t(s->index_written);
    return PCO_B200_OK;
  }
  switch (s->device_status) {
    case PCO_B200_ASYNC_TOO_MANY_FILES:
      return fail(kind, std::to_string(s->n_files) + " files, more than the plan's max_files");
    case PCO_B200_ASYNC_FILE_TOO_LARGE: return file_fail(kind, size_t(s->file), "more numbers than the plan's max_file_n");
    case PCO_B200_ASYNC_NUMS_CAP: return file_fail(kind, size_t(s->file), "the files up to this one hold more numbers than the plan's nums_cap");
    case PCO_B200_ASYNC_FILES_DST_FULL:
    case PCO_B200_ASYNC_FILES_INDEX_FULL:
      return fail(kind, "failed to write whole buffer (need " + std::to_string(s->dst_bytes) + " file bytes and " + std::to_string(s->index_bytes) +
                            " index bytes)");
    default: return fail(kind, "asynchronous batch compress failed (device status " + std::to_string(s->device_status) + ")");
  }
}

// ---- asynchronous batch compress into wrapped chunks (pco_b200_compress_wrapped_async; kernels in async_compress_wrapped.cuh).  The
// launches of pco_b200_compress_files_async up to pack_kernel with bare chunks staged in the workspace, then lens, scan, refs, split,
// finish.

PcoB200Error pco_b200_compress_wrapped_async_plan(unsigned char dtype, const PcoB200ChunkConfig* config, size_t max_arrays, size_t nums_cap,
                                                  size_t max_array_n, size_t metas_cap, size_t pages_cap, PcoB200AsyncCompressWrappedPlan* plan) {
  if (!nt_valid(dtype)) return fail(PCO_B200_INVALID_TYPE, "unknown number type byte: " + std::to_string(dtype));
  if (!plan) return fail(PCO_B200_INVALID_ARGUMENT, "null plan");
  PcoB200ChunkConfig cfg;
  ConfigCheck ck;
  uint64_t max_chunks = 0;
  if (PcoB200Error e = acf_plan_checks(dtype, config, max_arrays, nums_cap, max_array_n, "array", &cfg, &ck, &max_chunks)) return e;
  std::memset(plan, 0, sizeof(*plan));
  plan->dtype = dtype;
  fill_explicit_spec(plan, ck);
  plan->level = cfg.compression_level;
  plan->max_arrays = max_arrays;
  plan->nums_cap = nums_cap;
  plan->max_array_n = max_array_n;
  plan->max_page_n = cfg.max_page_n;
  plan->max_chunks = max_chunks;
  plan->metas_cap = metas_cap;
  plan->pages_cap = pages_cap;
  // the bounds the header comment derives
  const uint64_t lbits = nt_bits(dtype), obb = offset_bits_bits(uint32_t(lbits));
  const uint64_t mode_bits = plan->mode == MODE_CLASSIC ? 0 : plan->mode == MODE_FLOAT_QUANT ? 8 : lbits;
  const uint64_t meta_max = (4 + mode_bits + (4 + 5 + 5 + 64 + 32 * 32) + plan->n_vars * (4 + 15 + 256 * (15 + lbits + obb)) + 7) / 8;
  plan->pages_bound = max_chunks * (1 + baseline_chunk_meta_size(uint32_t(lbits))) + (uint64_t(nums_cap) * lbits + 7) / 8;
  plan->metas_bound = std::min<uint64_t>(max_chunks * meta_max, plan->pages_bound);
  plan->workspace_bytes = acw_plan_geom(*plan).l.total;
  return async_encode_setup<true>(dtype, {(const void*)acf_files_kernel, (const void*)acf_scan_kernel, (const void*)acf_place_kernel, (const void*)acf_init_kernel,
                                          (const void*)acf_bytes_kernel, (const void*)acf_bytes_scan_kernel, (const void*)acf_offsets_kernel,
                                          (const void*)acw_lens_kernel, (const void*)acw_scan_kernel, (const void*)acw_refs_kernel,
                                          (const void*)acw_split_kernel, (const void*)acw_finish_kernel});
}

PcoB200Error pco_b200_compress_wrapped_async(const PcoB200AsyncCompressWrappedPlan* plan, const void* nums, const uint64_t* array_ns,
                                             const uint64_t* n_arrays, void* metas, void* pages, PcoB200PageRef* refs, uint64_t* first_chunk,
                                             void* workspace, PcoB200AsyncCompressWrappedStatus* status, void* cuda_stream) {
  if (!plan || !array_ns || !n_arrays || !refs || !first_chunk || !workspace || !status || (!nums && plan->nums_cap) || (!metas && plan->metas_cap) ||
      (!pages && plan->pages_cap))
    return fail(PCO_B200_INVALID_ARGUMENT, "null buffer");
  AcwPlanGeom pg;
  if (PcoB200Error e = acw_check_plan(plan, &pg)) return e;
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail(PCO_B200_INVALID_ARGUMENT, "the workspace is not 256-byte aligned");
  if (reinterpret_cast<uintptr_t>(refs) & 7 || reinterpret_cast<uintptr_t>(first_chunk) & 7)
    return fail(PCO_B200_INVALID_ARGUMENT, "refs and first_chunk must be 8-byte aligned");
  AsyncLaunch ln;
  if (PcoB200Error e = open_async_launch(cuda_stream, &ln)) return e;
  const PcoB200AsyncCompressFilesPlan fp = acw_files_plan(*plan);
  AcwArgs w;
  std::memset(&w, 0, sizeof(w));
  w.f = acf_args(fp, pg.f, workspace, static_cast<uint8_t*>(workspace) + pg.l.stage, nullptr, array_ns, n_arrays, nullptr, 0);
  w.l = pg.l;
  w.metas = static_cast<uint8_t*>(metas);
  w.pages = static_cast<uint8_t*>(pages);
  w.refs = refs;
  w.first_chunk = first_chunk;
  w.metas_cap = plan->metas_cap;
  w.pages_cap = plan->pages_cap;
  w.dtype = plan->dtype;
  dispatch_latent(plan->dtype, [&](auto tag) {
    acw_launch<decltype(tag)>(*plan, pg, w, nums, status, ln);
    return 0;
  });
  PCOB_CUDA_TRY(cudaGetLastError());
  return PCO_B200_OK;  // spans stay pending until pco_b200_profile_last reads them
}

PcoB200Error pco_b200_compress_wrapped_async_result(const PcoB200AsyncCompressWrappedStatus* s, size_t* metas_len, size_t* pages_len, size_t* n_chunks) {
  if (!s) return fail(PCO_B200_INVALID_ARGUMENT, "null status");
  const PcoB200Error kind = async_result_kind(s->kind);
  if (kind == PCO_B200_OK) {
    if (metas_len) *metas_len = size_t(s->metas_written);
    if (pages_len) *pages_len = size_t(s->pages_written);
    if (n_chunks) *n_chunks = size_t(s->n_chunks);
    return PCO_B200_OK;
  }
  const std::string array = "array " + std::to_string(s->array) + ": ";
  switch (s->device_status) {
    case PCO_B200_ASYNC_TOO_MANY_FILES: return fail(kind, std::to_string(s->n_arrays) + " arrays, more than the plan's max_arrays");
    case PCO_B200_ASYNC_FILE_TOO_LARGE: return fail(kind, array + "more numbers than the plan's max_array_n");
    case PCO_B200_ASYNC_NUMS_CAP: return fail(kind, array + "the arrays up to this one hold more numbers than the plan's nums_cap");
    case PCO_B200_ASYNC_FILES_DST_FULL:
      return fail(kind, "failed to write whole buffer (need " + std::to_string(s->metas_bytes) + " meta bytes and " + std::to_string(s->pages_bytes) +
                            " page bytes)");
    case ST_CORRUPTION: return fail(kind, "compressor returned chunks that do not split into meta and page");
    default: return fail(kind, "asynchronous wrapped compress failed (device status " + std::to_string(s->device_status) + ")");
  }
}

PcoB200Error pco_b200_build_index(const void* compressed, size_t compressed_len, unsigned char dtype, void* index, size_t index_cap,
                                  size_t* index_len, uint32_t flags, void* cuda_stream) {
  if (!nt_valid(dtype)) return fail(PCO_B200_INVALID_TYPE, "unknown number type byte");
  Context& c = ctx();
  if (PcoB200Error e = ensure_device(c)) return e;
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  const bool src_dev = flags & PCO_B200_SRC_ON_DEVICE;
  StandaloneHeader hdr;
  if (PcoB200Error e = read_heads(compressed, compressed_len, src_dev, nullptr, 0, false, nullptr, &hdr, stream)) return e;
  const uint8_t* d_src;
  if (PcoB200Error e = stage_in(c.src, compressed, compressed_len, src_dev, stream, &d_src)) return e;
  const FileParams fp{d_src, compressed_len, dtype, hdr.uniform_type, hdr.format_major};
  if (index_cap < sizeof(IndexHeader) + sizeof(IndexChunk) + 64) return fail(PCO_B200_IO, "index buffer too small");
  // Split the caller's capacity: chunk records sized from a lower bound on chunk bytes, the rest for entries.
  uint64_t max_chunks = std::min<uint64_t>(uint64_t(compressed_len) / 5 + 2, (index_cap - sizeof(IndexHeader)) / (4 * sizeof(IndexChunk)));
  max_chunks = std::max<uint64_t>(1, std::min<uint64_t>(max_chunks, 0x7fffffffull));
  const uint64_t chunks_offset = sizeof(IndexHeader);
  uint64_t entries_begin = (chunks_offset + max_chunks * sizeof(IndexChunk) + 15) & ~uint64_t(15);
  if (entries_begin > index_cap) return fail(PCO_B200_IO, "index buffer too small");
  PCOB_CUDA_TRY(c.index.reserve(index_cap));
  PCOB_CUDA_TRY(c.misc.reserve(sizeof(WalkResult)));
  uint8_t* d_index = c.index.as<uint8_t>();
  // The walk writes only the records and entries of the file's chunks, but the bytes returned also hold the unused record slots and
  // the padding before the entries: zeroed, so the index is the same on every call instead of carrying what the thread's scratch held.
  PCOB_CUDA_TRY(cudaMemsetAsync(d_index, 0, index_cap, stream));
  walk_kernel<12><<<1, WALK_THREADS, sizeof(WalkSmem<12>), stream>>>(fp, d_index, chunks_offset, uint32_t(max_chunks), entries_begin, index_cap, hdr.first_chunk_byte,
                                                    0, ~uint64_t(0), nullptr, c.misc.as<WalkResult>(), 1);
  PCOB_CUDA_TRY(cudaGetLastError());
  WalkResult res;
  PCOB_CUDA_TRY(cudaMemcpyAsync(&res, c.misc.p, sizeof(res), cudaMemcpyDeviceToHost, stream));
  PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
  if (res.status == ST_INDEX_FULL) return fail(PCO_B200_IO, "index buffer too small");
  if (res.status != ST_TERMINATOR) return status_to_error(res.status, ("chunk " + std::to_string(res.n_chunks)).c_str());
  IndexHeader ih;
  std::memset(&ih, 0, sizeof(ih));
  ih.magic = INDEX_MAGIC;
  ih.version = 1;
  ih.n_chunks = res.n_chunks;
  ih.n_total = res.n_total;
  ih.file_len = compressed_len;
  ih.chunks_offset = chunks_offset;
  ih.end_byte = res.next_byte;
  size_t used = std::max<uint64_t>(res.entries_end, entries_begin);
  std::memcpy(index, &ih, sizeof(ih));
  if (used > sizeof(ih)) {
    PCOB_CUDA_TRY(cudaMemcpyAsync(static_cast<uint8_t*>(index) + sizeof(ih), d_index + sizeof(ih), used - sizeof(ih), cudaMemcpyDeviceToHost, stream));
    PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
  }
  if (index_len) *index_len = used;
  return PCO_B200_OK;
}

// ---- asynchronous side index of a standalone file (pco_b200_build_index_async; kernels in async_index_kernels.cuh)
// The plan fixes what the launches take by value and every grid size (from src_cap and max_chunks); the file's length comes from the
// device.  A call is a fixed sequence of launches: head, two rounds of seven, serial, place, copy, finish.

// Every grid of a call stays within 2^31 - 1 CTAs: the candidate walks launch max_chunks + AI_SPARE_CANDS, the find grid one CTA per
// AI_FIND_SPAN bytes of src_cap.
constexpr uint64_t AI_MAX_CHUNKS = 0x7fffffffull - AI_SPARE_CANDS;
constexpr uint64_t AI_MAX_SRC_CAP = 0x7fffffffull * AI_FIND_SPAN;

static bool ai_plan_ok(const PcoB200AsyncIndexPlan* p) {
  return nt_valid(p->dtype) && p->max_chunks >= 1 && p->max_chunks <= AI_MAX_CHUNKS && p->src_cap <= AI_MAX_SRC_CAP &&
         p->workspace_bytes == ai_layout(p->src_cap, p->index_cap, p->max_chunks).total;
}

PcoB200Error pco_b200_build_index_async_plan(const void* head, size_t head_len, unsigned char dtype, size_t src_cap, size_t index_cap, size_t max_chunks,
                                             PcoB200AsyncIndexPlan* plan) {
  StandaloneHeader hdr;
  if (PcoB200Error e = check_async_head(head, head_len, dtype, plan, &hdr)) return e;
  if (max_chunks == 0 || uint64_t(max_chunks) > AI_MAX_CHUNKS) return fail(PCO_B200_INVALID_ARGUMENT, "max_chunks must be 1 .. 2^31 - 9");
  if (uint64_t(src_cap) > AI_MAX_SRC_CAP) return fail(PCO_B200_INVALID_ARGUMENT, "src_cap above (2^31 - 1) x 4096 bytes");
  std::memset(plan, 0, sizeof(*plan));
  plan->dtype = dtype;
  plan->uniform_type = hdr.uniform_type;
  plan->format_major = hdr.format_major;
  plan->src_cap = src_cap;
  plan->index_cap = index_cap;
  plan->max_chunks = max_chunks;
  plan->workspace_bytes = ai_layout(src_cap, index_cap, max_chunks).total;
  Context& c = ctx();
  if (PcoB200Error e = ensure_device(c)) return e;
  PCOB_CUDA_TRY(cudaFuncSetAttribute(ai_walk_kernel<12>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(WalkSmem<12>)));
  PCOB_CUDA_TRY(cudaFuncSetAttribute(ai_serial_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(WalkSmem<12>)));
  return load_kernels({(const void*)ai_head_kernel, (const void*)ai_round_kernel, (const void*)ai_count_kernel, (const void*)ai_scan_kernel,
                       (const void*)ai_scatter_kernel, (const void*)ai_walk_kernel<SMALL_MAX_SIZE_LOG>, (const void*)ai_walk_kernel<12>,
                       (const void*)ai_chain_kernel, (const void*)ai_serial_kernel, (const void*)ai_place_kernel, (const void*)ai_copy_kernel,
                       (const void*)ai_finish_kernel});
}

PcoB200Error pco_b200_build_index_async(const PcoB200AsyncIndexPlan* plan, const void* src, const uint64_t* src_len, void* index, void* workspace,
                                        PcoB200AsyncIndexStatus* status, void* cuda_stream) {
  if (!plan || !src || !src_len || !index || !workspace || !status) return fail(PCO_B200_INVALID_ARGUMENT, "null buffer");
  if (!ai_plan_ok(plan)) return fail(PCO_B200_INVALID_ARGUMENT, "the plan was not made by pco_b200_build_index_async_plan");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail(PCO_B200_INVALID_ARGUMENT, "the workspace is not 256-byte aligned");
  if (reinterpret_cast<uintptr_t>(index) & 15) return fail(PCO_B200_INVALID_ARGUMENT, "the index is not 16-byte aligned");
  AsyncLaunch ln;
  if (PcoB200Error e = open_async_launch(cuda_stream, &ln)) return e;
  const cudaStream_t stream = ln.stream;

  const AiLayout lay = ai_layout(plan->src_cap, plan->index_cap, plan->max_chunks);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  AiState* state = reinterpret_cast<AiState*>(ws);
  uint64_t* parts = reinterpret_cast<uint64_t*>(ws + lay.parts);
  AiArgs g;
  g.src = static_cast<const uint8_t*>(src);
  g.src_len = src_len;
  g.index = static_cast<uint8_t*>(index);
  g.ws = ws;
  g.src_cap = plan->src_cap;
  g.index_cap = plan->index_cap;
  g.max_chunks = plan->max_chunks;
  g.dtype = plan->dtype;
  g.uniform_type = plan->uniform_type;
  g.format_major = plan->format_major;
  const uint32_t find = uint32_t(ai_find_ctas(plan->src_cap));
  const uint32_t cands = uint32_t(plan->max_chunks + AI_SPARE_CANDS), chunks = uint32_t(plan->max_chunks + 1);

  ln.begin("ai_head_kernel");
  ai_head_kernel<<<1, 1, 0, stream>>>(g, state);
  ln.end();
  for (int round = 0; round < AI_ROUNDS; round++) {
    ln.begin("ai_round_kernel");
    ai_round_kernel<<<1, 1, 0, stream>>>(g, state);
    ln.end();
    ln.begin("ai_count_kernel");
    ai_count_kernel<<<find, AI_THREADS, 0, stream>>>(g, state, parts);
    ln.end();
    ln.begin("ai_scan_kernel");
    ai_scan_kernel<<<1, AI_SCAN_THREADS, 0, stream>>>(g, state, parts);
    ln.end();
    ln.begin("ai_scatter_kernel");
    ai_scatter_kernel<<<find, AI_THREADS, 0, stream>>>(g, state, parts, reinterpret_cast<uint64_t*>(ws + lay.cand), reinterpret_cast<IndexChunk*>(ws + lay.crec));
    ln.end();
    ln.begin("ai_walk_kernel<10>");
    ai_walk_kernel<SMALL_MAX_SIZE_LOG><<<cands, WALK_THREADS, sizeof(WalkSmem<SMALL_MAX_SIZE_LOG>), stream>>>(
        g, state, reinterpret_cast<uint32_t*>(ws + lay.cst), reinterpret_cast<uint64_t*>(ws + lay.cend));
    ln.end();
    ln.begin("ai_walk_kernel<12>");
    ai_walk_kernel<12><<<cands, WALK_THREADS, sizeof(WalkSmem<12>), stream>>>(g, state, reinterpret_cast<uint32_t*>(ws + lay.cst),
                                                                              reinterpret_cast<uint64_t*>(ws + lay.cend));
    ln.end();
    ln.begin("ai_chain_kernel");
    ai_chain_kernel<<<1, AI_THREADS, 0, stream>>>(g, state);
    ln.end();
  }
  ln.begin("ai_serial_kernel");
  ai_serial_kernel<<<1, WALK_THREADS, sizeof(WalkSmem<12>), stream>>>(g, state);
  ln.end();
  ln.begin("ai_place_kernel");
  ai_place_kernel<<<1, AI_SCAN_THREADS, 0, stream>>>(g, state);
  ln.end();
  ln.begin("ai_copy_kernel");
  ai_copy_kernel<<<chunks, AI_THREADS, 0, stream>>>(g, state);
  ln.end();
  ln.begin("ai_finish_kernel");
  ai_finish_kernel<<<1, 1, 0, stream>>>(g, state, status);
  ln.end();
  PCOB_CUDA_TRY(cudaGetLastError());
  return PCO_B200_OK;  // spans stay pending until pco_b200_profile_last reads them
}

PcoB200Error pco_b200_build_index_async_result(const PcoB200AsyncIndexStatus* s, size_t* index_len) {
  if (!s) return fail(PCO_B200_INVALID_ARGUMENT, "null status");
  const PcoB200Error kind = async_result_kind(s->kind);
  if (kind == PCO_B200_OK) {
    if (index_len) *index_len = size_t(s->index_bytes);
    return PCO_B200_OK;
  }
  if (const char* h = async_header_refusal(s->device_status)) return fail(kind, h);
  switch (s->device_status) {
    case PCO_B200_ASYNC_FILE_OUTSIDE: return fail(kind, "the file length *src_len exceeds the plan's src_cap");
    case PCO_B200_ASYNC_TOO_MANY_CHUNKS: return fail(kind, "the file has more chunks than the plan's max_chunks");
    case PCO_B200_ASYNC_FILES_INDEX_FULL: return fail(kind, "index buffer too small: the side index needs more than the plan's index_cap bytes");
    default:
      status_to_error(s->device_status, "this chunk");
      return fail(kind, "chunk " + std::to_string(s->chunk) + ": " + last_error_ref());
  }
}

// ---- asynchronous transcode of wrapped pages into an indexed standalone file (pco_b200_pages_to_file_async; kernels in
// async_pages_to_file_kernels.cuh).  A call is a fixed sequence of launches: the pages front end (enqueue_pages_front), the wide walk, the
// gate, the file writer, the index writer, the finish.

static bool pf_plan_ok(const PcoB200AsyncPagesToFilePlan* p) {
  constexpr uint64_t cap = uint64_t(1) << 56;
  return nt_valid(p->dtype) && (p->uniform_type == 0 || p->uniform_type == p->dtype) && p->max_pages >= 1 && p->max_pages <= 0x7fffffffull &&
         p->frame_cap <= cap && p->dst_cap <= cap && p->index_cap <= cap && p->workspace_bytes == pf_layout(p->max_pages, p->frame_cap, p->index_cap).total;
}

PcoB200Error pco_b200_pages_to_file_async_plan(unsigned char dtype, int uniform_type_header, size_t metas_cap, size_t pages_cap, size_t max_pages,
                                               size_t frame_cap, size_t dst_cap, size_t index_cap, PcoB200AsyncPagesToFilePlan* plan) {
  if (!nt_valid(dtype)) return fail(PCO_B200_INVALID_TYPE, "unknown number type byte: " + std::to_string(dtype));
  if (!plan) return fail(PCO_B200_INVALID_ARGUMENT, "null plan");
  if (max_pages == 0 || uint64_t(max_pages) > 0x7fffffffull) return fail(PCO_B200_INVALID_ARGUMENT, "max_pages must be 1 .. 2^31 - 1");
  if (uint64_t(frame_cap) > (uint64_t(1) << 56)) return fail(PCO_B200_INVALID_ARGUMENT, "frame_cap above 2^56 bytes");
  if (uint64_t(dst_cap) > (uint64_t(1) << 56)) return fail(PCO_B200_INVALID_ARGUMENT, "dst_cap above 2^56 bytes");
  if (uint64_t(index_cap) > (uint64_t(1) << 56)) return fail(PCO_B200_INVALID_ARGUMENT, "index_cap above 2^56 bytes");
  std::memset(plan, 0, sizeof(*plan));
  plan->dtype = dtype;
  plan->uniform_type = uniform_type_header ? dtype : 0;
  plan->metas_cap = metas_cap;
  plan->pages_cap = pages_cap;
  plan->max_pages = max_pages;
  plan->frame_cap = frame_cap;
  plan->dst_cap = dst_cap;
  plan->index_cap = index_cap;
  plan->workspace_bytes = pf_layout(max_pages, frame_cap, index_cap).total;
  Context& c = ctx();
  if (PcoB200Error e = ensure_device(c)) return e;
  PCOB_CUDA_TRY(cudaFuncSetAttribute(pf_walk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(WalkSmem<12>)));
  return load_kernels({(const void*)ap_pages_kernel, (const void*)ap_scan_kernel, (const void*)ap_place_kernel, (const void*)frame_pages_kernel,
                       (const void*)walk_kernel<SMALL_MAX_SIZE_LOG>, (const void*)ap_route_kernel, (const void*)ap_rewalk_kernel,
                       (const void*)pf_walk_kernel, (const void*)pf_gate_kernel, (const void*)pf_file_kernel, (const void*)pf_index_kernel,
                       (const void*)pf_finish_kernel});
}

PcoB200Error pco_b200_pages_to_file_async(const PcoB200AsyncPagesToFilePlan* plan, const void* metas, const void* pages, const PcoB200PageRef* refs,
                                          const uint64_t* n_pages, void* dst, void* index, PcoB200FileRef* file_ref, void* workspace,
                                          PcoB200AsyncPagesToFileStatus* status, void* cuda_stream) {
  if (!plan || !metas || !pages || !refs || !n_pages || !dst || !index || !file_ref || !workspace || !status)
    return fail(PCO_B200_INVALID_ARGUMENT, "null buffer");
  if (!pf_plan_ok(plan)) return fail(PCO_B200_INVALID_ARGUMENT, "the plan was not made by pco_b200_pages_to_file_async_plan");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail(PCO_B200_INVALID_ARGUMENT, "the workspace is not 256-byte aligned");
  if (reinterpret_cast<uintptr_t>(index) & 15) return fail(PCO_B200_INVALID_ARGUMENT, "the index is not 16-byte aligned");
  AsyncLaunch ln;
  if (PcoB200Error e = open_async_launch(cuda_stream, &ln)) return e;
  const cudaStream_t stream = ln.stream;

  const uint32_t mp = uint32_t(plan->max_pages);
  const PfLayout lay = pf_layout(mp, plan->frame_cap, plan->index_cap);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  // no numbers are written: a number capacity that no batch of max_pages pages of at most 2^24 numbers reaches
  const ApArgs ag{static_cast<const uint8_t*>(metas), static_cast<const uint8_t*>(pages), refs, n_pages, plan->metas_cap, plan->pages_cap, NONE64,
                  plan->frame_cap, plan->dtype, mp};
  const PfArgs g{ws, static_cast<uint8_t*>(dst), static_cast<uint8_t*>(index), file_ref, plan->max_pages, plan->frame_cap, plan->dst_cap,
                 plan->index_cap, plan->dtype, plan->uniform_type};
  enqueue_pages_front(ln, ag, lay.ap, ws);
  ln.begin("pf_walk_kernel");
  pf_walk_kernel<<<mp, WALK_THREADS, sizeof(WalkSmem<12>), stream>>>(g);
  ln.end();
  ln.begin("pf_gate_kernel");
  pf_gate_kernel<<<1, AP_SCAN_THREADS, 0, stream>>>(g);
  ln.end();
  ln.begin("pf_file_kernel");
  pf_file_kernel<<<pf_file_ctas(plan->dst_cap), GATHER_THREADS, 0, stream>>>(g);
  ln.end();
  ln.begin("pf_index_kernel");
  pf_index_kernel<<<mp, AI_THREADS, 0, stream>>>(g);
  ln.end();
  ln.begin("pf_finish_kernel");
  pf_finish_kernel<<<1, 1, 0, stream>>>(g, status);
  ln.end();
  PCOB_CUDA_TRY(cudaGetLastError());
  return PCO_B200_OK;  // spans stay pending until pco_b200_profile_last reads them
}

PcoB200Error pco_b200_pages_to_file_async_result(const PcoB200AsyncPagesToFileStatus* s, size_t* file_len, size_t* index_len) {
  if (!s) return fail(PCO_B200_INVALID_ARGUMENT, "null status");
  const PcoB200Error kind = async_result_kind(s->kind);
  if (kind == PCO_B200_OK) {
    if (file_len) *file_len = size_t(s->file_len);
    if (index_len) *index_len = size_t(s->index_len);
    return PCO_B200_OK;
  }
  switch (s->device_status) {
    case PCO_B200_ASYNC_FILES_DST_FULL:
      return fail(kind, "the file needs " + std::to_string(s->file_needed) + " bytes, more than the plan's dst_cap");
    case PCO_B200_ASYNC_FILES_INDEX_FULL:
      if (s->index_needed == 0) return fail(kind, "the side index needs more than the walks' room, about twice the plan's index_cap bytes");
      return fail(kind, "the side index needs " + std::to_string(s->index_needed) + " bytes, more than the plan's index_cap");
    case ST_UNSUPPORTED:
      if (s->page != NONE64)
        return page_fail(kind, size_t(s->page), "neither walker takes this page (Dict, Lookback, Conv1, or tables above 2^12 states), so no side index can hold it");
      [[fallthrough]];
    default: {  // the pages call's words
      const PcoB200AsyncPagesStatus p{s->kind, s->device_status, s->page, 0, s->n_pages, s->frames_needed};
      return pco_b200_decompress_pages_async_result(&p, nullptr);
    }
  }
}

// ---------------------------------------------------------------------------
// Sharded writers (SURVEY.md 8e): device buffers other ranks can map, and the page gather (gather_kernels.cuh)
// ---------------------------------------------------------------------------
PcoB200Error pco_b200_ipc_alloc(size_t bytes, void** dev_ptr, unsigned char* handle64) {
  if (!dev_ptr || !handle64) return fail(PCO_B200_INVALID_ARGUMENT, "null argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "the handle travels as 64 bytes");
  Context& c = ctx();
  if (PcoB200Error e = ensure_device(c)) return e;
  void* p = nullptr;
  PCOB_CUDA_TRY(cudaMalloc(&p, bytes + 64));
  cudaIpcMemHandle_t h;
  cudaError_t ce = cudaIpcGetMemHandle(&h, p);
  if (ce != cudaSuccess) { cudaFree(p); return cuda_fail(ce, "cudaIpcGetMemHandle"); }
  std::memcpy(handle64, &h, 64);
  *dev_ptr = p;
  return PCO_B200_OK;
}
PcoB200Error pco_b200_ipc_open(const unsigned char* handle64, void** dev_ptr) {
  if (!dev_ptr || !handle64) return fail(PCO_B200_INVALID_ARGUMENT, "null argument");
  Context& c = ctx();
  if (PcoB200Error e = ensure_device(c)) return e;
  cudaIpcMemHandle_t h;
  std::memcpy(&h, handle64, 64);
  PCOB_CUDA_TRY(cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return PCO_B200_OK;
}
PcoB200Error pco_b200_ipc_close(void* dev_ptr) {
  if (dev_ptr) PCOB_CUDA_TRY(cudaIpcCloseMemHandle(dev_ptr));
  return PCO_B200_OK;
}
PcoB200Error pco_b200_ipc_free(void* dev_ptr) {
  if (dev_ptr) PCOB_CUDA_TRY(cudaFree(dev_ptr));
  return PCO_B200_OK;
}

PcoB200Error pco_b200_chunk_sizes(const void* index_dev, size_t index_len, uint64_t* sizes_dev, size_t n_chunks, void* cuda_stream) {
  if (n_chunks == 0) return PCO_B200_OK;
  if (!index_dev || !sizes_dev) return fail(PCO_B200_INVALID_ARGUMENT, "null argument");
  Context& c = ctx();
  if (PcoB200Error e = ensure_device(c)) return e;
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  PCOB_CUDA_TRY(c.misc.reserve(256));
  uint32_t* d_err = c.misc.as<uint32_t>() + 32;
  PCOB_CUDA_TRY(cudaMemsetAsync(d_err, 0, 4, stream));
  chunk_sizes_kernel<<<uint32_t(std::min<size_t>((n_chunks + 255) / 256, 1024)), 256, 0, stream>>>(static_cast<const uint8_t*>(index_dev), index_len, sizes_dev, uint32_t(n_chunks), d_err);
  PCOB_CUDA_TRY(cudaGetLastError());
  return PCO_B200_OK;  // asynchronous: a malformed index shows up as sizes the gather rejects (file length over capacity) or as d_err in pco_b200_gather_pages
}

PcoB200Error pco_b200_gather_pages(const void* chunks_dev, const uint64_t* all_sizes_dev, uint32_t world, uint32_t rank, size_t n_local, size_t n_total_numbers,
                                   unsigned char uniform_type, void* const* peer_files, size_t file_cap, uint64_t* file_len_dev, uint32_t max_ctas, void* cuda_stream) {
  if (world == 0 || world > uint32_t(GATHER_MAX_WORLD) || rank >= world) return fail(PCO_B200_INVALID_ARGUMENT, "world must be 1..16 and rank < world");
  if (!chunks_dev || !all_sizes_dev || !peer_files || !file_len_dev) return fail(PCO_B200_INVALID_ARGUMENT, "null argument");
  if (n_local > 0x7fffffffull) return fail(PCO_B200_INVALID_ARGUMENT, "too many chunks");
  Context& c = ctx();
  if (PcoB200Error e = ensure_device(c)) return e;
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  GatherPeers peers;
  for (uint32_t r = 0; r < uint32_t(GATHER_MAX_WORLD); r++) peers.file[r] = r < world ? static_cast<uint8_t*>(peer_files[r]) : nullptr;
  for (uint32_t r = 0; r < world; r++)
    if (!peers.file[r]) return fail(PCO_B200_INVALID_ARGUMENT, "peer file buffer " + std::to_string(r) + " is null");
  const std::vector<uint8_t> header = make_standalone_header(n_total_numbers, uniform_type);
  // scratch: [src_off | dst_off] (2 x n_local u64), header bytes, error word; owned by the calling thread's context and reused
  const size_t off_bytes = 2 * n_local * sizeof(uint64_t);
  PCOB_CUDA_TRY(c.gather.reserve(off_bytes + 256));
  uint64_t* d_src_off = c.gather.as<uint64_t>();
  uint64_t* d_dst_off = d_src_off + n_local;
  uint8_t* d_header = c.gather.as<uint8_t>() + off_bytes;
  uint32_t* d_err = reinterpret_cast<uint32_t*>(d_header + 128);
  PCOB_CUDA_TRY(cudaMemcpyAsync(d_header, header.data(), header.size(), cudaMemcpyHostToDevice, stream));
  PCOB_CUDA_TRY(cudaMemsetAsync(d_err, 0, 4, stream));
  c.gather_err = d_err;
  gather_offsets_kernel<<<1, 1024, 0, stream>>>(all_sizes_dev, world, rank, uint32_t(n_local), header.size(), d_src_off, d_dst_off, file_len_dev);
  const uint32_t ctas = std::max(1u, max_ctas ? max_ctas : uint32_t(c.sm_count));
  // (no profiler span here: the gather is meant to run asynchronously beside the caller's next calls, whose span resolution would wait for it)
  push_pages_kernel<<<ctas, GATHER_THREADS, 0, stream>>>(static_cast<const uint8_t*>(chunks_dev), all_sizes_dev, d_src_off, d_dst_off, file_len_dev, peers, world, rank,
                                                        uint32_t(n_local), file_cap, d_header, uint32_t(header.size()), d_err);
  PCOB_CUDA_TRY(cudaGetLastError());
  return PCO_B200_OK;  // asynchronous on `stream`; pco_b200_gather_status reports a file buffer that was too small
}

// Blocks until the calling thread's last pco_b200_gather_pages has finished on `cuda_stream` and reports it: PCO_B200_IO when a
// file buffer was too small for the gathered file, PCO_B200_INVALID_ARGUMENT for a malformed side index.
PcoB200Error pco_b200_gather_status(void* cuda_stream) {
  Context& c = ctx();
  if (!c.gather_err) return PCO_B200_OK;
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  uint32_t st = 0;
  PCOB_CUDA_TRY(cudaMemcpyAsync(&st, c.gather_err, 4, cudaMemcpyDeviceToHost, stream));
  PCOB_CUDA_TRY(cudaStreamSynchronize(stream));
  if (st == ST_INSUFFICIENT_DATA) return fail(PCO_B200_IO, "failed to write whole buffer: a rank's file buffer is smaller than the gathered file");
  if (st != ST_OK) return status_to_error(st, "the page gather");
  return PCO_B200_OK;
}

}  // extern "C"
