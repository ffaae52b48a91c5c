// Host-side support for libcpcodec.so: error state, device scratch cache, standalone header
// parse/write and size guarantees.  Independent of oracle/ (the product never links it).
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/pco_b200.h"
#include "codec_common.cuh"

namespace pcob200 {

// ---- thread-local error message (pco::errors::PcoError::message) -----------
inline std::string& last_error_ref() {
  static thread_local std::string s;
  return s;
}
inline PcoB200Error fail(PcoB200Error e, const std::string& msg) {
  last_error_ref() = msg;
  return e;
}
inline PcoB200Error cuda_fail(cudaError_t ce, const char* what) {
  return fail(PCO_B200_CUDA, std::string(what) + ": " + cudaGetErrorString(ce) +
                                 " (libcpcodec has no CPU fallback: a CUDA device is required)");
}
#define PCOB_CUDA_TRY(expr)                                   \
  do {                                                        \
    cudaError_t _ce = (expr);                                 \
    if (_ce != cudaSuccess) return cuda_fail(_ce, #expr);     \
  } while (0)

inline PcoB200Error status_to_error(uint32_t st, const char* where) {
  switch (st) {
    case ST_OK: return PCO_B200_OK;
    case ST_CORRUPTION: return fail(PCO_B200_CORRUPTION, std::string("corrupt data in ") + where);
    case ST_INSUFFICIENT_DATA: return fail(PCO_B200_INSUFFICIENT_DATA, std::string("insufficient data in ") + where);
    case ST_INVALID_ARGUMENT: return fail(PCO_B200_INVALID_ARGUMENT, std::string("invalid argument in ") + where);
    case ST_UNSUPPORTED:
      return fail(PCO_B200_UNSUPPORTED, std::string("valid pco outside the GPU hot path (dict/lookback/conv1, >256 bins or "
                                                    "ans_size_log > 10) in ") + where);
    default: return fail(PCO_B200_CORRUPTION, std::string("unexpected device status in ") + where);
  }
}

// ---- optional per-kernel timing (CUDA events on the launching stream; off by default) ----
inline std::atomic<bool>& profiler_enabled() {  // process-wide switch; spans and results are per thread
  static std::atomic<bool> on{false};
  return on;
}
struct Profiler {
  struct Span { std::string name; cudaEvent_t e0, e1; };
  std::vector<Span> spans;                              // of the call in flight
  std::vector<std::pair<std::string, float>> last;      // resolved spans of the last finished call
  void begin(const char* name, cudaStream_t s) {
    if (!profiler_enabled().load(std::memory_order_relaxed)) return;
    Span sp;
    sp.name = name;
    cudaEventCreate(&sp.e0);
    cudaEventCreate(&sp.e1);
    cudaEventRecord(sp.e0, s);
    spans.push_back(sp);
  }
  void end(cudaStream_t s) {
    if (spans.empty()) return;
    cudaEventRecord(spans.back().e1, s);
  }
  void resolve() {  // call after the stream has been synchronised
    if (spans.empty() && !profiler_enabled().load(std::memory_order_relaxed)) return;
    last.clear();
    for (auto& sp : spans) {
      float ms = 0.f;
      cudaEventSynchronize(sp.e1);
      cudaEventElapsedTime(&ms, sp.e0, sp.e1);
      last.push_back({sp.name, ms});
      cudaEventDestroy(sp.e0);
      cudaEventDestroy(sp.e1);
    }
    spans.clear();
  }
  void discard() {  // drops pending spans unread (the events are released once the device has passed them)
    for (auto& sp : spans) {
      cudaEventDestroy(sp.e0);
      cudaEventDestroy(sp.e1);
    }
    spans.clear();
  }
};
inline Profiler& profiler() {
  static thread_local Profiler p;
  return p;
}

// The caller's stream of an asynchronous call, and whether its launches record kernel spans: only outside a capture (an event record
// would become part of the graph).  Opening it drops the spans of an earlier call that nobody read.
struct AsyncLaunch {
  cudaStream_t stream;
  bool prof;
  void begin(const char* name) const { if (prof) profiler().begin(name, stream); }
  void end() const { if (prof) profiler().end(stream); }
};
inline PcoB200Error open_async_launch(void* cuda_stream, AsyncLaunch* ln) {
  cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  PCOB_CUDA_TRY(cudaStreamIsCapturing(stream, &cap));
  ln->stream = stream;
  ln->prof = cap == cudaStreamCaptureStatusNone && profiler_enabled().load(std::memory_order_relaxed);
  if (ln->prof) profiler().discard();
  return PCO_B200_OK;
}

// ---- PCOB200_TRACE=1: host-clock marks of a call's phases on stderr (one line per call; all threads share the epoch) ------------------
inline bool trace_enabled() {
  static const bool on = std::getenv("PCOB200_TRACE") != nullptr;
  return on;
}
struct CallTrace {
  std::string line;
  static double now_ms() {
    static const auto epoch = std::chrono::steady_clock::now();
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - epoch).count();
  }
  void mark(const char* what) {
    if (!trace_enabled()) return;
    char buf[64];
    std::snprintf(buf, sizeof(buf), " %s=%.2f", what, now_ms());
    line += buf;
  }
  void flush(const char* call) {
    if (!trace_enabled()) return;
    std::fprintf(stderr, "[pcob200 trace] %s%s\n", call, line.c_str());
    line.clear();
  }
};
inline CallTrace& call_trace() {
  static thread_local CallTrace t;
  return t;
}

// ---- large host <-> device copies: sliced, one slice in flight -----------------------------------------------------------------------
// Copies of one direction issued on different streams do not share the link slice by slice: a copy engine stays with the stream it is
// serving for as long as that stream has a copy queued (seen with PCOB200_TRACE: with a large upload running - whole, in 4 MB slices
// submitted in one go, or throttled to two slices in the queue - another host thread's upload waited until the last byte of the big
// one; the same in the other direction).  Two host threads that stream chunk
// groups through compress and decompress then wait for each other's big copy in turn and the two PCIe directions never overlap.  So a
// big copy goes out in 32 MB slices and the host submits a slice only when the previous one has finished: the stream's queue runs empty
// after every slice, the engine turns to whoever else is waiting, and the copies of two threads alternate.  Cost: the submit latency
// of one slice at a time when the thread has the link for itself (32 MB slices did better than 8 or 16 MB in the streamed e2e leg).
// Big copies of one direction take turns (bench.py e2e trace): two host threads that each stream chunk groups through compress
// start their uploads together, share the link slice by slice, finish together - and then both run their kernels and their small
// downloads while the upload direction idles, in lockstep for the rest of the array.  A process-wide turn
// per direction makes the second thread's big upload wait for the first one's: the threads fall out of step, one uploads while the
// other computes, and the link stays busy.  Small copies (a group's compressed bytes, at most two slices) do not take a turn: they slip
// in between two slices of whoever holds it.  PCOB200_COPY_FIFO=0 restores plain slice-by-slice sharing.
#ifndef PCOB_COPY_FIFO_DEFAULT
#define PCOB_COPY_FIFO_DEFAULT 1
#endif
inline std::mutex& big_copy_turn(cudaMemcpyKind kind) {
  static std::mutex turn[2];
  return turn[kind == cudaMemcpyDeviceToHost ? 1 : 0];
}
inline cudaError_t copy_sliced(void* dst, const void* src, size_t bytes, cudaMemcpyKind kind, cudaStream_t stream) {
  static const size_t SLICE = [] {  // PCOB200_COPY_SLICE_MB: experiments (0 = whole copies)
    const char* e = std::getenv("PCOB200_COPY_SLICE_MB");
    const long mb = e ? std::atol(e) : 32;
    return mb <= 0 ? ~size_t(0) / 4 : size_t(mb) << 20;
  }();
  static const bool FIFO = [] {
    const char* e = std::getenv("PCOB200_COPY_FIFO");
    return e ? e[0] != '0' : PCOB_COPY_FIFO_DEFAULT != 0;
  }();
  if (bytes <= 2 * SLICE) return cudaMemcpyAsync(dst, src, bytes, kind, stream);
  static thread_local cudaEvent_t ev = nullptr;
  if (!ev) {
    cudaError_t e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
    if (e != cudaSuccess) return e;
  }
  std::unique_lock<std::mutex> turn(big_copy_turn(kind), std::defer_lock);
  if (FIFO && (kind == cudaMemcpyHostToDevice || kind == cudaMemcpyDeviceToHost)) turn.lock();  // released when the last slice has been submitted
  for (size_t off = 0; off < bytes; off += SLICE) {
    if (off) {
      cudaError_t e = cudaEventSynchronize(ev);  // the previous slice is done
      if (e != cudaSuccess) return e;
    }
    const size_t len = bytes - off < SLICE ? bytes - off : SLICE;
    cudaError_t e = cudaMemcpyAsync(static_cast<uint8_t*>(dst) + off, static_cast<const uint8_t*>(src) + off, len, kind, stream);
    if (e == cudaSuccess) e = cudaEventRecord(ev, stream);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

// ---- small device -> host readbacks that do not queue on a copy engine --------------------------------------------------------------
// A call reads a few words back between its kernels (the one-pass front end's flags, the file size, the decode statuses) and waits for
// them.  As a cudaMemcpyAsync such a readback is an entry in the device-to-host copy queue - behind whatever 32 MB slice another host
// thread's download has in flight there, many times longer than the group's own kernels in the streamed e2e leg.  publish_kernel
// stores the words into a page-locked, device-
// mapped bounce buffer of the calling thread instead: an ordinary kernel on the call's stream, nothing in any copy queue; the stream
// synchronisation that follows makes the stores visible to the host.  Readbacks beyond the bounce buffer, and PCOB200_READBACK_KERNEL=0,
// take the copy.
__global__ void publish_kernel(uint32_t* __restrict__ dst_mapped, const uint32_t* __restrict__ src, uint32_t n_words) {
  for (uint32_t i = threadIdx.x; i < n_words; i += blockDim.x) dst_mapped[i] = src[i];
}
struct ReadbackBounce {
  void* host = nullptr;
  void* dev = nullptr;
  int device = -1;
  static constexpr size_t CAP = 64 << 10;
  void release() {
    if (host) cudaFreeHost(host);
    host = dev = nullptr;
    device = -1;
  }
};
inline ReadbackBounce& readback_bounce() {
  static thread_local ReadbackBounce b;
  return b;
}
// Copies `bytes` (a multiple of 4, 4-byte aligned source) from device memory to `host_dst` and returns with the stream synchronised.
inline cudaError_t readback_small_sync(void* host_dst, const void* dev_src, size_t bytes, cudaStream_t stream) {
  static const bool use_kernel = [] { const char* e = std::getenv("PCOB200_READBACK_KERNEL"); return !(e && e[0] == '0'); }();
  ReadbackBounce& b = readback_bounce();
  bool ok = use_kernel && bytes <= ReadbackBounce::CAP && (bytes & 3) == 0 && (reinterpret_cast<uintptr_t>(dev_src) & 3) == 0;
  if (ok) {
    int dev = -1;
    if (cudaGetDevice(&dev) != cudaSuccess) ok = false;
    if (ok && b.host && b.device != dev) b.release();
    if (ok && !b.host) {
      if (cudaHostAlloc(&b.host, ReadbackBounce::CAP, cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess || cudaHostGetDevicePointer(&b.dev, b.host, 0) != cudaSuccess) {
        cudaGetLastError();
        b.release();
        ok = false;
      } else {
        b.device = dev;
      }
    }
  }
  if (!ok) {
    cudaError_t e = cudaMemcpyAsync(host_dst, dev_src, bytes, cudaMemcpyDeviceToHost, stream);
    return e != cudaSuccess ? e : cudaStreamSynchronize(stream);
  }
  if (bytes) publish_kernel<<<1, 256, 0, stream>>>(static_cast<uint32_t*>(b.dev), static_cast<const uint32_t*>(dev_src), uint32_t(bytes / 4));
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
  if (e == cudaSuccess && bytes) std::memcpy(host_dst, b.host, bytes);
  return e;
}

// ---- in-place access to page-locked host buffers ("zero copy") -------------------------------------------------------------------------
// A caller's host buffer that is page-locked (cudaHostAlloc / cudaHostRegister: what torch's pin_memory, CuPy's pinned pool and most I/O
// stacks hand out) is addressable by the SMs through the same pointer under unified addressing.  The two big streams of the path are
// touched exactly once by exactly one kernel - the numbers by the split kernel of compress, the decoded numbers by the decode kernel of
// decompress - so those kernels can read / write the host buffer directly over PCIe: no staging buffer in HBM, no copy engine (copies of
// two host threads queue behind each other on an engine, see copy_sliced below; loads and stores of two kernels share the link word by
// word), and the transfer overlaps the kernel's own work.  Bit 0: compress reads its input in place; bit 1: decompress writes its output
// in place.  Pageable buffers (cudaMemoryTypeUnregistered) always take the staged path.  PCOB200_ZEROCOPY overrides the default mask.
#ifndef PCOB_ZEROCOPY_DEFAULT
#define PCOB_ZEROCOPY_DEFAULT 0
#endif
inline std::atomic<int>& zero_copy_mask() {
  static std::atomic<int> m{[] {
    const char* e = std::getenv("PCOB200_ZEROCOPY");
    return e ? std::atoi(e) : PCOB_ZEROCOPY_DEFAULT;
  }()};
  return m;
}
// the device alias of a page-locked host buffer, or nullptr when the buffer is pageable / not addressable from the current device
inline void* mapped_host_ptr(const void* host) {
  if (!host) return nullptr;
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, host) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  if (a.type != cudaMemoryTypeHost || a.devicePointer == nullptr) return nullptr;
  // the staging fallback of compress copies from the same pointer, so insist on the unified-addressing identity
  return a.devicePointer == host ? a.devicePointer : nullptr;
}

// ---- the chain of real chunks among the candidates of a speculative walk (host_api.cu speculative_walk_rounds) ---------------------
// chunk_chain (codec_common.cuh) with the verified chunks' indices collected in file order.
inline std::vector<uint32_t> follow_chunk_chain(const uint64_t* cand, const uint32_t* st, const uint64_t* ends, uint32_t m, uint64_t pos, uint64_t n0,
                                                uint64_t out_off, uint64_t dst_len, uint64_t src_len, uint64_t* next_pos) {
  std::vector<uint32_t> real;
  chunk_chain(cand, st, ends, m, pos, n0, out_off, dst_len, src_len, next_pos, [&](uint32_t k) { real.push_back(k); });
  return real;
}

// ---- grow-only device buffer -----------------------------------------------
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = n + (n >> 3) + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess) { e = cudaMalloc(&p, n); want = n; }
    if (e == cudaSuccess) cap = want;
    return e;
  }
  // grow while keeping the first `keep` bytes (device-to-device copy)
  cudaError_t grow_preserve(size_t n, size_t keep, cudaStream_t stream) {
    if (n <= cap) return cudaSuccess;
    void* np = nullptr;
    size_t want = n + (n >> 2) + 256;
    cudaError_t e = cudaMalloc(&np, want);
    if (e != cudaSuccess) { e = cudaMalloc(&np, n); want = n; }
    if (e != cudaSuccess) return e;
    if (p && keep) {
      e = cudaMemcpyAsync(np, p, keep, cudaMemcpyDeviceToDevice, stream);
      if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    }
    if (p) cudaFree(p);
    p = np;
    cap = want;
    return e;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  template <typename T> T* as() const { return static_cast<T*>(p); }
};

// ---- standalone header (docs/format.md:173-192; pco/src/standalone/decompressor.rs:85-148) ----
struct StandaloneHeader {
  uint32_t standalone_version = 0;
  uint32_t uniform_type = 0;
  uint64_t n_hint = 0;
  uint32_t format_major = 4, format_minor = 1;
  uint64_t first_chunk_byte = 0;
};

// Parses from the first bytes of the file (at most 32 are needed).  `avail` may be shorter than the file.
inline PcoB200Error parse_standalone_header(const uint8_t* b, size_t avail, size_t file_len, StandaloneHeader* h) {
  auto need = [&](size_t n) { return n <= file_len && n <= avail; };
  if (!need(4)) return fail(PCO_B200_INSUFFICIENT_DATA, "[BitReader] out of bounds reading magic header");
  static const uint8_t MAGIC[4] = {112, 99, 111, 33};
  if (std::memcmp(b, MAGIC, 4) != 0) return fail(PCO_B200_CORRUPTION, "magic header does not match \"pco!\"");
  size_t pos = 4;
  // The reference reads this section from a zero-padded buffer and bounds-checks afterwards.
  auto byte_at = [&](size_t i) -> uint8_t { return (i < file_len && i < avail) ? b[i] : 0; };
  uint32_t ver = byte_at(pos);
  if (ver < 2) {
    // versions 0/1 had no standalone header: this byte is the wrapped major version (decompressor.rs:101-107)
    h->standalone_version = ver;
  } else {
    pos += 1;
    h->standalone_version = ver;
    if (ver >= 3) {
      uint8_t t = byte_at(pos);
      pos += 1;
      if (t != 0) {
        if (!nt_valid(t)) return fail(PCO_B200_CORRUPTION, "unknown number type byte: " + std::to_string(t));
        h->uniform_type = t;
      }
    }
    // varint: 6 bits (power - 1), then `power` bits (standalone/decompressor.rs:14-19)
    unsigned __int128 wide = 0;
    for (int i = 0; i < 10; i++) wide |= (unsigned __int128)byte_at(pos + i) << (8 * i);
    uint32_t power = 1 + uint32_t(uint64_t(wide) & 63);
    unsigned __int128 v = wide >> 6;
    uint64_t n_hint = power >= 64 ? uint64_t(v) : uint64_t(v) & ((uint64_t(1) << power) - 1);
    uint32_t total_bits = 6 + power;
    uint32_t nbytes = (total_bits + 7) / 8;
    if (pos + nbytes > file_len) return fail(PCO_B200_INSUFFICIENT_DATA, "[BitReader] out of bounds in standalone header");
    uint32_t pad = nbytes * 8 - total_bits;
    if (pad) {
      uint32_t last = byte_at(pos + nbytes - 1);
      if ((last >> (8 - pad)) != 0) return fail(PCO_B200_CORRUPTION, "standalone size hint");
    }
    h->n_hint = n_hint;
    pos += nbytes;
  }
  if (pos > file_len) return fail(PCO_B200_INSUFFICIENT_DATA, "[BitReader] out of bounds in standalone header");
  if (h->standalone_version > 3)
    return fail(PCO_B200_CORRUPTION, "file's standalone version exceeds max supported (3); consider upgrading pco");
  // wrapped header (metadata/format_version.rs:65-85)
  uint8_t major = byte_at(pos);
  pos += 1;
  uint8_t minor = 0;
  if (major >= 4) { minor = byte_at(pos); pos += 1; }
  if (major > 4) return fail(PCO_B200_CORRUPTION, "file's format version cannot be decompressed by this library version");
  if (pos > file_len) return fail(PCO_B200_INSUFFICIENT_DATA, "[BitReader] out of bounds reading format version");
  h->format_major = major;
  h->format_minor = minor;
  h->first_chunk_byte = pos;
  return PCO_B200_OK;
}

// ---- size guarantees (pco/src/standalone/guarantee.rs:11-38, wrapped/guarantee.rs:11-37) ----
inline size_t standalone_header_size() { return 4 + 1 + (6 + 64 + 8 + 7) / 8 + 2; }
inline size_t baseline_chunk_meta_size(uint32_t latent_bits) {
  // mode 4 bits + DeltaEncoding::MAX_BIT_SIZE (4+5+5+64+32*32) + 4 + 15 + one bin (0 + L + log2(L)+1)
  size_t bits = 4 + (4 + 5 + 5 + 64 + 32 * 32) + 4 + 15 + (latent_bits + offset_bits_bits(latent_bits));
  return (bits + 7) / 8;
}
inline size_t wrapped_chunk_size_guarantee(uint32_t latent_bits, size_t n) {
  return baseline_chunk_meta_size(latent_bits) + (n * size_t(latent_bits) + 7) / 8;
}
inline size_t standalone_chunk_size_guarantee(uint32_t latent_bits, size_t n) { return 1 + 3 + wrapped_chunk_size_guarantee(latent_bits, n); }

}  // namespace pcob200
