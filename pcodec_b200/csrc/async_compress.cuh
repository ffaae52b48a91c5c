// Kernels and host steps of pco_b200_compress_async: an explicit-config compress with no host decision between launches, so the call can
// be queued behind other work or captured in a CUDA graph.  The plan fixes n, the chunk layout (EqualPagesUpTo: the first `rem` chunks
// hold low + 1 numbers, the others low), the mode, the delta order and one unoptimized_bins_log; everything that depends on the numbers
// is decided on the device.  The ordinary encode kernels run unchanged.  Each choice compress_typed makes on the host from a readback
// becomes a gate kernel that writes, per choice, a copy of the chunk starts that is either the real one or all zeros: a kernel launched
// with the zero copy sees chunks of 0 numbers and leaves at its first lines.  Choices and their gates:
//   one-pass or two-kernel front end (split_count_kernel's flag)  acomp_two_gate_kernel: split_delta_kernel's starts, ChunkEnc reset
//   counting or sorting planner, per var (the range bits)           acomp_var_gate_kernel: the counting probe, the sort path, bin_lut_kernel,
//                                                                   bin_kernel
//   16-bit keys or 64-bit latents in pack_kernel, per var           acomp_pack_gate_kernel: one copy of the ChunkEnc table per choice, whose
//                                                                   chunks the launches of the other choices find out of dst_cap
// acomp_init_kernel lays out the chunks, the header and the index header; acomp_finish_kernel writes the PcoB200AsyncCompressStatus.
// enqueue_encode_kernels and enqueue_pack make the gated launches, which the batch calls (async_compress_files.cuh) share.
#pragma once
#include "../../include/pco_b200.h"
#include "compress_host.cuh"

namespace pcob200 {

constexpr int ACOMP_THREADS = 256;
constexpr uint32_t ACOMP_GATES_PER_VAR = 4;  // counting probe, sort path, bin_lut_kernel, bin_kernel

// Chunk geometry of a plan: its EqualPages chunks, the largest chunk's size and the latent slots
struct AcompGeom {
  uint64_t n, n_chunks, low, rem, max_n, slots;
  uint32_t bpc, tiles;
};
inline AcompGeom acomp_geom(uint64_t n, uint64_t max_page_n) {
  const EqualPages ep = equal_pages(n, max_page_n);
  AcompGeom g = {};
  g.n = n;
  g.n_chunks = ep.n_chunks;
  g.low = ep.low;
  g.rem = ep.rem;
  g.max_n = ep.size(0);
  g.slots = ep.row_start(ep.n_chunks);
  g.bpc = n_batches_of(uint32_t(g.max_n));
  g.tiles = uint32_t((g.max_n + SPLIT_TILE - 1) / SPLIT_TILE);
  return g;
}

// Workspace of one in-flight call, byte offsets of 256-byte aligned regions.  head: split_count_kernel's flags (2 words), the range bits
// per var (2 words), the file size (u64 at byte 16), the standalone header (byte 64).
struct AcompLayout {
  uint64_t chunks, copies, starts, rows, gates, eoff, seg, plans, probes, ob_sum, ans_sum, entries;
  uint64_t lat[MAX_VARS], keys_a, keys_b, key16[MAX_VARS], sym[MAX_VARS], ans[MAX_VARS];
  uint64_t total;
};
inline uint64_t acomp_align(uint64_t x) { return (x + 255) & ~uint64_t(255); }
inline AcompLayout acomp_layout(const AcompGeom& g, uint32_t lbytes, uint32_t n_vars) {
  AcompLayout l = {};
  uint64_t at = 256;
  auto take = [&](uint64_t bytes) { const uint64_t o = at; at += acomp_align(bytes); return o; };
  const uint64_t nc = g.n_chunks, cvb = nc * MAX_VARS * g.bpc;
  l.chunks = take(nc * sizeof(ChunkEnc));
  l.copies = take((uint64_t(1) << n_vars) * nc * sizeof(ChunkEnc));
  l.starts = take((nc + 1) * 8);
  l.rows = take((nc + 1) * 8);
  l.gates = take((1 + ACOMP_GATES_PER_VAR * n_vars) * (nc + 1) * 8);
  l.eoff = take(nc * 8);
  l.seg = take(2 * nc * 8);
  l.plans = take(nc * MAX_VARS * sizeof(VarPlan));
  l.probes = take(nc * sizeof(PlanProbes));
  l.ob_sum = take(cvb * 4);
  l.ans_sum = take(cvb * 4);
  l.entries = take(cvb * sizeof(BatchEntry));
  // per number: the 64-bit path's latents and sort keys, the counting path's 16-bit keys, symbols and tANS fields (each + 64 bytes of
  // slack, as compress_typed reserves them)
  for (uint32_t v = 0; v < n_vars; v++) l.lat[v] = take(g.slots * lbytes + 64);
  l.keys_a = take(g.slots * lbytes + 64);
  l.keys_b = take(g.slots * lbytes + 64);
  for (uint32_t v = 0; v < n_vars; v++) {
    l.key16[v] = take(g.slots * 2 + 64);
    l.sym[v] = take(g.slots + 64);
    l.ans[v] = take(g.slots * 2 + 64);
  }
  l.total = at;
  return l;
}

// What the launches take by value
struct AcompArgs {
  uint64_t n, n_chunks, low, rem;
  uint64_t dst_cap, index_bytes;   // index_bytes: 0 = no index this call
  uint32_t header_bytes, n_vars;
  uint8_t* ws;
  uint8_t* dst;
  uint8_t* index;
  AcompLayout lay;
  uint8_t header[STANDALONE_HEADER_MAX];
};
struct AcompHead {
  uint32_t flags[2];      // split_count_kernel: [0] range bits, [1] some chunk spans 2^15 or more
  uint32_t range_bits[MAX_VARS];
  uint64_t total;         // file bytes (chunk_offsets_kernel)
};
__device__ inline uint64_t* acomp_gate(const AcompArgs& a, uint32_t g) { return reinterpret_cast<uint64_t*>(a.ws + a.lay.gates) + uint64_t(g) * (a.n_chunks + 1); }
// the chunk starts the init kernel wrote (acomp_init_kernel, or acf_init_kernel for a batch of files): the gates copy them
__device__ inline const uint64_t* acomp_starts(const AcompArgs& a) { return reinterpret_cast<const uint64_t*>(a.ws + a.lay.starts); }

// Grid-stride over every per-chunk and per-word job: ChunkEnc records, chunk starts and row bases, index entry offsets, the zeroed
// offset-bit sums (fallback chunks leave their secondary var's untouched) and the zeroed index body; thread 0 writes the head, the
// standalone header, the index header and, when n == 0, the whole file (header and terminator).
__global__ void __launch_bounds__(ACOMP_THREADS) acomp_init_kernel(AcompArgs a, uint32_t bpc) {
  const uint64_t nc = a.n_chunks;
  ChunkEnc* chunks = reinterpret_cast<ChunkEnc*>(a.ws + a.lay.chunks);
  uint64_t* starts = reinterpret_cast<uint64_t*>(a.ws + a.lay.starts);
  uint64_t* rows = reinterpret_cast<uint64_t*>(a.ws + a.lay.rows);
  uint64_t* eoff = reinterpret_cast<uint64_t*>(a.ws + a.lay.eoff);
  uint32_t* ob_sum = reinterpret_cast<uint32_t*>(a.ws + a.lay.ob_sum);
  const EqualPages ep = {nc, a.low, a.rem};
  const uint64_t n_sums = nc * MAX_VARS * bpc;
  const uint64_t idx_vecs = a.index_bytes > sizeof(IndexHeader) ? (a.index_bytes - sizeof(IndexHeader)) / 16 : 0;
  const uint64_t jobs = max(max(nc + 1, n_sums), idx_vecs);
  for (uint64_t t = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; t < jobs; t += uint64_t(gridDim.x) * blockDim.x) {
    if (t <= nc) {
      starts[t] = ep.start(t);
      rows[t] = ep.row_start(t);
      if (t < nc) {
        reset_chunk_enc(&chunks[t]);
        eoff[t] = ep.entries_offset(a.n_vars, t);
      }
    }
    if (t < n_sums) ob_sum[t] = 0;
    if (t < idx_vecs) reinterpret_cast<uint4*>(a.index + sizeof(IndexHeader))[t] = make_uint4(0, 0, 0, 0);
  }
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  AcompHead* h = reinterpret_cast<AcompHead*>(a.ws);
  h->flags[0] = h->flags[1] = 0;
  h->range_bits[0] = h->range_bits[1] = 0;
  h->total = a.n == 0 ? a.header_bytes + 1 : 0;  // n == 0: header and terminator only (standalone/simple.rs:62-91)
  for (uint32_t i = 0; i < a.header_bytes; i++) (a.ws + 64)[i] = a.header[i];
  if (a.n == 0 && a.header_bytes + 1 <= a.dst_cap) {
    for (uint32_t i = 0; i < a.header_bytes; i++) a.dst[i] = a.header[i];
    a.dst[a.header_bytes] = 0;
  }
  if (a.index_bytes) {
    IndexHeader ih;
    memset(&ih, 0, sizeof(ih));
    ih.magic = INDEX_MAGIC;
    ih.version = 1;
    ih.n_chunks = nc;
    ih.n_total = a.n;
    ih.chunks_offset = sizeof(IndexHeader);
    if (a.n == 0) ih.file_len = ih.end_byte = a.header_bytes + 1;  // with chunks, emit_index_kernel writes both
    *reinterpret_cast<IndexHeader*>(a.index) = ih;
  }
}

// Behind split_count_kernel (or first, for the two-var modes: always_two): the two-kernel front end runs when some chunk's latents span
// 2^15 or more.  Then the ChunkEnc records start over (init_chunks_kernel in plan_front) and split_delta_kernel sees the real starts.
__global__ void __launch_bounds__(ACOMP_THREADS) acomp_two_gate_kernel(AcompArgs a, uint32_t always_two) {
  const AcompHead* h = reinterpret_cast<const AcompHead*>(a.ws);
  const bool two = always_two || h->flags[1] != 0;
  ChunkEnc* chunks = reinterpret_cast<ChunkEnc*>(a.ws + a.lay.chunks);
  uint64_t* g = acomp_gate(a, 0);
  const uint64_t* starts = acomp_starts(a);
  for (uint64_t c = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; c <= a.n_chunks; c += uint64_t(gridDim.x) * blockDim.x) {
    g[c] = two ? starts[c] : 0;
    if (two && c < a.n_chunks) reset_chunk_enc(&chunks[c]);
  }
}

// One CTA, behind split_delta_kernel.  Per var: the range bits of the call (range_bits_kernel's maximum over the chunks, which also sets
// key_base = vmin, on the two-kernel path; split_count_kernel's flags[0] on the one-pass path), then the starts of the four gated
// launches: the counting probe (two-kernel path, range <= PLAN_MAX_COUNT_BITS), the sort path (range above), bin_lut_kernel (range <=)
// and bin_kernel (above).
__global__ void __launch_bounds__(1024) acomp_var_gate_kernel(AcompArgs a, uint32_t always_two) {
  __shared__ uint32_t s_bits;
  AcompHead* h = reinterpret_cast<AcompHead*>(a.ws);
  ChunkEnc* chunks = reinterpret_cast<ChunkEnc*>(a.ws + a.lay.chunks);
  const bool two = always_two || h->flags[1] != 0;
  for (uint32_t v = 0; v < a.n_vars; v++) {
    if (threadIdx.x == 0) s_bits = two ? 0u : h->flags[0];
    __syncthreads();
    if (two)
      for (uint64_t c = threadIdx.x; c < a.n_chunks; c += blockDim.x) {
        const uint64_t lo = chunks[c].vmin[v], hi = chunks[c].vmax[v];
        atomicMax(&s_bits, hi > lo ? 64 - __clzll((long long)(hi - lo)) : 0u);
        chunks[c].key_base[v] = lo;  // plan_probe_kernel's keys are latent - vmin
      }
    __syncthreads();
    const uint32_t bits = s_bits;
    if (threadIdx.x == 0) h->range_bits[v] = bits;
    const bool narrow = bits <= PLAN_MAX_COUNT_BITS;
    const bool on[ACOMP_GATES_PER_VAR] = {two && narrow, two && !narrow, narrow, !narrow};
    for (uint64_t c = threadIdx.x; c <= a.n_chunks; c += blockDim.x) {
      const uint64_t s = acomp_starts(a)[c];
      for (uint32_t k = 0; k < ACOMP_GATES_PER_VAR; k++) acomp_gate(a, 1 + ACOMP_GATES_PER_VAR * v + k)[c] = on[k] ? s : 0;
    }
    __syncthreads();
  }
}

// Behind chunk_offsets_kernel: copy k of the ChunkEnc table serves the pack_kernel launch whose var v reads 64-bit latents when bit v of k
// is set and 16-bit keys otherwise.  In the copies of the choices the range bits did not make, every chunk lies past dst_cap.
__global__ void __launch_bounds__(ACOMP_THREADS) acomp_pack_gate_kernel(AcompArgs a) {
  const AcompHead* h = reinterpret_cast<const AcompHead*>(a.ws);
  const ChunkEnc* chunks = reinterpret_cast<const ChunkEnc*>(a.ws + a.lay.chunks);
  ChunkEnc* copies = reinterpret_cast<ChunkEnc*>(a.ws + a.lay.copies);
  uint32_t live = 0;
  for (uint32_t v = 0; v < a.n_vars; v++) live |= (h->range_bits[v] > PLAN_MAX_COUNT_BITS ? 1u : 0u) << v;
  const uint64_t n_copies = uint64_t(1) << a.n_vars;
  for (uint64_t t = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; t < n_copies * a.n_chunks; t += uint64_t(gridDim.x) * blockDim.x) {
    const uint64_t k = t / a.n_chunks, c = t % a.n_chunks;
    ChunkEnc ch = chunks[c];
    if (k != live) ch.out_offset = ~uint64_t(0) - ch.chunk_bytes;  // out_offset + chunk_bytes exceeds any out_cap below 2^64 - 1
    copies[t] = ch;
  }
}

// One thread: the outcome.
__global__ void acomp_finish_kernel(AcompArgs a, PcoB200AsyncCompressStatus* __restrict__ out) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  const uint64_t total = reinterpret_cast<const AcompHead*>(a.ws)->total;
  PcoB200AsyncCompressStatus s;
  const bool fits = total <= a.dst_cap;
  s.kind = fits ? PCO_B200_OK : PCO_B200_IO;
  s.device_status = fits ? 0u : uint32_t(PCO_B200_ASYNC_DST_FULL);
  s.file_bytes = total;
  s.n_written = fits ? total : 0;
  s.index_bytes = a.index_bytes;
  *out = s;
}

// ---- host steps

// The clause every asynchronous compress plan check shares: the spec fields as the plan functions fill them (P: any of the three plans)
template <typename P>
inline bool acomp_spec_ok(const P* p) {
  return p && nt_valid(p->dtype) && p->mode <= MODE_FLOAT_QUANT && p->n_vars == (p->mode == MODE_CLASSIC ? 1u : 2u) && p->order <= MAX_ORDER;
}

inline PcoB200Error acomp_check_plan(const PcoB200AsyncCompressPlan* p, AcompGeom* g, AcompLayout* lay) {
  if (!acomp_spec_ok(p) || p->bins_log > ENC_NARROW_BINS_LOG || (p->index_cap != 0 && p->index_bytes > p->index_cap))
    return fail(PCO_B200_INVALID_ARGUMENT, "the plan was not made by pco_b200_compress_async_plan");
  *g = acomp_geom(p->n, p->max_page_n);
  *lay = acomp_layout(*g, nt_bits(p->dtype) / 8, p->n_vars);
  if (p->workspace_bytes != lay->total || p->index_bytes != equal_pages(p->n, p->max_page_n).index_bytes(p->n_vars))
    return fail(PCO_B200_INVALID_ARGUMENT, "the plan was not made by pco_b200_compress_async_plan");
  return PCO_B200_OK;
}

// The workspace regions of an AcompLayout as the encode kernels take them; the secondary var's are null for one var.
template <typename L>
struct AcompRegions {
  AcompHead* head;
  ChunkEnc *chunks, *copies;
  VarPlan* plans;
  PlanProbes* probes;
  uint64_t *gates, *seg_begin, *seg_end;
  L *lat[MAX_VARS], *keys_a, *keys_b;
  uint16_t *key16[MAX_VARS], *ans[MAX_VARS];
  uint8_t* sym[MAX_VARS];
  uint32_t *ob_sum, *ans_sum;
  BatchEntry* entries;
};
template <typename L>
AcompRegions<L> acomp_regions(const AcompArgs& a) {
  uint8_t* ws = a.ws;
  const AcompLayout& l = a.lay;
  const bool two = a.n_vars > 1;
  AcompRegions<L> r;
  r.head = reinterpret_cast<AcompHead*>(ws);
  r.chunks = reinterpret_cast<ChunkEnc*>(ws + l.chunks);
  r.copies = reinterpret_cast<ChunkEnc*>(ws + l.copies);
  r.plans = reinterpret_cast<VarPlan*>(ws + l.plans);
  r.probes = reinterpret_cast<PlanProbes*>(ws + l.probes);
  r.gates = reinterpret_cast<uint64_t*>(ws + l.gates);
  for (uint32_t v = 0; v < MAX_VARS; v++) {
    const bool on = v == 0 || two;
    r.lat[v] = on ? reinterpret_cast<L*>(ws + l.lat[v]) : nullptr;
    r.key16[v] = on ? reinterpret_cast<uint16_t*>(ws + l.key16[v]) : nullptr;
    r.sym[v] = on ? ws + l.sym[v] : nullptr;
    r.ans[v] = on ? reinterpret_cast<uint16_t*>(ws + l.ans[v]) : nullptr;
  }
  r.keys_a = reinterpret_cast<L*>(ws + l.keys_a);
  r.keys_b = reinterpret_cast<L*>(ws + l.keys_b);
  r.seg_begin = reinterpret_cast<uint64_t*>(ws + l.seg);
  r.seg_end = r.seg_begin + a.n_chunks;
  r.ob_sum = reinterpret_cast<uint32_t*>(ws + l.ob_sum);
  r.ans_sum = reinterpret_cast<uint32_t*>(ws + l.ans_sum);
  r.entries = reinterpret_cast<BatchEntry*>(ws + l.entries);
  return r;
}

// The EncParams of the encode stage: the spec fields of the plan (P: a compress_async or compress_files_async plan), the chunks of g,
// the starts and row bases the init kernel wrote, and the caller's n_total and unoptimized_bins_log (or level, for CHUNK_BINS).
template <typename P>
EncParams acomp_enc_params(const P& p, const AcompGeom& g, const AcompArgs& a, const void* nums, uint64_t n_total, uint32_t bins_log) {
  EncParams ep = enc_params(p.dtype, p.uniform_type_header ? p.dtype : 0, ModeSel{p.mode, p.mode_base, p.base_bits, p.inv_base_bits, p.mode_k}, p.order,
                            bins_log);
  ep.n_total = n_total;
  ep.n_chunks = uint32_t(g.n_chunks);
  ep.max_chunk_n = uint32_t(g.max_n);
  ep.nums = nums;
  ep.chunk_starts = reinterpret_cast<const uint64_t*>(a.ws + a.lay.starts);
  ep.row_base = reinterpret_cast<const uint64_t*>(a.ws + a.lay.rows);
  return ep;
}

// The gated encode kernels of every asynchronous compress, from the front end to layout_kernel, behind the init kernel that wrote the
// starts, row bases and head.  CHUNK_BINS: split_count_kernel and the planner kernels compute each chunk's unoptimized_bins_log from
// the level in ep.bins_log[0] and its n (a batch); otherwise they take ep.bins_log as it is.
template <typename L, bool CHUNK_BINS>
void enqueue_encode_kernels(const AcompGeom& g, const AcompArgs& a, const EncParams& ep, const AsyncLaunch& ln) {
  const cudaStream_t stream = ln.stream;
  const uint32_t nc = uint32_t(g.n_chunks), bpc = g.bpc, tiles = g.tiles, n_vars = ep.n_vars;
  constexpr uint32_t LBITS = sizeof(L) * 8;
  constexpr size_t RS_SMEM = size_t(RS_WARPS) * RS_BINS * sizeof(uint32_t);
  const AcompRegions<L> r = acomp_regions<L>(a);
  auto gated = [&](uint32_t gate) { EncParams e = ep; e.chunk_starts = r.gates + uint64_t(gate) * (g.n_chunks + 1); return e; };
  const uint32_t always_two = n_vars > 1 ? 1u : 0u;
  // ---- front end: the one-pass kernel for Classic, then the two-kernel path behind its flag (always, for the two-var modes)
  if (!always_two) {
    ln.begin("split_count_kernel");
    split_count_kernel<L, CHUNK_BINS><<<nc, SC_THREADS, size_t(SC_N) * 4, stream>>>(ep, r.chunks, r.probes, r.key16[0], r.head->flags);
    ln.end();
  }
  acomp_two_gate_kernel<<<(nc + ACOMP_THREADS) / ACOMP_THREADS, ACOMP_THREADS, 0, stream>>>(a, always_two);
  const EncParams e_two = gated(0);
  ln.begin("split_delta_kernel");
  switch (ep.mode) {
    case MODE_CLASSIC: split_delta_kernel<L, MODE_CLASSIC><<<nc * tiles, SPLIT_THREADS, 0, stream>>>(e_two, tiles, r.lat[0], r.lat[1], r.chunks); break;
    case MODE_INT_MULT: split_delta_kernel<L, MODE_INT_MULT><<<nc * tiles, SPLIT_THREADS, 0, stream>>>(e_two, tiles, r.lat[0], r.lat[1], r.chunks); break;
    case MODE_FLOAT_QUANT: split_delta_kernel<L, MODE_FLOAT_QUANT><<<nc * tiles, SPLIT_THREADS, 0, stream>>>(e_two, tiles, r.lat[0], r.lat[1], r.chunks); break;
    default: split_delta_kernel<L, MODE_FLOAT_MULT><<<nc * tiles, SPLIT_THREADS, 0, stream>>>(e_two, tiles, r.lat[0], r.lat[1], r.chunks); break;
  }
  ln.end();
  acomp_var_gate_kernel<<<1, 1024, 0, stream>>>(a, always_two);
  // ---- planner per var: counting probe or sort path (whichever the range bits gate on), then the solver on the probes either left
  // (the one-pass kernel writes var 0's probes itself).  The counting probe takes the counters of PLAN_MAX_COUNT_BITS and the sort all
  // bits of the number type: both give the probes of the narrower range, and the number of sort passes - so the buffer the sorted keys
  // end in - is fixed.
  const L* sorted = ((LBITS + RS_BITS - 1) / RS_BITS) & 1 ? r.keys_b : r.keys_a;
  for (uint32_t v = 0; v < n_vars; v++) {
    const EncParams e_count = gated(1 + ACOMP_GATES_PER_VAR * v), e_sort = gated(2 + ACOMP_GATES_PER_VAR * v);
    ln.begin("plan_probe_kernel_counting");
    plan_probe_kernel<L, true, false, CHUNK_BINS><<<nc, PLAN_THREADS, ((size_t(1) << PLAN_MAX_COUNT_BITS) + 1) * 4 + 16, stream>>>(
        e_count, r.lat[v], r.chunks, r.probes, int(v), PLAN_MAX_COUNT_BITS, r.key16[v]);
    ln.end();
    ln.begin("sort_keys_kernel");
    sort_keys_kernel<L><<<nc * tiles, 256, 0, stream>>>(e_sort, tiles, r.lat[v], r.keys_a, r.chunks, int(v));
    ln.end();
    segment_offsets_kernel<<<(nc + 255) / 256, 256, 0, stream>>>(e_sort, v == 0 ? ep.order : 0, r.seg_begin, r.seg_end);
    ln.begin("radix_sort_segments_kernel");
    radix_sort_segments_kernel<L><<<nc, RS_THREADS, RS_SMEM, stream>>>(r.keys_a, r.keys_b, r.seg_begin, r.seg_end, LBITS);
    ln.end();
    ln.begin("plan_probe_kernel_sorted");
    plan_probe_kernel<L, false, false, CHUNK_BINS><<<nc, PLAN_THREADS, 16, stream>>>(e_sort, sorted, r.chunks, r.probes, int(v), LBITS, nullptr);
    ln.end();
    ln.begin("plan_solve_kernel");
    plan_solve_kernel<L, CHUNK_BINS><<<nc, SOLVE_THREADS, 0, stream>>>(ep, r.probes, r.chunks, r.plans, int(v));
    ln.end();
  }
  fallback_kernel<false><<<(nc + 255) / 256, 256, 0, stream>>>(ep, r.plans, r.chunks, 0u);
  // ---- K3 per var: the lookup-table binning on the 16-bit keys, or the search over the 64-bit latents
  const uint32_t parts = (bpc + BINL_BATCHES - 1) / BINL_BATCHES, groups = (bpc + 7) / 8;
  for (uint32_t v = 0; v < n_vars; v++) {
    ln.begin("bin_lut_kernel");
    bin_lut_kernel<L><<<nc * parts, BINL_THREADS, (size_t(1) << PLAN_MAX_COUNT_BITS) + 16, stream>>>(gated(3 + ACOMP_GATES_PER_VAR * v), bpc, parts, r.key16[v],
                                                                                                    r.plans, r.chunks, r.sym[v], r.ob_sum, int(v), PLAN_MAX_COUNT_BITS);
    ln.end();
    ln.begin("bin_kernel");
    bin_kernel<L, false><<<nc * groups, BIN_THREADS, 0, stream>>>(gated(4 + ACOMP_GATES_PER_VAR * v), bpc, r.lat[v], r.plans, r.chunks, r.sym[v], r.ob_sum, int(v));
    ln.end();
  }
  ln.begin("ans_encode_kernel");
  ans_encode_kernel<false><<<nc * MAX_VARS, ANS_THREADS, 0, stream>>>(ep, bpc, r.plans, r.chunks, r.sym[0], r.sym[1], r.ans[0], r.ans[1], r.ans_sum, r.entries, nullptr);
  ln.end();
  ln.begin("layout_kernel");
  layout_kernel<false><<<nc, LAYOUT_THREADS, 0, stream>>>(ep, bpc, r.plans, r.chunks, r.ans_sum, r.ob_sum, r.entries);
  ln.end();
}

// K5, behind the launches that place each chunk (ChunkEnc::out_offset): the pack gate, then one pack_kernel per choice of keys or
// latents; only the one the range bits made finds its chunks inside dst_cap.
template <typename L>
void enqueue_pack(const AcompGeom& g, const AcompArgs& a, const EncParams& ep, const AsyncLaunch& ln) {
  const cudaStream_t stream = ln.stream;
  const AcompRegions<L> r = acomp_regions<L>(a);
  const uint64_t n_copies = uint64_t(1) << a.n_vars;
  acomp_pack_gate_kernel<<<uint32_t(std::min<uint64_t>(1024, (n_copies * g.n_chunks + ACOMP_THREADS - 1) / ACOMP_THREADS)), ACOMP_THREADS, 0, stream>>>(a);
  const uint64_t out_cap = std::min<uint64_t>(a.dst_cap, ~uint64_t(0) - 1);
  ln.begin("pack_kernel");
  for (uint64_t k = 0; k < n_copies; k++)
    pack_kernel<L><<<uint32_t(g.n_chunks), PACK_THREADS, sizeof(PackSmem), stream>>>(ep, g.bpc, r.lat[0], r.lat[1], r.plans, r.copies + k * g.n_chunks, r.sym[0],
                                                                                     r.sym[1], r.ans[0], r.ans[1], r.entries, a.dst, out_cap,
                                                                                     (k & 1) ? nullptr : r.key16[0], (a.n_vars > 1 && !(k & 2)) ? r.key16[1] : nullptr);
  ln.end();
}

template <typename L>
void acomp_launch(const PcoB200AsyncCompressPlan& p, const AcompGeom& g, const AcompArgs& a, const void* nums, PcoB200AsyncCompressStatus* status,
                  const AsyncLaunch& ln) {
  const cudaStream_t stream = ln.stream;
  const uint32_t nc = uint32_t(g.n_chunks);
  const uint32_t init_ctas = uint32_t(std::min<uint64_t>(1024, std::max<uint64_t>({g.n_chunks + 1, g.n_chunks * MAX_VARS * g.bpc, a.index_bytes / 16}) / ACOMP_THREADS + 1));
  ln.begin("acomp_init_kernel");
  acomp_init_kernel<<<init_ctas, ACOMP_THREADS, 0, stream>>>(a, g.bpc);
  ln.end();
  if (p.n > 0) {
    const EncParams ep = acomp_enc_params(p, g, a, nums, p.n, p.bins_log);
    const AcompRegions<L> r = acomp_regions<L>(a);
    enqueue_encode_kernels<L, false>(g, a, ep, ln);
    chunk_offsets_kernel<<<1, 1024, 0, stream>>>(r.chunks, nc, a.header_bytes, 1u, &r.head->total);
    enqueue_pack<L>(g, a, ep, ln);
    header_footer_kernel<<<1, 32, 0, stream>>>(a.dst, std::min<uint64_t>(a.dst_cap, ~uint64_t(0) - 1), a.ws + 64, a.header_bytes, &r.head->total);
    if (a.index_bytes)
      emit_index_kernel<<<nc, 256, 0, stream>>>(ep, g.bpc, r.chunks, r.entries, a.index, sizeof(IndexHeader), reinterpret_cast<const uint64_t*>(a.ws + a.lay.eoff),
                                                &r.head->total, 1u, 0u, 0, 1u);
  }
  ln.begin("acomp_finish_kernel");
  acomp_finish_kernel<<<1, 32, 0, stream>>>(a, status);
  ln.end();
}

}  // namespace pcob200
