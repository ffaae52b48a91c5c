// Kernels of pco_b200_filter_files_async: the files pco_b200_decompress_files_async decodes, with only the numbers inside a closed
// interval written out, in row order, with their positions in the files' concatenation.  The files call's launches (af_files_kernel ..
// af_finish_kernel, async_files_kernels.cuh) run unchanged with rows_cap in the role of dst_cap; around them:
//   ff_map_kernel        before the decode: the slot map (record r -> r) the FILT decode kernels read, and the cold list emptied;
//   fused_narrow_kernel<L, false, true>, symwalk_kernel<false>, decode_kernel<L, 1 / 2, false, true>  the FILT instantiations
//                        (decode_kernels.cuh, filt_store8), each batch's matches staged in its own slot;
//   ff_cold_list_kernel  between the decode stage and cold_chunks_kernel: the records the fast kernels left to the catch-all decoder;
//   cold_chunks_kernel<L>  unchanged, decoding those records into the value staging (each record's numbers at its rows);
//   ff_cold_kernel<L>    the cold list's records filtered in place into their slots;
//   fl_count_kernel, ff_finish_kernel, fl_gather_kernel  as pco_b200_filter_pages_async (async_filter_kernels.cuh), with the files call's
//                        outcome in place of the pages call's.
#pragma once
#include "async_filter_kernels.cuh"
#include "async_files_kernels.cuh"

namespace pcob200 {

constexpr int FF_THREADS = 256;    // ff_map_kernel and ff_cold_list_kernel: records per CTA
constexpr int FF_COLD_CTAS = 128;  // ff_cold_kernel's largest grid; its CTAs stride over the cold list

// Workspace of one in-flight call: the files call's (af_layout with dst_cap = rows_cap) | the files status | FlState | per slot: count,
// row | CTA sums of the counts | value staging (rows_cap numbers of elem bytes) | offset staging (rows_cap bytes) | the slot map
// (max_chunks words) | the cold list (its length, then up to max_chunks records).  Each region 256-byte aligned.  The batch slots are the
// pages filter's (fl_slots) with the records of the merged chunk table in the role of pages.
struct FfLayout : AfLayout {
  uint64_t fstatus, fstate, counts, rows, cparts, stage, soffs, slot_map, cold_list, ff_total;
};
__host__ __device__ inline FfLayout ff_layout(uint64_t max_files, uint64_t max_chunks, uint64_t rows_cap, uint32_t elem) {
  FfLayout l;
  static_cast<AfLayout&>(l) = af_layout(max_files, max_chunks, rows_cap);
  const uint64_t slots = fl_slots(max_chunks, rows_cap);
  l.fstatus = l.total;
  l.fstate = l.fstatus + async_align(sizeof(PcoB200AsyncFilesStatus));
  l.counts = l.fstate + async_align(sizeof(FlState));
  l.rows = l.counts + async_align(slots * sizeof(uint32_t));
  l.cparts = l.rows + async_align(slots * sizeof(uint64_t));
  l.stage = l.cparts + async_align(ctas_of<FL_THREADS>(slots) * sizeof(uint64_t));
  l.soffs = l.stage + async_align(rows_cap * elem);
  l.slot_map = l.soffs + async_align(rows_cap);
  l.cold_list = l.slot_map + async_align(max_chunks * sizeof(uint32_t));
  l.ff_total = l.cold_list + async_align((max_chunks + 1) * sizeof(uint32_t));
  return l;
}

// ceil(max_chunks / FF_THREADS) CTAs: map[r] = r, so the FILT decode kernels put batch b of record r (its numbers from row O) in slot
// O / 256 + r + b; and the cold list's length set to 0 for ff_cold_list_kernel.
__global__ void __launch_bounds__(FF_THREADS) ff_map_kernel(uint64_t max_chunks, uint32_t* __restrict__ map, uint32_t* __restrict__ cold_list) {
  const uint64_t r = uint64_t(blockIdx.x) * FF_THREADS + threadIdx.x;
  if (r < max_chunks) map[r] = uint32_t(r);
  if (r == 0) cold_list[0] = 0;
}

// ceil(max_chunks / FF_THREADS) CTAs, after the decode stage: the records of the chunks decoded ([0, chk->n_chunks)) that the fast kernels
// reported ST_UNSUPPORTED for - exactly those cold_chunks_kernel decodes next - appended to the cold list in any order.  Recorded here
// because cold_chunks_kernel overwrites their statuses.
__global__ void __launch_bounds__(FF_THREADS) ff_cold_list_kernel(const AsyncCheck* __restrict__ chk, const uint32_t* __restrict__ statuses,
                                                                  uint32_t* __restrict__ cold_list) {
  const uint64_t r = uint64_t(blockIdx.x) * FF_THREADS + threadIdx.x;
  if (r < chk->n_chunks && statuses[r] == ST_UNSUPPORTED) cold_list[1 + atomicAdd(&cold_list[0], 1u)] = uint32_t(r);
}

// min(max_chunks, FF_COLD_CTAS) CTAs striding over the cold list: each record, decoded into the value staging by cold_chunks_kernel,
// filtered in place.  A record whose decode failed is filtered too; the call then fails and gathers nothing.  AGG: reduced into the
// slots instead.
template <typename L, bool AGG = false>
__global__ void __launch_bounds__(FL_THREADS) ff_cold_kernel(const uint32_t* __restrict__ cold_list, const IndexChunk* __restrict__ table, FiltStage f,
                                                             uint32_t dtype, L* __restrict__ stage) {
  const uint32_t n_cold = cold_list[0];
  if (blockIdx.x >= n_cold) return;
  const FiltKey key = filt_bounds<L>(f.interval, dtype);
  for (uint32_t k = blockIdx.x; k < n_cold; k += gridDim.x) {
    const uint32_t r = cold_list[1 + k];
    const IndexChunk rec = table[r];
    fl_filter_in_place<L, AGG>(f, key, rec, r, stage);
  }
}

// One CTA: fl_finish_kernel with the files call's outcome: a refusal or failure as that call reports it (no matches), else success, or
// PCO_B200_IO when the matches outnumber out_cap (out_cap of them written).
__global__ void __launch_bounds__(FL_SCAN_THREADS) ff_finish_kernel(const PcoB200AsyncFilesStatus* __restrict__ fst, uint64_t* __restrict__ parts,
                                                                    uint64_t n_parts, uint64_t out_cap, FlState* __restrict__ fs,
                                                                    uint64_t* __restrict__ n_matches, PcoB200AsyncFilesFilterStatus* __restrict__ out) {
  const uint64_t total = fl_scan_parts(parts, n_parts);
  if (threadIdx.x != 0) return;
  const PcoB200AsyncFilesStatus p = *fst;
  PcoB200AsyncFilesFilterStatus r;
  r.kind = p.kind;
  r.device_status = p.device_status;
  r.file = p.file;
  r.chunk = p.chunk;
  r.n_written = p.n_written;
  r.n_files = p.n_files;
  fl_decide(p.kind == PCO_B200_OK, total, out_cap, r, fs, n_matches);
  *out = r;
}

}  // namespace pcob200
