// Kernels of pco_b200_decompress_ranges beyond the window-mode decode (decode_fused.cuh, decode_kernels.cuh: WinTask).
// A chunk that several ranges touch is decoded once, as the window [min lo, max hi), into a scratch slot; gather_ranges_kernel then
// copies every piece of a range from its slot to its place in the destination.  Byte copies go through cta_copy_bytes
// (gather_kernels.cuh): aligned 16-byte stores assembled from unaligned sources.
#pragma once
#include "gather_kernels.cuh"

namespace pcob200 {

constexpr int RANGES_THREADS = GATHER_THREADS;  // cta_copy_bytes strides by GATHER_THREADS

struct RangeCopy {
  uint64_t src;    // device address of the piece in its slot
  uint64_t dst;    // device address of the piece in the destination
  uint64_t bytes;
};

// one CTA per piece
__global__ void __launch_bounds__(RANGES_THREADS) gather_ranges_kernel(const RangeCopy* __restrict__ copies) {
  const RangeCopy cp = copies[blockIdx.x];
  cta_copy_bytes(reinterpret_cast<uint8_t*>(cp.dst), reinterpret_cast<const uint8_t*>(cp.src), cp.bytes);
}

}  // namespace pcob200
