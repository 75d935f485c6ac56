// line_starts.cuh -- line starts of a text buffer in device memory, shared by the tokenizers
// (libsvm_device.cu, criteo_feature.cu).
//
// Kernels: (1) count '\n' per 4 KB block; (2) scan the block counts; (3) emit line starts.
// They live in an anonymous namespace so that every translation unit that includes this header owns its copy.
#pragma once
#include "common.cuh"

namespace ctr {
namespace {

constexpr int LS_THREADS = 256, LS_BYTES_PER_THREAD = 16, LS_BLOCK_BYTES = LS_THREADS * LS_BYTES_PER_THREAD;

__device__ __forceinline__ int count_nl16(const unsigned char* __restrict__ t, int64_t pos, int64_t len, uint32_t& mask) {
  mask = 0;
  if (pos + 16 <= len && ((reinterpret_cast<uintptr_t>(t + pos) & 15) == 0)) {
    const uint4 w = __ldg(reinterpret_cast<const uint4*>(t + pos));
    const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
#pragma unroll
      for (int b = 0; b < 4; ++b)
        if (((ws[k] >> (8 * b)) & 0xFFu) == '\n') mask |= 1u << (4 * k + b);
    }
  } else {
    for (int b = 0; b < 16; ++b)
      if (pos + b < len && t[pos + b] == '\n') mask |= 1u << b;
  }
  return __popc(mask);
}

__global__ void __launch_bounds__(LS_THREADS) ls_count_kernel(const unsigned char* __restrict__ text, int64_t len,
                                                             int32_t* __restrict__ block_counts) {
  __shared__ int warp_tot[LS_THREADS / 32];
  const int64_t pos = ((int64_t)blockIdx.x * LS_THREADS + threadIdx.x) * LS_BYTES_PER_THREAD;
  uint32_t mask;
  int c = pos < len ? count_nl16(text, pos, len, mask) : 0;
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(FULL_MASK, c, o);
  if ((threadIdx.x & 31) == 0) warp_tot[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int w = 0; w < LS_THREADS / 32; ++w) s += warp_tot[w];
    block_counts[blockIdx.x] = s;
  }
}

// exclusive scan of block_counts (one CTA, sequential over tiles of 1024); total -> info_lines[0]
__global__ void __launch_bounds__(1024) ls_scan_kernel(int32_t* __restrict__ block_counts, int n_blocks,
                                                       int64_t* __restrict__ n_newlines) {
  __shared__ int64_t warp_sum_s[32];
  __shared__ int64_t carry_s;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  for (int base = 0; base < n_blocks; base += 1024) {
    const int i = base + threadIdx.x;
    const int64_t v = i < n_blocks ? block_counts[i] : 0;
    int64_t x = v;
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t y = __shfl_up_sync(FULL_MASK, x, o);
      if ((threadIdx.x & 31) >= o) x += y;
    }
    if ((threadIdx.x & 31) == 31) warp_sum_s[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x < 32) {
      int64_t w = warp_sum_s[threadIdx.x];
      for (int o = 1; o < 32; o <<= 1) {
        const int64_t y = __shfl_up_sync(FULL_MASK, w, o);
        if (threadIdx.x >= o) w += y;
      }
      warp_sum_s[threadIdx.x] = w;   // inclusive over warps
    }
    __syncthreads();
    const int64_t before = carry_s + (threadIdx.x >= 32 ? warp_sum_s[(threadIdx.x >> 5) - 1] : 0) + (x - v);
    // block counts are < 2^31 in total for any buffer this API accepts (len < 2^31 * 1 byte per newline)
    if (i < n_blocks) block_counts[i] = (int32_t)before;
    __syncthreads();
    if (threadIdx.x == 1023) carry_s = before + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) n_newlines[0] = carry_s;
}

// line_start[k+1] = position just after the k-th '\n' (k < max_rows); line_start[0] = 0
__global__ void __launch_bounds__(LS_THREADS) ls_emit_kernel(const unsigned char* __restrict__ text, int64_t len,
                                                            const int32_t* __restrict__ block_offsets, int64_t max_rows,
                                                            int64_t* __restrict__ line_start) {
  __shared__ int warp_tot[LS_THREADS / 32];
  const int64_t pos = ((int64_t)blockIdx.x * LS_THREADS + threadIdx.x) * LS_BYTES_PER_THREAD;
  uint32_t mask = 0;
  const int c = pos < len ? count_nl16(text, pos, len, mask) : 0;
  int x = c;
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(FULL_MASK, x, o);
    if ((threadIdx.x & 31) >= o) x += y;
  }
  if ((threadIdx.x & 31) == 31) warp_tot[threadIdx.x >> 5] = x;
  __syncthreads();
  int before = x - c;
  for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) before += warp_tot[w];
  int64_t k = (int64_t)block_offsets[blockIdx.x] + before;
  if (blockIdx.x == 0 && threadIdx.x == 0) line_start[0] = 0;
  while (mask) {
    const int b = __ffs(mask) - 1;
    mask &= mask - 1;
    if (k < max_rows) line_start[k + 1] = pos + b + 1;
    ++k;
  }
}

}  // namespace
}  // namespace ctr
