// scan_sort.cuh -- the one-CTA exclusive scan and the stable LSD radix sort over device-resident counts, shared by the
// text pipelines (line_starts.cuh, criteo_feature.cu, aliccp_sample.cu, smart_feature.cu).
//
// The sort takes uint64 keys with an optional uint32 value, 8-bit digits: per-CTA digit histograms, a one-CTA scan of
// the digit-major histogram, then a scatter that keeps index order within a CTA (warp match + per-warp digit counts).
// Multi-word keys are sorted word by word from the least significant one, carrying a permutation (iota / gather).
// They live in an anonymous namespace so that every translation unit that includes this header owns its copy.
#pragma once
#include "common.cuh"

namespace ctr {
namespace {

constexpr int LSD_THREADS = 256, LSD_WARPS = LSD_THREADS / 32;
constexpr int LSD_TILE = 16 * LSD_THREADS;   // items per CTA in the radix passes

// exclusive scan of a[0, n) in place (one CTA, tiles of 1024); n = *count when count is given; total -> *total
template <typename T>
__global__ void __launch_bounds__(1024) cta_scan_kernel(T* __restrict__ a, const int64_t* __restrict__ count,
                                                        int64_t n_fixed, int64_t* __restrict__ total) {
  __shared__ int64_t warp_sum_s[32];
  __shared__ int64_t carry_s;
  const int64_t n = count ? count[0] : n_fixed;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  for (int64_t base = 0; base < n; base += 1024) {
    const int64_t i = base + threadIdx.x;
    const int64_t v = i < n ? (int64_t)a[i] : 0;
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
      warp_sum_s[threadIdx.x] = w;
    }
    __syncthreads();
    const int64_t before = carry_s + (threadIdx.x >= 32 ? warp_sum_s[(threadIdx.x >> 5) - 1] : 0) + (x - v);
    if (i < n) a[i] = (T)before;
    __syncthreads();
    if (threadIdx.x == 1023) carry_s = before + v;
    __syncthreads();
  }
  if (threadIdx.x == 0 && total) total[0] = carry_s;
}

// hist[d * nb + b] = items of CTA b with digit d
__global__ void __launch_bounds__(LSD_THREADS) lsd_hist_kernel(const uint64_t* __restrict__ keys,
                                                              const int64_t* __restrict__ n_dev, int pass,
                                                              int32_t* __restrict__ hist,
                                                              int64_t* __restrict__ hist_count) {
  __shared__ int h[256];
  const int64_t n = n_dev[0], nb = (n + LSD_TILE - 1) / LSD_TILE;
  if (blockIdx.x == 0 && threadIdx.x == 0) hist_count[0] = 256 * nb;
  if (blockIdx.x >= nb) return;
  h[threadIdx.x] = 0;
  __syncthreads();
  for (int r = 0; r < LSD_TILE / LSD_THREADS; ++r) {
    const int64_t i = (int64_t)blockIdx.x * LSD_TILE + r * LSD_THREADS + threadIdx.x;
    if (i < n) atomicAdd(&h[(keys[i] >> (8 * pass)) & 0xFF], 1);
  }
  __syncthreads();
  hist[(int64_t)threadIdx.x * nb + blockIdx.x] = h[threadIdx.x];
}

// within a CTA the items go in index order (warp match + per-warp digit counts); vals may be null
__global__ void __launch_bounds__(LSD_THREADS) lsd_scatter_kernel(const uint64_t* __restrict__ keys,
                                                                 const uint32_t* __restrict__ vals,
                                                                 const int64_t* __restrict__ n_dev, int pass,
                                                                 const int32_t* __restrict__ hist,
                                                                 uint64_t* __restrict__ keys2,
                                                                 uint32_t* __restrict__ vals2) {
  __shared__ int base[256];
  __shared__ int wcnt[LSD_WARPS][256];
  const int64_t n = n_dev[0], nb = (n + LSD_TILE - 1) / LSD_TILE;
  if (blockIdx.x >= nb) return;
  const int lane = lane_id(), warp = threadIdx.x >> 5;
  base[threadIdx.x] = hist[(int64_t)threadIdx.x * nb + blockIdx.x];
  for (int w = 0; w < LSD_WARPS; ++w) wcnt[w][threadIdx.x] = 0;
  __syncthreads();
  for (int r = 0; r < LSD_TILE / LSD_THREADS; ++r) {
    const int64_t i = (int64_t)blockIdx.x * LSD_TILE + r * LSD_THREADS + threadIdx.x;
    const bool live = i < n;
    uint64_t k = 0;
    uint32_t v = 0;
    int d = 256;   // no digit: dead lanes match only each other and are not counted
    if (live) { k = keys[i]; v = vals ? vals[i] : 0; d = (int)((k >> (8 * pass)) & 0xFF); }
    const uint32_t peers = __match_any_sync(FULL_MASK, d);
    const int rank = __popc(peers & lanemask_lt());
    if (live && rank == 0) wcnt[warp][d] = __popc(peers);
    __syncthreads();
    if (live) {
      int pos = base[d] + rank;
      for (int w = 0; w < warp; ++w) pos += wcnt[w][d];
      keys2[pos] = k;
      if (vals) vals2[pos] = v;
    }
    __syncthreads();
    int add = 0;
    for (int w = 0; w < LSD_WARPS; ++w) { add += wcnt[w][threadIdx.x]; wcnt[w][threadIdx.x] = 0; }
    base[threadIdx.x] += add;
    __syncthreads();
  }
}

__global__ void lsd_iota_kernel(uint32_t* __restrict__ perm, const int64_t* __restrict__ n_dev) {
  const int64_t n = n_dev[0];
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    perm[i] = (uint32_t)i;
}

__global__ void lsd_gather_kernel(const uint64_t* __restrict__ src, const uint32_t* __restrict__ perm,
                                  const int64_t* __restrict__ n_dev, uint64_t* __restrict__ dst) {
  const int64_t n = n_dev[0];
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    dst[i] = src[perm ? perm[i] : i];
}

// (keys, vals) sorted stably by the low 8 * passes bits of keys, n = *n_dev <= cap; the result is in keys / vals
// (passes even) or keys2 / vals2 (odd): *out_keys / *out_vals.  hist holds 256 * ceil(cap / LSD_TILE) int32.
static int lsd_sort(uint64_t* keys, uint32_t* vals, uint64_t* keys2, uint32_t* vals2, const int64_t* n_dev, int64_t cap,
                    int passes, int32_t* hist, int64_t* hist_count, cudaStream_t st, const char* what,
                    uint64_t** out_keys, uint32_t** out_vals) {
  const unsigned nb = (unsigned)ceil_div64(cap > 0 ? cap : 1, LSD_TILE);
  uint64_t* k[2] = {keys, keys2};
  uint32_t* v[2] = {vals, vals2};
  int cur = 0;
  for (int pass = 0; pass < passes; ++pass, cur ^= 1) {
    lsd_hist_kernel<<<nb, LSD_THREADS, 0, st>>>(k[cur], n_dev, pass, hist, hist_count);
    CTR_LAUNCHED(what);
    cta_scan_kernel<int32_t><<<1, 1024, 0, st>>>(hist, hist_count, 0, nullptr);
    CTR_LAUNCHED(what);
    lsd_scatter_kernel<<<nb, LSD_THREADS, 0, st>>>(k[cur], v[cur], n_dev, pass, hist, k[cur ^ 1], v[cur ^ 1]);
    CTR_LAUNCHED(what);
  }
  *out_keys = k[cur];
  if (out_vals) *out_vals = v[cur];
  return CTR_OK;
}

}  // namespace
}  // namespace ctr
