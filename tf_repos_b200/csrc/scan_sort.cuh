// scan_sort.cuh -- the integer prefix scans and the stable LSD radix sort over device-resident counts, shared by the
// text pipelines (line_starts.cuh, criteo_feature.cu, smart_feature.cu, aliccp_tfrecord.cu, aliccp_sample.cu,
// tfrecord_device.cu).
//
// Scans, each level built on the one below: warp_scan_excl (N values per lane), block_scan_excl (N values per thread
// of a CTA), and cta_scan_kernel (N arrays of one device-resident length scanned by one CTA), launched by cta_scan.
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

// exclusive scan of each v[k] across the warp, in place; total[k] = the warp's sum of v[k], on every lane.
// Every lane of the warp calls it.
template <int N, typename T>
__device__ __forceinline__ void warp_scan_excl(T (&v)[N], T (&total)[N]) {
  const int lane = lane_id();
  T x[N];
#pragma unroll
  for (int k = 0; k < N; ++k) x[k] = v[k];
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
#pragma unroll
    for (int k = 0; k < N; ++k) {
      const T y = __shfl_up_sync(FULL_MASK, x[k], o);
      if (lane >= o) x[k] += y;
    }
  }
#pragma unroll
  for (int k = 0; k < N; ++k) {
    total[k] = __shfl_sync(FULL_MASK, x[k], 31);
    v[k] = x[k] - v[k];
  }
}

template <typename T>
__device__ __forceinline__ T warp_scan_excl(T v, T& total) {
  T a[1] = {v}, t[1];
  warp_scan_excl(a, t);
  total = t[0];
  return a[0];
}

// exclusive scan of each v[k] across a CTA of THREADS threads, in place; total[k] = the CTA's sum of v[k], on every
// thread.  Every thread of the CTA calls it; it ends with __syncthreads(), so calls may follow each other.
template <int THREADS, int N, typename T>
__device__ __forceinline__ void block_scan_excl(T (&v)[N], T (&total)[N]) {
  constexpr int WARPS = THREADS / 32;
  static_assert(THREADS % 32 == 0 && WARPS <= 32, "block_scan_excl: whole warps, at most 1024 threads");
  __shared__ T warp_s[N][WARPS];
  const int lane = lane_id(), warp = threadIdx.x >> 5;
  warp_scan_excl(v, total);
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < N; ++k) warp_s[k][warp] = total[k];
  }
  __syncthreads();
  T w[N];   // every warp scans the warp sums and takes its own warp's offset
#pragma unroll
  for (int k = 0; k < N; ++k) w[k] = lane < WARPS ? warp_s[k][lane] : T(0);
  warp_scan_excl(w, total);
#pragma unroll
  for (int k = 0; k < N; ++k) v[k] += __shfl_sync(FULL_MASK, w[k], warp);
  __syncthreads();
}

template <typename T, int N>
struct CtaScanArrays {
  T* a[N];
  int64_t* total[N];
};

// exclusive scans of s.a[k][0, n) in place, n = (count ? *count : 0) + extra; one CTA of 1024 threads, tiles of 1024.
// Values are summed in int64 and written back as T; the sum of s.a[k] -> *s.total[k] where that is not null.
template <typename T, int N>
__global__ void __launch_bounds__(1024) cta_scan_kernel(CtaScanArrays<T, N> s, const int64_t* __restrict__ count,
                                                        int64_t extra) {
  const int64_t n = (count ? count[0] : 0) + extra;
  int64_t carry[N] = {};
  for (int64_t base = 0; base < n; base += 1024) {
    const int64_t i = base + threadIdx.x;
    int64_t v[N], tot[N];
#pragma unroll
    for (int k = 0; k < N; ++k) v[k] = i < n ? (int64_t)s.a[k][i] : 0;
    block_scan_excl<1024>(v, tot);
#pragma unroll
    for (int k = 0; k < N; ++k) {
      if (i < n) s.a[k][i] = (T)(carry[k] + v[k]);
      carry[k] += tot[k];
    }
  }
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < N; ++k)
      if (s.total[k]) *s.total[k] = carry[k];
  }
}

// launches cta_scan_kernel over the arrays a (totals -> total, each may be null) and checks the launch
template <typename T, int N>
static int cta_scan(T* const (&a)[N], int64_t* const (&total)[N], const int64_t* count, int64_t extra, cudaStream_t st,
                    const char* what) {
  CtaScanArrays<T, N> s;
  for (int k = 0; k < N; ++k) { s.a[k] = a[k]; s.total[k] = total[k]; }
  cta_scan_kernel<T, N><<<1, 1024, 0, st>>>(s, count, extra);
  CTR_LAUNCHED(what);
  return CTR_OK;
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
    if (int rc = cta_scan({hist}, {nullptr}, hist_count, 0, st, what)) return rc;
    lsd_scatter_kernel<<<nb, LSD_THREADS, 0, st>>>(k[cur], v[cur], n_dev, pass, hist, k[cur ^ 1], v[cur ^ 1]);
    CTR_LAUNCHED(what);
  }
  *out_keys = k[cur];
  if (out_vals) *out_vals = v[cur];
  return CTR_OK;
}

}  // namespace
}  // namespace ctr
