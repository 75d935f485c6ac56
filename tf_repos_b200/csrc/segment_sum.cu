// segment_sum.cu -- K3b: per-unique-id sum of the per-occurrence gradient rows.
//
// Replaces tf.unsorted_segment_sum inside optimizer._deduplicate_indexed_slices
// (reached from optimizer.minimize, DeepFM.py:213) [TF-sem].
//
// Two fixed-shape paths, no float atomics => bit-reproducible run to run:
//   short runs (<= CTR_LONG_SEG occurrences): LPR = K/4 lanes per run, sequential in occurrence
//     order (== TF's CPU summation order), 4 independent row loads in flight per lane;
//   long runs (the 13 always-present continuous-feature ids of the Criteo layout occur once per
//     sample, i.e. B times): one CTA per run, 256/LPR lane groups stride the run, then a fixed
//     binary tree over the groups in shared memory.
#include "common.cuh"

namespace ctr {

template <int LPR, int VEC>
__global__ void __launch_bounds__(256)
segsum_short_kernel(const float* __restrict__ g_rows, const float* __restrict__ g_w,
                    const int32_t* __restrict__ perm, const int32_t* __restrict__ seg_offsets,
                    const int32_t* __restrict__ n_uniq, int64_t n, float* __restrict__ g_uniq,
                    float* __restrict__ gw_uniq) {
  constexpr int K = 4 * LPR * VEC;
  const int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / LPR;
  const int c = threadIdx.x % LPR;
  if (u >= n || u >= n_uniq[0]) return;
  const int start = seg_offsets[u];
  const int len = seg_offsets[u + 1] - start;
  if (len > CTR_LONG_SEG) return;
  float4 acc[VEC];
#pragma unroll
  for (int v = 0; v < VEC; ++v) acc[v] = f4_zero();
  float accw = 0.f;
  int i = 0;
  for (; i + 4 <= len; i += 4) {
    int32_t p[4];
    float4 r[4][VEC];
    float w[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) p[j] = perm[start + i + j];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float4* row = reinterpret_cast<const float4*>(g_rows + (int64_t)p[j] * K) + c;
#pragma unroll
      for (int v = 0; v < VEC; ++v) r[j][v] = row[v * LPR];
      w[j] = (g_w && c == 0) ? g_w[p[j]] : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
#pragma unroll
      for (int v = 0; v < VEC; ++v) acc[v] = f4_add(acc[v], r[j][v]);
      accw += w[j];
    }
  }
  for (; i < len; ++i) {
    const int32_t p = perm[start + i];
    const float4* row = reinterpret_cast<const float4*>(g_rows + (int64_t)p * K) + c;
#pragma unroll
    for (int v = 0; v < VEC; ++v) acc[v] = f4_add(acc[v], row[v * LPR]);
    if (g_w && c == 0) accw += g_w[p];
  }
  float4* o = reinterpret_cast<float4*>(g_uniq + u * K) + c;
#pragma unroll
  for (int v = 0; v < VEC; ++v) o[v * LPR] = acc[v];
  if (gw_uniq && c == 0) gw_uniq[u] = accw;
}

template <int LPR, int VEC>
__global__ void __launch_bounds__(256)
segsum_long_kernel(const float* __restrict__ g_rows, const float* __restrict__ g_w,
                   const int32_t* __restrict__ perm, const int32_t* __restrict__ seg_offsets,
                   const int32_t* __restrict__ long_list, float* __restrict__ g_uniq,
                   float* __restrict__ gw_uniq) {
  constexpr int K = 4 * LPR * VEC;
  constexpr int G = 256 / LPR;  // lane groups per CTA
  __shared__ float4 sm[VEC][256];
  __shared__ float smw[G];
  const int g = threadIdx.x / LPR, c = threadIdx.x % LPR;
  const int n_long = long_list[0];
  for (int li = blockIdx.x; li < n_long; li += gridDim.x) {
    const int u = long_list[1 + li];
    const int start = seg_offsets[u];
    const int len = seg_offsets[u + 1] - start;
    float4 acc[VEC];
#pragma unroll
    for (int v = 0; v < VEC; ++v) acc[v] = f4_zero();
    float accw = 0.f;
    int i = g;
    for (; i + 3 * G < len; i += 4 * G) {
      int32_t p[4];
      float4 r[4][VEC];
      float w[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) p[j] = perm[start + i + j * G];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float4* row = reinterpret_cast<const float4*>(g_rows + (int64_t)p[j] * K) + c;
#pragma unroll
        for (int v = 0; v < VEC; ++v) r[j][v] = row[v * LPR];
        w[j] = (g_w && c == 0) ? g_w[p[j]] : 0.f;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int v = 0; v < VEC; ++v) acc[v] = f4_add(acc[v], r[j][v]);
        accw += w[j];
      }
    }
    for (; i < len; i += G) {
      const int32_t p = perm[start + i];
      const float4* row = reinterpret_cast<const float4*>(g_rows + (int64_t)p * K) + c;
#pragma unroll
      for (int v = 0; v < VEC; ++v) acc[v] = f4_add(acc[v], row[v * LPR]);
      if (g_w && c == 0) accw += g_w[p];
    }
#pragma unroll
    for (int v = 0; v < VEC; ++v) sm[v][threadIdx.x] = acc[v];
    if (c == 0) smw[g] = accw;
    __syncthreads();
    for (int half = G / 2; half > 0; half >>= 1) {
      if (g < half) {
#pragma unroll
        for (int v = 0; v < VEC; ++v)
          sm[v][threadIdx.x] = f4_add(sm[v][threadIdx.x], sm[v][threadIdx.x + half * LPR]);
        if (c == 0) smw[g] += smw[g + half];
      }
      __syncthreads();
    }
    if (g == 0) {
      float4* o = reinterpret_cast<float4*>(g_uniq + (int64_t)u * K) + c;
#pragma unroll
      for (int v = 0; v < VEC; ++v) o[v * LPR] = sm[v][threadIdx.x];
      if (gw_uniq && c == 0) gw_uniq[u] = smw[0];
    }
    __syncthreads();
  }
}

// Long runs split into chunks of SEG_CHUNK occurrences (the 13 continuous-feature ids of the Criteo layout occur B
// times; DIN's padding id occurs ~10^6 times per step): segsum_long_plan_kernel gives every long run a range of partial
// rows, segsum_long_split_kernel sums chunk c of run li with the lane-group striding + fixed tree,
// segsum_long_final_kernel adds a run's partials in chunk order.  A run that does not get a range (scratch exhausted)
// is summed by one CTA in the same kernel -- a different tree, so which runs get a range must not depend on launch
// order: long_list is filled by atomics in no fixed order, so the plan hands out rows in ascending u instead.  A run's
// base is the chunk count of all long runs with a smaller u; it gets no range when base + chunks > cap_rows.  Fixed
// shapes and a plan that is a function of the segments alone => bit-reproducible.
constexpr int SEG_CHUNK = 1024;

// per long run li: plan[1 + 2*li] = base row (-1: no range), plan[2 + 2*li] = number of chunks.  One CTA; each run
// counts the chunks of the runs before it in u order from shared-memory tiles of long_list (n_long^2 / 256
// shared-memory adds per thread; n_long is 13 in the Criteo layout and 1 in DIN's).
constexpr int PLAN_THREADS = 256;
__device__ __forceinline__ int seg_chunks(const int32_t* __restrict__ seg_offsets, int u) {
  return (seg_offsets[u + 1] - seg_offsets[u] + SEG_CHUNK - 1) / SEG_CHUNK;
}
__global__ void __launch_bounds__(PLAN_THREADS)
segsum_long_plan_kernel(const int32_t* __restrict__ seg_offsets, const int32_t* __restrict__ long_list, int max_long,
                        int cap_rows, int32_t* __restrict__ plan) {
  __shared__ int su[PLAN_THREADS], sc[PLAN_THREADS];
  const int n_long = min(long_list[0], max_long);
  for (int li0 = 0; li0 < n_long; li0 += PLAN_THREADS) {
    const int li = li0 + threadIdx.x;
    const int u = li < n_long ? long_list[1 + li] : 0;
    int chunks = li < n_long ? seg_chunks(seg_offsets, u) : 0;
    int base = 0;
    for (int t0 = 0; t0 < n_long; t0 += PLAN_THREADS) {
      __syncthreads();
      const int tj = t0 + threadIdx.x;
      if (tj < n_long) {
        su[threadIdx.x] = long_list[1 + tj];
        sc[threadIdx.x] = seg_chunks(seg_offsets, su[threadIdx.x]);
      }
      __syncthreads();
      const int m = min(PLAN_THREADS, n_long - t0);
      for (int j = 0; j < m; ++j) base += su[j] < u ? sc[j] : 0;
    }
    if (li < n_long) {
      if (base + chunks > cap_rows) { base = -1; chunks = 1; }   // no room: whole run by one CTA, straight to the output
      plan[1 + 2 * li] = base;
      plan[2 + 2 * li] = chunks;
    }
  }
}

template <int LPR, int VEC>
__global__ void __launch_bounds__(256)
segsum_long_split_kernel(const float* __restrict__ g_rows, const float* __restrict__ g_w,
                         const int32_t* __restrict__ perm, const int32_t* __restrict__ seg_offsets,
                         const int32_t* __restrict__ long_list, int max_long, const int32_t* __restrict__ plan,
                         float* __restrict__ partial, float* __restrict__ g_uniq, float* __restrict__ gw_uniq) {
  constexpr int K = 4 * LPR * VEC;
  constexpr int G = 256 / LPR;
  __shared__ float4 sm[VEC][256];
  __shared__ float smw[G];
  const int g = threadIdx.x / LPR, c = threadIdx.x % LPR;
  const int n_long = min(long_list[0], max_long);
  for (int li = blockIdx.y; li < n_long; li += gridDim.y) {
    const int u = long_list[1 + li];
    const int start0 = seg_offsets[u];
    const int len0 = seg_offsets[u + 1] - start0;
    const int base = plan[1 + 2 * li], chunks = plan[2 + 2 * li];
    for (int chunk = blockIdx.x; chunk < chunks; chunk += gridDim.x) {
      const int lo = base < 0 ? 0 : chunk * SEG_CHUNK, hi = base < 0 ? len0 : min(len0, lo + SEG_CHUNK);
      const int start = start0 + lo, len = hi - lo;
      float4 acc[VEC];
#pragma unroll
      for (int v = 0; v < VEC; ++v) acc[v] = f4_zero();
      float accw = 0.f;
      for (int i = g; i < len; i += G) {
        const int32_t p = perm[start + i];
        const float4* row = reinterpret_cast<const float4*>(g_rows + (int64_t)p * K) + c;
#pragma unroll
        for (int v = 0; v < VEC; ++v) acc[v] = f4_add(acc[v], row[v * LPR]);
        if (g_w && c == 0) accw += g_w[p];
      }
#pragma unroll
      for (int v = 0; v < VEC; ++v) sm[v][threadIdx.x] = acc[v];
      if (c == 0) smw[g] = accw;
      __syncthreads();
      for (int half = G / 2; half > 0; half >>= 1) {
        if (g < half) {
#pragma unroll
          for (int v = 0; v < VEC; ++v)
            sm[v][threadIdx.x] = f4_add(sm[v][threadIdx.x], sm[v][threadIdx.x + half * LPR]);
          if (c == 0) smw[g] += smw[g + half];
        }
        __syncthreads();
      }
      if (g == 0) {
        float* prow = base < 0 ? nullptr : partial + (int64_t)(base + chunk) * (K + 4);
        float4* o = base < 0 ? reinterpret_cast<float4*>(g_uniq + (int64_t)u * K) + c : reinterpret_cast<float4*>(prow) + c;
#pragma unroll
        for (int v = 0; v < VEC; ++v) o[v * LPR] = sm[v][threadIdx.x];
        if (c == 0) {
          if (base < 0) { if (gw_uniq) gw_uniq[u] = smw[0]; }
          else prow[K] = smw[0];
        }
      }
      __syncthreads();
    }
  }
}

__global__ void segsum_long_final_kernel(const float* __restrict__ partial, const int32_t* __restrict__ long_list,
                                         int max_long, const int32_t* __restrict__ plan, int K,
                                         float* __restrict__ g_uniq, float* __restrict__ gw_uniq) {
  const int n_long = min(long_list[0], max_long);
  for (int li = blockIdx.x; li < n_long; li += gridDim.x) {
    const int base = plan[1 + 2 * li], chunks = plan[2 + 2 * li];
    if (base < 0) continue;
    const int u = long_list[1 + li];
    for (int k = threadIdx.x; k <= K; k += blockDim.x) {
      if (k == K && !gw_uniq) continue;
      float s = 0.f;
      for (int ch = 0; ch < chunks; ++ch) s += partial[(int64_t)(base + ch) * (K + 4) + k];
      if (k < K) g_uniq[(int64_t)u * K + k] = s;
      else gw_uniq[u] = s;
    }
  }
}

// any K: one warp per run, lanes stride k.  (long runs are summed sequentially here.)
__global__ void __launch_bounds__(256)
segsum_generic_kernel(const float* __restrict__ g_rows, const float* __restrict__ g_w,
                      const int32_t* __restrict__ perm, const int32_t* __restrict__ seg_offsets,
                      const int32_t* __restrict__ n_uniq, int64_t n, int K,
                      float* __restrict__ g_uniq, float* __restrict__ gw_uniq) {
  const int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (u >= n || u >= n_uniq[0]) return;
  const int start = seg_offsets[u];
  const int len = seg_offsets[u + 1] - start;
  for (int k = lane; k < K; k += 32) {
    float acc = 0.f;
    for (int i = 0; i < len; ++i) acc += g_rows[(int64_t)perm[start + i] * K + k];
    g_uniq[u * K + k] = acc;
  }
  if (g_w && gw_uniq && lane == 0) {
    float acc = 0.f;
    for (int i = 0; i < len; ++i) acc += g_w[perm[start + i]];
    gw_uniq[u] = acc;
  }
}

}  // namespace ctr

using namespace ctr;

extern "C" int ctr_segment_sum_rows(const float* g_rows, const float* g_w, const int32_t* perm,
                                    const int32_t* seg_offsets, const int32_t* n_uniq,
                                    const int32_t* long_list, int64_t n, int K, float* g_uniq,
                                    float* gw_uniq, void* ws, size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE(n >= 0 && K > 0, CTR_ERR_INVALID_ARG, "ctr_segment_sum_rows: bad n/K");
  if (n == 0) return CTR_OK;
  CTR_REQUIRE(g_rows && perm && seg_offsets && n_uniq && long_list && g_uniq, CTR_ERR_INVALID_ARG,
              "ctr_segment_sum_rows: null buffer");
  CTR_REQUIRE((g_w == nullptr) == (gw_uniq == nullptr), CTR_ERR_INVALID_ARG,
              "ctr_segment_sum_rows: g_w and gw_uniq must both be given or both be NULL");
  cudaStream_t st = as_stream(stream);
  const int long_grid = 2 * sm_count();
  // optional scratch (the K3 workspace is free by now): long runs are cut into chunks of SEG_CHUNK occurrences.
  // layout: int32 plan[1 + 2*max_long] (plan[0] unused) | float partial[cap_rows][K+4]
  const int64_t max_long = n / (CTR_LONG_SEG + 1) + 1;
  const size_t plan_bytes = ((size_t)(1 + 2 * max_long) * sizeof(int32_t) + 15) & ~(size_t)15;
  const int64_t want_rows = n / SEG_CHUNK + max_long;       // every run: its full chunks + at most one partial chunk
  int64_t cap_rows = 0;
  if (ws && ws_bytes > plan_bytes && ((uintptr_t)ws & 15) == 0)
    cap_rows = (int64_t)((ws_bytes - plan_bytes) / ((size_t)(K + 4) * sizeof(float)));
  if (cap_rows > want_rows) cap_rows = want_rows;
  const bool split = cap_rows >= 16;
  int32_t* plan = reinterpret_cast<int32_t*>(ws);
  float* partial = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(ws) + plan_bytes);
#define SEG_CASE(KK, LPR, VEC)                                                                      \
  case KK: {                                                                                        \
    unsigned blocks = (unsigned)ceil_div64(n * LPR, 256);                                           \
    segsum_short_kernel<LPR, VEC><<<blocks, 256, 0, st>>>(g_rows, g_w, perm, seg_offsets, n_uniq,   \
                                                          n, g_uniq, gw_uniq);                      \
    CTR_LAUNCHED("segsum_short");                                                                   \
    if (split) {                                                                                    \
      segsum_long_plan_kernel<<<1, PLAN_THREADS, 0, st>>>(seg_offsets, long_list, (int)max_long, (int)cap_rows, \
                                                          plan);                                    \
      CTR_LAUNCHED("segsum_long_plan");                                                             \
      segsum_long_split_kernel<LPR, VEC><<<dim3(64, 16), 256, 0, st>>>(                             \
          g_rows, g_w, perm, seg_offsets, long_list, (int)max_long, plan, partial, g_uniq, gw_uniq); \
      CTR_LAUNCHED("segsum_long_split");                                                            \
      segsum_long_final_kernel<<<64, 128, 0, st>>>(partial, long_list, (int)max_long, plan, K,      \
                                                   g_uniq, gw_uniq);                                \
      CTR_LAUNCHED("segsum_long_final");                                                            \
    } else {                                                                                        \
      segsum_long_kernel<LPR, VEC><<<long_grid, 256, 0, st>>>(g_rows, g_w, perm, seg_offsets,       \
                                                              long_list, g_uniq, gw_uniq);          \
      CTR_LAUNCHED("segsum_long");                                                                  \
    }                                                                                               \
    break;                                                                                          \
  }
  switch (K) {
    SEG_CASE(4, 1, 1)
    SEG_CASE(8, 2, 1)
    SEG_CASE(16, 4, 1)
    SEG_CASE(32, 8, 1)
    SEG_CASE(64, 16, 1)
    SEG_CASE(128, 32, 1)
    SEG_CASE(256, 32, 2)
    default: {
      unsigned blocks = (unsigned)ceil_div64(n * 32, 256);
      segsum_generic_kernel<<<blocks, 256, 0, st>>>(g_rows, g_w, perm, seg_offsets, n_uniq, n, K,
                                                    g_uniq, gw_uniq);
      CTR_LAUNCHED("segsum_generic");
    }
  }
#undef SEG_CASE
  return CTR_OK;
}
