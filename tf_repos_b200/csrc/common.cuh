// common.cuh -- shared helpers for libctr_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>

#include "../../include/ctr_b200.h"

namespace ctr {

// ---- error plumbing (thread-local message, never throws) -------------------------------------
void set_error(const char* fmt, ...);
extern std::atomic<int64_t> g_launches;
int sm_count();

#define CTR_REQUIRE(cond, code, ...)        \
  do {                                      \
    if (!(cond)) {                          \
      ::ctr::set_error(__VA_ARGS__);        \
      return (code);                        \
    }                                       \
  } while (0)

// call after every kernel launch: counts it and surfaces launch-configuration errors
#define CTR_LAUNCHED(name)                                                        \
  do {                                                                            \
    ::ctr::g_launches.fetch_add(1, std::memory_order_relaxed);                    \
    cudaError_t e__ = cudaPeekAtLastError();                                      \
    if (e__ != cudaSuccess) {                                                     \
      ::ctr::set_error("%s: launch failed: %s", name, cudaGetErrorString(e__));   \
      return CTR_ERR_CUDA;                                                        \
    }                                                                             \
  } while (0)

static inline cudaStream_t as_stream(ctr_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }

// ---- device helpers ----------------------------------------------------------------------------
#define FULL_MASK 0xffffffffu

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL_MASK, v, o);
  return v;
}

// streaming (evict-first) 128-bit accesses for data touched once per step
__device__ __forceinline__ float4 ld_stream4(const float4* p) { return __ldcs(p); }
__device__ __forceinline__ void st_stream4(float4* p, float4 v) { __stcs(p, v); }

__device__ __forceinline__ float4 f4_zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ float4 f4_scale(float4 a, float s) {
  return make_float4(a.x * s, a.y * s, a.z * s, a.w * s);
}
__device__ __forceinline__ float4 f4_add(float4 a, float4 b) {
  return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
}
__device__ __forceinline__ float4 f4_sub(float4 a, float4 b) {
  return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w);
}
__device__ __forceinline__ float4 f4_mul(float4 a, float4 b) {
  return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w);
}
__device__ __forceinline__ float4 f4_fma(float4 a, float4 b, float4 c) {
  return make_float4(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y), fmaf(a.z, b.z, c.z),
                     fmaf(a.w, b.w, c.w));
}
__device__ __forceinline__ float4 f4_shfl_xor(float4 a, int o) {
  return make_float4(__shfl_xor_sync(FULL_MASK, a.x, o), __shfl_xor_sync(FULL_MASK, a.y, o),
                     __shfl_xor_sync(FULL_MASK, a.z, o), __shfl_xor_sync(FULL_MASK, a.w, o));
}
__device__ __forceinline__ float f4_hsum(float4 a) { return (a.x + a.y) + (a.z + a.w); }

static inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

}  // namespace ctr
