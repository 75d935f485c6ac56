// lib.cu -- library-level entry points: version, error text, launch counter, small utilities.
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

namespace ctr {

static thread_local char g_err[512] = "";
std::atomic<int64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int sm_count() {
  static int cached = 0;
  if (cached > 0) return cached;
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
    return 132;
  cached = n;
  return n;
}

// ---- fill / truncated-normal init ---------------------------------------------------------------
__global__ void fill_kernel(float* __restrict__ t, int64_t n, float v) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) t[i] = v;
}

// counter-based generator: splitmix64 of (seed, element, attempt) -> two uniforms -> Box-Muller.
__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

// tf.truncated_normal semantics: redraw until |z| <= 2 (glorot_normal_initializer in TF 1.4 draws
// a truncated normal, SURVEY.md A.2).  The stream is NOT TF's Philox stream; parity tests inject
// weights, this only has to have the right distribution.
__global__ void trunc_normal_kernel(float* __restrict__ t, int64_t n, float stddev, uint64_t seed) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    float z = 0.f;
    for (uint32_t attempt = 0; attempt < 16; ++attempt) {
      uint64_t r = splitmix64(seed ^ splitmix64((uint64_t)i * 16ull + attempt));
      float u1 = ((uint32_t)(r >> 40) + 1u) * (1.0f / 16777217.0f);  // (0,1]
      float u2 = ((uint32_t)(r & 0xFFFFFFu)) * (1.0f / 16777216.0f); // [0,1)
      z = sqrtf(-2.0f * __logf(u1)) * __cosf(6.283185307f * u2);
      if (fabsf(z) <= 2.0f) break;
      z = 0.f;
    }
    t[i] = z * stddev;
  }
}

}  // namespace ctr

using namespace ctr;

extern "C" {

int ctr_abi_version(void) { return 1; }
const char* ctr_last_error(void) { return ctr::g_err; }
int64_t ctr_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
int ctr_device_sm_count(void) { return sm_count(); }

int ctr_fill(float* t, int64_t n, float value, ctr_stream_t stream) {
  CTR_REQUIRE(n >= 0, CTR_ERR_INVALID_ARG, "ctr_fill: n < 0");
  if (n == 0) return CTR_OK;
  CTR_REQUIRE(t != nullptr, CTR_ERR_INVALID_ARG, "ctr_fill: null tensor");
  int64_t blocks = ceil_div64(n, 256 * 8);
  int grid = (int)(blocks < (int64_t)sm_count() * 16 ? blocks : (int64_t)sm_count() * 16);
  fill_kernel<<<grid, 256, 0, as_stream(stream)>>>(t, n, value);
  CTR_LAUNCHED("ctr_fill");
  return CTR_OK;
}

int ctr_init_trunc_normal(float* t, int64_t n, float stddev, uint64_t seed, ctr_stream_t stream) {
  CTR_REQUIRE(n >= 0, CTR_ERR_INVALID_ARG, "ctr_init_trunc_normal: n < 0");
  if (n == 0) return CTR_OK;
  CTR_REQUIRE(t != nullptr, CTR_ERR_INVALID_ARG, "ctr_init_trunc_normal: null tensor");
  int64_t blocks = ceil_div64(n, 256 * 8);
  int grid = (int)(blocks < (int64_t)sm_count() * 16 ? blocks : (int64_t)sm_count() * 16);
  trunc_normal_kernel<<<grid, 256, 0, as_stream(stream)>>>(t, n, stddev, seed);
  CTR_LAUNCHED("ctr_init_trunc_normal");
  return CTR_OK;
}

}  // extern "C"
