// optim.cu -- K4: optimizer apply, TF-1.x arithmetic (every product/sum individually rounded:
// __fmul_rn/__fadd_rn never contract to FMA, IEEE sqrt/div), so that given the same gradient the
// CUDA result is bit-identical to oracle/tf_semantics.py on the CPU.
//
// Replaces optimizer.minimize -> apply_gradients (DeepFM.py:204-213) [TF-sem]:
//   tf.train.AdamOptimizer._apply_sparse_shared  (m*b1 ; scatter_add g*(1-b1) ; ... ; dense var update)
//   tf.train.AdagradOptimizer / MomentumOptimizer / FtrlOptimizer sparse applies
//   training_ops.apply_{adam,adagrad,momentum,ftrl} for dense variables (MLP weights).
// Because tf.nn.l2_loss(table) (DeepFM.py:189-190) contributes a DENSE gradient l2*table, TF
// updates EVERY row each step: rows gathered this step get g = segment_sum + l2*var, all others
// g = l2*var.  `ctr_opt_dense_sweep` is that full-table pass: a pure HBM stream
// (read var,slot0,slot1; write var,slot0,slot1) -- 24 B/element for Adam.
#include <stdlib.h>

#include "optim_steps.cuh"

namespace ctr {

// ---- sparse rows --------------------------------------------------------------------------------
// LPR lanes per row.  g = g_uniq + l2*var (the l2 term is a separate IndexedSlices entry in TF,
// summed by the de-duplication).
template <int OPT, int LPR, int VEC>
__global__ void __launch_bounds__(256)
opt_sparse_rows_kernel(float* __restrict__ var, float* __restrict__ slot0, float* __restrict__ slot1,
                       const int32_t* __restrict__ uniq, const int32_t* __restrict__ n_uniq,
                       const float* __restrict__ g_uniq, int64_t n_max,
                       const float* __restrict__ hyper, float* __restrict__ stage) {
  constexpr int K = 4 * LPR * VEC;
  constexpr bool two = OptTraits<OPT>::slots == 2;
  const int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / LPR;
  const int c = threadIdx.x % LPR;
  if (u >= n_max || u >= n_uniq[0]) return;
  const Hyper h = load_hyper(hyper);
  const int64_t row = (int64_t)uniq[u] * K;
#pragma unroll
  for (int v = 0; v < VEC; ++v) {
    const int64_t e = row + (c + v * LPR) * 4;
    float4 x = *reinterpret_cast<const float4*>(var + e);
    float4 a = *reinterpret_cast<const float4*>(slot0 + e);
    float4 b2 = two ? *reinterpret_cast<const float4*>(slot1 + e) : f4_zero();
    float4 g = *reinterpret_cast<const float4*>(g_uniq + u * K + (c + v * LPR) * 4);
    g = make_float4(__fadd_rn(g.x, __fmul_rn(h.l2, x.x)), __fadd_rn(g.y, __fmul_rn(h.l2, x.y)),
                    __fadd_rn(g.z, __fmul_rn(h.l2, x.z)), __fadd_rn(g.w, __fmul_rn(h.l2, x.w)));
    step_sparse4<OPT>(x, a, b2, g, h);
    if (stage) {
      const int64_t so = u * K + (c + v * LPR) * 4;
      *reinterpret_cast<float4*>(stage + so) = x;
      *reinterpret_cast<float4*>(stage + n_max * K + so) = a;
      if (two) *reinterpret_cast<float4*>(stage + 2 * n_max * K + so) = b2;
    } else {
      *reinterpret_cast<float4*>(var + e) = x;
      *reinterpret_cast<float4*>(slot0 + e) = a;
      if (two) *reinterpret_cast<float4*>(slot1 + e) = b2;
    }
  }
}

// scalar rows / any K: one thread per (row, k)
template <int OPT>
__global__ void __launch_bounds__(256)
opt_sparse_generic_kernel(float* __restrict__ var, float* __restrict__ slot0, float* __restrict__ slot1,
                          const int32_t* __restrict__ uniq, const int32_t* __restrict__ n_uniq,
                          const float* __restrict__ g_uniq, int64_t n_max, int K,
                          const float* __restrict__ hyper, float* __restrict__ stage) {
  constexpr bool two = OptTraits<OPT>::slots == 2;
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t u = t / K;
  const int k = (int)(t % K);
  if (u >= n_max || u >= n_uniq[0]) return;
  const Hyper h = load_hyper(hyper);
  const int64_t e = (int64_t)uniq[u] * K + k;
  float x = var[e], a = slot0[e], b2 = two ? slot1[e] : 0.f;
  float g = __fadd_rn(g_uniq[u * K + k], __fmul_rn(h.l2, x));
  step_sparse<OPT>(x, a, b2, g, h);
  if (stage) {
    stage[u * K + k] = x;
    stage[n_max * K + u * K + k] = a;
    if (two) stage[2 * n_max * K + u * K + k] = b2;
  } else {
    var[e] = x; slot0[e] = a;
    if (two) slot1[e] = b2;
  }
}

__global__ void __launch_bounds__(256)
opt_patch_rows_kernel(float* __restrict__ var, float* __restrict__ slot0, float* __restrict__ slot1,
                      const int32_t* __restrict__ uniq, const int32_t* __restrict__ n_uniq,
                      const float* __restrict__ stage, int64_t n_max, int K, int n_slots) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t u = t / K;
  const int k = (int)(t % K);
  if (u >= n_max || u >= n_uniq[0]) return;
  const int64_t e = (int64_t)uniq[u] * K + k;
  var[e] = stage[u * K + k];
  slot0[e] = stage[n_max * K + u * K + k];
  if (n_slots > 1) slot1[e] = stage[2 * n_max * K + u * K + k];
}

// ---- dense sweep (the dominant kernel of an exact-TF step: pure HBM stream) -----------------------
constexpr int SWEEP_THREADS = 256;

// UNROLL float4 triples in flight per thread; MINB = resident CTAs per SM the register budget is
// squeezed for: the kernel is a pure stream, so what matters is bytes
// in flight per SM = MINB * 256 threads * UNROLL * 48 B.
template <int OPT, int SWEEP_UNROLL, int MINB>
__global__ void __launch_bounds__(SWEEP_THREADS, MINB)
opt_dense_sweep_kernel(float* __restrict__ var, float* __restrict__ slot0, float* __restrict__ slot1,
                       int64_t n4, int64_t n_elem, const float* __restrict__ hyper,
                       float* __restrict__ sumsq_partials) {
  constexpr bool two = OptTraits<OPT>::slots == 2;
  const Hyper h = load_hyper(hyper);
  float4* v4 = reinterpret_cast<float4*>(var);
  float4* a4 = reinterpret_cast<float4*>(slot0);
  float4* b4 = reinterpret_cast<float4*>(slot1);
  float ss = 0.f;
  const int64_t stride = (int64_t)gridDim.x * SWEEP_THREADS;
  int64_t i = (int64_t)blockIdx.x * SWEEP_THREADS + threadIdx.x;
  for (; i + (SWEEP_UNROLL - 1) * stride < n4; i += SWEEP_UNROLL * stride) {
    float4 x[SWEEP_UNROLL], a[SWEEP_UNROLL], b[SWEEP_UNROLL];
#pragma unroll
    for (int j = 0; j < SWEEP_UNROLL; ++j) {
      x[j] = ld_stream4(v4 + i + j * stride);
      a[j] = ld_stream4(a4 + i + j * stride);
      b[j] = two ? ld_stream4(b4 + i + j * stride) : f4_zero();
    }
#pragma unroll
    for (int j = 0; j < SWEEP_UNROLL; ++j) {
      ss += (x[j].x * x[j].x + x[j].y * x[j].y) + (x[j].z * x[j].z + x[j].w * x[j].w);
      float4 g = make_float4(__fmul_rn(h.l2, x[j].x), __fmul_rn(h.l2, x[j].y),
                             __fmul_rn(h.l2, x[j].z), __fmul_rn(h.l2, x[j].w));
      step_sparse4<OPT>(x[j], a[j], b[j], g, h);
      st_stream4(v4 + i + j * stride, x[j]);
      st_stream4(a4 + i + j * stride, a[j]);
      if (two) st_stream4(b4 + i + j * stride, b[j]);
    }
  }
  for (; i < n4; i += stride) {
    float4 x = ld_stream4(v4 + i), a = ld_stream4(a4 + i), b = two ? ld_stream4(b4 + i) : f4_zero();
    ss += (x.x * x.x + x.y * x.y) + (x.z * x.z + x.w * x.w);
    float4 g = make_float4(__fmul_rn(h.l2, x.x), __fmul_rn(h.l2, x.y), __fmul_rn(h.l2, x.z),
                           __fmul_rn(h.l2, x.w));
    step_sparse4<OPT>(x, a, b, g, h);
    st_stream4(v4 + i, x);
    st_stream4(a4 + i, a);
    if (two) st_stream4(b4 + i, b);
  }
  // scalar tail (n_elem % 4)
  if (blockIdx.x == 0 && threadIdx.x < (int)(n_elem - n4 * 4)) {
    const int64_t e = n4 * 4 + threadIdx.x;
    float x = var[e], a = slot0[e], b = two ? slot1[e] : 0.f;
    ss += x * x;
    step_sparse<OPT>(x, a, b, __fmul_rn(h.l2, x), h);
    var[e] = x; slot0[e] = a;
    if (two) slot1[e] = b;
  }
  if (sumsq_partials) {
    __shared__ float wsum[SWEEP_THREADS / 32];
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = ss;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < SWEEP_THREADS / 32; ++w) t += wsum[w];
      sumsq_partials[blockIdx.x] = t;
    }
  }
}

template <int OPT>
__global__ void __launch_bounds__(256)
opt_dense_grad_kernel(float* __restrict__ var, float* __restrict__ slot0, float* __restrict__ slot1,
                      const float* __restrict__ grad, int64_t n, const float* __restrict__ hyper) {
  constexpr bool two = OptTraits<OPT>::slots == 2;
  const Hyper h = load_hyper(hyper);
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    float x = var[i], a = slot0[i], b = two ? slot1[i] : 0.f;
    float g = grad[i];
    if (h.l2 != 0.f) g = __fadd_rn(g, __fmul_rn(h.l2, x));
    step_dense<OPT>(x, a, b, g, h);
    var[i] = x; slot0[i] = a;
    if (two) slot1[i] = b;
  }
}

// AdamOptimizer: lr_t from the current beta powers, then _finish() advances them (fp32 products)
__global__ void adam_tick_kernel(float* __restrict__ state, float* __restrict__ hyper, int n_hyper) {
  const float b1p = state[0], b2p = state[1], lr = state[2];
  const float lr_t = __fdiv_rn(__fmul_rn(lr, __fsqrt_rn(__fsub_rn(1.f, b2p))), __fsub_rn(1.f, b1p));
  for (int r = 0; r < n_hyper; ++r) hyper[8 * r] = lr_t;
  state[0] = __fmul_rn(b1p, hyper[1]);
  state[1] = __fmul_rn(b2p, hyper[2]);
  state[3] = state[3] + 1.f;  // global_step (exact below 2^24)
}

// ---- deterministic reductions -----------------------------------------------------------------------
constexpr int RED_THREADS = 256;
constexpr int RED_MAX_BLOCKS = 1024;

template <bool SQUARE>
__global__ void __launch_bounds__(RED_THREADS)
reduce_partial_kernel(const float* __restrict__ in, int64_t n, float* __restrict__ partials) {
  __shared__ float wsum[RED_THREADS / 32];
  float s = 0.f;
  const int64_t stride = (int64_t)gridDim.x * RED_THREADS;
  for (int64_t i = (int64_t)blockIdx.x * RED_THREADS + threadIdx.x; i < n; i += stride) {
    const float v = in[i];
    s += SQUARE ? v * v : v;
  }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < RED_THREADS / 32; ++w) t += wsum[w];
    partials[blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(RED_THREADS)
reduce_final_kernel(const float* __restrict__ partials, int n, float scale, float* __restrict__ out) {
  __shared__ float wsum[RED_THREADS / 32];
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += RED_THREADS) s += partials[i];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < RED_THREADS / 32; ++w) t += wsum[w];
    out[0] = t * scale;
  }
}

static int reduce_grid(int64_t n) {
  int64_t b = ceil_div64(n, RED_THREADS * 8);
  if (b < 1) b = 1;
  return (int)(b > RED_MAX_BLOCKS ? RED_MAX_BLOCKS : b);
}

}  // namespace ctr

using namespace ctr;

extern "C" {

int ctr_opt_sparse_rows(int opt, float* var, float* slot0, float* slot1, const int32_t* uniq,
                        const int32_t* n_uniq, const float* g_uniq, int64_t n_max, int K,
                        const float* hyper, float* stage, ctr_stream_t stream) {
  CTR_REQUIRE(n_max >= 0 && K > 0, CTR_ERR_INVALID_ARG, "ctr_opt_sparse_rows: bad n_max/K");
  if (n_max == 0) return CTR_OK;
  CTR_REQUIRE(var && slot0 && uniq && n_uniq && g_uniq && hyper, CTR_ERR_INVALID_ARG,
              "ctr_opt_sparse_rows: null buffer");
  CTR_REQUIRE(n_slots_of(opt) == 1 || slot1, CTR_ERR_INVALID_ARG, "ctr_opt_sparse_rows: slot1 required");
  cudaStream_t st = as_stream(stream);
#define ROWS_K(OPT, KK, LPR, VEC)                                                                 \
  case KK:                                                                                        \
    opt_sparse_rows_kernel<OPT, LPR, VEC><<<(unsigned)ceil_div64(n_max * LPR, 256), 256, 0, st>>>( \
        var, slot0, slot1, uniq, n_uniq, g_uniq, n_max, hyper, stage);                            \
    break;
#define ROWS_CALL(OPT)                                                                            \
  switch (K) {                                                                                    \
    ROWS_K(OPT, 4, 1, 1) ROWS_K(OPT, 8, 2, 1) ROWS_K(OPT, 16, 4, 1) ROWS_K(OPT, 32, 8, 1)         \
    ROWS_K(OPT, 64, 16, 1) ROWS_K(OPT, 128, 32, 1) ROWS_K(OPT, 256, 32, 2)                        \
    default:                                                                                      \
      opt_sparse_generic_kernel<OPT><<<(unsigned)ceil_div64(n_max * K, 256), 256, 0, st>>>(       \
          var, slot0, slot1, uniq, n_uniq, g_uniq, n_max, K, hyper, stage);                       \
  }
  CTR_OPT_SWITCH(opt, ROWS_CALL)
#undef ROWS_CALL
#undef ROWS_K
  CTR_LAUNCHED("ctr_opt_sparse_rows");
  return CTR_OK;
}

int ctr_opt_dense_sweep(int opt, float* var, float* slot0, float* slot1, int64_t n_elem,
                        const float* hyper, float* sumsq_partials, int* n_partials_host,
                        ctr_stream_t stream) {
  CTR_REQUIRE(n_elem >= 0, CTR_ERR_INVALID_ARG, "ctr_opt_dense_sweep: n_elem < 0");
  // tuning hook (tools/tune_sweep.py): CTR_SWEEP_CFG = 0..3 selects (unroll, CTAs/SM)
  static int cfg = -1;
  if (cfg < 0) {
    const char* e = getenv("CTR_SWEEP_CFG");
    cfg = e ? atoi(e) : 0;
    if (cfg < 0 || cfg > 3) cfg = 0;
  }
  static const int kBlocksPerSm[4] = {2, 4, 3, 6};
  const int grid = sm_count() * kBlocksPerSm[cfg];
  if (n_partials_host) *n_partials_host = sm_count() * 8;
  if (n_elem == 0) return CTR_OK;
  CTR_REQUIRE(var && slot0 && hyper, CTR_ERR_INVALID_ARG, "ctr_opt_dense_sweep: null buffer");
  CTR_REQUIRE(n_slots_of(opt) == 1 || slot1, CTR_ERR_INVALID_ARG, "ctr_opt_dense_sweep: slot1 required");
  CTR_REQUIRE(((uintptr_t)var & 15) == 0 && ((uintptr_t)slot0 & 15) == 0 && ((uintptr_t)slot1 & 15) == 0,
              CTR_ERR_INVALID_ARG, "ctr_opt_dense_sweep: tensors must be 16-byte aligned");
  cudaStream_t st = as_stream(stream);
  const int64_t n4 = n_elem / 4;
#define SWEEP_LAUNCH(OPT, U, MB)                                                                   \
  opt_dense_sweep_kernel<OPT, U, MB><<<grid, SWEEP_THREADS, 0, st>>>(var, slot0, slot1, n4, n_elem, \
                                                                     hyper, sumsq_partials)
#define SWEEP_CALL(OPT)                                   \
  switch (cfg) {                                          \
    case 1: SWEEP_LAUNCH(OPT, 2, 4); break;               \
    case 2: SWEEP_LAUNCH(OPT, 4, 3); break;               \
    case 3: SWEEP_LAUNCH(OPT, 1, 6); break;               \
    default: SWEEP_LAUNCH(OPT, 4, 2); break;              \
  }
  CTR_OPT_SWITCH(opt, SWEEP_CALL)
#undef SWEEP_CALL
#undef SWEEP_LAUNCH
  CTR_LAUNCHED("ctr_opt_dense_sweep");
  return CTR_OK;
}

int ctr_opt_patch_rows(float* var, float* slot0, float* slot1, const int32_t* uniq,
                       const int32_t* n_uniq, const float* stage, int64_t n_max, int K, int n_slots,
                       ctr_stream_t stream) {
  CTR_REQUIRE(n_max >= 0 && K > 0 && (n_slots == 1 || n_slots == 2), CTR_ERR_INVALID_ARG,
              "ctr_opt_patch_rows: bad n_max/K/n_slots");
  if (n_max == 0) return CTR_OK;
  CTR_REQUIRE(var && slot0 && uniq && n_uniq && stage && (n_slots == 1 || slot1), CTR_ERR_INVALID_ARG,
              "ctr_opt_patch_rows: null buffer");
  opt_patch_rows_kernel<<<(unsigned)ceil_div64(n_max * K, 256), 256, 0, as_stream(stream)>>>(
      var, slot0, slot1, uniq, n_uniq, stage, n_max, K, n_slots);
  CTR_LAUNCHED("ctr_opt_patch_rows");
  return CTR_OK;
}

int ctr_opt_dense_grad(int opt, float* var, float* slot0, float* slot1, const float* grad,
                       int64_t n_elem, const float* hyper, ctr_stream_t stream) {
  CTR_REQUIRE(n_elem >= 0, CTR_ERR_INVALID_ARG, "ctr_opt_dense_grad: n_elem < 0");
  if (n_elem == 0) return CTR_OK;
  CTR_REQUIRE(var && slot0 && grad && hyper, CTR_ERR_INVALID_ARG, "ctr_opt_dense_grad: null buffer");
  CTR_REQUIRE(n_slots_of(opt) == 1 || slot1, CTR_ERR_INVALID_ARG, "ctr_opt_dense_grad: slot1 required");
  cudaStream_t st = as_stream(stream);
  int64_t b = ceil_div64(n_elem, 256);
  const int grid = (int)(b > (int64_t)sm_count() * 8 ? (int64_t)sm_count() * 8 : b);
#define DG_CALL(OPT) opt_dense_grad_kernel<OPT><<<grid, 256, 0, st>>>(var, slot0, slot1, grad, n_elem, hyper);
  CTR_OPT_SWITCH(opt, DG_CALL)
#undef DG_CALL
  CTR_LAUNCHED("ctr_opt_dense_grad");
  return CTR_OK;
}

int ctr_adam_tick(float* state, float* hyper, int n_hyper, ctr_stream_t stream) {
  CTR_REQUIRE(state && hyper && n_hyper >= 1, CTR_ERR_INVALID_ARG, "ctr_adam_tick: bad args");
  adam_tick_kernel<<<1, 1, 0, as_stream(stream)>>>(state, hyper, n_hyper);
  CTR_LAUNCHED("ctr_adam_tick");
  return CTR_OK;
}

int ctr_reduce_sum(const float* in, int64_t n, float scale, float* out, float* ws, size_t ws_bytes,
                   ctr_stream_t stream) {
  CTR_REQUIRE(n >= 0 && out, CTR_ERR_INVALID_ARG, "ctr_reduce_sum: bad args");
  cudaStream_t st = as_stream(stream);
  const int grid = reduce_grid(n);
  CTR_REQUIRE(ws && ws_bytes >= (size_t)grid * 4, CTR_ERR_WORKSPACE, "ctr_reduce_sum: workspace too small");
  CTR_REQUIRE(n == 0 || in, CTR_ERR_INVALID_ARG, "ctr_reduce_sum: null input");
  reduce_partial_kernel<false><<<grid, RED_THREADS, 0, st>>>(in, n, ws);
  CTR_LAUNCHED("reduce_partial");
  reduce_final_kernel<<<1, RED_THREADS, 0, st>>>(ws, grid, scale, out);
  CTR_LAUNCHED("reduce_final");
  return CTR_OK;
}

size_t ctr_l2_loss_workspace_bytes(int64_t n) { return (size_t)RED_MAX_BLOCKS * 4; }

int ctr_l2_loss(const float* t, int64_t n, float scale, float* out, void* ws, size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE(n >= 0 && out, CTR_ERR_INVALID_ARG, "ctr_l2_loss: bad args");
  cudaStream_t st = as_stream(stream);
  const int grid = reduce_grid(n);
  CTR_REQUIRE(ws && ws_bytes >= (size_t)grid * 4, CTR_ERR_WORKSPACE, "ctr_l2_loss: workspace too small");
  CTR_REQUIRE(n == 0 || t, CTR_ERR_INVALID_ARG, "ctr_l2_loss: null input");
  reduce_partial_kernel<true><<<grid, RED_THREADS, 0, st>>>(t, n, reinterpret_cast<float*>(ws));
  CTR_LAUNCHED("l2_partial");
  reduce_final_kernel<<<1, RED_THREADS, 0, st>>>(reinterpret_cast<float*>(ws), grid, 0.5f * scale, out);
  CTR_LAUNCHED("l2_final");
  return CTR_OK;
}

}  // extern "C"
