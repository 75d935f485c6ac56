// fm_embed.cu -- K1/K2: sparse-id -> embedding gather, value scaling, FM first/second order
// (or NFM bi-interaction, or plain gather), emit x; and the backward w.r.t. the gathered rows.
//
// Replaces (reference, relative to deep_ctr/Model_pipeline/):
//   DeepFM.py:125-127  First-order   y_w = sum_f W[ids]*vals
//   DeepFM.py:129-135  Second-order  e = V[ids]*vals ; y_v = 0.5*sum_k((sum_f e)^2 - sum_f e^2)
//   DeepFM.py:151      deep_inputs = reshape(e, [B, F*K])
//   NFM.py:122-128     bi = 0.5*((sum_f e)^2 - sum_f e^2)          (mode NFM)
//   DCN.py:135-138, PNN.py:134-136, AFM.py:128-130   e only       (mode PLAIN)
//
// Layout / mapping (HBM-bound, no reuse => no smem):
//   one warp per sample.  A row of K floats is read by LPR = K/4 lanes as one 128-bit load each
//   (K=16: 4 lanes x 16 B = one 64 B row = two full 32 B sectors), so a warp has 32/LPR rows in
//   flight per load instruction and the whole field loop is unrolled => all row loads of a sample
//   are issued before the first use.  ids/vals are read coalesced (one field per lane) and
//   broadcast with shuffles; the first-order scalar gather is done one-field-per-lane as well
//   (32 independent 4 B gathers in flight).  x is written as float4 (sample-contiguous, coalesced).
#include <stdlib.h>

#include "common.cuh"

namespace ctr {

template <typename IdT>
__device__ __forceinline__ int64_t load_id(const void* ids, int64_t i) {
  return (int64_t) reinterpret_cast<const IdT*>(ids)[i];
}

// LPR lanes per row, VEC float4 per lane: K = 4*LPR*VEC
template <int LPR, int VEC, typename IdT>
__global__ void __launch_bounds__(128)
fm_embed_fwd_kernel(const void* __restrict__ ids, const float* __restrict__ vals,
                    const float* __restrict__ V, const float* __restrict__ W, int64_t N, int B,
                    int F, int mode, float* __restrict__ x, float* __restrict__ y_w,
                    float* __restrict__ y2, float* __restrict__ S, int32_t* __restrict__ oob) {
  constexpr int K = 4 * LPR * VEC;
  constexpr int RPW = 32 / LPR;                       // rows per warp-wide load
  constexpr int ITERS = 32 / RPW;                     // iterations per 32-field chunk (== LPR)
  constexpr int UNROLL = (ITERS <= 8) ? ITERS : 8;
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  const int slot = lane / LPR;
  const int c = lane % LPR;

  float4 s[VEC], q[VEC];
#pragma unroll
  for (int v = 0; v < VEC; ++v) { s[v] = f4_zero(); q[v] = f4_zero(); }
  float yw = 0.f;

  const int64_t base = (int64_t)b * F;
  for (int fbase = 0; fbase < F; fbase += 32) {
    const int fl = fbase + lane;
    int64_t id_l = 0;
    float val_l = 0.f;
    if (fl < F) {
      id_l = load_id<IdT>(ids, base + fl);
      val_l = vals[base + fl];
      if (id_l < 0 || id_l >= N) {                    // TF: InvalidArgument on CPU; here: count it
        if (oob) { if (atomicAdd(&oob[0], 1) == 0) oob[1] = (int32_t)id_l; }
        id_l = 0; val_l = 0.f;
      }
      if (W) yw = fmaf(__ldg(W + id_l), val_l, yw);
    }
    const int nf = min(32, F - fbase);
#pragma unroll UNROLL
    for (int it = 0; it < ITERS; ++it) {
      const int fj = it * RPW + slot;                 // field inside this chunk
      const int64_t id = __shfl_sync(FULL_MASK, id_l, fj);
      const float val = __shfl_sync(FULL_MASK, val_l, fj);
      if (fj < nf) {
        const float4* row = reinterpret_cast<const float4*>(V + id * K) + c;
        float4 e[VEC];
#pragma unroll
        for (int v = 0; v < VEC; ++v) e[v] = f4_scale(__ldg(row + v * LPR), val);
#pragma unroll
        for (int v = 0; v < VEC; ++v) {
          s[v] = f4_add(s[v], e[v]);
          q[v] = f4_fma(e[v], e[v], q[v]);
        }
        if (x) {
          float4* xr = reinterpret_cast<float4*>(x + (base + fbase + fj) * K) + c;
#pragma unroll
          for (int v = 0; v < VEC; ++v) xr[v * LPR] = e[v];
        }
      }
    }
  }

  if (W && y_w) {
    yw = warp_sum(yw);
    if (lane == 0) y_w[b] = yw;
  }
  if (mode == CTR_FM_PLAIN) return;

  // combine the RPW row slots
#pragma unroll
  for (int o = LPR; o < 32; o <<= 1) {
#pragma unroll
    for (int v = 0; v < VEC; ++v) { s[v] = f4_add(s[v], f4_shfl_xor(s[v], o)); q[v] = f4_add(q[v], f4_shfl_xor(q[v], o)); }
  }
  if (S && slot == 0) {
    float4* Sr = reinterpret_cast<float4*>(S + (int64_t)b * K) + c;
#pragma unroll
    for (int v = 0; v < VEC; ++v) Sr[v * LPR] = s[v];
  }
  // d = S*S - q, with S*S rounded first (as tf.square then tf.subtract do): a sample with a single
  // active field gives exactly 0, like the reference.
  float4 d[VEC];
#pragma unroll
  for (int v = 0; v < VEC; ++v)
    d[v] = make_float4(__fmul_rn(s[v].x, s[v].x) - q[v].x, __fmul_rn(s[v].y, s[v].y) - q[v].y,
                       __fmul_rn(s[v].z, s[v].z) - q[v].z, __fmul_rn(s[v].w, s[v].w) - q[v].w);
  if (mode == CTR_FM_NFM) {
    if (slot == 0) {
      float4* o = reinterpret_cast<float4*>(y2 + (int64_t)b * K) + c;
#pragma unroll
      for (int v = 0; v < VEC; ++v) o[v * LPR] = f4_scale(d[v], 0.5f);
    }
  } else {
    float t = 0.f;
#pragma unroll
    for (int v = 0; v < VEC; ++v) t += f4_hsum(d[v]);
#pragma unroll
    for (int o = 1; o < LPR; o <<= 1) t += __shfl_xor_sync(FULL_MASK, t, o);
    if (lane == 0) y2[b] = 0.5f * t;
  }
}


// ---- K1 with the rows staged in shared memory by the TMA engine (1-D bulk copies) -----------------------------
// north_star: "TMA staging of embedding rows into shared memory".  Same mapping and the same arithmetic order as
// fm_embed_fwd_kernel (=> bit-identical outputs); the only difference is how a row travels: one lane per field
// issues cp.async.bulk global -> shared (K*4 bytes, completion counted on the warp's mbarrier) instead of K/4
// lanes issuing 128-bit loads into registers.  Selected with CTR_FM_EMBED_TMA=1 (tools/bench_kernels.py measures
// both; DESIGN.md records the result).  One warp per sample, F <= 64, K in {16, 32, 64, 128}.
__device__ __forceinline__ uint32_t fe_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

template <int LPR, int VEC, typename IdT>
__global__ void __launch_bounds__(128)
fm_embed_fwd_tma_kernel(const void* __restrict__ ids, const float* __restrict__ vals,
                        const float* __restrict__ V, const float* __restrict__ W, int64_t N, int B,
                        int F, int mode, float* __restrict__ x, float* __restrict__ y_w,
                        float* __restrict__ y2, float* __restrict__ S, int32_t* __restrict__ oob) {
  constexpr int K = 4 * LPR * VEC;
  constexpr int RPW = 32 / LPR;
  constexpr int ITERS = 32 / RPW;
  constexpr int UNROLL = (ITERS <= 8) ? ITERS : 8;
  extern __shared__ __align__(128) uint8_t fe_smem[];
  __shared__ __align__(8) uint64_t bars[4];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.x * (blockDim.x >> 5) + warp;
  float* rows = reinterpret_cast<float*>(fe_smem) + (size_t)warp * F * K;      // [F][K] of this warp's sample
  const uint32_t bar = fe_smem_u32(&bars[warp]);
  if (lane == 0) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncwarp();
  if (b >= B) return;
  const int slot = lane / LPR;
  const int c = lane % LPR;
  const int64_t base = (int64_t)b * F;
  float yw = 0.f;
  int64_t id_l[2] = {0, 0};
  float val_l[2] = {0.f, 0.f};
  if (lane == 0) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"((uint32_t)(F * K * 4)) : "memory");
  }
  __syncwarp();
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int fl = h * 32 + lane;
    if (fl < F) {
      int64_t id = load_id<IdT>(ids, base + fl);
      float val = vals[base + fl];
      if (id < 0 || id >= N) {
        if (oob) { if (atomicAdd(&oob[0], 1) == 0) oob[1] = (int32_t)id; }
        id = 0; val = 0.f;
      }
      id_l[h] = id; val_l[h] = val;
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                       fe_smem_u32(rows + (size_t)fl * K)),
                   "l"(V + id * K), "r"((uint32_t)(K * 4)), "r"(bar)
                   : "memory");
      if (W) yw = fmaf(__ldg(W + id), val, yw);
    }
  }
  {  // wait for all F rows of this sample
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "FE_WAIT:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n\t"
        "@p bra FE_DONE;\n\t"
        "bra FE_WAIT;\n\t"
        "FE_DONE:\n\t"
        "}" ::"r"(bar) : "memory");
  }
  float4 s[VEC], q[VEC];
#pragma unroll
  for (int v = 0; v < VEC; ++v) { s[v] = f4_zero(); q[v] = f4_zero(); }
  for (int fbase = 0, h = 0; fbase < F; fbase += 32, ++h) {
    const int nf = min(32, F - fbase);
#pragma unroll UNROLL
    for (int it = 0; it < ITERS; ++it) {
      const int fj = it * RPW + slot;
      const float val = __shfl_sync(FULL_MASK, h == 0 ? val_l[0] : val_l[1], fj);
      if (fj < nf) {
        const float4* row = reinterpret_cast<const float4*>(rows + (size_t)(fbase + fj) * K) + c;
        float4 e[VEC];
#pragma unroll
        for (int v = 0; v < VEC; ++v) e[v] = f4_scale(row[v * LPR], val);
#pragma unroll
        for (int v = 0; v < VEC; ++v) {
          s[v] = f4_add(s[v], e[v]);
          q[v] = f4_fma(e[v], e[v], q[v]);
        }
        if (x) {
          float4* xr = reinterpret_cast<float4*>(x + (base + fbase + fj) * K) + c;
#pragma unroll
          for (int v = 0; v < VEC; ++v) xr[v * LPR] = e[v];
        }
      }
    }
  }
  if (W && y_w) {
    yw = warp_sum(yw);
    if (lane == 0) y_w[b] = yw;
  }
  if (mode == CTR_FM_PLAIN) return;
#pragma unroll
  for (int o = LPR; o < 32; o <<= 1) {
#pragma unroll
    for (int v = 0; v < VEC; ++v) { s[v] = f4_add(s[v], f4_shfl_xor(s[v], o)); q[v] = f4_add(q[v], f4_shfl_xor(q[v], o)); }
  }
  if (S && slot == 0) {
    float4* Sr = reinterpret_cast<float4*>(S + (int64_t)b * K) + c;
#pragma unroll
    for (int v = 0; v < VEC; ++v) Sr[v * LPR] = s[v];
  }
  float4 d[VEC];
#pragma unroll
  for (int v = 0; v < VEC; ++v)
    d[v] = make_float4(__fmul_rn(s[v].x, s[v].x) - q[v].x, __fmul_rn(s[v].y, s[v].y) - q[v].y,
                       __fmul_rn(s[v].z, s[v].z) - q[v].z, __fmul_rn(s[v].w, s[v].w) - q[v].w);
  if (mode == CTR_FM_NFM) {
    if (slot == 0) {
      float4* o = reinterpret_cast<float4*>(y2 + (int64_t)b * K) + c;
#pragma unroll
      for (int v = 0; v < VEC; ++v) o[v * LPR] = f4_scale(d[v], 0.5f);
    }
  } else {
    float t = 0.f;
#pragma unroll
    for (int v = 0; v < VEC; ++v) t += f4_hsum(d[v]);
#pragma unroll
    for (int o = 1; o < LPR; o <<= 1) t += __shfl_xor_sync(FULL_MASK, t, o);
    if (lane == 0) y2[b] = 0.5f * t;
  }
}

// any K: one warp per sample, lanes stride over k, fields sequential.  Correct, not fast.
template <typename IdT>
__global__ void __launch_bounds__(128)
fm_embed_fwd_generic_kernel(const void* __restrict__ ids, const float* __restrict__ vals,
                            const float* __restrict__ V, const float* __restrict__ W, int64_t N,
                            int B, int F, int K, int mode, float* __restrict__ x,
                            float* __restrict__ y_w, float* __restrict__ y2, float* __restrict__ S,
                            int32_t* __restrict__ oob) {
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  const int64_t base = (int64_t)b * F;
  float yw = 0.f, yv = 0.f;
  for (int k0 = 0; k0 < K; k0 += 32) {
    const int k = k0 + lane;
    float s = 0.f, q = 0.f;
    for (int f = 0; f < F; ++f) {
      int64_t id = load_id<IdT>(ids, base + f);
      float val = vals[base + f];
      if (id < 0 || id >= N) {
        if (oob && lane == 0 && k0 == 0) { if (atomicAdd(&oob[0], 1) == 0) oob[1] = (int32_t)id; }
        id = 0; val = 0.f;
      }
      if (W && k == 0) yw = fmaf(__ldg(W + id), val, yw);
      if (k < K) {
        float e = __ldg(V + id * K + k) * val;
        s += e;
        q = fmaf(e, e, q);
        if (x) x[(base + f) * K + k] = e;
      }
    }
    if (mode != CTR_FM_PLAIN && k < K) {
      if (S) S[(int64_t)b * K + k] = s;
      float d = __fmul_rn(s, s) - q;
      if (mode == CTR_FM_NFM) y2[(int64_t)b * K + k] = 0.5f * d;
      else yv += d;
    }
  }
  if (W && y_w && lane == 0) y_w[b] = yw;
  if (mode == CTR_FM_DEEPFM) {
    yv = warp_sum(yv);
    if (lane == 0) y2[b] = 0.5f * yv;
  }
}

// ---- backward ----------------------------------------------------------------------------------
// g_e = dy2*(S - e) + dX   (DeepFM: dy2 scalar per sample; NFM: dy2 per (sample,k); PLAIN: dX only)
// g_rows = g_e * val ; g_w = dyw * val.   Everything is a coalesced stream (x was saved by fwd).
template <int LPR, int VEC>
__global__ void __launch_bounds__(128)
fm_embed_bwd_kernel(const float* __restrict__ vals, const float* __restrict__ x,
                    const float* __restrict__ S, const float* __restrict__ dX,
                    const float* __restrict__ dy2, const float* __restrict__ dyw, int B, int F,
                    int mode, float* __restrict__ g_rows, float* __restrict__ g_w) {
  constexpr int K = 4 * LPR * VEC;
  constexpr int RPW = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  const int slot = lane / LPR;
  const int c = lane % LPR;
  const int64_t base = (int64_t)b * F;

  float4 s[VEC], w2[VEC];
#pragma unroll
  for (int v = 0; v < VEC; ++v) { s[v] = f4_zero(); w2[v] = f4_zero(); }
  if (mode != CTR_FM_PLAIN) {
    const float4* Sr = reinterpret_cast<const float4*>(S + (int64_t)b * K) + c;
#pragma unroll
    for (int v = 0; v < VEC; ++v) s[v] = Sr[v * LPR];
    if (mode == CTR_FM_DEEPFM) {
      const float d = dy2[b];
#pragma unroll
      for (int v = 0; v < VEC; ++v) w2[v] = make_float4(d, d, d, d);
    } else {
      const float4* dr = reinterpret_cast<const float4*>(dy2 + (int64_t)b * K) + c;
#pragma unroll
      for (int v = 0; v < VEC; ++v) w2[v] = dr[v * LPR];
    }
  }
  if (g_w) {
    const float d = dyw[b];
    for (int f = lane; f < F; f += 32) g_w[base + f] = d * vals[base + f];
  }
#pragma unroll 4
  for (int f = slot; f < F; f += RPW) {
    const float val = vals[base + f];
    const int64_t off = (base + f) * K;
    float4 g[VEC];
#pragma unroll
    for (int v = 0; v < VEC; ++v) g[v] = f4_zero();
    if (dX) {
      const float4* dr = reinterpret_cast<const float4*>(dX + off) + c;
#pragma unroll
      for (int v = 0; v < VEC; ++v) g[v] = ld_stream4(dr + v * LPR);
    }
    if (mode != CTR_FM_PLAIN) {
      const float4* xr = reinterpret_cast<const float4*>(x + off) + c;
#pragma unroll
      for (int v = 0; v < VEC; ++v) g[v] = f4_fma(w2[v], f4_sub(s[v], xr[v * LPR]), g[v]);
    }
    float4* o = reinterpret_cast<float4*>(g_rows + off) + c;
#pragma unroll
    for (int v = 0; v < VEC; ++v) o[v * LPR] = f4_scale(g[v], val);
  }
}

__global__ void __launch_bounds__(128)
fm_embed_bwd_generic_kernel(const float* __restrict__ vals, const float* __restrict__ x,
                            const float* __restrict__ S, const float* __restrict__ dX,
                            const float* __restrict__ dy2, const float* __restrict__ dyw, int B,
                            int F, int K, int mode, float* __restrict__ g_rows,
                            float* __restrict__ g_w) {
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  const int64_t base = (int64_t)b * F;
  if (g_w) {
    const float d = dyw[b];
    for (int f = lane; f < F; f += 32) g_w[base + f] = d * vals[base + f];
  }
  for (int k = lane; k < K; k += 32) {
    float s = 0.f, w2 = 0.f;
    if (mode != CTR_FM_PLAIN) {
      s = S[(int64_t)b * K + k];
      w2 = (mode == CTR_FM_DEEPFM) ? dy2[b] : dy2[(int64_t)b * K + k];
    }
    for (int f = 0; f < F; ++f) {
      const int64_t off = (base + f) * K + k;
      float g = dX ? dX[off] : 0.f;
      if (mode != CTR_FM_PLAIN) g = fmaf(w2, s - x[off], g);
      g_rows[off] = g * vals[base + f];
    }
  }
}

template <typename IdT>
static int launch_fwd(const void* ids, const float* vals, const float* V, const float* W, int64_t N,
                      int B, int F, int K, int mode, float* x, float* y_w, float* y2, float* S,
                      int32_t* oob, cudaStream_t st) {
  const int wpb = 4;
  dim3 grid((B + wpb - 1) / wpb), block(wpb * 32);
  // bulk copies pay off only for long rows => default: TMA staging for K == 128 (512 B rows) only; CTR_FM_EMBED_TMA=0/1 forces
  static int use_tma = -2;
  if (use_tma == -2) { const char* e = getenv("CTR_FM_EMBED_TMA"); use_tma = e ? atoi(e) : -1; }
  const bool tma = use_tma == 1 || (use_tma == -1 && K == 128);
  if (tma && F <= 64 && (K == 16 || K == 32 || K == 64 || K == 128)) {
    const size_t smem = (size_t)wpb * F * K * 4;
#define TMA_CASE(KK, LPR, VEC)                                                                             \
  case KK: {                                                                                               \
    static size_t set = 0;                                                                                 \
    if (smem > set) {                                                                                      \
      cudaFuncSetAttribute(fm_embed_fwd_tma_kernel<LPR, VEC, IdT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
      set = smem;                                                                                          \
    }                                                                                                      \
    fm_embed_fwd_tma_kernel<LPR, VEC, IdT><<<grid, block, smem, st>>>(ids, vals, V, W, N, B, F, mode, x, y_w, y2, S, oob); \
  } break;
    if (smem <= 200 * 1024) {
      switch (K) {
        TMA_CASE(16, 4, 1)
        TMA_CASE(32, 8, 1)
        TMA_CASE(64, 16, 1)
        TMA_CASE(128, 32, 1)
      }
#undef TMA_CASE
      CTR_LAUNCHED("ctr_fm_embed_fwd(tma)");
      return CTR_OK;
    }
  }
#define FWD_CASE(KK, LPR, VEC)                                                                     \
  case KK:                                                                                         \
    fm_embed_fwd_kernel<LPR, VEC, IdT><<<grid, block, 0, st>>>(ids, vals, V, W, N, B, F, mode, x,  \
                                                               y_w, y2, S, oob);                   \
    break;
  switch (K) {
    FWD_CASE(4, 1, 1)
    FWD_CASE(8, 2, 1)
    FWD_CASE(16, 4, 1)
    FWD_CASE(32, 8, 1)
    FWD_CASE(64, 16, 1)
    FWD_CASE(128, 32, 1)
    FWD_CASE(256, 32, 2)
    default:
      fm_embed_fwd_generic_kernel<IdT><<<grid, block, 0, st>>>(ids, vals, V, W, N, B, F, K, mode, x,
                                                               y_w, y2, S, oob);
  }
#undef FWD_CASE
  CTR_LAUNCHED("ctr_fm_embed_fwd");
  return CTR_OK;
}

}  // namespace ctr

using namespace ctr;

extern "C" {

int ctr_fm_embed_fwd(const void* ids, int id_bits, const float* vals, const float* V, const float* W,
                     int64_t N, int B, int F, int K, int mode, float* x, float* y_w, float* y2,
                     float* S, int32_t* oob, ctr_stream_t stream) {
  CTR_REQUIRE(B >= 0 && F >= 0 && K > 0 && N > 0, CTR_ERR_INVALID_ARG,
              "ctr_fm_embed_fwd: bad shape B=%d F=%d K=%d N=%lld", B, F, K, (long long)N);
  CTR_REQUIRE(id_bits == 32 || id_bits == 64, CTR_ERR_INVALID_ARG,
              "ctr_fm_embed_fwd: id_bits must be 32 or 64, got %d", id_bits);
  CTR_REQUIRE(mode >= CTR_FM_DEEPFM && mode <= CTR_FM_PLAIN, CTR_ERR_INVALID_ARG,
              "ctr_fm_embed_fwd: bad mode %d", mode);
  if (B == 0) return CTR_OK;
  CTR_REQUIRE(ids && vals && V, CTR_ERR_INVALID_ARG, "ctr_fm_embed_fwd: null ids/vals/V");
  CTR_REQUIRE((W == nullptr) == (y_w == nullptr), CTR_ERR_INVALID_ARG,
              "ctr_fm_embed_fwd: W and y_w must both be given or both be NULL");
  CTR_REQUIRE(mode == CTR_FM_PLAIN || (y2 && S), CTR_ERR_INVALID_ARG,
              "ctr_fm_embed_fwd: y2 and S are required unless mode is PLAIN");
  CTR_REQUIRE(mode != CTR_FM_PLAIN || x, CTR_ERR_INVALID_ARG,
              "ctr_fm_embed_fwd: x is required in PLAIN mode");
  if (id_bits == 32)
    return launch_fwd<int32_t>(ids, vals, V, W, N, B, F, K, mode, x, y_w, y2, S, oob, as_stream(stream));
  return launch_fwd<int64_t>(ids, vals, V, W, N, B, F, K, mode, x, y_w, y2, S, oob, as_stream(stream));
}

int ctr_fm_embed_bwd(const float* vals, const float* x, const float* S, const float* dX,
                     const float* dy2, const float* dyw, int B, int F, int K, int mode,
                     float* g_rows, float* g_w, ctr_stream_t stream) {
  CTR_REQUIRE(B >= 0 && F >= 0 && K > 0, CTR_ERR_INVALID_ARG, "ctr_fm_embed_bwd: bad shape");
  CTR_REQUIRE(mode >= CTR_FM_DEEPFM && mode <= CTR_FM_PLAIN, CTR_ERR_INVALID_ARG,
              "ctr_fm_embed_bwd: bad mode %d", mode);
  if (B == 0 || F == 0) return CTR_OK;
  CTR_REQUIRE(vals && g_rows, CTR_ERR_INVALID_ARG, "ctr_fm_embed_bwd: null vals/g_rows");
  CTR_REQUIRE(mode == CTR_FM_PLAIN || (x && S && dy2), CTR_ERR_INVALID_ARG,
              "ctr_fm_embed_bwd: x, S, dy2 required unless mode is PLAIN");
  CTR_REQUIRE(mode != CTR_FM_PLAIN || dX, CTR_ERR_INVALID_ARG,
              "ctr_fm_embed_bwd: dX required in PLAIN mode");
  CTR_REQUIRE((g_w == nullptr) == (dyw == nullptr), CTR_ERR_INVALID_ARG,
              "ctr_fm_embed_bwd: g_w and dyw must both be given or both be NULL");
  cudaStream_t st = as_stream(stream);
  const int wpb = 4;
  dim3 grid((B + wpb - 1) / wpb), block(wpb * 32);
#define BWD_CASE(KK, LPR, VEC)                                                                    \
  case KK:                                                                                        \
    fm_embed_bwd_kernel<LPR, VEC><<<grid, block, 0, st>>>(vals, x, S, dX, dy2, dyw, B, F, mode,   \
                                                          g_rows, g_w);                           \
    break;
  switch (K) {
    BWD_CASE(4, 1, 1)
    BWD_CASE(8, 2, 1)
    BWD_CASE(16, 4, 1)
    BWD_CASE(32, 8, 1)
    BWD_CASE(64, 16, 1)
    BWD_CASE(128, 32, 1)
    BWD_CASE(256, 32, 2)
    default:
      fm_embed_bwd_generic_kernel<<<grid, block, 0, st>>>(vals, x, S, dX, dy2, dyw, B, F, K, mode,
                                                          g_rows, g_w);
  }
#undef BWD_CASE
  CTR_LAUNCHED("ctr_fm_embed_bwd");
  return CTR_OK;
}

}  // extern "C"
