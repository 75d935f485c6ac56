// pairwise.cu -- K7/K8: all-pairs feature interactions of PNN and AFM.
//
// Replaces (pair order: i < j, row-major, PNN.py:144-147 / AFM.py:134-136; P = F(F-1)/2):
//   PNN.py:148-153  Inner:  inner[b,p] = <e_i, e_j>;   deep_inputs = concat([x, inner])
//   PNN.py:164-167  Outer:  outer[b,p,:,:] = e_i (x) e_j;  deep_inputs = concat([x, outer])  ("NOT ready yet")
//   AFM.py:132-138  element-wise products  pw[b,p,:] = e_i * e_j
//   AFM.py:151-162  softmax over the P pairs, dropout, attention-weighted sum -> y_emb [B,K]
// and their autodiff.  e = x.reshape(B,F,K) are the scaled embeddings K1 produced.
// One warp per sample; the sample's F*K floats are staged in shared memory (row stride K+1: the
// lanes of a warp read different rows at the same k => conflict-free).
#include "common.cuh"

namespace ctr {

constexpr int PW_WARPS = 4;

__device__ __forceinline__ void pair_of(int p, int F, int& i, int& j) {
  // p -> (i, j), i < j, row-major.  Solve by walking rows (F is small: <= a few hundred).
  int row = 0, rem = p, len = F - 1;
  while (rem >= len) { rem -= len; --len; ++row; }
  i = row; j = row + 1 + rem;
}

// z[b] = [x[b] (F*K) | tail], tail = inner (P) or outer (P*K*K)
template <bool OUTER>
__global__ void __launch_bounds__(PW_WARPS * 32)
pnn_fwd_kernel(const float* __restrict__ x, int B, int F, int K, float* __restrict__ z) {
  extern __shared__ float sm[];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int b = blockIdx.x * PW_WARPS + wid;
  const int FK = F * K, P = F * (F - 1) / 2, KP = K + 1;
  float* e = sm + (int64_t)wid * F * KP;
  if (b >= B) return;
  const int64_t ldz = FK + (OUTER ? (int64_t)P * K * K : P);
  float* zr = z + (int64_t)b * ldz;
  for (int t = lane; t < FK; t += 32) {
    const float v = x[(int64_t)b * FK + t];
    e[(t / K) * KP + (t % K)] = v;
    zr[t] = v;
  }
  __syncwarp();
  if (!OUTER) {
    for (int p = lane; p < P; p += 32) {
      int i, j;
      pair_of(p, F, i, j);
      float s = 0.f;
      for (int k = 0; k < K; ++k) s = fmaf(e[i * KP + k], e[j * KP + k], s);
      zr[FK + p] = s;
    }
  } else {
    const int KK = K * K;
    for (int p = 0; p < P; ++p) {
      int i, j;
      pair_of(p, F, i, j);
      for (int t = lane; t < KK; t += 32) zr[FK + (int64_t)p * KK + t] = e[i * KP + t / K] * e[j * KP + t % K];
    }
  }
}

// dX[b] = dz[b, :FK] + sum over pairs of the product-rule terms
template <bool OUTER>
__global__ void __launch_bounds__(PW_WARPS * 32)
pnn_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dz, int B, int F, int K,
               float* __restrict__ dX) {
  extern __shared__ float sm[];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int b = blockIdx.x * PW_WARPS + wid;
  const int FK = F * K, P = F * (F - 1) / 2, KP = K + 1;
  float* e = sm + (int64_t)wid * 2 * F * KP;
  float* g = e + F * KP;
  if (b >= B) return;
  const int64_t ldz = FK + (OUTER ? (int64_t)P * K * K : P);
  const float* dzr = dz + (int64_t)b * ldz;
  for (int t = lane; t < FK; t += 32) {
    e[(t / K) * KP + (t % K)] = x[(int64_t)b * FK + t];
    g[(t / K) * KP + (t % K)] = dzr[t];
  }
  __syncwarp();
  // lanes own elements t = (field f, k); each accumulates over the F-1 pairs that contain f
  for (int t = lane; t < FK; t += 32) {
    const int f = t / K, k = t % K;
    float acc = 0.f;
    for (int o = 0; o < F; ++o) {
      if (o == f) continue;
      const int i = min(f, o), j = max(f, o);
      const int p = i * (2 * F - i - 1) / 2 + (j - i - 1);
      if (!OUTER) {
        acc = fmaf(dzr[FK + p], e[o * KP + k], acc);
      } else {
        const float* d = dzr + FK + (int64_t)p * K * K;   // d[a*K + c] multiplies e_i[a]*e_j[c]
        if (f == i) { for (int c = 0; c < K; ++c) acc = fmaf(d[k * K + c], e[o * KP + c], acc); }
        else        { for (int a = 0; a < K; ++a) acc = fmaf(d[a * K + k], e[o * KP + a], acc); }
      }
    }
    dX[(int64_t)b * FK + t] = g[f * KP + k] + acc;
  }
}

// AFM: pw[b,p,:] = e_i * e_j
__global__ void __launch_bounds__(256)
afm_pairs_fwd_kernel(const float* __restrict__ x, int B, int F, int K, float* __restrict__ pw) {
  const int P = F * (F - 1) / 2;
  const int64_t n = (int64_t)B * P * K;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += stride) {
    const int k = (int)(t % K);
    const int64_t bp = t / K;
    const int p = (int)(bp % P);
    const int64_t b = bp / P;
    int i, j;
    pair_of(p, F, i, j);
    const float* xr = x + b * F * K;
    pw[t] = xr[i * K + k] * xr[j * K + k];
  }
}

// dX[b,f,k] = sum_{o != f} dpw[b, pair(f,o), k] * e[b,o,k]
__global__ void __launch_bounds__(256)
afm_pairs_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dpw, int B, int F, int K,
                     float* __restrict__ dX) {
  const int P = F * (F - 1) / 2;
  const int64_t n = (int64_t)B * F * K;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += stride) {
    const int k = (int)(t % K);
    const int f = (int)((t / K) % F);
    const int64_t b = t / ((int64_t)F * K);
    const float* xr = x + b * F * K;
    const float* dr = dpw + b * P * K;
    float acc = 0.f;
    for (int o = 0; o < F; ++o) {
      if (o == f) continue;
      const int i = min(f, o), j = max(f, o);
      const int p = i * (2 * F - i - 1) / 2 + (j - i - 1);
      acc = fmaf(dr[(int64_t)p * K + k], xr[o * K + k], acc);
    }
    dX[t] = acc;
  }
}

// softmax over the P pair logits of a sample, dropout on the weights, weighted sum of pw -> y_emb.
// att_out[b,p] = softmax (pre-dropout, saved for the backward)
__global__ void __launch_bounds__(256)
afm_pool_fwd_kernel(const float* __restrict__ pw, const float* __restrict__ logit, const float* __restrict__ mask,
                    float keep, int B, int P, int K, float* __restrict__ att_out, float* __restrict__ y_emb) {
  __shared__ float red[256];
  extern __shared__ float w_s[];  // [P] weights after dropout
  const int b = blockIdx.x, tid = threadIdx.x;
  const float* lg = logit + (int64_t)b * P;
  float m = -INFINITY;
  for (int p = tid; p < P; p += 256) m = fmaxf(m, lg[p]);
  red[tid] = m; __syncthreads();
  for (int o = 128; o > 0; o >>= 1) { if (tid < o) red[tid] = fmaxf(red[tid], red[tid + o]); __syncthreads(); }
  m = red[0]; __syncthreads();
  float s = 0.f;
  for (int p = tid; p < P; p += 256) { const float ex = expf(lg[p] - m); w_s[p] = ex; s += ex; }
  red[tid] = s; __syncthreads();
  for (int o = 128; o > 0; o >>= 1) { if (tid < o) red[tid] += red[tid + o]; __syncthreads(); }
  s = red[0]; __syncthreads();
  for (int p = tid; p < P; p += 256) {
    const float a = __fdiv_rn(w_s[p], s);
    att_out[(int64_t)b * P + p] = a;
    w_s[p] = mask ? __fdiv_rn(a, keep) * mask[(int64_t)b * P + p] : a;
  }
  __syncthreads();
  for (int k = tid; k < K; k += 256) {
    float acc = 0.f;
    for (int p = 0; p < P; ++p) acc = fmaf(w_s[p], pw[((int64_t)b * P + p) * K + k], acc);
    y_emb[(int64_t)b * K + k] = acc;
  }
}

// backward of the above: dpw = w * dy_emb ; dlogit = softmax-backward of d w
__global__ void __launch_bounds__(256)
afm_pool_bwd_kernel(const float* __restrict__ pw, const float* __restrict__ att, const float* __restrict__ mask,
                    float keep, const float* __restrict__ dy_emb, int B, int P, int K, float* __restrict__ dpw,
                    float* __restrict__ dlogit) {
  __shared__ float red[256];
  extern __shared__ float da_s[];  // [P] gradient w.r.t. the softmax output
  const int b = blockIdx.x, tid = threadIdx.x;
  const float* dy = dy_emb + (int64_t)b * K;
  // d w_p = <pw_p, dy> ; d a_p = d w_p * mask/keep ; dpw_p = w_p * dy
  for (int p = tid; p < P; p += 256) {
    const float a = att[(int64_t)b * P + p];
    const float mk = mask ? mask[(int64_t)b * P + p] : 1.f;
    const float w = mask ? __fdiv_rn(a, keep) * mk : a;
    const float* pr = pw + ((int64_t)b * P + p) * K;
    float* dr = dpw + ((int64_t)b * P + p) * K;
    float dot = 0.f;
    for (int k = 0; k < K; ++k) { dot = fmaf(pr[k], dy[k], dot); dr[k] = w * dy[k]; }
    da_s[p] = mask ? __fdiv_rn(dot * mk, keep) : dot;
  }
  __syncthreads();
  float s = 0.f;
  for (int p = tid; p < P; p += 256) s = fmaf(da_s[p], att[(int64_t)b * P + p], s);
  red[tid] = s; __syncthreads();
  for (int o = 128; o > 0; o >>= 1) { if (tid < o) red[tid] += red[tid + o]; __syncthreads(); }
  s = red[0];
  for (int p = tid; p < P; p += 256) {
    const float a = att[(int64_t)b * P + p];
    dlogit[(int64_t)b * P + p] = a * (da_s[p] - s);
  }
}

// out = x / keep * mask  (tf.nn.dropout on a tensor that is not the output of one of our GEMMs)
__global__ void dropout_apply_kernel(const float* __restrict__ x, const float* __restrict__ mask, float keep, int64_t n,
                                     float* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    out[i] = __fdiv_rn(x[i], keep) * mask[i];
}

}  // namespace ctr

using namespace ctr;

extern "C" {

int ctr_pnn_product_fwd(const float* x, int B, int F, int K, int outer, float* z, ctr_stream_t stream) {
  CTR_REQUIRE(B >= 0 && F >= 2 && K > 0, CTR_ERR_INVALID_ARG, "ctr_pnn_product_fwd: bad shape");
  const size_t smem = (size_t)PW_WARPS * F * (K + 1) * sizeof(float);
  CTR_REQUIRE(smem <= 200 * 1024, CTR_ERR_UNSUPPORTED,
              "ctr_pnn_product_fwd: F*K too large for shared memory (got F=%d K=%d)", F, K);
  if (B == 0) return CTR_OK;
  CTR_REQUIRE(x && z, CTR_ERR_INVALID_ARG, "ctr_pnn_product_fwd: null buffer");
  cudaStream_t st = as_stream(stream);
  const int grid = (B + PW_WARPS - 1) / PW_WARPS;
  if (outer) {
    cudaFuncSetAttribute(pnn_fwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    pnn_fwd_kernel<true><<<grid, PW_WARPS * 32, smem, st>>>(x, B, F, K, z);
  } else {
    cudaFuncSetAttribute(pnn_fwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    pnn_fwd_kernel<false><<<grid, PW_WARPS * 32, smem, st>>>(x, B, F, K, z);
  }
  CTR_LAUNCHED("ctr_pnn_product_fwd");
  return CTR_OK;
}

int ctr_pnn_product_bwd(const float* x, const float* dz, int B, int F, int K, int outer, float* dX,
                        ctr_stream_t stream) {
  CTR_REQUIRE(B >= 0 && F >= 2 && K > 0, CTR_ERR_INVALID_ARG, "ctr_pnn_product_bwd: bad shape");
  const size_t smem = (size_t)PW_WARPS * 2 * F * (K + 1) * sizeof(float);
  CTR_REQUIRE(smem <= 200 * 1024, CTR_ERR_UNSUPPORTED,
              "ctr_pnn_product_bwd: F*K too large for shared memory (got F=%d K=%d)", F, K);
  if (B == 0) return CTR_OK;
  CTR_REQUIRE(x && dz && dX, CTR_ERR_INVALID_ARG, "ctr_pnn_product_bwd: null buffer");
  cudaStream_t st = as_stream(stream);
  const int grid = (B + PW_WARPS - 1) / PW_WARPS;
  if (outer) {
    cudaFuncSetAttribute(pnn_bwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    pnn_bwd_kernel<true><<<grid, PW_WARPS * 32, smem, st>>>(x, dz, B, F, K, dX);
  } else {
    cudaFuncSetAttribute(pnn_bwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    pnn_bwd_kernel<false><<<grid, PW_WARPS * 32, smem, st>>>(x, dz, B, F, K, dX);
  }
  CTR_LAUNCHED("ctr_pnn_product_bwd");
  return CTR_OK;
}

static int ew_grid(int64_t n) {
  int64_t b = ceil_div64(n, 256 * 4);
  return (int)(b < (int64_t)sm_count() * 16 ? (b < 1 ? 1 : b) : (int64_t)sm_count() * 16);
}

int ctr_afm_pairs_fwd(const float* x, int B, int F, int K, float* pw, ctr_stream_t stream) {
  CTR_REQUIRE(B >= 0 && F >= 2 && K > 0, CTR_ERR_INVALID_ARG, "ctr_afm_pairs_fwd: bad shape");
  if (B == 0) return CTR_OK;
  CTR_REQUIRE(x && pw, CTR_ERR_INVALID_ARG, "ctr_afm_pairs_fwd: null buffer");
  afm_pairs_fwd_kernel<<<ew_grid((int64_t)B * (F * (F - 1) / 2) * K), 256, 0, as_stream(stream)>>>(x, B, F, K, pw);
  CTR_LAUNCHED("ctr_afm_pairs_fwd");
  return CTR_OK;
}

int ctr_afm_pairs_bwd(const float* x, const float* dpw, int B, int F, int K, float* dX, ctr_stream_t stream) {
  CTR_REQUIRE(B >= 0 && F >= 2 && K > 0, CTR_ERR_INVALID_ARG, "ctr_afm_pairs_bwd: bad shape");
  if (B == 0) return CTR_OK;
  CTR_REQUIRE(x && dpw && dX, CTR_ERR_INVALID_ARG, "ctr_afm_pairs_bwd: null buffer");
  afm_pairs_bwd_kernel<<<ew_grid((int64_t)B * F * K), 256, 0, as_stream(stream)>>>(x, dpw, B, F, K, dX);
  CTR_LAUNCHED("ctr_afm_pairs_bwd");
  return CTR_OK;
}

int ctr_afm_pool_fwd(const float* pw, const float* logit, const float* mask, float keep, int B, int P, int K,
                     float* att, float* y_emb, ctr_stream_t stream) {
  CTR_REQUIRE(B >= 0 && P > 0 && K > 0, CTR_ERR_INVALID_ARG, "ctr_afm_pool_fwd: bad shape");
  CTR_REQUIRE((size_t)P * 4 <= 40 * 1024, CTR_ERR_UNSUPPORTED,
              "ctr_afm_pool_fwd: too many pairs (got P=%d, the limit is 10240)", P);
  if (B == 0) return CTR_OK;
  CTR_REQUIRE(pw && logit && att && y_emb, CTR_ERR_INVALID_ARG, "ctr_afm_pool_fwd: null buffer");
  afm_pool_fwd_kernel<<<B, 256, (size_t)P * 4, as_stream(stream)>>>(pw, logit, mask, keep, B, P, K, att, y_emb);
  CTR_LAUNCHED("ctr_afm_pool_fwd");
  return CTR_OK;
}

int ctr_afm_pool_bwd(const float* pw, const float* att, const float* mask, float keep, const float* dy_emb, int B,
                     int P, int K, float* dpw, float* dlogit, ctr_stream_t stream) {
  CTR_REQUIRE(B >= 0 && P > 0 && K > 0, CTR_ERR_INVALID_ARG, "ctr_afm_pool_bwd: bad shape");
  CTR_REQUIRE((size_t)P * 4 <= 40 * 1024, CTR_ERR_UNSUPPORTED,
              "ctr_afm_pool_bwd: too many pairs (got P=%d, the limit is 10240)", P);
  if (B == 0) return CTR_OK;
  CTR_REQUIRE(pw && att && dy_emb && dpw && dlogit, CTR_ERR_INVALID_ARG, "ctr_afm_pool_bwd: null buffer");
  afm_pool_bwd_kernel<<<B, 256, (size_t)P * 4, as_stream(stream)>>>(pw, att, mask, keep, dy_emb, B, P, K, dpw, dlogit);
  CTR_LAUNCHED("ctr_afm_pool_bwd");
  return CTR_OK;
}

int ctr_dropout_apply(const float* x, const float* mask, float keep, int64_t n, float* out, ctr_stream_t stream) {
  CTR_REQUIRE(n >= 0 && keep > 0.f, CTR_ERR_INVALID_ARG, "ctr_dropout_apply: bad args");
  if (n == 0) return CTR_OK;
  CTR_REQUIRE(x && mask && out, CTR_ERR_INVALID_ARG, "ctr_dropout_apply: null buffer");
  dropout_apply_kernel<<<ew_grid(n), 256, 0, as_stream(stream)>>>(x, mask, keep, n, out);
  CTR_LAUNCHED("ctr_dropout_apply");
  return CTR_OK;
}

}  // extern "C"
