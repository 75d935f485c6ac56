// din.cu -- K6/K9: the pieces of DIN's embedding + field-wise pooling layers that are not GEMMs.
//
// Replaces (DIN.py):
//   :143-147  tf.nn.embedding_lookup(Feat_Emb, feat_ids / a_catids / ...)     -> gather_scale_rows
//   :148,180-183  tf.nn.embedding_lookup_sparse(..., combiner="sum")          -> bag_sum fwd/bwd
//   :153-159  sparse_tensor_to_dense ids/weights, lookup, multiply            -> gather_scale_rows
//   :165-172  sigmoid attention weight, mask (id > 0), weighted sum over P    -> din_pool fwd/bwd
// The attention MLP itself ([e, e-a, a] @ W, DIN.py:161-169) runs on the fc.cu GEMM with the
// algebraic split  [e, e-a, a] @ [W1;W2;W3] = e @ (W1+W2) + a @ (W3-W2):  the position-wise product
// shrinks from 3K to K and the ad part becomes one row per sample (3x fewer FLOPs, same value up to
// fp32 rounding).  All kernels here are HBM-bound gathers/streams.
#include "common.cuh"

namespace ctr {

// out[(i / G) * ld_group + (i % G) * K + k] = V[ids[i]][k] * (wgt ? wgt[i] : 1)
template <int LPR, int VEC>
__global__ void __launch_bounds__(256)
gather_scale_rows_kernel(const int32_t* __restrict__ ids, const float* __restrict__ wgt,
                         const float* __restrict__ V, int64_t N, int64_t n, int G, int64_t ld_group,
                         float* __restrict__ out, int32_t* __restrict__ oob) {
  constexpr int K = 4 * LPR * VEC;
  const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / LPR;
  const int c = threadIdx.x % LPR;
  if (i >= n) return;
  int64_t id = ids[i];
  float w = wgt ? wgt[i] : 1.f;
  if (id < 0 || id >= N) {
    if (oob && c == 0) { if (atomicAdd(&oob[0], 1) == 0) oob[1] = (int32_t)id; }
    id = 0; w = 0.f;
  }
  const float4* row = reinterpret_cast<const float4*>(V + id * K) + c;
  float4* o = reinterpret_cast<float4*>(out + (i / G) * ld_group + (i % G) * K) + c;
#pragma unroll
  for (int v = 0; v < VEC; ++v) o[v * LPR] = f4_scale(__ldg(row + v * LPR), w);
}

// out[b*ld + k] = sum_{i in [off[b], off[b+1])} V[ids[i]][k] * w_i      (one lane group per bag)
// ids outside [0, N) add nothing and are counted into oob like gather_scale_rows_kernel
template <int LPR, int VEC>
__global__ void __launch_bounds__(256)
bag_sum_fwd_kernel(const int32_t* __restrict__ ids, const float* __restrict__ wgt,
                   const int32_t* __restrict__ offsets, const float* __restrict__ V, int64_t N, int B,
                   int64_t ld, float* __restrict__ out, int32_t* __restrict__ oob) {
  constexpr int K = 4 * LPR * VEC;
  const int b = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / LPR);
  const int c = threadIdx.x % LPR;
  if (b >= B) return;
  float4 acc[VEC];
#pragma unroll
  for (int v = 0; v < VEC; ++v) acc[v] = f4_zero();
  for (int i = offsets[b]; i < offsets[b + 1]; ++i) {
    int64_t id = ids[i];
    float w = wgt ? wgt[i] : 1.f;
    if (id < 0 || id >= N) {
      if (oob && c == 0) { if (atomicAdd(&oob[0], 1) == 0) oob[1] = (int32_t)id; }
      id = 0; w = 0.f;
    }
    const float4* row = reinterpret_cast<const float4*>(V + id * K) + c;
#pragma unroll
    for (int v = 0; v < VEC; ++v) acc[v] = f4_fma(__ldg(row + v * LPR), make_float4(w, w, w, w), acc[v]);
  }
  float4* o = reinterpret_cast<float4*>(out + (int64_t)b * ld) + c;
#pragma unroll
  for (int v = 0; v < VEC; ++v) o[v * LPR] = acc[v];
}

// g_rows[i][k] = d_out[b(i)*ld + k] * w_i
template <int LPR, int VEC>
__global__ void __launch_bounds__(256)
bag_sum_bwd_kernel(const float* __restrict__ d_out, int64_t ld, const float* __restrict__ wgt,
                   const int32_t* __restrict__ offsets, int B, float* __restrict__ g_rows) {
  constexpr int K = 4 * LPR * VEC;
  const int b = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / LPR);
  const int c = threadIdx.x % LPR;
  if (b >= B) return;
  const float4* d = reinterpret_cast<const float4*>(d_out + (int64_t)b * ld) + c;
  float4 g[VEC];
#pragma unroll
  for (int v = 0; v < VEC; ++v) g[v] = d[v * LPR];
  for (int i = offsets[b]; i < offsets[b + 1]; ++i) {
    const float w = wgt ? wgt[i] : 1.f;
    float4* o = reinterpret_cast<float4*>(g_rows + (int64_t)i * K) + c;
#pragma unroll
    for (int v = 0; v < VEC; ++v) o[v * LPR] = f4_scale(g[v], w);
  }
}

// out[i][:] = (x[(i/G)*ld_group + (i%G)*K + :] + (add ? add[i][:] : 0)) * (w ? w[i] : 1)
// (un-concatenates a slice of d x_deep into per-occurrence gradient rows)
template <int LPR, int VEC>
__global__ void __launch_bounds__(256)
scale_rows_kernel(const float* __restrict__ x, const float* __restrict__ add, const float* __restrict__ w,
                  int64_t n, int G, int64_t ld_group, float* __restrict__ out) {
  constexpr int K = 4 * LPR * VEC;
  const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / LPR;
  const int c = threadIdx.x % LPR;
  if (i >= n) return;
  const float ww = w ? w[i] : 1.f;
  const float4* p = reinterpret_cast<const float4*>(x + (i / G) * ld_group + (i % G) * K) + c;
  const float4* q = add ? reinterpret_cast<const float4*>(add + i * K) + c : nullptr;
  float4* o = reinterpret_cast<float4*>(out + i * K) + c;
#pragma unroll
  for (int v = 0; v < VEC; ++v) {
    float4 t = p[v * LPR];
    if (q) t = f4_add(t, q[v * LPR]);
    o[v * LPR] = f4_scale(t, ww);
  }
}

// attention pooling forward: att = sigmoid(z); u[b] = sum_p (id > 0) * att * E[b,p,:]    (DIN.py:169-172)
// one warp per sample; LPR lanes per row, 32/LPR positions per iteration
template <int LPR, int VEC>
__global__ void __launch_bounds__(128)
din_pool_fwd_kernel(const float* __restrict__ E, const float* __restrict__ z, const int32_t* __restrict__ ids,
                    int B, int P, float* __restrict__ att, float* __restrict__ u, int64_t ld_u) {
  constexpr int K = 4 * LPR * VEC;
  constexpr int RPW = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  const int slot = lane / LPR, c = lane % LPR;
  float4 acc[VEC];
#pragma unroll
  for (int v = 0; v < VEC; ++v) acc[v] = f4_zero();
  for (int p0 = 0; p0 < P; p0 += RPW) {
    const int p = p0 + slot;
    if (p < P) {
      const int64_t i = (int64_t)b * P + p;
      const float a = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-z[i])));
      if (c == 0) att[i] = a;
      const float m = (ids[i] > 0) ? a : 0.f;
      const float4* row = reinterpret_cast<const float4*>(E + i * K) + c;
#pragma unroll
      for (int v = 0; v < VEC; ++v) acc[v] = f4_fma(row[v * LPR], make_float4(m, m, m, m), acc[v]);
    }
  }
#pragma unroll
  for (int o = LPR; o < 32; o <<= 1)
#pragma unroll
    for (int v = 0; v < VEC; ++v) acc[v] = f4_add(acc[v], f4_shfl_xor(acc[v], o));
  if (slot == 0) {
    float4* up = reinterpret_cast<float4*>(u + (int64_t)b * ld_u) + c;
#pragma unroll
    for (int v = 0; v < VEC; ++v) up[v * LPR] = acc[v];
  }
}

// backward: dE[b,p,:] = m*att*du ; dz[b,p] = m * att*(1-att) * (E[b,p,:] . du)      (m = id > 0)
template <int LPR, int VEC>
__global__ void __launch_bounds__(128)
din_pool_bwd_kernel(const float* __restrict__ E, const float* __restrict__ att, const int32_t* __restrict__ ids,
                    const float* __restrict__ du, int64_t ld_u, int B, int P, float* __restrict__ dE,
                    float* __restrict__ dz) {
  constexpr int K = 4 * LPR * VEC;
  constexpr int RPW = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  const int slot = lane / LPR, c = lane % LPR;
  float4 g[VEC];
  const float4* dp = reinterpret_cast<const float4*>(du + (int64_t)b * ld_u) + c;
#pragma unroll
  for (int v = 0; v < VEC; ++v) g[v] = dp[v * LPR];
  for (int p0 = 0; p0 < P; p0 += RPW) {
    const int p = p0 + slot;
    const bool ok = p < P;
    const int64_t i = (int64_t)b * P + (ok ? p : 0);
    const float a = ok ? att[i] : 0.f;
    const float m = (ok && ids[i] > 0) ? 1.f : 0.f;
    float dot = 0.f;
    if (ok) {
      const float4* row = reinterpret_cast<const float4*>(E + i * K) + c;
      float4* o = reinterpret_cast<float4*>(dE + i * K) + c;
      const float s = m * a;
#pragma unroll
      for (int v = 0; v < VEC; ++v) {
        const float4 e = row[v * LPR];
        dot += (e.x * g[v].x + e.y * g[v].y) + (e.z * g[v].z + e.w * g[v].w);
        o[v * LPR] = f4_scale(g[v], s);
      }
    }
#pragma unroll
    for (int o = 1; o < LPR; o <<= 1) dot += __shfl_xor_sync(FULL_MASK, dot, o);
    if (ok && c == 0) dz[i] = m * a * (1.f - a) * dot;
  }
}

// out = alpha*a + beta*b
__global__ void axpby_kernel(const float* __restrict__ a, float alpha, const float* __restrict__ b, float beta,
                             int64_t n, float* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = alpha * a[i] + beta * b[i];
}

}  // namespace ctr

using namespace ctr;

#define DIN_K_SWITCH(K, CALL)                                                                      \
  switch (K) {                                                                                     \
    case 4: { CALL(1, 1) } break;   case 8: { CALL(2, 1) } break;   case 16: { CALL(4, 1) } break;  \
    case 32: { CALL(8, 1) } break;  case 64: { CALL(16, 1) } break; case 128: { CALL(32, 1) } break; \
    case 256: { CALL(32, 2) } break;                                                               \
    default:                                                                                       \
      set_error("K=%d unsupported here (must be one of 4,8,16,32,64,128,256)", K);                 \
      return CTR_ERR_UNSUPPORTED;                                                                  \
  }


// ---- attention unit backward, the [B*P, H] hidden layer in ONE pass ------------------------------------------
// Replaces three passes over the hidden activations of a behaviour field (autodiff of DIN.py:164-169):
//   fc1_bwd   dHh[r][c] = dz[r]*w2[c]                      (+ gw2 = sum_r dz[r]*Hh[r][c], gb2 = sum_r dz[r])
//   fc_dz     dZ = dHh*mask/keep * (Hh > 0)                (+ db1 = colsum dZ)
//   sum_p     dU[b][c] = sum_p dZ[b*P+p][c]              (the group-bias gradient)
// One CTA per sample (its P rows are contiguous); a thread owns column(s) c, walks the P rows, writes dZ, and keeps
// sum_p dZ (= dU row b; db1 = colsum(dU)) and sum_p dz*Hh (gw2 partial row b) in registers: no atomics, fixed order.
__global__ void __launch_bounds__(256)
din_att_dz_kernel(const float* __restrict__ Hh, const float* __restrict__ mask, float keep, const float* __restrict__ dz,
                  const float* __restrict__ w2, int P, int H, float* __restrict__ dZ, float* __restrict__ dU,
                  float* __restrict__ gw2_part) {
  const int b = blockIdx.x;
  const int64_t row0 = (int64_t)b * P;
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    const float wc = w2[c];
    float su = 0.f, sg = 0.f;
    for (int p = 0; p < P; ++p) {
      const int64_t i = (row0 + p) * H + c;
      const float d0 = dz[row0 + p], h = Hh[i];
      float d = d0 * wc;
      if (mask) d = __fdiv_rn(d * mask[i], keep);
      if (!(h > 0.f)) d = 0.f;
      dZ[i] = d;
      su += d;
      sg = fmaf(h, d0, sg);
    }
    dU[(int64_t)b * H + c] = su;
    gw2_part[(int64_t)b * H + c] = sg;
  }
}

extern "C" {

int ctr_gather_scale_rows(const int32_t* ids, const float* wgt, const float* V, int64_t N, int64_t n, int K,
                          int G, int64_t ld_group, float* out, int32_t* oob, ctr_stream_t stream) {
  CTR_REQUIRE(n >= 0 && K > 0 && G >= 1 && N > 0, CTR_ERR_INVALID_ARG, "ctr_gather_scale_rows: bad args");
  if (n == 0) return CTR_OK;
  CTR_REQUIRE(ids && V && out, CTR_ERR_INVALID_ARG, "ctr_gather_scale_rows: null buffer");
  CTR_REQUIRE(ld_group % 4 == 0, CTR_ERR_INVALID_ARG, "ctr_gather_scale_rows: ld_group must be a multiple of 4");
  cudaStream_t st = as_stream(stream);
#define GS(LPR, VEC)                                                                                     \
  gather_scale_rows_kernel<LPR, VEC><<<(unsigned)ceil_div64(n * LPR, 256), 256, 0, st>>>(ids, wgt, V, N, n, G, \
                                                                                         ld_group, out, oob);
  DIN_K_SWITCH(K, GS)
#undef GS
  CTR_LAUNCHED("ctr_gather_scale_rows");
  return CTR_OK;
}

int ctr_bag_sum_fwd_oob(const int32_t* ids, const float* wgt, const int32_t* offsets, const float* V, int64_t N,
                        int B, int K, int64_t ld, float* out, int32_t* oob, ctr_stream_t stream) {
  CTR_REQUIRE(B >= 0 && K > 0 && N > 0, CTR_ERR_INVALID_ARG, "ctr_bag_sum_fwd_oob: bad args");
  if (B == 0) return CTR_OK;
  CTR_REQUIRE(offsets && V && out, CTR_ERR_INVALID_ARG, "ctr_bag_sum_fwd_oob: null buffer");
  cudaStream_t st = as_stream(stream);
#define BF(LPR, VEC)                                                                                                   \
  bag_sum_fwd_kernel<LPR, VEC><<<(unsigned)ceil_div64((int64_t)B * LPR, 256), 256, 0, st>>>(ids, wgt, offsets, V, N, B, \
                                                                                            ld, out, oob);
  DIN_K_SWITCH(K, BF)
#undef BF
  CTR_LAUNCHED("ctr_bag_sum_fwd_oob");
  return CTR_OK;
}

int ctr_bag_sum_bwd(const float* d_out, int64_t ld, const float* wgt, const int32_t* offsets, int B, int K,
                    float* g_rows, ctr_stream_t stream) {
  CTR_REQUIRE(B >= 0 && K > 0, CTR_ERR_INVALID_ARG, "ctr_bag_sum_bwd: bad args");
  if (B == 0) return CTR_OK;
  CTR_REQUIRE(d_out && offsets && g_rows, CTR_ERR_INVALID_ARG, "ctr_bag_sum_bwd: null buffer");
  cudaStream_t st = as_stream(stream);
#define BB(LPR, VEC) \
  bag_sum_bwd_kernel<LPR, VEC><<<(unsigned)ceil_div64((int64_t)B * LPR, 256), 256, 0, st>>>(d_out, ld, wgt, offsets, B, g_rows);
  DIN_K_SWITCH(K, BB)
#undef BB
  CTR_LAUNCHED("ctr_bag_sum_bwd");
  return CTR_OK;
}

int ctr_scale_rows(const float* x, const float* add, const float* w, int64_t n, int K, int G, int64_t ld_group,
                   float* out, ctr_stream_t stream) {
  CTR_REQUIRE(n >= 0 && K > 0 && G >= 1, CTR_ERR_INVALID_ARG, "ctr_scale_rows: bad args");
  if (n == 0) return CTR_OK;
  CTR_REQUIRE(x && out, CTR_ERR_INVALID_ARG, "ctr_scale_rows: null buffer");
  cudaStream_t st = as_stream(stream);
#define SR(LPR, VEC) \
  scale_rows_kernel<LPR, VEC><<<(unsigned)ceil_div64(n * LPR, 256), 256, 0, st>>>(x, add, w, n, G, ld_group, out);
  DIN_K_SWITCH(K, SR)
#undef SR
  CTR_LAUNCHED("ctr_scale_rows");
  return CTR_OK;
}

int ctr_din_pool_fwd(const float* E, const float* z, const int32_t* ids, int B, int P, int K, float* att, float* u,
                     int64_t ld_u, ctr_stream_t stream) {
  CTR_REQUIRE(B >= 0 && P >= 0 && K > 0, CTR_ERR_INVALID_ARG, "ctr_din_pool_fwd: bad args");
  if (B == 0) return CTR_OK;
  CTR_REQUIRE(E && z && ids && att && u, CTR_ERR_INVALID_ARG, "ctr_din_pool_fwd: null buffer");
  cudaStream_t st = as_stream(stream);
#define PF(LPR, VEC) din_pool_fwd_kernel<LPR, VEC><<<(B + 3) / 4, 128, 0, st>>>(E, z, ids, B, P, att, u, ld_u);
  DIN_K_SWITCH(K, PF)
#undef PF
  CTR_LAUNCHED("ctr_din_pool_fwd");
  return CTR_OK;
}

int ctr_din_pool_bwd(const float* E, const float* att, const int32_t* ids, const float* du, int64_t ld_u, int B,
                     int P, int K, float* dE, float* dz, ctr_stream_t stream) {
  CTR_REQUIRE(B >= 0 && P >= 0 && K > 0, CTR_ERR_INVALID_ARG, "ctr_din_pool_bwd: bad args");
  if (B == 0) return CTR_OK;
  CTR_REQUIRE(E && att && ids && du && dE && dz, CTR_ERR_INVALID_ARG, "ctr_din_pool_bwd: null buffer");
  cudaStream_t st = as_stream(stream);
#define PB(LPR, VEC) din_pool_bwd_kernel<LPR, VEC><<<(B + 3) / 4, 128, 0, st>>>(E, att, ids, du, ld_u, B, P, dE, dz);
  DIN_K_SWITCH(K, PB)
#undef PB
  CTR_LAUNCHED("ctr_din_pool_bwd");
  return CTR_OK;
}

int ctr_din_att_dz(const float* Hh, const float* drop_mask, float keep_prob, const float* dz, const float* w2, int B, int P,
                   int H, float* dZ, float* dU, float* gw2_part, ctr_stream_t stream) {
  CTR_REQUIRE(B >= 0 && P > 0 && H > 0, CTR_ERR_INVALID_ARG, "ctr_din_att_dz: bad shape");
  if (B == 0) return CTR_OK;
  CTR_REQUIRE(Hh && dz && w2 && dZ && dU && gw2_part, CTR_ERR_INVALID_ARG, "ctr_din_att_dz: null buffer");
  CTR_REQUIRE(!drop_mask || keep_prob > 0.f, CTR_ERR_INVALID_ARG, "ctr_din_att_dz: keep_prob must be > 0 with a mask");
  din_att_dz_kernel<<<B, 256, 0, as_stream(stream)>>>(Hh, drop_mask, keep_prob, dz, w2, P, H, dZ, dU, gw2_part);
  CTR_LAUNCHED("ctr_din_att_dz");
  return CTR_OK;
}

int ctr_axpby(const float* a, float alpha, const float* b, float beta, int64_t n, float* out, ctr_stream_t stream) {
  CTR_REQUIRE(n >= 0, CTR_ERR_INVALID_ARG, "ctr_axpby: n < 0");
  if (n == 0) return CTR_OK;
  CTR_REQUIRE(a && b && out, CTR_ERR_INVALID_ARG, "ctr_axpby: null buffer");
  int64_t blocks = ceil_div64(n, 256 * 4);
  const int grid = (int)(blocks < (int64_t)sm_count() * 8 ? blocks : (int64_t)sm_count() * 8);
  axpby_kernel<<<grid, 256, 0, as_stream(stream)>>>(a, alpha, b, beta, n, out);
  CTR_LAUNCHED("ctr_axpby");
  return CTR_OK;
}

}  // extern "C"
