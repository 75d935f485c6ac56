// esmm.cu -- ESMM (DeepCvrMTL): the shared embedding layer over CSR bags and the multi-task head.
//
// Replaces (DeepMTL/Model_pipeline/DeepCvrMTL.py):
//   :153-164  embedding_lookup(feat_ids / a_*ids), embedding_lookup_sparse(u_*ids, u_*vals, "sum"),
//             embedding_lookup_sparse(a_intids, None, "sum") and the concat          -> esmm_embed_fwd
//             and their autodiff (per-occurrence gradient rows)                       -> esmm_embed_bwd
//   :205-223  pctr, pcvr, pctcvr = pctr*pcvr, the two task losses and their autodiff  -> esmm_head
//
// Batch layout (one CSR over 5B bags, bag j*B + b = field j of sample b, j = u_cat, u_shop, u_brand, u_int, a_int):
//   occurrences [bag_off[j*B+b], bag_off[j*B+b+1]) of bag_ids / bag_wgt; bag_off[5B] = nnz.  a_int is unweighted
//   (sp_weights=None, :159): its bag_wgt entries are never read.
// x [B, (F'+8)K] = [common F'K | u_cat | u_shop | u_brand | u_int | a_cat | a_shop | a_brand | a_int]   (:164)
// g_rows (the model's ids_all order) = [common B*F' (row b*F'+f) | a_cat B | a_shop B | a_brand B | occurrences nnz |
//   zero rows up to n_rows].
//
// Numerics of the bags: acc = +0; for each occurrence in order: acc = acc + (e * w), two IEEE-rounded ops (no FMA:
// TF multiplies the gathered rows by the weights, then segment-sums).  An empty bag is a +0 row; id 0 is a real row.
// The backward writes dx_slice * w (one rounded multiply; TF's gradient of segment_sum followed by `*= weights`).
// An id outside [0, N) is counted into oob[0] (oob[1] = the first one seen) like gather_scale_rows and contributes
// a zero row, so the host's check_ids() raises.
//
// Mapping: one lane group of K/4 lanes (float4 each; K = 256 uses 32 lanes x 2 float4) per (segment, sample), where
// segment 0 is the F'+3 plain lookups of the sample and segments 1..5 are its five bags.  The sums are sequential per
// bag, but U rows are loaded before any of them is added, so a long bag keeps U independent loads in flight.
#include "common.cuh"

namespace ctr {

constexpr int ESMM_BAGS = 5;           // u_cat, u_shop, u_brand, u_int, a_int
constexpr int ESMM_HEAD_THREADS = 1024;
constexpr float ESMM_LOG_EPS = 1e-7f;  // tf.losses.log_loss default epsilon

__device__ __forceinline__ float4 f4_mul_rn(float4 a, float s) {
  return make_float4(__fmul_rn(a.x, s), __fmul_rn(a.y, s), __fmul_rn(a.z, s), __fmul_rn(a.w, s));
}
__device__ __forceinline__ float4 f4_add_rn(float4 a, float4 b) {
  return make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z), __fadd_rn(a.w, b.w));
}

// column of bag kind j inside a row of x
__device__ __forceinline__ int64_t esmm_bag_col(int j, int Fp, int K) {
  return (int64_t)(j < 4 ? Fp + j : Fp + 7) * K;
}

__device__ __forceinline__ bool esmm_id_ok(int64_t id, int64_t N, int32_t* oob, bool count) {
  if (id >= 0 && id < N) return true;
  if (oob && count) { if (atomicAdd(&oob[0], 1) == 0) oob[1] = (int32_t)id; }
  return false;
}

template <int LPR, int VEC>
__global__ void __launch_bounds__(256)
esmm_embed_fwd_kernel(const int32_t* __restrict__ feat_ids, const int32_t* __restrict__ a_ids,
                      const int32_t* __restrict__ bag_ids, const float* __restrict__ bag_wgt,
                      const int32_t* __restrict__ bag_off, const float* __restrict__ V, int64_t N, int B, int Fp,
                      float* __restrict__ x, int32_t* __restrict__ oob) {
  constexpr int K = 4 * LPR * VEC;
  constexpr int U = 8 / VEC;           // rows in flight per lane group
  const int64_t t = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / LPR;
  const int c = threadIdx.x % LPR;
  if (t >= (int64_t)(ESMM_BAGS + 1) * B) return;
  const int seg = (int)(t / B), b = (int)(t % B);
  float* xr = x + (int64_t)b * (Fp + 8) * K;
  if (seg == 0) {                      // F' common lookups, then a_cat, a_shop, a_brand
    const int n = Fp + 3;
    for (int f0 = 0; f0 < n; f0 += U) {
      float4 r[U][VEC];
      bool ok[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int f = f0 + u;
        ok[u] = false;
        if (f < n) {
          const int64_t id = f < Fp ? feat_ids[(int64_t)b * Fp + f] : a_ids[(int64_t)(f - Fp) * B + b];
          ok[u] = esmm_id_ok(id, N, oob, c == 0);
          const float4* row = reinterpret_cast<const float4*>(V + (ok[u] ? id : 0) * K) + c;
#pragma unroll
          for (int v = 0; v < VEC; ++v) r[u][v] = ok[u] ? __ldg(row + v * LPR) : f4_zero();
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int f = f0 + u;
        if (f < n) {
          float4* o = reinterpret_cast<float4*>(xr + (int64_t)(f < Fp ? f : Fp + 4 + (f - Fp)) * K) + c;
#pragma unroll
          for (int v = 0; v < VEC; ++v) o[v * LPR] = r[u][v];
        }
      }
    }
    return;
  }
  const int j = seg - 1;
  const bool weighted = j < 4;
  const int beg = bag_off[(int64_t)j * B + b], end = bag_off[(int64_t)j * B + b + 1];
  float4 acc[VEC];
#pragma unroll
  for (int v = 0; v < VEC; ++v) acc[v] = f4_zero();
  for (int i0 = beg; i0 < end; i0 += U) {
    float4 r[U][VEC];
    float w[U];
    bool ok[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = i0 + u;
      ok[u] = false;
      w[u] = 1.f;
      if (i < end) {
        const int64_t id = bag_ids[i];
        ok[u] = esmm_id_ok(id, N, oob, c == 0);
        if (weighted) w[u] = bag_wgt[i];
        const float4* row = reinterpret_cast<const float4*>(V + (ok[u] ? id : 0) * K) + c;
#pragma unroll
        for (int v = 0; v < VEC; ++v) r[u][v] = ok[u] ? __ldg(row + v * LPR) : f4_zero();
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {      // occurrence order: acc = acc + e*w
      if (ok[u]) {
#pragma unroll
        for (int v = 0; v < VEC; ++v) acc[v] = f4_add_rn(acc[v], weighted ? f4_mul_rn(r[u][v], w[u]) : r[u][v]);
      }
    }
  }
  float4* o = reinterpret_cast<float4*>(xr + esmm_bag_col(j, Fp, K)) + c;
#pragma unroll
  for (int v = 0; v < VEC; ++v) o[v * LPR] = acc[v];
}

template <int LPR, int VEC>
__global__ void __launch_bounds__(256)
esmm_embed_bwd_kernel(const float* __restrict__ dx, const float* __restrict__ bag_wgt,
                      const int32_t* __restrict__ bag_off, int B, int Fp, int64_t n_rows, float* __restrict__ g) {
  constexpr int K = 4 * LPR * VEC;
  const int64_t t = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / LPR;
  const int64_t groups = (int64_t)gridDim.x * blockDim.x / LPR;
  const int c = threadIdx.x % LPR;
  const int64_t occ0 = (int64_t)B * (Fp + 3);            // first occurrence row
  if (t < (int64_t)(ESMM_BAGS + 1) * B) {
    const int seg = (int)(t / B), b = (int)(t % B);
    const float* dr = dx + (int64_t)b * (Fp + 8) * K;
    if (seg == 0) {
      for (int f = 0; f < Fp + 3; ++f) {
        const int64_t row = f < Fp ? (int64_t)b * Fp + f : (int64_t)B * Fp + (int64_t)(f - Fp) * B + b;
        const float4* s = reinterpret_cast<const float4*>(dr + (int64_t)(f < Fp ? f : Fp + 4 + (f - Fp)) * K) + c;
        float4* o = reinterpret_cast<float4*>(g + row * K) + c;
#pragma unroll
        for (int v = 0; v < VEC; ++v) o[v * LPR] = s[v * LPR];
      }
    } else {
      const int j = seg - 1;
      const bool weighted = j < 4;
      const int beg = bag_off[(int64_t)j * B + b], end = bag_off[(int64_t)j * B + b + 1];
      const float4* s = reinterpret_cast<const float4*>(dr + esmm_bag_col(j, Fp, K)) + c;
      float4 d[VEC];
#pragma unroll
      for (int v = 0; v < VEC; ++v) d[v] = s[v * LPR];
      for (int i = beg; i < end && occ0 + i < n_rows; ++i) {
        const float w = weighted ? bag_wgt[i] : 1.f;
        float4* o = reinterpret_cast<float4*>(g + (occ0 + i) * K) + c;
#pragma unroll
        for (int v = 0; v < VEC; ++v) o[v * LPR] = weighted ? f4_mul_rn(d[v], w) : d[v];
      }
    }
  }
  // slots past the batch's occurrences: zero rows (every lane group takes a strided share)
  for (int64_t row = occ0 + bag_off[(int64_t)ESMM_BAGS * B] + t; row < n_rows; row += groups) {
    float4* o = reinterpret_cast<float4*>(g + row * K) + c;
#pragma unroll
    for (int v = 0; v < VEC; ++v) o[v * LPR] = f4_zero();
  }
}

__device__ __forceinline__ float esmm_block_sum(float v, float* sh) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
  if (threadIdx.x < 32) t = warp_sum(sh[threadIdx.x]);
  __syncthreads();
  return t;  // valid in warp 0
}

__device__ __forceinline__ float esmm_sigmoid(float y) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-y))); }

// See ctr_esmm_head in include/ctr_b200.h for the formulas.  Every operation of the gradient chain is one explicitly
// rounded fp32 op in TF's order (nothing is contracted to an FMA).
__global__ void __launch_bounds__(ESMM_HEAD_THREADS)
esmm_head_kernel(const float* __restrict__ y_ctr, const float* __restrict__ y_cvr, const float* __restrict__ y,
                 const float* __restrict__ z, int B, int n, float w_ctr, float w_cvr, float* __restrict__ pctr,
                 float* __restrict__ pcvr, float* __restrict__ pctcvr, float* __restrict__ losses,
                 float* __restrict__ d_ctr, float* __restrict__ d_cvr) {
  __shared__ float sh[32];
  const bool train = y != nullptr;
  const float g_ctr = __fdiv_rn(w_ctr, (float)n);      // MeanGrad of w*reduce_mean(CE)
  const float g_cvr = __fdiv_rn(w_cvr, (float)n);      // (1-w) * log_loss's sum / num_present
  float l_ctr = 0.f, l_cvr = 0.f;
  for (int i = threadIdx.x; i < B; i += ESMM_HEAD_THREADS) {
    const float a = y_ctr[i], c = y_cvr[i];
    const float pt = esmm_sigmoid(a), pv = esmm_sigmoid(c);
    const float p = __fmul_rn(pt, pv);
    if (pctr) pctr[i] = pt;
    if (pcvr) pcvr[i] = pv;
    if (pctcvr) pctcvr[i] = p;
    if (!train) continue;
    if (i >= n) {
      if (d_ctr) d_ctr[i] = 0.f;
      if (d_cvr) d_cvr[i] = 0.f;
      continue;
    }
    const float t = y[i], zz = z[i], nz = __fsub_rn(1.f, zz);
    const float q1 = __fadd_rn(p, ESMM_LOG_EPS), q2 = __fadd_rn(__fsub_rn(1.f, p), ESMM_LOG_EPS);
    l_ctr += __fadd_rn(__fsub_rn(fmaxf(a, 0.f), __fmul_rn(a, t)), log1pf(expf(-fabsf(a))));
    l_cvr += __fsub_rn(-__fmul_rn(zz, logf(q1)), __fmul_rn(nz, logf(q2)));
    const float ng = -g_cvr;
    const float c1 = __fmul_rn(__fmul_rn(ng, zz), __frcp_rn(q1));       // through log(p + eps)
    const float c2 = -__fmul_rn(__fmul_rn(ng, nz), __frcp_rn(q2));      // through log(1 - p + eps)
    const float dp = __fadd_rn(c1, c2);
    const float dv = __fmul_rn(__fmul_rn(__fmul_rn(dp, pt), pv), __fsub_rn(1.f, pv));   // SigmoidGrad(pcvr, dp*pctr)
    const float ds = __fmul_rn(__fmul_rn(__fmul_rn(dp, pv), pt), __fsub_rn(1.f, pt));   // SigmoidGrad(pctr, dp*pcvr)
    const float dce = __fmul_rn(__fsub_rn(pt, t), g_ctr);
    if (d_ctr) d_ctr[i] = __fadd_rn(dce, ds);
    if (d_cvr) d_cvr[i] = dv;
  }
  if (train) {
    const float sc = esmm_block_sum(l_ctr, sh);
    const float sv = esmm_block_sum(l_cvr, sh);
    if (threadIdx.x == 0 && losses) {
      losses[0] = __fdiv_rn(sc, (float)n);
      losses[1] = __fdiv_rn(sv, (float)n);
    }
  }
}

}  // namespace ctr

using namespace ctr;

#define ESMM_K_SWITCH(K, CALL)                                                                     \
  switch (K) {                                                                                     \
    case 4: { CALL(1, 1) } break;   case 8: { CALL(2, 1) } break;   case 16: { CALL(4, 1) } break;  \
    case 32: { CALL(8, 1) } break;  case 64: { CALL(16, 1) } break; case 128: { CALL(32, 1) } break; \
    case 256: { CALL(32, 2) } break;                                                               \
    default:                                                                                       \
      set_error("%s: K=%d unsupported (must be one of 4,8,16,32,64,128,256)", fn, K);              \
      return CTR_ERR_UNSUPPORTED;                                                                  \
  }

static int esmm_lanes(int K) { return K >= 128 ? 32 : K / 4; }

extern "C" {

int ctr_esmm_embed_fwd(const int32_t* feat_ids, const int32_t* a_ids, const int32_t* bag_ids, const float* bag_wgt,
                       const int32_t* bag_off, const float* V, int64_t N, int B, int Fp, int K, float* x, int32_t* oob,
                       ctr_stream_t stream) {
  const char* fn = "ctr_esmm_embed_fwd";
  CTR_REQUIRE(B >= 0 && Fp >= 0 && K > 0 && N > 0, CTR_ERR_INVALID_ARG, "%s: bad args (B=%d F'=%d K=%d)", fn, B, Fp, K);
  if (B == 0) return CTR_OK;
  CTR_REQUIRE(a_ids && bag_off && V && x && (Fp == 0 || feat_ids), CTR_ERR_INVALID_ARG, "%s: null buffer", fn);
  cudaStream_t st = as_stream(stream);
  const int64_t threads = (int64_t)(ESMM_BAGS + 1) * B * esmm_lanes(K);
#define EF(LPR, VEC)                                                                                      \
  esmm_embed_fwd_kernel<LPR, VEC><<<(unsigned)ceil_div64(threads, 256), 256, 0, st>>>(                    \
      feat_ids, a_ids, bag_ids, bag_wgt, bag_off, V, N, B, Fp, x, oob);
  ESMM_K_SWITCH(K, EF)
#undef EF
  CTR_LAUNCHED(fn);
  return CTR_OK;
}

int ctr_esmm_embed_bwd(const float* dx, const float* bag_wgt, const int32_t* bag_off, int B, int Fp, int K,
                       int64_t n_rows, float* g_rows, ctr_stream_t stream) {
  const char* fn = "ctr_esmm_embed_bwd";
  CTR_REQUIRE(B >= 0 && Fp >= 0 && K > 0, CTR_ERR_INVALID_ARG, "%s: bad args (B=%d F'=%d K=%d)", fn, B, Fp, K);
  if (B == 0) return CTR_OK;
  CTR_REQUIRE(n_rows >= (int64_t)B * (Fp + 3), CTR_ERR_INVALID_ARG, "%s: n_rows %lld < B*(F'+3)", fn, (long long)n_rows);
  CTR_REQUIRE(dx && bag_off && g_rows, CTR_ERR_INVALID_ARG, "%s: null buffer", fn);
  cudaStream_t st = as_stream(stream);
  const int64_t threads = (int64_t)(ESMM_BAGS + 1) * B * esmm_lanes(K);
#define EB(LPR, VEC)                                                                                      \
  esmm_embed_bwd_kernel<LPR, VEC><<<(unsigned)ceil_div64(threads, 256), 256, 0, st>>>(dx, bag_wgt, bag_off, B, \
                                                                                       Fp, n_rows, g_rows);
  ESMM_K_SWITCH(K, EB)
#undef EB
  CTR_LAUNCHED(fn);
  return CTR_OK;
}

int ctr_esmm_head(const float* y_ctr, const float* y_cvr, const float* y, const float* z, int B, int n, float w_ctr,
                  float w_cvr, float* pctr, float* pcvr, float* pctcvr, float* losses, float* d_ctr, float* d_cvr,
                  ctr_stream_t stream) {
  CTR_REQUIRE(B >= 0, CTR_ERR_INVALID_ARG, "ctr_esmm_head: B < 0");
  if (B == 0) return CTR_OK;
  CTR_REQUIRE(y_ctr && y_cvr, CTR_ERR_INVALID_ARG, "ctr_esmm_head: null logits");
  CTR_REQUIRE(!y || (z && n >= 1 && n <= B), CTR_ERR_INVALID_ARG,
              "ctr_esmm_head: training needs both labels and 1 <= n <= B (n=%d B=%d)", n, B);
  esmm_head_kernel<<<1, ESMM_HEAD_THREADS, 0, as_stream(stream)>>>(y_ctr, y_cvr, y, z, B, y ? n : 1, w_ctr, w_cvr,
                                                                   pctr, pcvr, pctcvr, losses, d_ctr, d_cvr);
  CTR_LAUNCHED("ctr_esmm_head");
  return CTR_OK;
}

}  // extern "C"
