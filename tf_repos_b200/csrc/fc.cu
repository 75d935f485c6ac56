// fc.cu -- the dense 'Deep-part': fully_connected layers (DeepFM.py:152-167), forward and backward,
// with fused epilogues (bias + relu + dropout; dZ + bias-gradient).  The products run on the tensor cores
// (tc_gemm.cu, 3xTF32); the fp32 SIMT tiles below are the CTR_GEMM=simt alternative.
//
// One templated tile kernel serves the three products of a layer:
//   forward   out[M,N]  = act(in[M,K] @ W[K,N] + b)          (A reduce-contiguous, B row-contiguous)
//   backward  dIn[M,K]  = dZ[M,N] @ W[K,N]^T                 (A reduce-contiguous, B reduce-contiguous)
//             dW[K,N]   = in[M,K]^T @ dZ[M,N]  (split over M, deterministic two-pass reduction)
// Accumulation order over the reduction dimension is fixed => bit-reproducible run to run.
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace ctr {

constexpr int GEMM_BK = 16;

// C[i][j] = sum_r A(i,r) * B(r,j),  i < M, j < N, r < R.
//   A_RC (reduce-contiguous): A(i,r) = A[i*lda + r]   else  A(i,r) = A[r*lda + i]
//   B_RC (reduce-contiguous): B(r,j) = B[j*ldb + r]   else  B(r,j) = B[r*ldb + j]
// blockIdx.z splits R into gridDim.z chunks; chunk z writes C + z*M*N (EPI 0) .
// EPI 1: C = act(acc + bias[j] + gbias[i / gP][j]) (/keep * mask[i][j])   (act: 0 identity, 1 relu)
//        gbias: optional per-row-group bias (DIN: one row per sample, shared by its P positions)
// EPI 2: C += acc
template <int BM, int BN, int TM, int TN, bool A_RC, bool B_RC, int EPI>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
gemm_tile_kernel(const float* __restrict__ A, int lda, const float* __restrict__ B, int ldb,
                 float* __restrict__ C, int ldc, int M, int N, int R, const float* __restrict__ bias,
                 int act, const float* __restrict__ mask, float keep, const float* __restrict__ gbias,
                 int gP) {
  constexpr int NT = (BM / TM) * (BN / TN);
  __shared__ __align__(16) float As[2][GEMM_BK][BM + 4];
  __shared__ __align__(16) float Bs[2][GEMM_BK][BN + 4];
  const int tid = threadIdx.x;
  const int tx = tid % (BN / TN), ty = tid / (BN / TN);
  const int i0 = blockIdx.y * BM, j0 = blockIdx.x * BN;
  const int r_chunk = (R + gridDim.z - 1) / gridDim.z;
  const int r_begin = blockIdx.z * r_chunk;
  const int r_end = min(R, r_begin + r_chunk);

  float acc[TM][TN];
#pragma unroll
  for (int a = 0; a < TM; ++a)
#pragma unroll
    for (int b = 0; b < TN; ++b) acc[a][b] = 0.f;

  // cooperative tile loads (scalar, bounds-checked; the tiles are small and L2-resident)
  auto load_tiles = [&](int buf, int r0) {
    for (int e = tid; e < BM * GEMM_BK; e += NT) {
      int i, r;
      if (A_RC) { r = e % GEMM_BK; i = e / GEMM_BK; } else { i = e % BM; r = e / BM; }
      const int gi = i0 + i, gr = r0 + r;
      float v = 0.f;
      if (gi < M && gr < r_end) v = A_RC ? A[(int64_t)gi * lda + gr] : A[(int64_t)gr * lda + gi];
      As[buf][r][i] = v;
    }
    for (int e = tid; e < BN * GEMM_BK; e += NT) {
      int j, r;
      if (B_RC) { r = e % GEMM_BK; j = e / GEMM_BK; } else { j = e % BN; r = e / BN; }
      const int gj = j0 + j, gr = r0 + r;
      float v = 0.f;
      if (gj < N && gr < r_end) v = B_RC ? B[(int64_t)gj * ldb + gr] : B[(int64_t)gr * ldb + gj];
      Bs[buf][r][j] = v;
    }
  };

  int buf = 0;
  if (r_begin < r_end) load_tiles(0, r_begin);
  __syncthreads();
  for (int r0 = r_begin; r0 < r_end; r0 += GEMM_BK) {
    if (r0 + GEMM_BK < r_end) load_tiles(buf ^ 1, r0 + GEMM_BK);
#pragma unroll
    for (int r = 0; r < GEMM_BK; ++r) {
      float a[TM], b[TN];
#pragma unroll
      for (int u = 0; u < TM; u += 4) {
        const float4 t = *reinterpret_cast<const float4*>(&As[buf][r][ty * TM + u]);
        a[u] = t.x; a[u + 1] = t.y; a[u + 2] = t.z; a[u + 3] = t.w;
      }
#pragma unroll
      for (int u = 0; u < TN; u += 4) {
        const float4 t = *reinterpret_cast<const float4*>(&Bs[buf][r][tx * TN + u]);
        b[u] = t.x; b[u + 1] = t.y; b[u + 2] = t.z; b[u + 3] = t.w;
      }
#pragma unroll
      for (int u = 0; u < TM; ++u)
#pragma unroll
        for (int w = 0; w < TN; ++w) acc[u][w] = fmaf(a[u], b[w], acc[u][w]);
    }
    __syncthreads();
    buf ^= 1;
  }

  float* Cz = C + (EPI == 0 ? (int64_t)blockIdx.z * M * ldc : 0);
#pragma unroll
  for (int u = 0; u < TM; ++u) {
    const int gi = i0 + ty * TM + u;
    if (gi >= M) continue;
#pragma unroll
    for (int w = 0; w < TN; ++w) {
      const int gj = j0 + tx * TN + w;
      if (gj >= N) continue;
      float v = acc[u][w];
      if (EPI == 2) v += Cz[(int64_t)gi * ldc + gj];
      if (EPI == 1) {
        if (bias) v += bias[gj];
        if (gbias) v += gbias[(int64_t)(gi / gP) * N + gj];
        if (act == 1) v = fmaxf(v, 0.f);
        if (mask) v = __fdiv_rn(v, keep) * mask[(int64_t)gi * ldc + gj];  // tf.nn.dropout: x/keep*binary
      }
      Cz[(int64_t)gi * ldc + gj] = v;
    }
  }
}

// out[k][n] = sum_z partial[z][k][n]  (fixed order)
__global__ void splitk_reduce_kernel(const float* __restrict__ partial, int S, int64_t n, float* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    float s = 0.f;
    for (int z = 0; z < S; ++z) s += partial[(int64_t)z * n + i];
    out[i] = s;
  }
}

// out[k][n] = sum_z partial[z][n][k]: reduce split-R partials of the TRANSPOSED product (dW^T = dZ^T @ in)
__global__ void splitk_reduce_t_kernel(const float* __restrict__ partial, int S, int Kd, int Nd, float* __restrict__ out) {
  const int64_t n = (int64_t)Kd * Nd;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int k = (int)(i / Nd), c = (int)(i % Nd);
    float s = 0.f;
    for (int z = 0; z < S; ++z) s += partial[(int64_t)z * n + (int64_t)c * Kd + k];
    out[i] = s;
  }
}

// dZ = (dOut * mask / keep) * (out > 0) in place, plus partial column sums (bias gradient)
constexpr int DZ_ROWS = 128;
__global__ void __launch_bounds__(256)
fc_dz_kernel(float* __restrict__ dOut, const float* __restrict__ out, const float* __restrict__ mask, float keep,
             int M, int N, int act, float* __restrict__ colsum_partial /*[chunks][N]*/) {
  const int col = blockIdx.x * 32 + (threadIdx.x & 31);
  const int rl = threadIdx.x >> 5;  // 8 row lanes
  const int r0 = blockIdx.y * DZ_ROWS;
  __shared__ float red[8][33];
  float s = 0.f;
  if (col < N) {
    for (int r = r0 + rl; r < min(M, r0 + DZ_ROWS); r += 8) {
      const int64_t i = (int64_t)r * N + col;
      float d = dOut[i];
      if (mask) d = __fdiv_rn(d * mask[i], keep);
      if (act == 1 && !(out[i] > 0.f)) d = 0.f;
      dOut[i] = d;
      s += d;
    }
  }
  red[rl][threadIdx.x & 31] = s;
  __syncthreads();
  if (rl == 0 && col < N) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += red[k][threadIdx.x & 31];
    colsum_partial[(int64_t)blockIdx.y * N + col] = t;
  }
}

// ---- N = 1 output layer: y = [in_a | in_b] @ w + b   (DeepFM.py:165 deep_out; DCN.py:180 out_layer) ----
__global__ void __launch_bounds__(256)
fc1_fwd_kernel(const float* __restrict__ in_a, int Ka, const float* __restrict__ in_b, int Kb,
               const float* __restrict__ w, const float* __restrict__ b, int M, float* __restrict__ y) {
  const int lane = threadIdx.x & 31;
  const int m = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (m >= M) return;
  float s = 0.f;
  for (int k = lane; k < Ka; k += 32) s = fmaf(in_a[(int64_t)m * Ka + k], w[k], s);
  for (int k = lane; k < Kb; k += 32) s = fmaf(in_b[(int64_t)m * Kb + k], w[Ka + k], s);
  s = warp_sum(s);
  if (lane == 0) y[m] = s + (b ? b[0] : 0.f);
}

// d_in[m][k] = dy[m]*w[k]; dw partials over row chunks; db = sum dy (chunk partial)
constexpr int FC1_ROWS = 64;
__global__ void __launch_bounds__(256)
fc1_bwd_kernel(const float* __restrict__ in_a, int Ka, const float* __restrict__ in_b, int Kb,
               const float* __restrict__ w, const float* __restrict__ dy, int M, float* __restrict__ d_a,
               float* __restrict__ d_b, float* __restrict__ dw_partial /*[chunks][Ka+Kb+1]*/) {
  const int Kt = Ka + Kb;
  const int r0 = blockIdx.x * FC1_ROWS, r1 = min(M, r0 + FC1_ROWS);
  for (int k = threadIdx.x; k < Kt + 1; k += blockDim.x) {
    float s = 0.f;
    if (k < Kt) {
      const float wk = w[k];
      for (int r = r0; r < r1; ++r) {
        const float d = dy[r];
        if (k < Ka) {
          s = fmaf(in_a[(int64_t)r * Ka + k], d, s);
          if (d_a) d_a[(int64_t)r * Ka + k] = d * wk;
        } else {
          s = fmaf(in_b[(int64_t)r * Kb + (k - Ka)], d, s);
          if (d_b) d_b[(int64_t)r * Kb + (k - Ka)] = d * wk;
        }
      }
    } else {
      for (int r = r0; r < r1; ++r) s += dy[r];
    }
    dw_partial[(int64_t)blockIdx.x * (Kt + 1) + k] = s;
  }
}

// out[k] = sum_c part[c*ld + k] for many partial rows (thousands when M = B*P): 32 columns x 8 row groups per CTA,
// each group adds rows g, g+8, ... in order, then a fixed 8-way tree.  Columns [0, na) go to out_a, the rest to out_b.
__global__ void __launch_bounds__(256)
colsum_rows_kernel(const float* __restrict__ part, int chunks, int ld, int ncols, int na, float* __restrict__ out_a,
                   float* __restrict__ out_b) {
  __shared__ float red[8][33];
  const int k = blockIdx.x * 32 + (threadIdx.x & 31), g = threadIdx.x >> 5;
  float s = 0.f;
  if (k < ncols) for (int c = g; c < chunks; c += 8) s += part[(int64_t)c * ld + k];
  red[g][threadIdx.x & 31] = s;
  __syncthreads();
  if (g == 0 && k < ncols) {
    float t = 0.f;
#pragma unroll
    for (int q = 0; q < 8; ++q) t += red[q][threadIdx.x];
    if (k < na) out_a[k] = t; else out_b[k - na] = t;
  }
}

// binary keep mask (1.0 / 0.0) from a counter-based hash: tf.nn.dropout's floor(keep + U[0,1))
__device__ __forceinline__ uint64_t mix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
__global__ void dropout_mask_kernel(float* __restrict__ mask, int64_t n, float keep, uint64_t seed,
                                    const float* __restrict__ step_dev) {
  const uint64_t step = step_dev ? (uint64_t)step_dev[0] : 0ull;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint64_t r = mix64(seed ^ mix64(step * 0x100000001B3ull + (uint64_t)i));
    const float u = (float)(r >> 40) * (1.0f / 16777216.0f);
    mask[i] = (u < keep) ? 1.f : 0.f;
  }
}

// tc_gemm.cu: the same products on wgmma tensor cores (3xTF32).  CTR_GEMM=simt selects the SIMT tiles.
int tc_gemm_dispatch(int kind, int epi, const float* A, int lda, const float* B, int ldb, float* C, int ldc, int M, int N,
                     int R, int S, const float* bias, int act, const float* mask, float keep, const float* gbias, int gP,
                     cudaStream_t st);

static bool use_tc() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("CTR_GEMM");
    v = (e && strcmp(e, "simt") == 0) ? 0 : 1;
  }
  return v == 1;
}

static int pick_split(int M, int N, int R) {
  // dW-style product: few output tiles, long reduction => split R so that >= ~2 waves of CTAs exist
  const int t = use_tc() ? 128 : 64;
  const int tiles = ((M + t - 1) / t) * ((N + t - 1) / t);
  int s = (2 * sm_count() + tiles - 1) / tiles;
  if (s < 1) s = 1;
  const int max_s = (R + 255) / 256;
  if (s > max_s) s = max_s;
  if (s > 64) s = 64;
  return s < 1 ? 1 : s;
}

}  // namespace ctr

using namespace ctr;

extern "C" {

int ctr_fc_fwd_grouped(const float* in, const float* Wt, const float* b, const float* group_bias, int group_P,
                       const float* drop_mask, float keep_prob, int M, int Kd, int Nd, int act, float* out,
                       ctr_stream_t stream);

int ctr_fc_fwd(const float* in, const float* Wt, const float* b, const float* drop_mask, float keep_prob,
               int M, int Kd, int Nd, int act, float* out, ctr_stream_t stream) {
  return ctr_fc_fwd_grouped(in, Wt, b, nullptr, 1, drop_mask, keep_prob, M, Kd, Nd, act, out, stream);
}

int ctr_fc_fwd_grouped(const float* in, const float* Wt, const float* b, const float* group_bias, int group_P,
                       const float* drop_mask, float keep_prob, int M, int Kd, int Nd, int act, float* out,
                       ctr_stream_t stream) {
  CTR_REQUIRE(M >= 0 && Kd > 0 && Nd > 0 && (act == 0 || act == 1) && group_P >= 1, CTR_ERR_INVALID_ARG,
              "ctr_fc_fwd: bad shape/act");
  if (M == 0) return CTR_OK;
  CTR_REQUIRE(in && Wt && out, CTR_ERR_INVALID_ARG, "ctr_fc_fwd: null buffer");
  CTR_REQUIRE(!drop_mask || keep_prob > 0.f, CTR_ERR_INVALID_ARG, "ctr_fc_fwd: keep_prob must be > 0");
  cudaStream_t st = as_stream(stream);
  if (use_tc()) {
    tc_gemm_dispatch(0, 1, in, Kd, Wt, Nd, out, Nd, M, Nd, Kd, 1, b, act, drop_mask, keep_prob, group_bias, group_P, st);
  } else if (Nd >= 128) {
    dim3 grid((Nd + 127) / 128, (M + 63) / 64, 1);
    gemm_tile_kernel<64, 128, 4, 8, true, false, 1><<<grid, 256, 0, st>>>(in, Kd, Wt, Nd, out, Nd, M, Nd, Kd, b, act,
                                                                          drop_mask, keep_prob, group_bias, group_P);
  } else {
    dim3 grid((Nd + 63) / 64, (M + 63) / 64, 1);
    gemm_tile_kernel<64, 64, 4, 4, true, false, 1><<<grid, 256, 0, st>>>(in, Kd, Wt, Nd, out, Nd, M, Nd, Kd, b, act,
                                                                         drop_mask, keep_prob, group_bias, group_P);
  }
  CTR_LAUNCHED("ctr_fc_fwd");
  return CTR_OK;
}

size_t ctr_fc_bwd_workspace_bytes(int M, int Kd, int Nd) {
  if (M <= 0 || Kd <= 0 || Nd <= 0) return 0;
  const size_t chunks = (size_t)(M + DZ_ROWS - 1) / DZ_ROWS;
  const size_t split = 64;
  return (chunks * (size_t)Nd + split * (size_t)Kd * (size_t)Nd) * sizeof(float);
}

int ctr_fc_bwd(const float* in, const float* Wt, const float* out, const float* drop_mask, float keep_prob,
               float* dOut, int M, int Kd, int Nd, int act, float* dIn, int accumulate_din, float* dW, float* db,
               void* ws, size_t ws_bytes, ctr_stream_t stream) {
  // act == 2: dOut already holds dZ and the caller has the bias gradient (ctr_din_att_dz): skip the dZ pass
  CTR_REQUIRE(M >= 0 && Kd > 0 && Nd > 0 && (act == 0 || act == 1 || act == 2), CTR_ERR_INVALID_ARG, "ctr_fc_bwd: bad shape/act");
  if (M == 0) return CTR_OK;
  CTR_REQUIRE(in && Wt && dOut && dW && (act == 2 || (out && db)), CTR_ERR_INVALID_ARG, "ctr_fc_bwd: null buffer");
  CTR_REQUIRE(ws && ws_bytes >= ctr_fc_bwd_workspace_bytes(M, Kd, Nd), CTR_ERR_WORKSPACE,
              "ctr_fc_bwd: workspace too small");
  cudaStream_t st = as_stream(stream);
  float* colsum = reinterpret_cast<float*>(ws);
  const int chunks = (M + DZ_ROWS - 1) / DZ_ROWS;
  float* dw_part = colsum + (size_t)chunks * Nd;
  // 1. dZ in place + bias gradient
  if (act != 2) {
    fc_dz_kernel<<<dim3((Nd + 31) / 32, chunks), 256, 0, st>>>(dOut, out, drop_mask, keep_prob, M, Nd, act, colsum);
    CTR_LAUNCHED("fc_dz");
    colsum_rows_kernel<<<(Nd + 31) / 32, 256, 0, st>>>(colsum, chunks, Nd, Nd, Nd, db, nullptr);
    CTR_LAUNCHED("fc_db_reduce");
  }
  // 2. dW[Kd,Nd] = in^T @ dZ, split over M
  // narrow layer input (DIN attention: Kd = 32, Nd = 256, M = B*P = 409600): as in^T @ dZ the 128-row MMA tile
  // would be 3/4 padding; the transposed product dW^T[Nd,Kd] = dZ^T @ in fills it (and its N = Kd MMAs are 4x smaller)
  const bool dw_transposed = use_tc() && Kd <= 64 && Nd >= 128;
  const int S = dw_transposed ? pick_split(Nd, Kd, M) : pick_split(Kd, Nd, M);
  if (dw_transposed) {
    tc_gemm_dispatch(2, 0, dOut, Nd, in, Kd, dw_part, Kd, Nd, Kd, M, S, nullptr, 0, nullptr, 1.f, nullptr, 1, st);
    CTR_LAUNCHED("fc_dw(t)");
    const int64_t n = (int64_t)Kd * Nd;
    splitk_reduce_t_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(dw_part, S, Kd, Nd, dW);
    CTR_LAUNCHED("fc_dw_reduce(t)");
  } else {
    if (use_tc()) {
      tc_gemm_dispatch(2, 0, in, Kd, dOut, Nd, S == 1 ? dW : dw_part, Nd, Kd, Nd, M, S, nullptr, 0, nullptr, 1.f, nullptr, 1, st);
    } else {
      dim3 grid((Nd + 63) / 64, (Kd + 63) / 64, S);
      gemm_tile_kernel<64, 64, 4, 4, false, false, 0><<<grid, 256, 0, st>>>(in, Kd, dOut, Nd, S == 1 ? dW : dw_part, Nd,
                                                                            Kd, Nd, M, nullptr, 0, nullptr, 1.f, nullptr, 1);
    }
    CTR_LAUNCHED("fc_dw");
    if (S > 1) {
      const int64_t n = (int64_t)Kd * Nd;
      splitk_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(dw_part, S, n, dW);
      CTR_LAUNCHED("fc_dw_reduce");
    }
  }
  // 3. dIn[M,Kd] = dZ @ W^T
  if (dIn && use_tc()) {
    tc_gemm_dispatch(1, accumulate_din ? 2 : 0, dOut, Nd, Wt, Nd, dIn, Kd, M, Kd, Nd, 1, nullptr, 0, nullptr, 1.f, nullptr, 1, st);
    CTR_LAUNCHED("fc_din");
  } else if (dIn) {
    dim3 grid((Kd + 127) / 128, (M + 63) / 64, 1);
    if (accumulate_din)
      gemm_tile_kernel<64, 128, 4, 8, true, true, 2><<<grid, 256, 0, st>>>(dOut, Nd, Wt, Nd, dIn, Kd, M, Kd, Nd, nullptr,
                                                                           0, nullptr, 1.f, nullptr, 1);
    else
      gemm_tile_kernel<64, 128, 4, 8, true, true, 0><<<grid, 256, 0, st>>>(dOut, Nd, Wt, Nd, dIn, Kd, M, Kd, Nd, nullptr,
                                                                           0, nullptr, 1.f, nullptr, 1);
    CTR_LAUNCHED("fc_din");
  }
  return CTR_OK;
}

int ctr_colsum_rows(const float* part, int rows, int ld, int ncols, float* out, ctr_stream_t stream) {
  CTR_REQUIRE(rows >= 0 && ncols > 0 && ld >= ncols, CTR_ERR_INVALID_ARG, "ctr_colsum_rows: bad shape");
  CTR_REQUIRE(part && out, CTR_ERR_INVALID_ARG, "ctr_colsum_rows: null buffer");
  colsum_rows_kernel<<<(ncols + 31) / 32, 256, 0, as_stream(stream)>>>(part, rows, ld, ncols, ncols, out, nullptr);
  CTR_LAUNCHED("ctr_colsum_rows");
  return CTR_OK;
}

int ctr_fc1_fwd(const float* in_a, int Ka, const float* in_b, int Kb, const float* w, const float* b, int M,
                float* y, ctr_stream_t stream) {
  CTR_REQUIRE(M >= 0 && Ka > 0 && Kb >= 0, CTR_ERR_INVALID_ARG, "ctr_fc1_fwd: bad shape");
  if (M == 0) return CTR_OK;
  CTR_REQUIRE(in_a && w && y && (Kb == 0 || in_b), CTR_ERR_INVALID_ARG, "ctr_fc1_fwd: null buffer");
  fc1_fwd_kernel<<<(M + 7) / 8, 256, 0, as_stream(stream)>>>(in_a, Ka, in_b, Kb, w, b, M, y);
  CTR_LAUNCHED("ctr_fc1_fwd");
  return CTR_OK;
}

size_t ctr_fc1_bwd_workspace_bytes(int M, int Ka, int Kb) {
  if (M <= 0) return 0;
  return (size_t)((M + FC1_ROWS - 1) / FC1_ROWS) * (size_t)(Ka + Kb + 1) * sizeof(float);
}

int ctr_fc1_bwd(const float* in_a, int Ka, const float* in_b, int Kb, const float* w, const float* dy, int M,
                float* d_a, float* d_b, float* dw, float* db, void* ws, size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE(M >= 0 && Ka > 0 && Kb >= 0, CTR_ERR_INVALID_ARG, "ctr_fc1_bwd: bad shape");
  if (M == 0) return CTR_OK;
  CTR_REQUIRE(in_a && w && dy && dw && db && (Kb == 0 || in_b), CTR_ERR_INVALID_ARG, "ctr_fc1_bwd: null buffer");
  CTR_REQUIRE(ws && ws_bytes >= ctr_fc1_bwd_workspace_bytes(M, Ka, Kb), CTR_ERR_WORKSPACE,
              "ctr_fc1_bwd: workspace too small");
  cudaStream_t st = as_stream(stream);
  const int chunks = (M + FC1_ROWS - 1) / FC1_ROWS;
  float* part = reinterpret_cast<float*>(ws);
  fc1_bwd_kernel<<<chunks, 256, 0, st>>>(in_a, Ka, in_b, Kb, w, dy, M, d_a, d_b, part);
  CTR_LAUNCHED("fc1_bwd");
  const int Kt = Ka + Kb;
  colsum_rows_kernel<<<(Kt + 1 + 31) / 32, 256, 0, st>>>(part, chunks, Kt + 1, Kt + 1, Kt, dw, db);   // rows are [dw(Kt) | db(1)]
  CTR_LAUNCHED("fc1_reduce");
  return CTR_OK;
}

int ctr_dropout_mask(float* mask, int64_t n, float keep_prob, uint64_t seed, const float* step_dev,
                     ctr_stream_t stream) {
  CTR_REQUIRE(n >= 0 && keep_prob > 0.f && keep_prob <= 1.f, CTR_ERR_INVALID_ARG, "ctr_dropout_mask: bad args");
  if (n == 0) return CTR_OK;
  CTR_REQUIRE(mask, CTR_ERR_INVALID_ARG, "ctr_dropout_mask: null mask");
  int64_t blocks = ceil_div64(n, 256 * 4);
  const int grid = (int)(blocks < (int64_t)sm_count() * 8 ? blocks : (int64_t)sm_count() * 8);
  dropout_mask_kernel<<<grid, 256, 0, as_stream(stream)>>>(mask, n, keep_prob, seed, step_dev);
  CTR_LAUNCHED("ctr_dropout_mask");
  return CTR_OK;
}

}  // extern "C"
