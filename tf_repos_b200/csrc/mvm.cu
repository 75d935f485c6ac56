// mvm.cu -- the DeepMVM multi-view product, forward and backward.
//
// Replaces DeepMVM.py:144-150:  all_order = tf.add(embeddings, MVM_B)              # [B,F,K] + [F,K]
//                               x_mvm = all_order[:,0,:]
//                               for i in range(1, field_size): x_mvm = tf.multiply(x_mvm, all_order[:,i,:])
// and its autodiff.  embeddings = x = reshape(mvm_w[ids]*vals, [B, F*K]) comes from K1 (CTR_FM_PLAIN).
//
// Numerics: every add and multiply is one IEEE-rounded fp32 op (__fadd_rn / __fmul_rn: nothing is contracted to an
// FMA), the product runs in field order, and denormals are kept (the library is built without -ftz).  At the
// reference's glorot initialisation most x_mvm elements are denormal (DESIGN.md 2.2), so flushing them would change
// the results.  With these three properties x_mvm and d_e are bit-identical to a sequential fp32 restatement.
//
// Mapping: a CTA of T = R*K threads (R = max(1, 128/K) sample rows); thread (r, k) owns column k of the samples
// r, r + R*gridDim, ... so that, for a fixed field, the K threads of a sample read K consecutive floats.  mvm_b [F,K]
// is staged in shared memory.  The backward recomputes the prefix products P_f = a_0*...*a_f (the forward's own
// roundings) into a per-thread shared-memory column, then walks the fields backwards:
//     da_i = g*P_{i-1};  g = g*a_i   (i = F-1 .. 1);   da_0 = g;   d_e = da + dX
// which is the autodiff of the left-to-right chain and needs no division (exact zeros in `a` are fine).
// d mvm_b = sum over samples of da: per-thread sums in shared memory, summed over the CTA's rows in a fixed order into
// a per-CTA slab of the workspace, then over the CTAs in a fixed order by mvm_merge_kernel (no float atomics, so the
// result is deterministic for a given B).
// HBM traffic per sample: fwd reads x and writes x_mvm (4(F+1)K B); bwd reads x, dX, d_xmvm and writes d_e
// (4(3F+1)K B).  The backward walk re-reads x, from L1.
#include "common.cuh"

namespace ctr {

constexpr int MVM_MAX_F = 64;
constexpr int MVM_MAX_K = 256;
constexpr int MVM_CTAS_PER_SM = 4;

static int mvm_rows(int K) { return K >= 128 ? 1 : 128 / K; }

static int mvm_grid(int B, int K) {
  const int R = mvm_rows(K);
  const int64_t need = ((int64_t)B + R - 1) / R;
  const int64_t cap = (int64_t)sm_count() * MVM_CTAS_PER_SM;
  return (int)(need < cap ? need : cap);
}

// shared memory of the backward: mvm_b [F*K] + prefix products [F-1][T] + d mvm_b sums [F][T]
static size_t mvm_bwd_smem(int F, int K) {
  const size_t T = (size_t)mvm_rows(K) * K;
  return ((size_t)F * K + (size_t)(F - 1) * T + (size_t)F * T) * sizeof(float);
}

__global__ void __launch_bounds__(256)
mvm_fwd_kernel(const float* __restrict__ x, const float* __restrict__ mb, int B, int F, int K, int R,
               float* __restrict__ xm) {
  extern __shared__ float sb[];
  for (int i = threadIdx.x; i < F * K; i += blockDim.x) sb[i] = mb[i];
  __syncthreads();
  const int r = threadIdx.x / K, k = threadIdx.x - r * K;
  const int64_t FK = (int64_t)F * K;
  for (int64_t b = (int64_t)blockIdx.x * R + r; b < B; b += (int64_t)gridDim.x * R) {
    const float* xr = x + b * FK + k;
    float p = __fadd_rn(xr[0], sb[k]);                                   // a_0 = e_0 + b_0
#pragma unroll 4
    for (int f = 1; f < F; ++f) p = __fmul_rn(p, __fadd_rn(xr[(int64_t)f * K], sb[f * K + k]));
    xm[b * K + k] = p;
  }
}

__global__ void __launch_bounds__(256)
mvm_bwd_kernel(const float* __restrict__ x, const float* __restrict__ mb, const float* __restrict__ gx,
               const float* __restrict__ dX, int B, int F, int K, int R, float* __restrict__ de,
               float* __restrict__ partial) {
  extern __shared__ float smem[];
  const int T = R * K, tid = threadIdx.x;
  float* sb = smem;                      // mvm_b [F][K]
  float* sp = sb + F * K;                // P_{f-1} at [f-1][tid], f = 1..F-1
  float* sa = sp + (F - 1) * T;          // this thread's sum of da_f at [f][tid]
  for (int i = tid; i < F * K; i += blockDim.x) sb[i] = mb[i];
  for (int i = tid; i < F * T; i += blockDim.x) sa[i] = 0.f;
  __syncthreads();
  const int r = tid / K, k = tid - r * K;
  const int64_t FK = (int64_t)F * K;
  for (int64_t b = (int64_t)blockIdx.x * R + r; b < B; b += (int64_t)gridDim.x * R) {
    const float* xr = x + b * FK + k;
    float p = __fadd_rn(xr[0], sb[k]);
#pragma unroll 4
    for (int f = 1; f < F; ++f) {
      sp[(f - 1) * T + tid] = p;
      p = __fmul_rn(p, __fadd_rn(xr[(int64_t)f * K], sb[f * K + k]));
    }
    float g = gx[b * K + k];
    float* dr = de + b * FK + k;
    const float* dxr = dX ? dX + b * FK + k : nullptr;
#pragma unroll 4
    for (int f = F - 1; f >= 1; --f) {
      const float da = __fmul_rn(g, sp[(f - 1) * T + tid]);                // d a_f = g * P_{f-1}
      sa[f * T + tid] = __fadd_rn(sa[f * T + tid], da);
      dr[(int64_t)f * K] = dxr ? __fadd_rn(da, dxr[(int64_t)f * K]) : da;
      g = __fmul_rn(g, __fadd_rn(xr[(int64_t)f * K], sb[f * K + k]));     // d P_{f-1} = g * a_f
    }
    sa[tid] = __fadd_rn(sa[tid], g);                                     // d a_0 = g
    dr[0] = dxr ? __fadd_rn(g, dxr[0]) : g;
  }
  __syncthreads();
  float* out = partial + (int64_t)blockIdx.x * FK;
  for (int i = tid; i < F * K; i += blockDim.x) {
    const int f = i / K, kk = i - f * K;
    float s = 0.f;
    for (int rr = 0; rr < R; ++rr) s += sa[f * T + rr * K + kk];
    out[i] = s;
  }
}

// out[i] = sum over c = 0..n-1 of partial[c][i]: 8 fixed strided slices per column, then the slices in order
__global__ void __launch_bounds__(256)
mvm_merge_kernel(const float* __restrict__ partial, int n, int FK, float* __restrict__ out) {
  __shared__ float red[8][33];
  const int i = blockIdx.x * 32 + threadIdx.x;
  float s = 0.f;
  if (i < FK)
    for (int c = threadIdx.y; c < n; c += 8) s += partial[(int64_t)c * FK + i];
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && i < FK) {
    float t = red[0][threadIdx.x];
    for (int y = 1; y < 8; ++y) t += red[y][threadIdx.x];
    out[i] = t;
  }
}

}  // namespace ctr

using namespace ctr;

extern "C" {

int ctr_mvm_fwd(const float* x, const float* mvm_b, int B, int F, int K, float* x_mvm, ctr_stream_t stream) {
  CTR_REQUIRE(B >= 0 && F > 0 && K > 0, CTR_ERR_INVALID_ARG, "ctr_mvm_fwd: bad shape (B=%d F=%d K=%d)", B, F, K);
  CTR_REQUIRE(F <= MVM_MAX_F && K <= MVM_MAX_K, CTR_ERR_UNSUPPORTED,
              "ctr_mvm_fwd: needs F <= %d and K <= %d (got F=%d K=%d)", MVM_MAX_F, MVM_MAX_K, F, K);
  if (B == 0) return CTR_OK;
  CTR_REQUIRE(x && mvm_b && x_mvm, CTR_ERR_INVALID_ARG, "ctr_mvm_fwd: null buffer");
  const int R = mvm_rows(K);
  const size_t smem = (size_t)F * K * sizeof(float);
  if (smem > 48 * 1024)
    cudaFuncSetAttribute(mvm_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  mvm_fwd_kernel<<<mvm_grid(B, K), R * K, smem, as_stream(stream)>>>(x, mvm_b, B, F, K, R, x_mvm);
  CTR_LAUNCHED("ctr_mvm_fwd");
  return CTR_OK;
}

size_t ctr_mvm_bwd_workspace_bytes(int B, int F, int K) {
  if (B <= 0 || F <= 0 || K <= 0 || F > MVM_MAX_F || K > MVM_MAX_K) return 16;
  return (size_t)mvm_grid(B, K) * F * K * sizeof(float);
}

int ctr_mvm_bwd(const float* x, const float* mvm_b, const float* d_xmvm, const float* dX, int B, int F, int K,
                float* d_e, float* d_mvm_b, void* ws, size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE(B >= 0 && F > 0 && K > 0, CTR_ERR_INVALID_ARG, "ctr_mvm_bwd: bad shape (B=%d F=%d K=%d)", B, F, K);
  CTR_REQUIRE(F <= MVM_MAX_F && K <= MVM_MAX_K, CTR_ERR_UNSUPPORTED,
              "ctr_mvm_bwd: needs F <= %d and K <= %d (got F=%d K=%d)", MVM_MAX_F, MVM_MAX_K, F, K);
  CTR_REQUIRE(d_mvm_b, CTR_ERR_INVALID_ARG, "ctr_mvm_bwd: null d_mvm_b");
  CTR_REQUIRE(B == 0 || (x && mvm_b && d_xmvm && d_e), CTR_ERR_INVALID_ARG, "ctr_mvm_bwd: null buffer");
  CTR_REQUIRE(B == 0 || (ws && ws_bytes >= ctr_mvm_bwd_workspace_bytes(B, F, K)), CTR_ERR_WORKSPACE,
              "ctr_mvm_bwd: workspace too small");
  cudaStream_t st = as_stream(stream);
  const int FK = F * K;
  const int grid = B > 0 ? mvm_grid(B, K) : 0;
  float* partial = reinterpret_cast<float*>(ws);
  if (B > 0) {
    const int R = mvm_rows(K);
    const size_t smem = mvm_bwd_smem(F, K);
    if (smem > 48 * 1024)
      cudaFuncSetAttribute(mvm_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    mvm_bwd_kernel<<<grid, R * K, smem, st>>>(x, mvm_b, d_xmvm, dX, B, F, K, R, d_e, partial);
    CTR_LAUNCHED("ctr_mvm_bwd");
  }
  mvm_merge_kernel<<<(FK + 31) / 32, dim3(32, 8), 0, st>>>(partial, grid, FK, d_mvm_b);   // B == 0: zeros
  CTR_LAUNCHED("mvm_merge");
  return CTR_OK;
}

}  // extern "C"
