// cross.cu -- K5: the DCN cross network, forward and backward.
//
// Replaces DCN.py:140-145:   for l in range(cross_layers):
//                                xlw = tf.matmul(xl, wl)            # [B,1]   (wl = cross_w[l], [D,1])
//                                xl  = x0 * xlw + xl + cross_b[l]   # [B,D]
// and its autodiff.  x0 = reshape(emb[ids]*vals, [B, D]) with D = field_size*embedding_size.
//
// Mapping: one warp per sample, x0 and x_l live in registers (NV float4 per lane, D <= 128*NV), the
// L dot products are warp-shuffle reductions, w/b rows come from L1/L2 (L*D*8 B = 30 KB at config 3).
// HBM traffic: forward reads x0 and writes x_L (2 x 4D B/sample); only the L scalars s_l = x_l.w_l
// are saved.  The backward recomputes x_l from x0 and the saved scalars (O(L^2) FMAs, free next to
// the 3 x 4D B/sample of traffic) and accumulates dw/db in per-warp shared-memory slabs that a
// second kernel reduces in a fixed order (no float atomics => deterministic).
#include "common.cuh"

namespace ctr {

template <int NV>
__global__ void __launch_bounds__(128)
cross_fwd_kernel(const float* __restrict__ x0g, const float* __restrict__ w, const float* __restrict__ b,
                 int B, int D, int L, float* __restrict__ xL, float* __restrict__ s_out) {
  const int lane = threadIdx.x & 31;
  const int smp = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (smp >= B) return;
  const int D4 = D >> 2;
  const float4* x0p = reinterpret_cast<const float4*>(x0g + (int64_t)smp * D);
  float4 x0[NV], x[NV];
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    const int i = lane + 32 * v;
    x0[v] = (i < D4) ? ld_stream4(x0p + i) : f4_zero();
    x[v] = x0[v];
  }
  for (int l = 0; l < L; ++l) {
    const float4* wl = reinterpret_cast<const float4*>(w + (int64_t)l * D);
    const float4* bl = reinterpret_cast<const float4*>(b + (int64_t)l * D);
    float dot = 0.f;
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      const int i = lane + 32 * v;
      if (i < D4) {
        const float4 ww = __ldg(wl + i);
        dot = fmaf(x[v].x, ww.x, dot); dot = fmaf(x[v].y, ww.y, dot);
        dot = fmaf(x[v].z, ww.z, dot); dot = fmaf(x[v].w, ww.w, dot);
      }
    }
    dot = warp_sum(dot);
    if (lane == 0 && s_out) s_out[(int64_t)smp * L + l] = dot;
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      const int i = lane + 32 * v;
      if (i < D4) {
        const float4 bb = __ldg(bl + i);
        // (x0*xlw + xl) + b, each op rounded like the reference's separate TF ops
        x[v].x = __fadd_rn(__fadd_rn(__fmul_rn(x0[v].x, dot), x[v].x), bb.x);
        x[v].y = __fadd_rn(__fadd_rn(__fmul_rn(x0[v].y, dot), x[v].y), bb.y);
        x[v].z = __fadd_rn(__fadd_rn(__fmul_rn(x0[v].z, dot), x[v].z), bb.z);
        x[v].w = __fadd_rn(__fadd_rn(__fmul_rn(x0[v].w, dot), x[v].w), bb.w);
      }
    }
  }
  float4* op = reinterpret_cast<float4*>(xL + (int64_t)smp * D);
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    const int i = lane + 32 * v;
    if (i < D4) op[i] = x[v];
  }
}

// backward.  slab layout per warp: [2][L][D]  (0: dw, 1: db)
template <int NV>
__global__ void __launch_bounds__(128)
cross_bwd_kernel(const float* __restrict__ x0g, const float* __restrict__ w, const float* __restrict__ b,
                 const float* __restrict__ s_in, const float* __restrict__ dxL, const float* __restrict__ dx_in,
                 int B, int D, int L, float* __restrict__ dx0, float* __restrict__ partial, int warps_per_cta) {
  extern __shared__ __align__(16) float slab_all[];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int D4 = D >> 2;
  float4* slab = reinterpret_cast<float4*>(slab_all + (int64_t)wid * 2 * L * D);
  for (int i = lane; i < 2 * L * D4; i += 32) slab[i] = f4_zero();
  __syncwarp();
  const int n_warps = gridDim.x * warps_per_cta;
  const int gw = blockIdx.x * warps_per_cta + wid;
  for (int smp = gw; smp < B; smp += n_warps) {
    const float4* x0p = reinterpret_cast<const float4*>(x0g + (int64_t)smp * D);
    const float4* gp = reinterpret_cast<const float4*>(dxL + (int64_t)smp * D);
    float4 x0[NV], g[NV], acc[NV];
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      const int i = lane + 32 * v;
      x0[v] = (i < D4) ? ld_stream4(x0p + i) : f4_zero();
      g[v] = (i < D4) ? ld_stream4(gp + i) : f4_zero();
      acc[v] = f4_zero();
    }
    const float s_mine = (lane < L) ? s_in[(int64_t)smp * L + lane] : 0.f;  // L <= 32
    for (int l = L - 1; l >= 0; --l) {
      // recompute x_l = forward recursion from x0 with the saved scalars
      float4 x[NV];
#pragma unroll
      for (int v = 0; v < NV; ++v) x[v] = x0[v];
      for (int t = 0; t < l; ++t) {
        const float st = __shfl_sync(FULL_MASK, s_mine, t);
        const float4* bt = reinterpret_cast<const float4*>(b + (int64_t)t * D);
#pragma unroll
        for (int v = 0; v < NV; ++v) {
          const int i = lane + 32 * v;
          if (i < D4) {
            const float4 bb = __ldg(bt + i);
            x[v].x = __fadd_rn(__fadd_rn(__fmul_rn(x0[v].x, st), x[v].x), bb.x);
            x[v].y = __fadd_rn(__fadd_rn(__fmul_rn(x0[v].y, st), x[v].y), bb.y);
            x[v].z = __fadd_rn(__fadd_rn(__fmul_rn(x0[v].z, st), x[v].z), bb.z);
            x[v].w = __fadd_rn(__fadd_rn(__fmul_rn(x0[v].w, st), x[v].w), bb.w);
          }
        }
      }
      const float sl = __shfl_sync(FULL_MASK, s_mine, l);
      float ds = 0.f;  // d s_l = g . x0
#pragma unroll
      for (int v = 0; v < NV; ++v) {
        ds = fmaf(g[v].x, x0[v].x, ds); ds = fmaf(g[v].y, x0[v].y, ds);
        ds = fmaf(g[v].z, x0[v].z, ds); ds = fmaf(g[v].w, x0[v].w, ds);
      }
      ds = warp_sum(ds);
      const float4* wl = reinterpret_cast<const float4*>(w + (int64_t)l * D);
      float4* dwl = slab + (int64_t)l * D4;
      float4* dbl = slab + (int64_t)(L + l) * D4;
#pragma unroll
      for (int v = 0; v < NV; ++v) {
        const int i = lane + 32 * v;
        if (i < D4) {
          dbl[i] = f4_add(dbl[i], g[v]);                                   // d b_l += g
          dwl[i] = f4_fma(make_float4(ds, ds, ds, ds), x[v], dwl[i]);      // d w_l += ds * x_l
          acc[v] = f4_fma(g[v], make_float4(sl, sl, sl, sl), acc[v]);      // d x0  += g * s_l
          const float4 ww = __ldg(wl + i);
          g[v] = f4_fma(make_float4(ds, ds, ds, ds), ww, g[v]);            // d x_l  = g + ds * w_l
        }
      }
    }
    float4* op = reinterpret_cast<float4*>(dx0 + (int64_t)smp * D);
    const float4* ip = dx_in ? reinterpret_cast<const float4*>(dx_in + (int64_t)smp * D) : nullptr;
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      const int i = lane + 32 * v;
      if (i < D4) {
        float4 o = f4_add(acc[v], g[v]);                                   // x_0 = x0 : + d x_0
        if (ip) o = f4_add(o, ip[i]);
        op[i] = o;
      }
    }
  }
  __syncwarp();
  float4* outp = reinterpret_cast<float4*>(partial) + (int64_t)gw * 2 * L * D4;
  for (int i = lane; i < 2 * L * D4; i += 32) outp[i] = slab[i];
}

// dw[l][d] = sum over warps (fixed order); out = [dw | db] each [L*D]
__global__ void cross_reduce_kernel(const float* __restrict__ partial, int n_warps, int64_t LD, float* __restrict__ dw,
                                    float* __restrict__ db) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 2 * LD) return;
  float s = 0.f;
  for (int wv = 0; wv < n_warps; ++wv) s += partial[(int64_t)wv * 2 * LD + i];
  if (i < LD) dw[i] = s; else db[i - LD] = s;
}

static int bwd_warps_per_cta(int D, int L) {
  const size_t per_warp = (size_t)2 * L * D * sizeof(float);
  int wpc = (int)((200u * 1024u) / per_warp);
  if (wpc > 4) wpc = 4;
  return wpc;
}

}  // namespace ctr

using namespace ctr;

#define CROSS_NV_SWITCH(NVV, CALL)                                                     \
  switch (NVV) {                                                                       \
    case 1: { CALL(1) } break;  case 2: { CALL(2) } break;  case 3: { CALL(3) } break;  \
    case 4: { CALL(4) } break;  case 5: { CALL(5) } break;  case 6: { CALL(6) } break;  \
    case 7: case 8: { CALL(8) } break;                                                 \
    case 9: case 10: { CALL(10) } break;                                               \
    case 11: case 12: { CALL(12) } break;                                              \
    default: { CALL(16) } break;                                                       \
  }

extern "C" {

int ctr_cross_fwd(const float* x0, const float* w, const float* b, int B, int D, int L, float* xL, float* s,
                  ctr_stream_t stream) {
  CTR_REQUIRE(B >= 0 && D > 0 && L >= 0, CTR_ERR_INVALID_ARG, "ctr_cross_fwd: bad shape");
  CTR_REQUIRE(D % 4 == 0 && D <= 2048 && L <= 32, CTR_ERR_UNSUPPORTED,
              "ctr_cross_fwd: needs D %% 4 == 0, D <= 2048, L <= 32 (got D=%d L=%d)", D, L);
  if (B == 0) return CTR_OK;
  CTR_REQUIRE(x0 && xL && (L == 0 || (w && b)), CTR_ERR_INVALID_ARG, "ctr_cross_fwd: null buffer");
  const int nv = (D / 4 + 31) / 32;
  dim3 grid((B + 3) / 4), block(128);
#define FWD(NV) cross_fwd_kernel<NV><<<grid, block, 0, as_stream(stream)>>>(x0, w, b, B, D, L, xL, s);
  CROSS_NV_SWITCH(nv, FWD)
#undef FWD
  CTR_LAUNCHED("ctr_cross_fwd");
  return CTR_OK;
}

size_t ctr_cross_bwd_workspace_bytes(int B, int D, int L) {
  if (D <= 0 || L <= 0) return 16;
  const int wpc = bwd_warps_per_cta(D, L);
  if (wpc < 1) return 0;
  return (size_t)sm_count() * wpc * 2 * L * D * sizeof(float);
}

int ctr_cross_bwd(const float* x0, const float* w, const float* b, const float* s, const float* dxL,
                  const float* dx_in, int B, int D, int L, float* dx0, float* dw, float* db, void* ws,
                  size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE(B >= 0 && D > 0 && L > 0, CTR_ERR_INVALID_ARG, "ctr_cross_bwd: bad shape");
  CTR_REQUIRE(D % 4 == 0 && D <= 2048 && L <= 32, CTR_ERR_UNSUPPORTED,
              "ctr_cross_bwd: needs D %% 4 == 0, D <= 2048, L <= 32 (got D=%d L=%d)", D, L);
  const int wpc = bwd_warps_per_cta(D, L);
  CTR_REQUIRE(wpc >= 1, CTR_ERR_UNSUPPORTED,
              "ctr_cross_bwd: L*D too large for the shared-memory slabs (got D=%d L=%d)", D, L);
  if (B == 0) return CTR_OK;
  CTR_REQUIRE(x0 && w && b && s && dxL && dx0 && dw && db, CTR_ERR_INVALID_ARG, "ctr_cross_bwd: null buffer");
  CTR_REQUIRE(ws && ws_bytes >= ctr_cross_bwd_workspace_bytes(B, D, L), CTR_ERR_WORKSPACE,
              "ctr_cross_bwd: workspace too small");
  cudaStream_t st = as_stream(stream);
  const int grid = sm_count();
  const size_t smem = (size_t)wpc * 2 * L * D * sizeof(float);
  const int nv = (D / 4 + 31) / 32;
  float* partial = reinterpret_cast<float*>(ws);
#define BWD(NV)                                                                                         \
  cudaFuncSetAttribute(cross_bwd_kernel<NV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);   \
  cross_bwd_kernel<NV><<<grid, wpc * 32, smem, st>>>(x0, w, b, s, dxL, dx_in, B, D, L, dx0, partial, wpc);
  CROSS_NV_SWITCH(nv, BWD)
#undef BWD
  CTR_LAUNCHED("ctr_cross_bwd");
  const int64_t LD = (int64_t)L * D;
  cross_reduce_kernel<<<(unsigned)((2 * LD + 255) / 256), 256, 0, st>>>(partial, grid * wpc, LD, dw, db);
  CTR_LAUNCHED("cross_reduce");
  return CTR_OK;
}

}  // extern "C"
