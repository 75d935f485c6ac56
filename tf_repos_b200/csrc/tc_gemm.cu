// tc_gemm.cu -- the dense GEMMs of the MLP / attention layers on the Hopper tensor cores (wgmma, fp32
// accumulators in registers), at fp32-class accuracy through a 3xTF32 split.  This is the only GEMM path:
// fc.cu launches every layer product, at every shape, through tc_gemm_dispatch.
//
// Why 3xTF32: the parity target is 1e-5 relative on the logits; a plain TF32 (10-bit mantissa) or
// BF16 product loses 1e-3.  Each fp32 operand is split on the fly into hi = rn_tf32(a) and
// lo = a - hi (exact); D += A_lo*B_hi + A_hi*B_lo + A_hi*B_hi on the tensor cores recovers ~2^-21
// relative accuracy with fp32 accumulation, at 1/3 of the TF32 rate (still several times the fp32
// SIMT pipe).
//
// Structure of one CTA (256 threads = two warpgroups, one 128 x BN output tile, BN in {32, 64, 128}):
//   loop over 32-wide reduction slices, 2-stage shared-memory ring (1 stage when the reduction is one slice):
//     all threads  : registers (loaded one slice ahead, coalesced for either operand orientation)
//                    -> hi/lo split -> st.shared in the canonical K-major SWIZZLE_128B layout
//                    fence.proxy.async ; __syncthreads ; issue the NEXT slice's global loads
//     warpgroup w  : rows 64w..64w+63: 4 k-steps x 3 wgmma.m64nBNk8.tf32 ; commit ; wait
//                    (the stage is refilled two slices later, after every warpgroup has waited on it)
//   epilogue       : accumulator fragments -> staging tile in shared memory ->
//                    whole rows per warp: bias / group bias / relu / dropout / accumulate -> 512 B coalesced stores
// Operands are staged by plain loads rather than TMA because the three products of a layer need
// three different operand orientations of fp32 data that must be split anyway.
#include <stdlib.h>

#include "common.cuh"

namespace ctr {

constexpr int TC_BM = 128, TC_BK = 32, TC_THREADS = 256;
constexpr int TC_TILE_BYTES = TC_BM * TC_BK * 4;            // 16 KB: one 128 x 32 fp32 operand tile
constexpr int TC_STAGE_BYTES = 4 * TC_TILE_BYTES;           // A_hi, A_lo, B_hi, B_lo

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// K-major, SWIZZLE_128B shared-memory matrix descriptor (sm_90 wgmma):
//   start_address[0,14) = addr>>4 ; LBO[16,30) = 1 (unused for swizzled K-major) ; SBO[32,46) = 1024 B >> 4
//   layout_type[62,64) = 1 (SWIZZLE_128B)
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// D[64 x N] += A[64 x 8] * B[8 x N], both operands K-major in shared memory, fp32 accumulators in registers:
// thread t of the warpgroup holds rows 16*(t/32) + (t%32)/4 (+8) and columns 8j + 2*(t%4) (+1), j < N/8
template <int N>
__device__ __forceinline__ void wgmma_tf32(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc);

template <>
__device__ __forceinline__ void wgmma_tf32<32>(float (&d)[16], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t"
      "}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(1));
}

template <>
__device__ __forceinline__ void wgmma_tf32<64>(float (&d)[32], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t"
      "}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(1));
}

template <>
__device__ __forceinline__ void wgmma_tf32<128>(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t"
      "}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(1));
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accesses of the accumulators across the asynchronous wgmma window
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

__device__ __forceinline__ float tf32_hi(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

// byte offset of (row, 16-byte chunk c) inside a K-major SWIZZLE_128B tile of 32 fp32 per row
__device__ __forceinline__ uint32_t sw128_off(int row, int chunk) {
  return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((chunk ^ (row & 7)) << 4));
}


// ---- operand staging -----------------------------------------------------------------------------------------
// One 128 x 32 fp32 operand tile = 4 float4 per thread of the 256.  RC (the reduction index is the contiguous one in
// global memory): a warp reads 4 rows x 128 B per instruction (8 lanes per row) -- coalesced -- and the same
// (row, 16-byte chunk) assignment makes the swizzled shared-memory stores conflict-free.  !RC (the tile row
// index is the contiguous one): thread t owns tile row t%128 and half t/128 of the slice.
template <bool RC>
__device__ __forceinline__ void load_tile(float4 (&r)[4], const float* __restrict__ P, int ld, int row0, int n_rows,
                                             int r0, int r_end, int tid) {
  if (RC) {
    const int sub = (tid & 31) >> 3, ch = tid & 7, wrow = (tid >> 5) * 16;
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const int g = row0 + wrow + it * 4 + sub, k0 = r0 + ch * 4;
      const float* p = P + (int64_t)g * ld + k0;
      if (g < n_rows && k0 + 4 <= r_end && ((((uintptr_t)p) & 15) == 0)) {
        r[it] = __ldg(reinterpret_cast<const float4*>(p));
      } else {
        const bool in = g < n_rows;
        r[it].x = (in && k0 < r_end) ? p[0] : 0.f;
        r[it].y = (in && k0 + 1 < r_end) ? p[1] : 0.f;
        r[it].z = (in && k0 + 2 < r_end) ? p[2] : 0.f;
        r[it].w = (in && k0 + 3 < r_end) ? p[3] : 0.f;
      }
    }
  } else {
    const int g = row0 + (tid & 127), half = tid >> 7;
    const bool in = g < n_rows;
    const float* p = P + (int64_t)r0 * ld + g;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int cc = half * 4 + c;
      r[c].x = (in && r0 + 4 * cc < r_end) ? p[(int64_t)(4 * cc) * ld] : 0.f;
      r[c].y = (in && r0 + 4 * cc + 1 < r_end) ? p[(int64_t)(4 * cc + 1) * ld] : 0.f;
      r[c].z = (in && r0 + 4 * cc + 2 < r_end) ? p[(int64_t)(4 * cc + 2) * ld] : 0.f;
      r[c].w = (in && r0 + 4 * cc + 3 < r_end) ? p[(int64_t)(4 * cc + 3) * ld] : 0.f;
    }
  }
}

// Interior tiles and full 32-wide slices (all of a layer but its edges): no bounds logic, pointers advanced by the
// caller.  `base` already points at this thread's first element of slice 0 (RC: row (wrow+sub), 16 B chunk ch;
// !RC: tile row tid&127, reduction index (tid>>7)*16); r0 is the slice's offset along the reduction.
template <bool RC>
__device__ __forceinline__ void load_tile_fast(float4 (&r)[4], const float* __restrict__ base, int ld, int r0) {
  if (RC) {
    const float* p = base + r0;
#pragma unroll
    for (int it = 0; it < 4; ++it) r[it] = __ldg(reinterpret_cast<const float4*>(p + (int64_t)(it * 4) * ld));
  } else {
    const float* p = base + (int64_t)r0 * ld;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      r[c].x = __ldg(p + (int64_t)(4 * c) * ld);
      r[c].y = __ldg(p + (int64_t)(4 * c + 1) * ld);
      r[c].z = __ldg(p + (int64_t)(4 * c + 2) * ld);
      r[c].w = __ldg(p + (int64_t)(4 * c + 3) * ld);
    }
  }
}

// hi/lo split + store with the swizzled offsets precomputed once per thread (they do not depend on the slice)
__device__ __forceinline__ void store_tile_fast(const float4 (&r)[4], uint8_t* hi_tile, uint8_t* lo_tile,
                                                   const uint32_t (&off)[4]) {
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    float4 hi, lo;
    hi.x = tf32_hi(r[it].x); hi.y = tf32_hi(r[it].y); hi.z = tf32_hi(r[it].z); hi.w = tf32_hi(r[it].w);
    lo.x = r[it].x - hi.x; lo.y = r[it].y - hi.y; lo.z = r[it].z - hi.z; lo.w = r[it].w - hi.w;
    *reinterpret_cast<float4*>(hi_tile + off[it]) = hi;
    *reinterpret_cast<float4*>(lo_tile + off[it]) = lo;
  }
}

constexpr int TC_STG_PITCH = TC_BM + 4;                          // epilogue staging row pitch (floats)
constexpr int TC_STG_BYTES = TC_BM * TC_STG_PITCH * 4;
constexpr int tc_smem_bytes(int stages) { return (stages * TC_STAGE_BYTES > TC_STG_BYTES ? stages * TC_STAGE_BYTES : TC_STG_BYTES) + 1024; }

// ---- epilogue: NW warps write whole rows of the staged tile (lane l <-> columns 4l..4l+3, 512 B
// coalesced): bias / group bias / relu / dropout (EPI 1), accumulate (EPI 2).  When a row needs a global read first
// (dropout mask, old C) the reads of 4 rows are issued together: one dependent load per row made the masked forward of
// DIN's attention layer latency-bound at 1.1 TB/s.
template <int EPI, int NW>
__device__ __forceinline__ void tc_epilogue_rows(const float* __restrict__ stg, float* __restrict__ Cz, int ldc, int M, int N,
                                                 int i0, int j0, int n_here, int warp, int lane,
                                                 const float* __restrict__ bias, int act, const float* __restrict__ mask,
                                                 float keep, const float* __restrict__ gbias, int gP) {
  const int col = lane * 4, gj = j0 + col;
  const bool vec = ((ldc & 3) == 0) && ((((uintptr_t)Cz) & 15) == 0) && (EPI != 1 || !mask || ((((uintptr_t)mask) & 15) == 0));
  if (col >= n_here) return;
  float bv[4] = {0.f, 0.f, 0.f, 0.f};
  if (EPI == 1 && bias) {
#pragma unroll
    for (int q = 0; q < 4; ++q) bv[q] = (gj + q < N) ? bias[gj + q] : 0.f;
  }
  const int rows = min(TC_BM, M - i0);
  const bool full = vec && (col + 4 <= n_here);
  auto emit_row = [&](int row, const float4& mkv, const float4& ocv) {
    const int gi = i0 + row;
    const float4 t = *reinterpret_cast<const float4*>(stg + row * TC_STG_PITCH + col);
    float v[4] = {t.x, t.y, t.z, t.w};
    float* cp = Cz + (int64_t)gi * ldc + gj;
    if (EPI == 2) {
      if (full) { v[0] += ocv.x; v[1] += ocv.y; v[2] += ocv.z; v[3] += ocv.w; }
      else {
#pragma unroll
        for (int q = 0; q < 4; ++q) if (col + q < n_here) v[q] += cp[q];
      }
    }
    if (EPI == 1) {
      const float* gb = gbias ? gbias + (int64_t)(gi / gP) * N + gj : nullptr;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        v[q] += bv[q];
        if (gb && col + q < n_here) v[q] += gb[q];
        if (act == 1) v[q] = fmaxf(v[q], 0.f);
      }
      if (mask) {
        const float* mp = mask + (int64_t)gi * ldc + gj;
        if (full) {
          v[0] = __fdiv_rn(v[0], keep) * mkv.x; v[1] = __fdiv_rn(v[1], keep) * mkv.y;
          v[2] = __fdiv_rn(v[2], keep) * mkv.z; v[3] = __fdiv_rn(v[3], keep) * mkv.w;
        } else {
#pragma unroll
          for (int q = 0; q < 4; ++q) if (col + q < n_here) v[q] = __fdiv_rn(v[q], keep) * mp[q];
        }
      }
    }
    if (full) {
      *reinterpret_cast<float4*>(cp) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
#pragma unroll
      for (int q = 0; q < 4; ++q) if (col + q < n_here) cp[q] = v[q];
    }
  };
  const float4 one = make_float4(1.f, 1.f, 1.f, 1.f), zero = f4_zero();
  if (full && ((EPI == 1 && mask) || EPI == 2)) {
    constexpr int UNR = 4;
    for (int row_base = warp; row_base < rows; row_base += NW * UNR) {
      float4 mk[UNR], oc[UNR];
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        const int row = row_base + u * NW;
        mk[u] = one; oc[u] = zero;
        if (row < rows) {
          const int64_t o = (int64_t)(i0 + row) * ldc + gj;
          if (EPI == 1) mk[u] = __ldg(reinterpret_cast<const float4*>(mask + o));
          if (EPI == 2) oc[u] = *reinterpret_cast<const float4*>(Cz + o);
        }
      }
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        const int row = row_base + u * NW;
        if (row < rows) emit_row(row, mk[u], oc[u]);
      }
    }
  } else {
    for (int row = warp; row < rows; row += NW) emit_row(row, one, zero);
  }
}

// C[i][j] = sum_r A(i,r) * B(r,j)
//   A_RC: A(i,r) = A[i*lda + r] else A[r*lda + i];  B_RC: B(r,j) = B[j*ldb + r] else B[r*ldb + j]
// EPI 0: store (split-R chunk z to C + z*M*ldc)  1: act(acc + bias + gbias[i/gP]) (/keep*mask)  2: C += acc
// BN: tile width (32 / 64 only when the whole of N fits: narrow products do not pay for a 128-wide MMA)
template <bool A_RC, bool B_RC, int EPI, int BN>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_gemm_kernel(const float* __restrict__ A, int lda, const float* __restrict__ B, int ldb, float* __restrict__ C,
               int ldc, int M, int N, int R, const float* __restrict__ bias, int act, const float* __restrict__ mask,
               float keep, const float* __restrict__ gbias, int gP) {
  extern __shared__ uint8_t smem_raw[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // SWIZZLE_128B wants 1024 B alignment
  const int i0 = blockIdx.y * TC_BM, j0 = blockIdx.x * BN;
  const int n_here = min(N - j0, BN);
  const int r_chunk = (R + gridDim.z - 1) / gridDim.z;
  const int r_begin = blockIdx.z * r_chunk, r_end = min(R, r_begin + r_chunk);
  const int KT = max((r_end - r_begin + TC_BK - 1) / TC_BK, 0);
  const int stages = KT > 1 ? 2 : 1;

  // per-thread constants of the operand staging
  const int sub = (tid & 31) >> 3, ch = tid & 7, wrow = (tid >> 5) * 16;
  uint32_t offA[4], offB[4];
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    offA[it] = A_RC ? sw128_off(wrow + it * 4 + sub, ch) : sw128_off(tid & 127, (tid >> 7) * 4 + it);
    offB[it] = B_RC ? sw128_off(wrow + it * 4 + sub, ch) : sw128_off(tid & 127, (tid >> 7) * 4 + it);
  }
  const float* baseA = A_RC ? A + (int64_t)(i0 + wrow + sub) * lda + ch * 4 : A + (int64_t)((tid >> 7) * 16) * lda + i0 + (tid & 127);
  const float* baseB = B_RC ? B + (int64_t)(j0 + wrow + sub) * ldb + ch * 4 : B + (int64_t)((tid >> 7) * 16) * ldb + j0 + (tid & 127);
  // interior tile, and 16 B alignment of every float4 the RC path reads
  const bool fullA = (i0 + TC_BM <= M) && (!A_RC || (((lda & 3) == 0) && ((((uintptr_t)A) & 15) == 0) && ((r_begin & 3) == 0)));
  const bool fullB = (j0 + TC_BM <= N) && (!B_RC || (((ldb & 3) == 0) && ((((uintptr_t)B) & 15) == 0) && ((r_begin & 3) == 0)));
  auto load_slice = [&](float4 (&a)[4], float4 (&b)[4], int kt) {
    const int r0 = r_begin + kt * TC_BK;
    const bool whole = r0 + TC_BK <= r_end;
    if (fullA && whole) load_tile_fast<A_RC>(a, baseA, lda, r0); else load_tile<A_RC>(a, A, lda, i0, M, r0, r_end, tid);
    if (fullB && whole) load_tile_fast<B_RC>(b, baseB, ldb, r0); else load_tile<B_RC>(b, B, ldb, j0, N, r0, r_end, tid);
  };

  // Two accumulators: the tensor core adds in fp32 with truncation, so every accumulation costs ~2^-24 of the
  // accumulator, with a bias.  The two cross terms (2^-11 of the result) go to their own accumulator: the main
  // one then sees one accumulation per k-step instead of three.
  float acc[BN / 2], acc2[BN / 2];
#pragma unroll
  for (int q = 0; q < BN / 2; ++q) { acc[q] = 0.f; acc2[q] = 0.f; }
  float4 ra[4], rb[4];
  if (KT > 0) load_slice(ra, rb, 0);
  for (int kt = 0; kt < KT; ++kt) {
    // stage kt%2 was last read by the MMAs of slice kt-2, which both warpgroups waited for before the barrier of kt-1
    uint8_t* st = smem + (kt % stages) * TC_STAGE_BYTES;
    store_tile_fast(ra, st, st + TC_TILE_BYTES, offA);
    store_tile_fast(rb, st + 2 * TC_TILE_BYTES, st + 3 * TC_TILE_BYTES, offB);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> visible to the tensor core
    __syncthreads();
    if (kt + 1 < KT) load_slice(ra, rb, kt + 1);   // next slice: global -> registers while the tensor core works
    const uint32_t a_hi = smem_u32(st) + wg * (TC_TILE_BYTES / 2), a_lo = a_hi + TC_TILE_BYTES;
    const uint32_t b_hi = smem_u32(st) + 2 * TC_TILE_BYTES, b_lo = b_hi + TC_TILE_BYTES;
    fence_regs(acc); fence_regs(acc2);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < TC_BK / 8; ++k) {                        // K = 8 tf32 = 32 bytes inside the 128 B swizzle atom
      const uint32_t ko = k * 32;
      wgmma_tf32<BN>(acc2, make_desc(a_lo + ko), make_desc(b_hi + ko));
      wgmma_tf32<BN>(acc2, make_desc(a_hi + ko), make_desc(b_lo + ko));
      wgmma_tf32<BN>(acc, make_desc(a_hi + ko), make_desc(b_hi + ko));
    }
    wgmma_commit();
    wgmma_wait_all();
    fence_regs(acc); fence_regs(acc2);
  }
  __syncthreads();   // every MMA has completed: the operand stages become the staging tile

  // ---- epilogue 1: fragments -> staging tile (row 64*wg + 16*(warp%4) + lane/4 (+8), columns 8j + 2*(lane%4))
  float* stg = reinterpret_cast<float*>(smem);
  const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = 8 * j + 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int q = 4 * j + 2 * h;
      *reinterpret_cast<float2*>(stg + (row0 + 8 * h) * TC_STG_PITCH + col) =
          make_float2(acc[q] + acc2[q], acc[q + 1] + acc2[q + 1]);
    }
  }
  __syncthreads();

  // ---- epilogue 2: a warp writes whole rows (lane l <-> columns 4l..4l+3): 512 B coalesced stores
  float* Cz = C + (EPI == 0 ? (int64_t)blockIdx.z * M * ldc : 0);
  tc_epilogue_rows<EPI, TC_THREADS / 32>(stg, Cz, ldc, M, N, i0, j0, n_here, warp, lane, bias, act, mask, keep, gbias, gP);
}

template <bool A_RC, bool B_RC, int EPI, int BN>
static int launch_tc_bn(const float* A, int lda, const float* B, int ldb, float* C, int ldc, int M, int N, int R, int S,
                        const float* bias, int act, const float* mask, float keep, const float* gbias, int gP,
                        cudaStream_t st) {
  static bool attr = false;
  constexpr int smem_max = tc_smem_bytes(2);
  if (!attr) {
    cudaFuncSetAttribute(tc_gemm_kernel<A_RC, B_RC, EPI, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max);
    attr = true;
  }
  const int r_chunk = (R + S - 1) / S;
  const int smem = tc_smem_bytes(r_chunk > TC_BK ? 2 : 1);   // one slice: one stage, so that more CTAs fit an SM
  dim3 grid((N + BN - 1) / BN, (M + TC_BM - 1) / TC_BM, S);
  tc_gemm_kernel<A_RC, B_RC, EPI, BN><<<grid, TC_THREADS, smem, st>>>(A, lda, B, ldb, C, ldc, M, N, R, bias, act, mask,
                                                                      keep, gbias, gP);
  return 0;
}

template <bool A_RC, bool B_RC, int EPI>
static int launch_tc(const float* A, int lda, const float* B, int ldb, float* C, int ldc, int M, int N, int R, int S,
                     const float* bias, int act, const float* mask, float keep, const float* gbias, int gP,
                     cudaStream_t st) {
  if (N <= 32) return launch_tc_bn<A_RC, B_RC, EPI, 32>(A, lda, B, ldb, C, ldc, M, N, R, S, bias, act, mask, keep, gbias, gP, st);
  if (N <= 64) return launch_tc_bn<A_RC, B_RC, EPI, 64>(A, lda, B, ldb, C, ldc, M, N, R, S, bias, act, mask, keep, gbias, gP, st);
  return launch_tc_bn<A_RC, B_RC, EPI, 128>(A, lda, B, ldb, C, ldc, M, N, R, S, bias, act, mask, keep, gbias, gP, st);
}

// entry used by fc.cu: kind 0 = forward (A_RC, !B_RC, EPI 1), 1 = dIn (A_RC, B_RC, EPI 0 / 2), 2 = dW (!A_RC, !B_RC, EPI 0)
int tc_gemm_dispatch(int kind, int epi, const float* A, int lda, const float* B, int ldb, float* C, int ldc, int M, int N,
                     int R, int S, const float* bias, int act, const float* mask, float keep, const float* gbias, int gP,
                     cudaStream_t st) {
  if (kind == 0) return launch_tc<true, false, 1>(A, lda, B, ldb, C, ldc, M, N, R, S, bias, act, mask, keep, gbias, gP, st);
  if (kind == 1 && epi == 2) return launch_tc<true, true, 2>(A, lda, B, ldb, C, ldc, M, N, R, S, bias, act, mask, keep, gbias, gP, st);
  if (kind == 1) return launch_tc<true, true, 0>(A, lda, B, ldb, C, ldc, M, N, R, S, bias, act, mask, keep, gbias, gP, st);
  return launch_tc<false, false, 0>(A, lda, B, ldb, C, ldc, M, N, R, S, bias, act, mask, keep, gbias, gP, st);
}

}  // namespace ctr
