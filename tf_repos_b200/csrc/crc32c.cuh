// crc32c.cuh -- warp-cooperative CRC-32C (Castagnoli) over device memory, shared by the TFRecord reader
// (tfrecord_device.cu) and writer (aliccp_tfrecord.cu).
//
// Each lane CRCs 1/32 of the bytes; the 32 remainders are combined with x^(8n) mod P.  The helpers live in an
// anonymous namespace so that every translation unit that includes this header owns its copy.
#pragma once
#include "common.cuh"

namespace ctr {
namespace {

constexpr uint32_t TR_POLY = 0x82F63B78u;  // CRC-32C, reflected

__device__ __forceinline__ uint32_t gf_mul(uint32_t a, uint32_t b) {   // reflected GF(2)[x] / P: bit 31 is x^0
  uint32_t p = 0;
#pragma unroll 4
  for (int i = 0; i < 32; ++i) {
    if (a & 0x80000000u) p ^= b;
    a <<= 1;
    b = (b & 1) ? (b >> 1) ^ TR_POLY : b >> 1;
  }
  return p;
}
__device__ __forceinline__ uint32_t gf_x8n(const uint32_t* x8, uint64_t n) {   // x^(8n) mod P; x8[k] = x^(8*2^k)
  uint32_t r = 0x80000000u;
  for (int k = 0; n; ++k, n >>= 1)
    if (n & 1) r = gf_mul(r, x8[k]);
  return r;
}

// The data is read as 32 equal segments of a stream with 32*seg - L zero bytes in front: leading zeros leave a CRC
// with zero initial value unchanged, so every segment is shifted by a multiple of seg bytes and the tree needs one
// constant per level.  load(d, p) returns byte p (CrcLdg or CrcPlain below).
template <class Load>
__device__ uint32_t crc32c_warp(const uint8_t* d, int64_t L, const uint32_t* tab, const uint32_t* x8, Load load) {
  const int lane = threadIdx.x & 31;
  const int64_t seg = (L + 31) >> 5, z = 32 * seg - L;
  int64_t lo = lane * seg - z, hi = lo + seg;
  lo = lo < 0 ? 0 : lo;
  uint32_t c = 0;
  for (int64_t p = lo; p < hi; ++p) c = tab[(c ^ load(d, p)) & 0xFF] ^ (c >> 8);
  uint32_t M = gf_x8n(x8, (uint64_t)seg);
  for (int k = 1; k < 32; k <<= 1) {
    const uint32_t partner = __shfl_down_sync(FULL_MASK, c, k);
    if ((lane & (2 * k - 1)) == 0) c = gf_mul(c, M) ^ partner;
    M = gf_mul(M, M);
  }
  c = __shfl_sync(FULL_MASK, c, 0);
  return c ^ gf_mul(0xFFFFFFFFu, gf_x8n(x8, (uint64_t)L)) ^ 0xFFFFFFFFu;
}

struct CrcLdg {     // through the read-only cache
  __device__ __forceinline__ uint32_t operator()(const uint8_t* d, int64_t p) const { return __ldg(d + p); }
};
struct CrcPlain {   // plain loads: bytes the calling warp has just stored
  __device__ __forceinline__ uint32_t operator()(const uint8_t* d, int64_t p) const { return d[p]; }
};

__device__ __forceinline__ uint32_t crc32c_mask(uint32_t c) { return ((c >> 15) | (c << 17)) + 0xA282EAD8u; }

// the byte table and x8[k] = x^(8*2^k) mod P in shared memory (every thread of the CTA calls this)
__device__ void tr_crc_tables(uint32_t* tab, uint32_t* x8) {
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    uint32_t c = i;
    for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ TR_POLY : c >> 1;
    tab[i] = c;
  }
  if (threadIdx.x == 0) {
    x8[0] = 0x00800000u;   // x^8
    for (int k = 1; k < 64; ++k) x8[k] = gf_mul(x8[k - 1], x8[k - 1]);
  }
  __syncthreads();
}

}  // namespace
}  // namespace ctr
