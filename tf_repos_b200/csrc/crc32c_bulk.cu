// crc32c_bulk.cu -- CRC-32C of whole device tensors (TensorFlow checkpoint bundles, tf_repos_b200/tf_checkpoint.py).
//
// Each range (address, length) is cut into chunks of CHUNK_BYTES that END at the last 16-byte boundary of the range,
// so the first chunk is the partial one and reads as leading zero bytes (a CRC with zero initial value is unchanged by
// leading zeros).  The bytes of the 16-byte word that holds the range's start but lie before it are masked to zero
// the same way; the < 16 bytes after the last boundary are folded in byte by byte at the end.
//
//   crc_chunks   persistent CTAs, one chunk at a time.  Thread t reads words t, t+T, t+2T, ... (coalesced 16-byte
//                loads) and keeps c_t = c_t * x^(128T) + crc(word): the shift is four table lookups, the word sixteen
//                (slicing by 16).  The chunk's CRC is the XOR of c_t * x^(128(T-1-t)).
//   crc_combine  one CTA per range: the chunk CRCs folded by x^(8*CHUNK_BYTES), the tail bytes, and the ~0 initial
//                value / final XOR of the standard CRC-32C.
#include "crc32c.cuh"

namespace ctr {
namespace {

constexpr int CRC_T = 256;                         // threads per CTA
constexpr int CRC_U = 32;                          // 16-byte words per thread and chunk
constexpr int64_t CHUNK_WORDS = (int64_t)CRC_T * CRC_U;
constexpr int64_t CHUNK_BYTES = CHUNK_WORDS * 16;  // 128 KiB

struct RangeLayout {   // chunk grid of one range
  uint64_t a, e;       // first / one past the last 16-byte aligned address of the body (e <= a: no body)
  int64_t chunks;
};

__device__ __forceinline__ RangeLayout range_layout(uint64_t p, int64_t len) {
  RangeLayout r;
  r.a = p & ~(uint64_t)15;
  r.e = (p + (uint64_t)len) & ~(uint64_t)15;
  r.chunks = (len > 0 && r.e > r.a) ? (int64_t)(((r.e - r.a) / 16 + CHUNK_WORDS - 1) / CHUNK_WORDS) : 0;
  return r;
}

// ws: int64 prefix[n + 1] (chunk index of each range's first chunk), then uint32 crc[chunks]
__global__ void crc_plan_kernel(const int64_t* __restrict__ ranges, int n, int64_t* __restrict__ prefix) {
  if (threadIdx.x != 0) return;
  int64_t s = 0;
  for (int i = 0; i < n; ++i) {
    prefix[i] = s;
    s += range_layout((uint64_t)ranges[2 * i], ranges[2 * i + 1]).chunks;
  }
  prefix[n] = s;
}

__global__ void __launch_bounds__(CRC_T) crc_chunks_kernel(const int64_t* __restrict__ ranges, int n,
                                                           const int64_t* __restrict__ prefix,
                                                           uint32_t* __restrict__ chunk_crc) {
  __shared__ uint32_t tab[256], x8[64];
  __shared__ uint32_t sl[16][256];   // sl[k][b]: crc of byte b followed by k zero bytes
  __shared__ uint32_t sh[4][256];    // sh[j][b]: (b << 8j) * x^(128(T-1))
  __shared__ uint32_t warp_c[CRC_T / 32];
  tr_crc_tables(tab, x8);
  const int t = threadIdx.x;
  {
    uint32_t c = tab[t];
    sl[0][t] = c;
    for (int k = 1; k < 16; ++k) { c = (c >> 8) ^ tab[c & 0xFF]; sl[k][t] = c; }
    const uint32_t K = gf_x8n(x8, 16ull * (CRC_T - 1));
    for (int j = 0; j < 4; ++j) sh[j][t] = gf_mul((uint32_t)t << (8 * j), K);
  }
  const uint32_t out_shift = gf_x8n(x8, 16ull * (CRC_T - 1 - t));   // this thread's words -> end of the chunk
  __syncthreads();
  const int64_t total = prefix[n];
  for (int64_t g = blockIdx.x; g < total; g += gridDim.x) {
    int lo = 0, hi = n - 1;   // the range whose chunks hold g: prefix[lo] <= g < prefix[lo + 1]
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (prefix[mid] <= g) lo = mid; else hi = mid - 1;
    }
    const uint64_t p = (uint64_t)ranges[2 * lo];
    const RangeLayout L = range_layout(p, ranges[2 * lo + 1]);
    // virtual start of this chunk (may lie below a: those words read as zero)
    const int64_t j = g - prefix[lo];
    const int64_t base = (int64_t)L.e - (L.chunks - j) * CHUNK_BYTES;
    uint32_t c = 0;
#pragma unroll 4
    for (int i = 0; i < CRC_U; ++i) {
      const int64_t addr = base + ((int64_t)i * CRC_T + t) * 16;
      uint4 w = make_uint4(0u, 0u, 0u, 0u);
      if (addr >= (int64_t)L.a) {
        w = __ldcs(reinterpret_cast<const uint4*>(addr));
        if (addr == (int64_t)L.a) {           // bytes before the range's start
          const uint32_t h = (uint32_t)(p - L.a);   // 0, 4, 8 or 12
          if (h > 0) w.x = 0u;
          if (h > 4) w.y = 0u;
          if (h > 8) w.z = 0u;
        }
      }
      c = sh[0][c & 0xFF] ^ sh[1][(c >> 8) & 0xFF] ^ sh[2][(c >> 16) & 0xFF] ^ sh[3][c >> 24];
      c ^= w.x;
      c = sl[15][c & 0xFF] ^ sl[14][(c >> 8) & 0xFF] ^ sl[13][(c >> 16) & 0xFF] ^ sl[12][c >> 24] ^
          sl[11][w.y & 0xFF] ^ sl[10][(w.y >> 8) & 0xFF] ^ sl[9][(w.y >> 16) & 0xFF] ^ sl[8][w.y >> 24] ^
          sl[7][w.z & 0xFF] ^ sl[6][(w.z >> 8) & 0xFF] ^ sl[5][(w.z >> 16) & 0xFF] ^ sl[4][w.z >> 24] ^
          sl[3][w.w & 0xFF] ^ sl[2][(w.w >> 8) & 0xFF] ^ sl[1][(w.w >> 16) & 0xFF] ^ sl[0][w.w >> 24];
    }
    c = gf_mul(c, out_shift);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c ^= __shfl_xor_sync(FULL_MASK, c, o);
    if ((t & 31) == 0) warp_c[t >> 5] = c;
    __syncthreads();
    if (t == 0) {
      uint32_t s = 0;
      for (int k = 0; k < CRC_T / 32; ++k) s ^= warp_c[k];
      chunk_crc[g] = s;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(CRC_T) crc_combine_kernel(const int64_t* __restrict__ ranges,
                                                            const int64_t* __restrict__ prefix,
                                                            const uint32_t* __restrict__ chunk_crc,
                                                            uint32_t* __restrict__ crc, uint32_t* __restrict__ masked) {
  __shared__ uint32_t tab[256], x8[64];
  __shared__ uint32_t warp_c[CRC_T / 32];
  tr_crc_tables(tab, x8);
  const int r = blockIdx.x, t = threadIdx.x;
  const uint64_t p = (uint64_t)ranges[2 * r];
  const int64_t len = ranges[2 * r + 1];
  const RangeLayout L = range_layout(p, len);
  const uint32_t* cc = chunk_crc + prefix[r];
  // thread t folds chunks [t*G - z, (t+1)*G - z): z leading virtual chunks of zeros make the groups equal
  const int64_t G = (L.chunks + CRC_T - 1) / CRC_T, z = G * CRC_T - L.chunks;
  const uint32_t M = gf_x8n(x8, (uint64_t)CHUNK_BYTES);
  uint32_t c = 0;
  for (int64_t v = t * G; v < (t + 1) * G; ++v)
    if (v >= z) c = gf_mul(c, M) ^ cc[v - z];
  if (c) c = gf_mul(c, gf_x8n(x8, (uint64_t)CHUNK_BYTES * G * (CRC_T - 1 - t)));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c ^= __shfl_xor_sync(FULL_MASK, c, o);
  if ((t & 31) == 0) warp_c[t >> 5] = c;
  __syncthreads();
  if (t != 0) return;
  uint32_t s = 0;
  for (int k = 0; k < CRC_T / 32; ++k) s ^= warp_c[k];
  const uint8_t* d = reinterpret_cast<const uint8_t*>(p);
  for (uint64_t q = (L.chunks ? L.e : p); q < p + (uint64_t)len; ++q) s = tab[(s ^ d[q - p]) & 0xFF] ^ (s >> 8);
  s ^= gf_mul(0xFFFFFFFFu, gf_x8n(x8, (uint64_t)len)) ^ 0xFFFFFFFFu;
  if (crc) crc[r] = s;
  if (masked) masked[r] = crc32c_mask(s);
}

size_t crc_ws_layout(int n, int64_t total_bytes, size_t* chunk_off) {
  const int64_t cap = total_bytes / CHUNK_BYTES + 2 * (int64_t)n + 1;   // a range's body spans <= len + 12 bytes
  *chunk_off = align256(sizeof(int64_t) * (size_t)(n + 1));
  return *chunk_off + align256(sizeof(uint32_t) * (size_t)cap);
}

}  // namespace
}  // namespace ctr

using namespace ctr;

extern "C" {

size_t ctr_crc32c_workspace_bytes(int n, int64_t total_bytes) {
  if (n < 0 || total_bytes < 0) return 0;
  size_t off;
  return crc_ws_layout(n, total_bytes, &off);
}

int ctr_crc32c_ranges(const int64_t* ranges, int n, int64_t total_bytes, uint32_t* crc, uint32_t* masked, void* ws,
                      size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE(n >= 0 && total_bytes >= 0, CTR_ERR_INVALID_ARG, "ctr_crc32c_ranges: n < 0 or total_bytes < 0");
  if (n == 0) return CTR_OK;
  CTR_REQUIRE(ranges != nullptr && ws != nullptr, CTR_ERR_INVALID_ARG, "ctr_crc32c_ranges: null ranges or workspace");
  CTR_REQUIRE(crc != nullptr || masked != nullptr, CTR_ERR_INVALID_ARG, "ctr_crc32c_ranges: no output");
  size_t chunk_off;
  const size_t need = crc_ws_layout(n, total_bytes, &chunk_off);
  CTR_REQUIRE(ws_bytes >= need, CTR_ERR_WORKSPACE, "ctr_crc32c_ranges: workspace %zu < %zu bytes", ws_bytes, need);
  int64_t* prefix = static_cast<int64_t*>(ws);
  uint32_t* chunk_crc = reinterpret_cast<uint32_t*>(static_cast<char*>(ws) + chunk_off);
  cudaStream_t s = as_stream(stream);
  crc_plan_kernel<<<1, 32, 0, s>>>(ranges, n, prefix);
  CTR_LAUNCHED("ctr_crc32c_ranges (plan)");
  const int64_t cap = total_bytes / CHUNK_BYTES + 2 * (int64_t)n + 1;
  crc_chunks_kernel<<<grid_for(cap, 1, 8), CRC_T, 0, s>>>(ranges, n, prefix, chunk_crc);
  CTR_LAUNCHED("ctr_crc32c_ranges (chunks)");
  crc_combine_kernel<<<n, CRC_T, 0, s>>>(ranges, prefix, chunk_crc, crc, masked);
  CTR_LAUNCHED("ctr_crc32c_ranges (combine)");
  return CTR_OK;
}

}  // extern "C"
