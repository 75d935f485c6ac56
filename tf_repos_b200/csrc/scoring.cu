// scoring.cu -- what the drop-in scripts do after the forward pass in --task_type=eval / infer (DESIGN.md §2.13).
//
//   auc_counts   tf.metrics.auc's confusion counts at 200 thresholds (DeepFM.py:194, DeepCvrMTL.py:229-233) as a
//                per-class histogram of "how many thresholds lie below p", accumulated across calls.  Each warp owns a
//                sub-histogram in shared memory; lanes that hit the same bin are merged with __match_any_sync first,
//                because CTR predictions crowd into a few bins.  One 64-bit global add per non-zero bin per CTA.
//   format       pred.txt's "%f\n" (or "%f\t%f\n") lines, the bytes of Python's "%f" % float(x) for every float32:
//                lengths per tile of FMT_TILE rows, the tile offsets by cta_scan (scan_sort.cuh), then each tile is
//                formatted into shared memory a sub-tile at a time and copied out in aligned 4-byte words at the
//                device-resident running offset, which a last one-thread kernel advances.
#include "scan_sort.cuh"

namespace ctr {
namespace {

constexpr int AUC_THREADS = 256, AUC_WARPS = AUC_THREADS / 32;
constexpr int AUC_N_THR = 200, AUC_BINS = AUC_N_THR + 1;
constexpr int AUC_KEYS = 512;   // class * 256 + bin

// number of thresholds t with t < p; a NaN p lies above every threshold (np.sort puts it last, and searchsorted(...,
// side="right") counts it above).  thr: 256 ascending values, the 56 past the real ones +inf.
__device__ __forceinline__ int auc_bin(const float* thr, float p) {
  if (isnan(p)) return AUC_N_THR;
  int pos = 0;
#pragma unroll
  for (int step = 128; step > 0; step >>= 1)
    if (thr[pos + step - 1] < p) pos += step;
  return pos;
}

// key = class * 256 + bin; a label is positive when it is non-zero (a NaN label too, as astype(bool) makes it)
__device__ __forceinline__ int auc_key(const float* thr, float p, float y) {
  return (y != 0.0f ? 256 : 0) + auc_bin(thr, p);
}

// one shared add per distinct key among the active lanes of the warp
__device__ __forceinline__ void auc_add(uint32_t* h, int key) {
  const unsigned peers = __match_any_sync(__activemask(), key);
  if ((peers & lanemask_lt()) == 0) atomicAdd(&h[key], (uint32_t)__popc(peers));
}

__global__ void __launch_bounds__(AUC_THREADS) auc_counts_kernel(const float* __restrict__ pred,
                                                                 const float* __restrict__ label, int64_t n,
                                                                 const float* __restrict__ thresholds,
                                                                 unsigned long long* __restrict__ counts) {
  __shared__ float s_thr[256];
  __shared__ uint32_t s_h[AUC_WARPS][AUC_KEYS];
  const int t = threadIdx.x, warp = t >> 5;
  s_thr[t] = t < AUC_N_THR ? thresholds[t] : __int_as_float(0x7f800000);
  for (int k = t; k < AUC_WARPS * AUC_KEYS; k += AUC_THREADS) (&s_h[0][0])[k] = 0;
  __syncthreads();
  uint32_t* h = s_h[warp];
  const float* thr = s_thr;
  const int64_t stride = (int64_t)gridDim.x * AUC_THREADS;
  const bool vec = ((reinterpret_cast<uintptr_t>(pred) | reinterpret_cast<uintptr_t>(label)) & 15) == 0;
  int64_t done = 0;
  if (vec) {
    const int64_t n4 = n >> 2;
    const float4* p4 = reinterpret_cast<const float4*>(pred);
    const float4* y4 = reinterpret_cast<const float4*>(label);
    for (int64_t i = (int64_t)blockIdx.x * AUC_THREADS + t; i < n4; i += stride) {
      const float4 p = __ldcs(p4 + i), y = __ldcs(y4 + i);
      const int k0 = auc_key(thr, p.x, y.x), k1 = auc_key(thr, p.y, y.y);
      const int k2 = auc_key(thr, p.z, y.z), k3 = auc_key(thr, p.w, y.w);
      auc_add(h, k0);
      auc_add(h, k1);
      auc_add(h, k2);
      auc_add(h, k3);
    }
    done = n4 << 2;
  }
  for (int64_t i = done + (int64_t)blockIdx.x * AUC_THREADS + t; i < n; i += stride)
    auc_add(h, auc_key(thr, __ldg(pred + i), __ldg(label + i)));
  __syncthreads();
  for (int k = t; k < AUC_KEYS; k += AUC_THREADS) {
    const int cls = k >> 8, bin = k & 255;
    if (bin >= AUC_BINS) continue;
    uint64_t s = 0;
#pragma unroll
    for (int w = 0; w < AUC_WARPS; ++w) s += s_h[w][k];
    if (s) atomicAdd(counts + cls * AUC_BINS + bin, (unsigned long long)s);
  }
}

// ---- "%f" of a float32 -------------------------------------------------------------------------------------------
// x = M * 2^E, M < 2^24.  E < 0: q = round-half-even((M * 10^6) / 2^-E), exact in 64 bits (M * 10^6 < 2^44); the
// integer part q / 10^6 < 2^25.  E >= 0: x is the integer M << E < 2^128, fraction .000000.  The integer part is held
// as five groups of nine decimal digits, least significant first.
constexpr int FMT_NAN = 1, FMT_INF = 2;
constexpr uint32_t E9 = 1000000000u;

struct Fixed6 {
  uint32_t g0, g1, g2, g3, g4;   // integer part, base 10^9 (scalars, not an array: no local memory)
  uint32_t frac;                 // the six fraction digits
  int ng;                        // groups in use (>= 1)
  int kind;                      // 0 finite, FMT_NAN, FMT_INF
  bool neg;
};

// w[3..0] (a 128-bit integer in 32-bit limbs) /= 10^9 -> the remainder
__device__ __forceinline__ uint32_t div_e9(uint32_t& w3, uint32_t& w2, uint32_t& w1, uint32_t& w0) {
  uint64_t cur = w3;
  w3 = (uint32_t)(cur / E9);
  cur = ((cur % E9) << 32) | w2;
  w2 = (uint32_t)(cur / E9);
  cur = ((cur % E9) << 32) | w1;
  w1 = (uint32_t)(cur / E9);
  cur = ((cur % E9) << 32) | w0;
  w0 = (uint32_t)(cur / E9);
  return (uint32_t)(cur % E9);
}

__device__ __forceinline__ Fixed6 fixed6(float x) {
  const uint32_t b = __float_as_uint(x);
  Fixed6 r;
  r.neg = (b >> 31) != 0;
  r.frac = 0;
  r.ng = 1;
  r.g0 = r.g1 = r.g2 = r.g3 = r.g4 = 0;
  const uint32_t e8 = (b >> 23) & 0xFF, m = b & 0x7FFFFF;
  if (e8 == 0xFF) {
    r.kind = m ? FMT_NAN : FMT_INF;
    return r;
  }
  r.kind = 0;
  const uint32_t M = e8 ? (m | 0x800000u) : m;
  const int E = e8 ? (int)e8 - 150 : -149;
  if (E < 0) {
    const int sh = -E;
    uint64_t q = 0;
    if (sh < 64) {   // a shift of 64 or more leaves < 2^-20: rounds to 0
      const uint64_t P = (uint64_t)M * 1000000ull;
      q = P >> sh;
      const uint64_t rem = P & ((1ull << sh) - 1), half = 1ull << (sh - 1);
      if (rem > half || (rem == half && (q & 1))) ++q;
    }
    r.frac = (uint32_t)(q % 1000000ull);
    r.g0 = (uint32_t)(q / 1000000ull);   // < 2^25 < 10^9
    return r;
  }
  // M << E in 32-bit limbs w3..w0
  const int ws = E >> 5;
  const uint64_t v = (uint64_t)M << (E & 31);
  const uint32_t lo = (uint32_t)v, hi = (uint32_t)(v >> 32);
  uint32_t w0 = ws == 0 ? lo : 0u;
  uint32_t w1 = ws == 1 ? lo : (ws == 0 ? hi : 0u);
  uint32_t w2 = ws == 2 ? lo : (ws == 1 ? hi : 0u);
  uint32_t w3 = ws == 3 ? lo : (ws == 2 ? hi : 0u);
  r.g0 = div_e9(w3, w2, w1, w0);
  r.g1 = div_e9(w3, w2, w1, w0);
  r.g2 = div_e9(w3, w2, w1, w0);
  r.g3 = div_e9(w3, w2, w1, w0);
  r.g4 = w0;   // M << E < 2^128 < 10^45: what is left is below 10^9
  r.ng = r.g4 ? 5 : r.g3 ? 4 : r.g2 ? 3 : r.g1 ? 2 : 1;
  return r;
}

__device__ __forceinline__ uint32_t fixed6_top(const Fixed6& f) {   // the most significant group
  return f.ng == 5 ? f.g4 : f.ng == 4 ? f.g3 : f.ng == 3 ? f.g2 : f.ng == 2 ? f.g1 : f.g0;
}

__device__ __forceinline__ int fixed6_len(const Fixed6& f) {
  if (f.kind == FMT_NAN) return 3;
  if (f.kind == FMT_INF) return 3 + f.neg;
  return (int)f.neg + 9 * (f.ng - 1) + dec_digits(fixed6_top(f)) + 7;
}

// writes the text at o[0, fixed6_len(f)) -> its length
__device__ __forceinline__ int fixed6_put(const Fixed6& f, char* o) {
  if (f.kind == FMT_NAN) { o[0] = 'n'; o[1] = 'a'; o[2] = 'n'; return 3; }
  int p = 0;
  if (f.neg) o[p++] = '-';
  if (f.kind == FMT_INF) { o[p] = 'i'; o[p + 1] = 'n'; o[p + 2] = 'f'; return p + 3; }
  p += put_dec<true>(fixed6_top(f), o + p);
  if (f.ng > 4) { put_dec(f.g3, o + p, 9); p += 9; }
  if (f.ng > 3) { put_dec(f.g2, o + p, 9); p += 9; }
  if (f.ng > 2) { put_dec(f.g1, o + p, 9); p += 9; }
  if (f.ng > 1) { put_dec(f.g0, o + p, 9); p += 9; }
  o[p++] = '.';
  put_dec(f.frac, o + p, 6);
  return p + 6;
}

constexpr int FMT_THREADS = 256;                  // one row per thread per sub-tile
constexpr int FMT_SUB = 8;                        // sub-tiles per tile
constexpr int FMT_TILE = FMT_THREADS * FMT_SUB;   // rows per tile (and per entry of the tile scan)
constexpr int FMT_ROW_MAX = 2 * 48;               // "%f\t%f\n" of two 47-character columns

__device__ __forceinline__ int row_len(const float* a, const float* b, int64_t r) {
  int len = fixed6_len(fixed6(__ldg(a + r))) + 1;
  if (b) len += fixed6_len(fixed6(__ldg(b + r))) + 1;
  return len;
}

__global__ void __launch_bounds__(FMT_THREADS) fmt_len_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                              int64_t n, int64_t* __restrict__ tile_len) {
  const int64_t base = (int64_t)blockIdx.x * FMT_TILE;
  int64_t v[1] = {0}, tot[1];
#pragma unroll 1
  for (int s = 0; s < FMT_SUB; ++s) {
    const int64_t r = base + s * FMT_THREADS + threadIdx.x;
    if (r < n) v[0] += row_len(a, b, r);
  }
  block_scan_excl<FMT_THREADS>(v, tot);
  if (threadIdx.x == 0) tile_len[blockIdx.x] = tot[0];
}

// out[d, d + len) = s[0, len), with 4-byte aligned word stores; bytes at or past out_bytes are not written
__device__ __forceinline__ void copy_out(const char* s, int len, char* out, int64_t d, int64_t out_bytes) {
  const int t = threadIdx.x;
  if (d + len > out_bytes) {
    for (int i = t; i < len; i += FMT_THREADS)
      if (d + i < out_bytes) out[d + i] = s[i];
    return;
  }
  const int head = min(len, (int)((4 - (reinterpret_cast<uintptr_t>(out + d) & 3)) & 3));
  const int words = (len - head) >> 2, tail = head + 4 * words;
  if (t < head) out[d + t] = s[t];
  uint32_t* o = reinterpret_cast<uint32_t*>(out + d + head);
  for (int i = t; i < words; i += FMT_THREADS) {
    const char* c = s + head + 4 * i;
    o[i] = (uint32_t)(uint8_t)c[0] | (uint32_t)(uint8_t)c[1] << 8 | (uint32_t)(uint8_t)c[2] << 16 |
           (uint32_t)(uint8_t)c[3] << 24;
  }
  if (t < len - tail) out[d + tail + t] = s[tail + t];
}

__global__ void __launch_bounds__(FMT_THREADS) fmt_write_kernel(const float* __restrict__ a,
                                                                const float* __restrict__ b, int64_t n,
                                                                const int64_t* __restrict__ tile_off,
                                                                const int64_t* __restrict__ offset,
                                                                char* __restrict__ out, int64_t out_bytes) {
  __shared__ char s_text[FMT_THREADS * FMT_ROW_MAX];
  const int t = threadIdx.x;
  const int64_t base = (int64_t)blockIdx.x * FMT_TILE;
  int64_t d = offset[0] + tile_off[blockIdx.x];
#pragma unroll 1
  for (int s = 0; s < FMT_SUB; ++s) {
    const int64_t r = base + s * FMT_THREADS + t;
    if (base + s * FMT_THREADS >= n) break;   // CTA-uniform
    int v[1] = {r < n ? row_len(a, b, r) : 0}, tot[1];
    block_scan_excl<FMT_THREADS>(v, tot);
    if (r < n) {   // decoded again rather than held across the scan
      char* o = s_text + v[0];
      int p = fixed6_put(fixed6(__ldg(a + r)), o);
      if (b) {
        o[p++] = '\t';
        p += fixed6_put(fixed6(__ldg(b + r)), o + p);
      }
      o[p] = '\n';
    }
    __syncthreads();
    copy_out(s_text, tot[0], out, d, out_bytes);
    d += tot[0];
    __syncthreads();
  }
}

__global__ void fmt_advance_kernel(int64_t* __restrict__ offset, const int64_t* __restrict__ total) {
  offset[0] += total[0];
}

struct FmtWs {   // int64 total, then int64 tile_len[tiles] (scanned in place into the tile offsets)
  int64_t* total;
  int64_t* tile;
  FmtWs(void* ws) : total(static_cast<int64_t*>(ws)), tile(static_cast<int64_t*>(ws) + 32) {}
};

}  // namespace
}  // namespace ctr

using namespace ctr;

extern "C" {

int ctr_auc_counts(const float* pred, const float* label, int64_t n, const float* thresholds, int64_t* counts,
                   ctr_stream_t stream) {
  CTR_REQUIRE(n >= 0 && n < (1ll << 40), CTR_ERR_INVALID_ARG, "ctr_auc_counts: n=%lld out of range [0, 2^40)",
              (long long)n);
  CTR_REQUIRE(thresholds && counts && (n == 0 || (pred && label)), CTR_ERR_INVALID_ARG,
              "ctr_auc_counts: null pointer");
  if (n == 0) return CTR_OK;
  auc_counts_kernel<<<grid_for(n, 4 * AUC_THREADS, 8), AUC_THREADS, 0, as_stream(stream)>>>(
      pred, label, n, thresholds, reinterpret_cast<unsigned long long*>(counts));
  CTR_LAUNCHED("ctr_auc_counts");
  return CTR_OK;
}

size_t ctr_format_preds_workspace_bytes(int64_t n) {
  const int64_t tiles = n > 0 ? ceil_div64(n, FMT_TILE) : 0;
  return align256((size_t)(32 + tiles) * sizeof(int64_t));
}

int ctr_format_preds(const float* a, const float* b, int64_t n, char* out, int64_t out_bytes, int64_t* offset,
                     void* ws, size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE(n >= 0 && n <= (1ll << 40), CTR_ERR_INVALID_ARG, "ctr_format_preds: n=%lld out of range [0, 2^40]",
              (long long)n);
  CTR_REQUIRE(offset && out_bytes >= 0 && (n == 0 || (a && out)), CTR_ERR_INVALID_ARG,
              "ctr_format_preds: bad arguments");
  CTR_REQUIRE(ws && ws_bytes >= ctr_format_preds_workspace_bytes(n), CTR_ERR_WORKSPACE,
              "ctr_format_preds: workspace too small");
  if (n == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  const FmtWs W(ws);
  const int64_t tiles = ceil_div64(n, FMT_TILE);
  CTR_REQUIRE(tiles < (1ll << 31), CTR_ERR_INVALID_ARG, "ctr_format_preds: too many rows");
  fmt_len_kernel<<<(unsigned)tiles, FMT_THREADS, 0, st>>>(a, b, n, W.tile);
  CTR_LAUNCHED("ctr_format_preds(lengths)");
  int64_t* const arr[1] = {W.tile};
  int64_t* const tot[1] = {W.total};
  if (int rc = cta_scan(arr, tot, nullptr, tiles, st, "ctr_format_preds(scan)")) return rc;
  fmt_write_kernel<<<(unsigned)tiles, FMT_THREADS, 0, st>>>(a, b, n, W.tile, offset, out, out_bytes);
  CTR_LAUNCHED("ctr_format_preds(write)");
  fmt_advance_kernel<<<1, 1, 0, st>>>(offset, W.total);
  CTR_LAUNCHED("ctr_format_preds(advance)");
  return CTR_OK;
}

}  // extern "C"
