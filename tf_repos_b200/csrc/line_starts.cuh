// line_starts.cuh -- line starts of a text buffer in device memory, and the warp-per-line splitting, shared by the
// tokenizers (libsvm_device.cu, csv_device.cu, criteo_feature.cu, aliccp_tfrecord.cu, aliccp_sample.cu,
// smart_feature.cu).
//
// Kernels: (1) count '\n' per 4 KB block; (2) scan the block counts (cta_scan_kernel); (3) emit line starts.
// LineStarts is their workspace and launches them; line_bounds / chunk_lines read the result in the per-line kernels.
// A kernel that gives each line a warp reads it in windows of 32 bytes: warp_strip is line.strip(), warp_seps the
// first separators of a line (its fields), warp_split its tokens.
// They live in an anonymous namespace so that every translation unit that includes this header owns its copy.
#pragma once
#include "common.cuh"
#include "scan_sort.cuh"

namespace ctr {
namespace {

constexpr int LS_THREADS = 256, LS_BYTES_PER_THREAD = 16, LS_BLOCK_BYTES = LS_THREADS * LS_BYTES_PER_THREAD;

__device__ __forceinline__ int count_nl16(const unsigned char* __restrict__ t, int64_t pos, int64_t len, uint32_t& mask) {
  mask = 0;
  if (pos + 16 <= len && ((reinterpret_cast<uintptr_t>(t + pos) & 15) == 0)) {
    const uint4 w = __ldg(reinterpret_cast<const uint4*>(t + pos));
    const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
#pragma unroll
      for (int b = 0; b < 4; ++b)
        if (((ws[k] >> (8 * b)) & 0xFFu) == '\n') mask |= 1u << (4 * k + b);
    }
  } else {
    for (int b = 0; b < 16; ++b)
      if (pos + b < len && t[pos + b] == '\n') mask |= 1u << b;
  }
  return __popc(mask);
}

__global__ void __launch_bounds__(LS_THREADS) ls_count_kernel(const unsigned char* __restrict__ text, int64_t len,
                                                             int32_t* __restrict__ block_counts) {
  __shared__ int warp_tot[LS_THREADS / 32];
  const int64_t pos = ((int64_t)blockIdx.x * LS_THREADS + threadIdx.x) * LS_BYTES_PER_THREAD;
  uint32_t mask;
  int c = pos < len ? count_nl16(text, pos, len, mask) : 0;
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(FULL_MASK, c, o);
  if ((threadIdx.x & 31) == 0) warp_tot[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int w = 0; w < LS_THREADS / 32; ++w) s += warp_tot[w];
    block_counts[blockIdx.x] = s;
  }
}

// line_start[k+1] = position just after the k-th '\n' (k < max_rows); line_start[0] = 0
__global__ void __launch_bounds__(LS_THREADS) ls_emit_kernel(const unsigned char* __restrict__ text, int64_t len,
                                                            const int32_t* __restrict__ block_offsets, int64_t max_rows,
                                                            int64_t* __restrict__ line_start) {
  const int64_t pos = ((int64_t)blockIdx.x * LS_THREADS + threadIdx.x) * LS_BYTES_PER_THREAD;
  uint32_t mask = 0;
  int before[1] = {pos < len ? count_nl16(text, pos, len, mask) : 0}, tot[1];
  block_scan_excl<LS_THREADS>(before, tot);
  int64_t k = (int64_t)block_offsets[blockIdx.x] + before[0];
  if (blockIdx.x == 0 && threadIdx.x == 0) line_start[0] = 0;
  while (mask) {
    const int b = __ffs(mask) - 1;
    mask &= mask - 1;
    if (k < max_rows) line_start[k + 1] = pos + b + 1;
    ++k;
  }
}

// line `row` of the chunk: [p, e), '\n' dropped (the last line of the chunk may have none)
__device__ __forceinline__ void line_bounds(const int64_t* line_start, int64_t nn, int64_t len, int64_t row,
                                            int64_t& p, int64_t& e) {
  p = line_start[row];
  e = row < nn ? line_start[row + 1] - 1 : len;
}

// lines of the chunk, nn = its '\n' count: an unterminated last line counts; at most cap
__device__ __forceinline__ int64_t chunk_lines(const uint8_t* __restrict__ t, int64_t len, int64_t nn,
                                               int64_t cap = INT64_MAX) {
  const int64_t n = nn + ((len > 0 && t[len - 1] != '\n') ? 1 : 0);
  return n < cap ? n : cap;
}

// ---- one warp per line: the line's bytes in windows of 32, one byte a lane, read by ballots ----

// line.strip() of [p, e) -> [s, te); s = te = e for a blank line.  Warp-uniform.
__device__ __forceinline__ void warp_strip(const uint8_t* t, int64_t p, int64_t e, int64_t& s, int64_t& te) {
  const int lane = lane_id();
  s = e; te = e;
  for (int64_t w = p; w < e; w += 32) {
    const int64_t q = w + lane;
    const unsigned m = __ballot_sync(FULL_MASK, q < e && !is_py_space(byte_at(t, q)));
    if (m) { s = w + __ffs(m) - 1; break; }
  }
  if (s == e) return;
  for (int64_t w = e; w > s; w -= 32) {
    const int64_t q = w - 32 + lane;
    const unsigned m = __ballot_sync(FULL_MASK, q >= s && !is_py_space(byte_at(t, q)));
    if (m) { te = w - 32 + (31 - __clz(m)) + 1; break; }
  }
}

// pos[n] = v for n < MAX, as a chain of constant indices so that pos stays in registers
template <int K = 0, int MAX>
__device__ __forceinline__ void seps_put(int64_t (&pos)[MAX], int n, int64_t v) {
  if (n == K) pos[K] = v;
  if constexpr (K + 1 < MAX) seps_put<K + 1>(pos, n, v);
}

// The first MAX bytes sep of [s, te) -> pos, nul = [s, te) holds a NUL byte (within the windows read); -> their count,
// MAX + 1 = more than MAX.  The walk stops at the window of separator MAX + 1.  Warp-uniform.
template <int MAX>
__device__ __forceinline__ int warp_seps(const uint8_t* t, int64_t s, int64_t te, uint32_t sep, int64_t (&pos)[MAX],
                                         bool& nul) {
  const int lane = lane_id();
  int n = 0;
  nul = false;
  for (int64_t w = s; w < te && n <= MAX; w += 32) {
    const int64_t q = w + lane;
    const uint32_t b = q < te ? byte_at(t, q) : 1u;
    unsigned m = __ballot_sync(FULL_MASK, b == sep);
    nul |= __ballot_sync(FULL_MASK, b == 0) != 0;
    while (m && n <= MAX) {
      const int c = __ffs(m) - 1;
      m &= m - 1;
      seps_put(pos, n, w + c);
      ++n;
    }
  }
  return n;
}

// [s, e) split at the bytes where is_sep(byte) holds, in windows of 32 bytes: visit(end, start, q, mask) once per
// window (warp-uniform), mask = the window's ballot of ends; lanes with `end` set end the token [start, q), the last
// one at q = e.
template <class IsSep, class Visit>
__device__ __forceinline__ void warp_split(const uint8_t* t, int64_t s, int64_t e, IsSep&& is_sep, Visit&& visit) {
  const int lane = lane_id();
  int64_t carry = s - 1;
  for (int64_t w = s; w <= e; w += 32) {
    const int64_t q = w + lane;
    const bool end = q <= e && (q == e || is_sep(byte_at(t, q)));
    const unsigned m = __ballot_sync(FULL_MASK, end);
    const unsigned below = m & lanemask_lt();
    visit(end, (below ? w + 31 - __clz(below) : carry) + 1, q, m);
    if (m) carry = w + 31 - __clz(m);
  }
}

// Workspace of a chunk of len bytes: block_counts int32[nb] | n_newlines int64[2] | line_start int64[max_rows + 1],
// each 256-B aligned; bytes = its end, where a caller's own arrays may follow.
struct LineStarts {
  int32_t* block_counts;
  int64_t *n_newlines, *line_start;
  int64_t max_rows;
  int n_blocks;
  size_t bytes;
  LineStarts(void* ws, size_t len, int64_t rows) : max_rows(rows) {
    uint8_t* b = reinterpret_cast<uint8_t*>(ws);
    n_blocks = (int)((len + LS_BLOCK_BYTES - 1) / LS_BLOCK_BYTES);
    size_t o = 0;
    block_counts = reinterpret_cast<int32_t*>(b + o); o += align256((size_t)n_blocks * 4);
    n_newlines = reinterpret_cast<int64_t*>(b + o); o += align256(16);
    line_start = reinterpret_cast<int64_t*>(b + o); o += align256((size_t)(max_rows + 1) * 8);
    bytes = o;
  }

  // n_newlines[0] = the '\n' count of text[0, len); line_start[0] = 0 and line_start[k + 1] = the position after the
  // k-th '\n' for k < max_rows
  int launch(const uint8_t* t, size_t len, cudaStream_t st, const char* what) const {
    ls_count_kernel<<<n_blocks, LS_THREADS, 0, st>>>(t, (int64_t)len, block_counts);
    CTR_LAUNCHED(what);
    if (int rc = cta_scan({block_counts}, {n_newlines}, nullptr, n_blocks, st, what)) return rc;
    ls_emit_kernel<<<n_blocks, LS_THREADS, 0, st>>>(t, (int64_t)len, block_counts, max_rows, line_start);
    CTR_LAUNCHED(what);
    return CTR_OK;
  }
};

}  // namespace
}  // namespace ctr
