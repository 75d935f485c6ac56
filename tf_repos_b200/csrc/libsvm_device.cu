// libsvm_device.cu -- libsvm tokenizer on the GPU (SURVEY.md 8f-1; replaces decode_libsvm, DeepFM.py:65-81,
// when the text is already in device memory).
//
// Contract: whatever this path accepts, it converts to EXACTLY the bits the host parser (libsvm_host.cu:
// strtof / strtol) produces; everything it is not sure about is counted in `info` and the caller re-parses
// that chunk on the host (tf_repos_b200/input_fn.py does).  "Not sure" =
//   * a blank line, a malformed line, a pair count != F            (host parser owns the error messages)
//   * a number outside the fast decimal path (decimal.cuh::parse_float, which states what it declines and why the
//     conversion is exact inside it)
//
// Kernels: (1)-(3) line starts (line_starts.cuh); (4) one thread per line walks its bytes (adjacent threads
// read adjacent lines, so sectors are shared through L1).
#include "decimal.cuh"
#include "line_starts.cuh"

namespace ctr {

// one thread per line.  status[0] = blank lines, [1] = malformed lines, [2] = lines with a number for the host
__global__ void __launch_bounds__(128) ls_parse_kernel(const unsigned char* __restrict__ text, int64_t len,
                                                      const int64_t* __restrict__ line_start,
                                                      const int64_t* __restrict__ n_newlines, int64_t max_rows, int F,
                                                      int final_chunk, int32_t* __restrict__ ids, float* __restrict__ vals,
                                                      float* __restrict__ labels, int64_t* __restrict__ info) {
  const int64_t nn = n_newlines[0];
  const bool tail = final_chunk && len > 0 && text[len - 1] != '\n';
  int64_t n_lines = nn + (tail ? 1 : 0);
  if (n_lines > max_rows) n_lines = max_rows;
  const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (row == 0) {
    info[0] = n_lines;
    info[1] = n_lines == 0 ? 0 : ((n_lines <= nn) ? line_start[n_lines] : len);   // bytes consumed
  }
  if (row >= n_lines) return;
  int64_t p = line_start[row];
  int64_t e = (row < nn) ? line_start[row + 1] - 1 : len;     // exclusive end, '\n' dropped
  if (e > p && text[e - 1] == '\r') --e;
  while (p < e && text[p] == ' ') ++p;
  if (p == e) { atomicAdd(reinterpret_cast<unsigned long long*>(&info[2]), 1ull); return; }
  int st = LS_OK;
  float lab = 0.f;
  st |= parse_float(text, p, e, lab);
  int f = 0;
  int32_t* id_row = ids + row * F;
  float* val_row = vals + row * F;
  while (st == LS_OK) {
    if (p < e && text[p] != ' ') { st = LS_BAD; break; }      // a number must be followed by a space or the end
    while (p < e && text[p] == ' ') ++p;
    if (p >= e) break;
    if (f >= F) { st = LS_BAD; break; }
    // id: [+-]digits ':'   (strtol; more than 9 digits could overflow int32 -> host)
    bool neg = false;
    if (text[p] == '+' || text[p] == '-') { neg = text[p] == '-'; ++p; }
    int64_t v = 0;
    int nd = 0;
    while (p < e && text[p] >= '0' && text[p] <= '9') { if (nd < 12) v = v * 10 + (text[p] - '0'); ++nd; ++p; }
    if (nd == 0 || p >= e || text[p] != ':') { st = LS_BAD; break; }
    if (nd > 9) { st = LS_HOST; break; }
    ++p;
    if (p < e && (text[p] == ' ' || text[p] == '\t')) { st = LS_HOST; break; }   // strtof would skip the blank
    float val = 0.f;
    st |= parse_float(text, p, e, val);
    if (st != LS_OK) break;
    id_row[f] = (int32_t)(neg ? -v : v);
    val_row[f] = val;
    ++f;
  }
  if (st == LS_OK && f != F) st = LS_BAD;
  if (st & LS_BAD) atomicAdd(reinterpret_cast<unsigned long long*>(&info[3]), 1ull);
  else if (st & LS_HOST) atomicAdd(reinterpret_cast<unsigned long long*>(&info[4]), 1ull);
  else labels[row] = lab;
}

}  // namespace ctr

using namespace ctr;

extern "C" {

size_t ctr_parse_libsvm_device_workspace_bytes(size_t len, int64_t max_rows) {
  return LineStarts(nullptr, len, max_rows).bytes;
}

int ctr_parse_libsvm_device(const char* text, size_t len, int F, int64_t max_rows, int final_chunk, int32_t* ids,
                            float* vals, float* labels, int64_t* info, void* ws, size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE(F > 0 && max_rows >= 0 && info && (len == 0 || text), CTR_ERR_INVALID_ARG,
              "ctr_parse_libsvm_device: bad arguments");
  CTR_REQUIRE(len < ((size_t)1 << 32), CTR_ERR_INVALID_ARG, "ctr_parse_libsvm_device: buffer too large (len < 2^32)");
  CTR_REQUIRE(max_rows == 0 || (ids && vals && labels), CTR_ERR_INVALID_ARG, "ctr_parse_libsvm_device: null output");
  CTR_REQUIRE(ws && ws_bytes >= ctr_parse_libsvm_device_workspace_bytes(len, max_rows), CTR_ERR_WORKSPACE,
              "ctr_parse_libsvm_device: workspace too small");
  cudaStream_t st = as_stream(stream);
  CTR_REQUIRE(cudaMemsetAsync(info, 0, 5 * sizeof(int64_t), st) == cudaSuccess, CTR_ERR_CUDA,
              "ctr_parse_libsvm_device: memset failed");
  if (len == 0 || max_rows == 0) return CTR_OK;
  const unsigned char* t = reinterpret_cast<const unsigned char*>(text);
  const LineStarts L(ws, len, max_rows);
  if (int rc = L.launch(t, len, st, "ctr_parse_libsvm_device(lines)")) return rc;
  ls_parse_kernel<<<(unsigned)ceil_div64(max_rows, 128), 128, 0, st>>>(
      t, (int64_t)len, L.line_start, L.n_newlines, max_rows, F, final_chunk, ids, vals, labels, info);
  CTR_LAUNCHED("ctr_parse_libsvm_device(parse)");
  return CTR_OK;
}

}  // extern "C"
