// csv_device.cu -- wide_n_deep's CSV tokenizer on the GPU (replaces the tf.decode_csv of input_fn,
// wide_n_deep.py:55-73, when the text is already in device memory).
//
// tf.decode_csv(line, record_defaults=[[0.0]] + 13*[[0.0]] + 26*[[0]]): n_float float columns (the first is the
// label) then n_int int columns, split on ','; an empty field takes its default (0.0 / 0).
//
// Contract: whatever this path accepts has EXACTLY the bits the host decoder (wide_deep_main.decode_csv_file: Python
// float() / int(), then a NumPy cast to fp32 / int32) produces; everything it is not sure about is counted in `info`
// and the caller re-parses that piece on the host, which owns every error message.  "Not sure" =
//   * a blank line (the host decoder skips it, which would shift the rows)
//   * a malformed line: a field count != n_float + n_int, or a '"', a blank or a tab anywhere in it
//   * a number for the host: a float outside the fast decimal path (decimal.cuh::parse_float) or one that does not
//     end at the end of its field; an int that is not [+-]?[0-9]{1,9}
// Any other byte in a field (a lone '\r', '_', a letter, a non-ASCII byte) fails one of the two number rules, so a
// line the kernel accepts is made of the characters of plain decimal numbers and ',' only.
//
// Why parse_float, written against strtof, is exact against this decoder too: inside the fast path the double
// d = m / 10^k (or m * 10^k) is ONE IEEE operation on exact operands, hence the correctly rounded double of the
// decimal -- which is what Python's float() returns -- and both sides then round that same d to fp32 (NumPy's cast
// and __double2float_rn are both round-to-nearest-even).  The guard band around fp32 rounding boundaries, which
// strtof's single rounding needs, only declines a few values more here.  "-0" is -0.0 on both sides.
//
// Ids are written as parsed: the identity column's out-of-range -> 0 rule stays in the feature-column kernel
// (wide_deep.cu).
//
// Kernels: (1)-(3) line starts (line_starts.cuh); (4) one thread per line walks its bytes (adjacent threads
// read adjacent lines, so sectors are shared through L1).
#include "decimal.cuh"
#include "line_starts.cuh"

namespace ctr {

// one thread per line.  info[2] = blank lines, [3] = malformed lines, [4] = lines with a number for the host
__global__ void __launch_bounds__(128) csv_parse_kernel(const unsigned char* __restrict__ text, int64_t len,
                                                       const int64_t* __restrict__ line_start,
                                                       const int64_t* __restrict__ n_newlines, int64_t max_rows,
                                                       int n_float, int n_int, int final_chunk,
                                                       float* __restrict__ labels, float* __restrict__ dense,
                                                       int32_t* __restrict__ cat, int64_t* __restrict__ info) {
  const int64_t nn = n_newlines[0];
  const int64_t n_lines = final_chunk ? chunk_lines(text, len, nn, max_rows) : (nn < max_rows ? nn : max_rows);
  const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (row == 0) {
    info[0] = n_lines;
    info[1] = n_lines == 0 ? 0 : ((n_lines <= nn) ? line_start[n_lines] : len);   // bytes consumed
  }
  if (row >= n_lines) return;
  int64_t p, e;
  line_bounds(line_start, nn, len, row, p, e);
  if (e > p && text[e - 1] == '\r') --e;
  if (p == e) { atomicAdd(reinterpret_cast<unsigned long long*>(&info[2]), 1ull); return; }
  const int64_t p0 = p;
  const int n_fields = n_float + n_int;
  float* dense_row = dense + row * (n_float - 1);
  int32_t* cat_row = cat + row * n_int;
  int st = LS_OK;
  for (int f = 0; f < n_fields; ++f) {
    if (f) {
      if (p >= e || text[p] != ',') { st = LS_BAD; break; }     // the previous field must end here
      ++p;
    }
    const bool empty = p >= e || text[p] == ',';
    if (f < n_float) {
      float v = 0.f;
      if (!empty && (st = parse_float(text, p, e, v)) != LS_OK) break;
      if (f == 0) labels[row] = v;
      else dense_row[f - 1] = v;
    } else {
      int32_t v = 0;
      if (!empty) {
        bool neg = false;
        if (text[p] == '+' || text[p] == '-') { neg = text[p] == '-'; ++p; }
        int nd = 0;
        while (p < e && text[p] >= '0' && text[p] <= '9') { if (nd < 9) v = v * 10 + (text[p] - '0'); ++nd; ++p; }
        if (nd == 0 || nd > 9) { st = LS_HOST; break; }         // more than 9 digits could overflow int32
        if (neg) v = -v;
      }
      cat_row[f - n_float] = v;
    }
  }
  if (st == LS_OK && p == e) return;
  // declined: malformed (field count, quote, blank, tab) or a number only the host decoder may decide
  int commas = 0;
  bool odd = false;
  for (int64_t q = p0; q < e; ++q) {
    const unsigned char c = text[q];
    commas += c == ',';
    odd |= c == '"' || c == ' ' || c == '\t';
  }
  const int slot = (odd || commas != n_fields - 1) ? 3 : 4;
  atomicAdd(reinterpret_cast<unsigned long long*>(&info[slot]), 1ull);
}

}  // namespace ctr

using namespace ctr;

extern "C" {

size_t ctr_parse_csv_device_workspace_bytes(size_t len, int64_t max_rows) {
  return LineStarts(nullptr, len, max_rows).bytes;
}

int ctr_parse_csv_device(const char* text, size_t len, int n_float, int n_int, int64_t max_rows, int final_chunk,
                         float* labels, float* dense, int32_t* cat, int64_t* info, void* ws, size_t ws_bytes,
                         ctr_stream_t stream) {
  CTR_REQUIRE(n_float >= 1 && n_int >= 0 && max_rows >= 0 && info && (len == 0 || text), CTR_ERR_INVALID_ARG,
              "ctr_parse_csv_device: bad arguments");
  CTR_REQUIRE(len < ((size_t)1 << 32), CTR_ERR_INVALID_ARG, "ctr_parse_csv_device: buffer too large (len < 2^32)");
  CTR_REQUIRE(max_rows == 0 || (labels && (dense || n_float == 1) && (cat || n_int == 0)), CTR_ERR_INVALID_ARG,
              "ctr_parse_csv_device: null output");
  CTR_REQUIRE(ws && ws_bytes >= ctr_parse_csv_device_workspace_bytes(len, max_rows), CTR_ERR_WORKSPACE,
              "ctr_parse_csv_device: workspace too small");
  cudaStream_t st = as_stream(stream);
  CTR_REQUIRE(cudaMemsetAsync(info, 0, 5 * sizeof(int64_t), st) == cudaSuccess, CTR_ERR_CUDA,
              "ctr_parse_csv_device: memset failed");
  if (len == 0 || max_rows == 0) return CTR_OK;
  const unsigned char* t = reinterpret_cast<const unsigned char*>(text);
  const LineStarts L(ws, len, max_rows);
  if (int rc = L.launch(t, len, st, "ctr_parse_csv_device(lines)")) return rc;
  csv_parse_kernel<<<(unsigned)ceil_div64(max_rows, 128), 128, 0, st>>>(
      t, (int64_t)len, L.line_start, L.n_newlines, max_rows, n_float, n_int, final_chunk, labels, dense, cat, info);
  CTR_LAUNCHED("ctr_parse_csv_device(parse)");
  return CTR_OK;
}

}  // extern "C"
