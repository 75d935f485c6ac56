// decimal.cuh -- decimal numbers in device text: the fast decimal-to-fp32 path of the text tokenizers
// (libsvm_device.cu, csv_device.cu), the powers of ten behind it (also aliccp_tfrecord.cu's values), and parse_u63,
// the id grammar of the Ali-CCP kernels (aliccp_tfrecord.cu, aliccp_sample.cu).
//
// parse_float converts what it is sure about and hands everything else to the host parser: > 15 significant digits,
// |decimal exponent| > 22, inf/nan/hex, a result outside the normal fp32 range, or a double that sits within one ulp
// of an fp32 rounding boundary (fp32(RN_double(m / 10^k)) could then differ from the correctly rounded strtof by
// double rounding; about 6e-9 of all values).
// Inside the fast path the conversion is exact: m < 2^53 and 10^k (k <= 22) are exact doubles, one IEEE
// double division/multiplication gives the correctly rounded double, and away from an fp32 boundary
// rounding that double to fp32 equals rounding the exact decimal value.
// The table lives in an anonymous namespace so that every translation unit that includes this header owns its copy.
#pragma once
#include "common.cuh"

namespace ctr {
namespace {

__constant__ double kPow10[23] = {1e0,  1e1,  1e2,  1e3,  1e4,  1e5,  1e6,  1e7,  1e8,  1e9,  1e10, 1e11,
                                  1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};

enum { LS_OK = 0, LS_BAD = 1, LS_HOST = 2 };

// decimal float at p (no leading spaces): [+-]digits[.digits][(e|E)[+-]digits].  Returns LS_OK and advances p,
// LS_BAD if no number starts here, LS_HOST if the host's strtof has to decide.
__device__ __forceinline__ int parse_float(const unsigned char* __restrict__ t, int64_t& p, int64_t e, float& out) {
  int64_t q = p;
  bool neg = false;
  if (q < e && (t[q] == '+' || t[q] == '-')) { neg = t[q] == '-'; ++q; }
  uint64_t m = 0;
  int sig = 0, exp10 = 0, any = 0;
  bool dropped = false;
  while (q < e && t[q] >= '0' && t[q] <= '9') {
    any = 1;
    const int d = t[q] - '0';
    if (sig < 18) { if (sig || d) { m = m * 10 + d; ++sig; } }
    else { dropped = true; ++exp10; }
    ++q;
  }
  if (q < e && t[q] == '.') {
    ++q;
    while (q < e && t[q] >= '0' && t[q] <= '9') {
      any = 1;
      const int d = t[q] - '0';
      if (sig < 18) { if (sig || d) { m = m * 10 + d; ++sig; } --exp10; }
      else dropped = true;
      ++q;
    }
  }
  if (!any) {
    // "inf", "nan", "0x..." and friends are the host's business; anything else is not a number
    const unsigned char c = q < e ? t[q] : 0;
    return (c == 'i' || c == 'I' || c == 'n' || c == 'N') ? LS_HOST : LS_BAD;
  }
  if (q < e && (t[q] == 'e' || t[q] == 'E')) {
    int64_t r = q + 1;
    bool eneg = false;
    if (r < e && (t[r] == '+' || t[r] == '-')) { eneg = t[r] == '-'; ++r; }
    if (r < e && t[r] >= '0' && t[r] <= '9') {
      int ex = 0;
      while (r < e && t[r] >= '0' && t[r] <= '9') { if (ex < 10000) ex = ex * 10 + (t[r] - '0'); ++r; }
      exp10 += eneg ? -ex : ex;
      q = r;
    }  // else: "1e" / "1e+" -> strtof stops before the 'e'
  }
  if (q < e && (t[q] == 'x' || t[q] == 'X')) return LS_HOST;   // "0x1p3": hex float
  p = q;
  if (m == 0) { out = neg ? -0.0f : 0.0f; return LS_OK; }
  if (dropped || sig > 15 || exp10 < -22 || exp10 > 22) return LS_HOST;
  const double d = exp10 < 0 ? __ddiv_rn((double)m, kPow10[-exp10]) : __dmul_rn((double)m, kPow10[exp10]);
  if (!(d >= 1.1754943508222875e-38 && d <= 3.4028234663852886e38)) return LS_HOST;   // fp32 subnormal / overflow
  const uint64_t low = (uint64_t)__double_as_longlong(d) & 0x1FFFFFFFull;              // bits below the fp32 mantissa
  if (low >= 0x0FFFFFFFull && low <= 0x10000001ull) return LS_HOST;                     // next to a rounding boundary
  const float f = __double2float_rn(d);
  out = neg ? -f : f;
  return LS_OK;
}

// [0-9]+ below 2^63 -> true and its value.  One thread.
__device__ __forceinline__ bool parse_u63(const uint8_t* t, int64_t s, int64_t e, uint64_t& v) {
  v = 0;
  if (e <= s) return false;
  for (int64_t p = s; p < e; ++p) {
    const uint32_t c = byte_at(t, p);
    if (c < '0' || c > '9') return false;
    const uint64_t d = c - '0';
    if (v > (0x7FFFFFFFFFFFFFFFull - d) / 10) return false;
    v = v * 10 + d;
  }
  return true;
}

}  // namespace
}  // namespace ctr
