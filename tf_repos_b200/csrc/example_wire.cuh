// example_wire.cuh -- the protobuf wire format of tf.Example as device code: the TFRecord reader (tfrecord_device.cu)
// and the wide_n_deep serving parser (wd_serving.cu) walk Example -> Features -> map entries with these.
// Warp-uniform: every lane calls them with the same arguments and gets the same result.  An anonymous namespace, so
// that every translation unit that includes this header owns its copy.
#pragma once
#include "common.cuh"

namespace ctr {
namespace {

__device__ __forceinline__ uint32_t tr_byte(const uint8_t* d, int64_t p) { return __ldg(d + p); }
__device__ __forceinline__ uint32_t tr_u32(const uint8_t* d, int64_t p) {
  return tr_byte(d, p) | tr_byte(d, p + 1) << 8 | tr_byte(d, p + 2) << 16 | tr_byte(d, p + 3) << 24;
}
__device__ __forceinline__ float tr_float(uint32_t bits) {   // float -> Python float -> float32 quiets a signalling NaN
  if ((bits & 0x7FFFFFFFu) > 0x7F800000u) bits |= 0x00400000u;
  return __uint_as_float(bits);
}

// -> the position after the varint, or -1 when it runs past e, is longer than 10 bytes or is >= 2^64
__device__ __forceinline__ int tr_varint(const uint8_t* d, int p, int e, uint64_t& v) {
  v = 0;
  for (int i = 0; i < 10; ++i) {
    if (p >= e) return -1;
    const uint32_t b = tr_byte(d, p++);
    if (i == 9 && b > 1) return -1;
    v |= (uint64_t)(b & 0x7F) << (7 * i);
    if (!(b & 0x80)) return p;
  }
  return -1;
}

struct TrField {
  int num, wt, vs, ve;   // payload [vs, ve) of wire types 1, 2, 5
  uint64_t v;            // value of wire type 0
};

// one field of the message [p, e) -> the position after it, or -1 (bad varint, wire type 3/4/6/7, payload past e)
__device__ __forceinline__ int tr_field(const uint8_t* d, int p, int e, TrField& f) {
  uint64_t key;
  p = tr_varint(d, p, e, key);
  if (p < 0) return -1;
  f.wt = (int)(key & 7);
  f.num = (key >> 3) > 0x7FFFFFFFull ? 0x7FFFFFFF : (int)(key >> 3);
  f.vs = f.ve = p;
  switch (f.wt) {
    case 0: return tr_varint(d, p, e, f.v);
    case 1: if (e - p < 8) return -1; f.ve = p + 8; return f.ve;
    case 5: if (e - p < 4) return -1; f.ve = p + 4; return f.ve;
    case 2: {
      uint64_t ln;
      p = tr_varint(d, p, e, ln);
      if (p < 0 || ln > (uint64_t)(e - p)) return -1;
      f.vs = p; f.ve = p + (int)ln;
      return f.ve;
    }
    default: return -1;
  }
}

// strict UTF-8 (what bytes.decode("utf-8") accepts)
__device__ bool tr_utf8(const uint8_t* d, int s, int e) {
  for (int p = s; p < e;) {
    const uint32_t c = tr_byte(d, p);
    if (c < 0x80) { ++p; continue; }
    int n;
    uint32_t lo = 0x80, hi = 0xBF;
    if (c >= 0xC2 && c <= 0xDF) {
      n = 1;
    } else if (c >= 0xE0 && c <= 0xEF) {
      n = 2; if (c == 0xE0) lo = 0xA0; if (c == 0xED) hi = 0x9F;
    } else if (c >= 0xF0 && c <= 0xF4) {
      n = 3; if (c == 0xF0) lo = 0x90; if (c == 0xF4) hi = 0x8F;
    } else {
      return false;
    }
    if (e - p - 1 < n) return false;
    const uint32_t c1 = tr_byte(d, p + 1);
    if (c1 < lo || c1 > hi) return false;
    for (int k = 2; k <= n; ++k)
      if ((tr_byte(d, p + k) & 0xC0) != 0x80) return false;
    p += n + 1;
  }
  return true;
}

}  // namespace
}  // namespace ctr
