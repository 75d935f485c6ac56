// example_wire.cuh -- the protobuf wire format of tf.Example as device code, and the one walk of Example -> Features ->
// map entries and the one Feature kind rule that the TFRecord reader, DIN serving (tfrecord_device.cu) and wide_n_deep
// serving (wd_serving.cu) share, so that all three agree byte for byte on what is well formed.  Both restate the host
// parser, tfrecord.parse_example / _parse_feature.  Warp-uniform: every lane calls them with the same arguments and
// gets the same result.  An anonymous namespace, so that every translation unit that includes this header owns its copy.
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

// Example -> Features -> map entries of [0, L), as the host parser reads them.  For each entry with a key:
// entry(match(ks, ke), fs, fe) -> ok, where match maps the key bytes [ks, ke) to the caller's key index (or -1) and
// [fs, fe) is the Feature (empty when the entry has no value field).  Entries come in order, so a caller that keeps the
// last entry of a key keeps the host's.  Every keyed entry reaches `entry`, schema key or not, because the host parses
// them all; an entry without a key is skipped unparsed; inside an entry the last key / value field wins.  Message
// fields must be length-delimited and a key must be UTF-8 (the host decodes every key).  false = malformed.  The
// __syncwarps publish to the whole warp what the caller wrote before and what `entry` writes.
template <class Match, class Entry>
__device__ __forceinline__ bool tr_map_entries(const uint8_t* d, int L, Match match, Entry entry) {
  __syncwarp();
  bool ok = true;
  for (int p = 0; p < L && ok;) {
    TrField f;
    p = tr_field(d, p, L, f);
    if (p < 0) { ok = false; break; }
    if (f.num != 1) continue;
    if (f.wt != 2) { ok = false; break; }
    for (int q = f.vs; q < f.ve;) {            // Features: map entries
      TrField g;
      q = tr_field(d, q, f.ve, g);
      if (q < 0 || (g.num == 1 && g.wt != 2)) { ok = false; break; }
      if (g.num != 1) continue;
      int ks = -1, ke = 0, fs = 0, fe = 0;     // no value field = an empty Feature
      for (int r = g.vs; r < g.ve;) {
        TrField h;
        r = tr_field(d, r, g.ve, h);
        if (r < 0 || ((h.num == 1 || h.num == 2) && h.wt != 2)) { ok = false; break; }
        if (h.num == 1) { ks = h.vs; ke = h.ve; }
        if (h.num == 2) { fs = h.vs; fe = h.ve; }
      }
      if (!ok) break;
      if (ks < 0) continue;                    // an entry without a key is skipped unparsed
      bool high = false;
      for (int i = ks + (threadIdx.x & 31); i < ke; i += 32) high |= tr_byte(d, i) >= 0x80;
      const int key = match(ks, ke);           // between the loads of the UTF-8 gate and its vote: they overlap
      if ((__any_sync(FULL_MASK, high) && !tr_utf8(d, ks, ke)) || !entry(key, fs, fe)) { ok = false; break; }
    }
  }
  __syncwarp();
  return ok;
}

// a Feature message [s, e) read as tfrecord._parse_feature does: its first field numbered 1..3 sets r.kind (1 bytes,
// 2 float, 3 int64) and must be length-delimited; its payload, the list message, goes to list(ls, le) -> ok with
// r.kind already set.  Later kind fields only set r.multi.  r.kind = 0 when there is none.  false = malformed.
template <class Slot, class List>
__device__ __forceinline__ bool tr_feature_kind(const uint8_t* d, int s, int e, Slot& r, List list) {
  r.kind = 0; r.multi = false;
  for (int p = s; p < e;) {
    TrField f;
    p = tr_field(d, p, e, f);
    if (p < 0) return false;
    if (f.num < 1 || f.num > 3) continue;
    if (r.kind != 0) { r.multi = true; continue; }
    if (f.wt != 2) return false;
    r.kind = f.num;
    if (!list(f.vs, f.ve)) return false;
  }
  return true;
}

}  // namespace
}  // namespace ctr
