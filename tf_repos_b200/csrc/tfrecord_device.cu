// tfrecord_device.cu -- DIN / ESMM TFRecord input on the GPU (DIN.py:57-99, DeepCvrMTL.py:63-105; DESIGN.md §2.5).
//
// Two passes over records the host has framed (ctr_tfrecord_frame, tfrecord_host.cu):
//   scan  one warp per record: masked CRC-32C of the data, then a walk of Example -> Features -> map entries that keeps
//         the last occurrence of each schema key, counts the values of every Feature, checks the protobuf is well
//         formed and runs the checks of din_main.decode_tfrecord_files in its order.  Writes the five bag lengths of
//         the record and folds one error word (smallest = the error the host decoder meets first).
//   emit  one warp per batch slot over a staging buffer of whole records: the same walk, then every value of the keys
//         the model reads is written where din_main.make_batch / esmm_main.make_batch puts it.
// The walk is warp-uniform (every lane parses the same bytes, so control flow never diverges); the per-byte work --
// the CRC, the varint terminators of packed Int64Lists, the float copies -- is spread over the lanes.  Nothing is
// reduced with atomics except the error word, so two runs write the same bits.
//
// Host semantics kept bit for bit (tfrecord.parse_example / _parse_feature):
//   the last map entry of a key wins; inside an entry the last key / value field wins; a Feature's kind is its first
//   field numbered 1..3; a list's values are its field-1 runs, packed (wire type 2) or not (varint / fixed32), in order;
//   an int64 id keeps its low 32 bits; a float keeps its bits except that a signalling NaN comes out quiet (the host
//   goes through a Python float).
// Error word (uint64, ~0 = none): (record << 16) | (check << 8) | arg, with check in the host's order:
//   0 data CRC | 1 malformed protobuf | 2 required key missing or empty (arg = key) | 3 feat_ids count |
//   4 u_*ids / u_*vals lengths differ (arg = field) | 5 wrong or several Feature kinds (arg = key) |
//   6 id outside [0, 2^31) (arg = key)
#include "common.cuh"

namespace ctr {

constexpr int TR_KEYS = 15;
constexpr int TR_THREADS = 256, TR_WARPS = TR_THREADS / 32;
constexpr uint32_t TR_POLY = 0x82F63B78u;  // CRC-32C, reflected
constexpr int TR_ALL = 0x7FFFFFFF;
enum { TK_Y = 0, TK_Z = 1, TK_FEAT = 2, TK_ACAT = 3, TK_AINT = 6, TK_UIDS = 7, TK_UVALS = 11 };
enum { TE_CRC = 0, TE_MALFORMED = 1, TE_REQUIRED = 2, TE_COUNT = 3, TE_MISMATCH = 4, TE_KIND = 5, TE_RANGE = 6 };
enum { KIND_NONE = 0, KIND_BYTES = 1, KIND_FLOAT = 2, KIND_INT = 3 };

__device__ const char kTrKey[TR_KEYS][12] = {"y",         "z",         "feat_ids",  "a_catids",   "a_shopids",
                                             "a_brandids", "a_intids",  "u_catids",  "u_shopids",  "u_brandids",
                                             "u_intids",  "u_catvals", "u_shopvals", "u_brandvals", "u_intvals"};
__device__ const int kTrKeyLen[TR_KEYS] = {1, 1, 8, 8, 9, 10, 8, 8, 9, 10, 8, 9, 10, 11, 9};
__device__ const int kTrKeyKind[TR_KEYS] = {2, 2, 3, 3, 3, 3, 3, 3, 3, 3, 3, 2, 2, 2, 2};

__device__ __forceinline__ int tr_lane() { return threadIdx.x & 31; }
__device__ __forceinline__ uint32_t tr_byte(const uint8_t* d, int64_t p) { return __ldg(d + p); }
__device__ __forceinline__ uint32_t tr_u32(const uint8_t* d, int64_t p) {
  return tr_byte(d, p) | tr_byte(d, p + 1) << 8 | tr_byte(d, p + 2) << 16 | tr_byte(d, p + 3) << 24;
}
__device__ __forceinline__ float tr_float(uint32_t bits) {   // float -> Python float -> float32 quiets a signalling NaN
  if ((bits & 0x7FFFFFFFu) > 0x7F800000u) bits |= 0x00400000u;
  return __uint_as_float(bits);
}

// ---- CRC-32C: each lane CRCs 1/32 of the record, the 32 remainders are combined with x^(8n) mod P ---------------
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
// constant per level.
__device__ uint32_t tr_crc32c(const uint8_t* d, int64_t L, const uint32_t* tab, const uint32_t* x8) {
  const int lane = tr_lane();
  const int64_t seg = (L + 31) >> 5, z = 32 * seg - L;
  int64_t lo = lane * seg - z, hi = lo + seg;
  lo = lo < 0 ? 0 : lo;
  uint32_t c = 0;
  for (int64_t p = lo; p < hi; ++p) c = tab[(c ^ tr_byte(d, p)) & 0xFF] ^ (c >> 8);
  uint32_t M = gf_x8n(x8, (uint64_t)seg);
  for (int k = 1; k < 32; k <<= 1) {
    const uint32_t partner = __shfl_down_sync(FULL_MASK, c, k);
    if ((lane & (2 * k - 1)) == 0) c = gf_mul(c, M) ^ partner;
    M = gf_mul(M, M);
  }
  c = __shfl_sync(FULL_MASK, c, 0);
  return c ^ gf_mul(0xFFFFFFFFu, gf_x8n(x8, (uint64_t)L)) ^ 0xFFFFFFFFu;
}

// ---- protobuf wire format (warp-uniform: every lane calls these with the same arguments) -------------------------
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

struct TrFeat {
  int kind, count;
  bool multi, range_bad;
};

// A packed Int64List run [s, e) whose first value is value number `base` of the list, decoded 32 bytes per step:
// a ballot of the terminators gives every varint's index (prefix popcount) and its start (the terminator before it);
// each terminating lane assembles its value.  Value i < range_n must lie in [0, 2^31) (else range_bad); value i < limit
// is written to out[i].  -> values in the run, or -1 when a varint is unterminated, > 10 bytes or >= 2^64.
__device__ int tr_packed_ints(const uint8_t* d, int s, int e, int base, int range_n, int32_t* out, int limit,
                              bool& range_bad) {
  const int lane = tr_lane();
  const unsigned below_mask = (1u << lane) - 1;
  int count = 0, carry = s - 1;
  bool bad = false, rbad = false;
  for (int w = s; w < e; w += 32) {
    const int p = w + lane;
    const uint32_t b = p < e ? tr_byte(d, p) : 0x80u;
    const bool term = !(b & 0x80);
    const unsigned m = __ballot_sync(FULL_MASK, term);
    if (term) {
      const unsigned below = m & below_mask;
      const int prev = below ? w + 31 - __clz(below) : carry;
      const int n = p - prev;
      if (n > 10 || (n == 10 && b > 1)) {
        bad = true;
      } else {
        uint64_t v = 0;
        for (int k = 0; k < n; ++k) v |= (uint64_t)(tr_byte(d, prev + 1 + k) & 0x7F) << (7 * k);
        const int i = base + count + __popc(below);
        if (i < range_n && (v >> 31)) rbad = true;
        if (out && i < limit) out[i] = (int32_t)(uint32_t)v;
      }
    }
    count += __popc(m);
    if (m) carry = w + 31 - __clz(m);
  }
  if (e > s && carry != e - 1) bad = true;
  if (__any_sync(FULL_MASK, rbad)) range_bad = true;
  return __any_sync(FULL_MASK, bad) ? -1 : count;
}

// the field-1 runs of a BytesList / FloatList / Int64List [s, e) of kind r.kind, appended to r.count
__device__ bool tr_list(const uint8_t* d, int s, int e, TrFeat& r, void* out, int limit, int range_n) {
  const int lane = tr_lane();
  for (int p = s; p < e;) {
    TrField f;
    p = tr_field(d, p, e, f);
    if (p < 0) return false;
    if (f.num != 1) continue;
    if (r.kind == KIND_BYTES) {
      ++r.count;
    } else if (r.kind == KIND_FLOAT) {
      float* o = static_cast<float*>(out);
      if (f.wt == 2) {
        if ((f.ve - f.vs) & 3) return false;   // np.frombuffer raises
        const int n = (f.ve - f.vs) >> 2;
        if (o)
          for (int i = lane; i < n && r.count + i < limit; i += 32) o[r.count + i] = tr_float(tr_u32(d, f.vs + 4 * i));
        r.count += n;
      } else if (f.wt == 5) {
        if (o && lane == 0 && r.count < limit) o[r.count] = tr_float(tr_u32(d, f.vs));
        ++r.count;
      }
    } else {
      int32_t* o = static_cast<int32_t*>(out);
      if (f.wt == 2) {
        const int n = tr_packed_ints(d, f.vs, f.ve, r.count, range_n, o, limit, r.range_bad);
        if (n < 0) return false;
        r.count += n;
      } else if (f.wt == 0) {
        if (r.count < range_n && (f.v >> 31)) r.range_bad = true;
        if (o && lane == 0 && r.count < limit) o[r.count] = (int32_t)(uint32_t)f.v;
        ++r.count;
      }
    }
  }
  return true;
}

// a Feature message [s, e) read as tfrecord._parse_feature does: its first field numbered 1..3 sets the kind and the
// values; later kind fields only set `multi`.  false = malformed.
__device__ bool tr_feature(const uint8_t* d, int s, int e, TrFeat& r, void* out, int limit, int range_n) {
  r.kind = KIND_NONE; r.count = 0; r.multi = false; r.range_bad = false;
  for (int p = s; p < e;) {
    TrField f;
    p = tr_field(d, p, e, f);
    if (p < 0) return false;
    if (f.num < 1 || f.num > 3) continue;
    if (r.kind != KIND_NONE) { r.multi = true; continue; }
    if (f.wt != 2) return false;
    r.kind = f.num;
    if (!tr_list(d, f.vs, f.ve, r, out, limit, range_n)) return false;
  }
  return true;
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

// schema key of the map key [s, e): lane k compares key k.  -1 = not a schema key, -2 = not UTF-8 (the host raises)
__device__ int tr_match_key(const uint8_t* d, int s, int e, bool want_z) {
  const int lane = tr_lane(), n = e - s;
  bool hit = false, high = false;
  if (lane < TR_KEYS && n == kTrKeyLen[lane] && (lane != TK_Z || want_z)) {
    hit = true;
    for (int i = 0; i < n && hit; ++i) hit = tr_byte(d, s + i) == (uint32_t)(uint8_t)kTrKey[lane][i];
  }
  for (int i = lane; i < n; i += 32) high |= tr_byte(d, s + i) >= 0x80;
  const unsigned m = __ballot_sync(FULL_MASK, hit);
  if (__any_sync(FULL_MASK, high) && !tr_utf8(d, s, e)) return -2;
  return m ? __ffs(m) - 1 : -1;
}

struct TrSlot {
  int fs, fe;   // the last occurrence's Feature bytes; fs < 0 = key absent
  TrFeat r;     // its kind and counts (scan only)
};

__device__ __forceinline__ int tr_range_n(int key) {
  return key == TK_FEAT || key == TK_AINT || (key >= TK_UIDS && key < TK_UVALS) ? TR_ALL
         : (key >= TK_ACAT && key < TK_AINT)                                    ? 1
                                                                                : 0;
}

// Example -> Features -> map entries of the record [0, L): slot[k] = the last entry of schema key k.  scan: every keyed
// entry's Feature is parsed (the host parses them all) and slot[k].r holds the counts.  false = malformed.
__device__ bool tr_walk(const uint8_t* d, int L, TrSlot* slot, bool want_z, bool scan) {
  const int lane = tr_lane();
  if (lane < TR_KEYS) slot[lane].fs = -1;
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
      const int key = tr_match_key(d, ks, ke, want_z);
      if (key == -2) { ok = false; break; }
      TrFeat r{};
      if (scan && !tr_feature(d, fs, fe, r, nullptr, 0, key >= 0 ? tr_range_n(key) : 0)) { ok = false; break; }
      if (key >= 0 && lane == 0) { slot[key].fs = fs; slot[key].fe = fe; slot[key].r = r; }
    }
  }
  __syncwarp();
  return ok;
}

// the checks of decode_tfrecord_files, in its order, then the deviations -> (check << 8) | arg, or -1
__device__ int tr_checks(const TrSlot* slot, int F, int labels_mask) {
  auto cnt = [&](int k) { return slot[k].fs < 0 ? 0 : slot[k].r.count; };
  for (int k = TK_Y; k <= TK_FEAT + 3; ++k) {
    if (k <= TK_Z && !(labels_mask >> k & 1)) continue;
    if (cnt(k) == 0) return TE_REQUIRED << 8 | k;
  }
  if (cnt(TK_FEAT) != F) return TE_COUNT << 8;
  for (int f = 0; f < 4; ++f)
    if (cnt(TK_UIDS + f) != cnt(TK_UVALS + f)) return TE_MISMATCH << 8 | f;
  for (int k = 0; k < TR_KEYS; ++k) {
    if (slot[k].fs < 0) continue;
    const TrFeat& r = slot[k].r;
    if (r.multi || (r.kind != KIND_NONE && r.kind != kTrKeyKind[k])) return TE_KIND << 8 | k;
  }
  for (int k = 0; k < TR_KEYS; ++k)
    if (slot[k].fs >= 0 && slot[k].r.range_bad) return TE_RANGE << 8 | k;
  return -1;
}

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

__global__ void __launch_bounds__(TR_THREADS) tr_scan_kernel(const uint8_t* __restrict__ chunk,
                                                             const int64_t* __restrict__ rec_off, int64_t n_rec,
                                                             int64_t record_base, int F, int labels_mask,
                                                             int32_t* __restrict__ lens,
                                                             unsigned long long* __restrict__ err) {
  __shared__ uint32_t tab[256], x8[64];
  __shared__ TrSlot slots[TR_WARPS][TR_KEYS];
  tr_crc_tables(tab, x8);
  const int lane = tr_lane(), wib = threadIdx.x >> 5;
  TrSlot* slot = slots[wib];
  const int64_t stride = (int64_t)gridDim.x * TR_WARPS;
  for (int64_t i = (int64_t)blockIdx.x * TR_WARPS + wib; i < n_rec; i += stride) {
    const uint8_t* h = chunk + rec_off[i];
    const int64_t L = (int64_t)tr_u32(h, 0) | (int64_t)tr_u32(h, 4) << 32;   // framed (< 2^31) by the host
    const uint8_t* d = h + 12;
    int word = -1;
    const uint32_t c = tr_crc32c(d, L, tab, x8);
    if ((((c >> 15) | (c << 17)) + 0xA282EAD8u) != tr_u32(d, L)) {
      word = TE_CRC << 8;
    } else if (!tr_walk(d, (int)L, slot, labels_mask & 2, true)) {
      word = TE_MALFORMED << 8;
    } else {
      word = tr_checks(slot, F, labels_mask);
    }
    int len = 0;
    if (word < 0 && lane < 5) {
      const int k = lane < 4 ? TK_UIDS + lane : TK_AINT;
      len = slot[k].fs < 0 ? 0 : slot[k].r.count;
    }
    if (lane < 5) lens[i * 5 + lane] = len;
    if (word >= 0 && lane == 0) atomicMin(err, (unsigned long long)(record_base + i) << 16 | (unsigned)word);
    __syncwarp();
  }
}

__device__ __forceinline__ void tr_zero(int32_t* o, int from, int to) {
  for (int i = from + tr_lane(); i < to; i += 32) o[i] = 0;
}
__device__ __forceinline__ void tr_zero(float* o, int from, int to) {
  for (int i = from + tr_lane(); i < to; i += 32) o[i] = 0.f;
}
__device__ __forceinline__ int tr_emit_key(const uint8_t* d, const TrSlot* slot, int k, void* out, int limit) {
  if (slot[k].fs < 0) return 0;
  TrFeat r;
  tr_feature(d, slot[k].fs, slot[k].fe, r, out, limit, 0);
  return r.count < limit ? r.count : limit;
}

// make_batch of din_main (DIN.py:57-99): one warp per slot b
__global__ void __launch_bounds__(TR_THREADS) tr_emit_din_kernel(
    const uint8_t* __restrict__ stage, const int64_t* __restrict__ slot_off, const int32_t* __restrict__ slot_len, int B,
    int F, int P, const int32_t* __restrict__ a_int_off, int32_t* __restrict__ feat_ids, int32_t* __restrict__ a_ids,
    int32_t* __restrict__ a_int_ids, int32_t* __restrict__ u_ids, float* __restrict__ u_wgt, float* __restrict__ y) {
  __shared__ TrSlot slots[TR_WARPS][TR_KEYS];
  const int wib = threadIdx.x >> 5;
  TrSlot* slot = slots[wib];
  for (int b = blockIdx.x * TR_WARPS + wib; b < B; b += gridDim.x * TR_WARPS) {
    const uint8_t* d = stage + slot_off[b];
    tr_walk(d, slot_len[b], slot, false, false);
    tr_emit_key(d, slot, TK_FEAT, feat_ids + (int64_t)b * F, F);
    for (int j = 0; j < 3; ++j) tr_emit_key(d, slot, TK_ACAT + j, a_ids + (int64_t)j * B + b, 1);
    tr_emit_key(d, slot, TK_AINT, a_int_ids + a_int_off[b], a_int_off[b + 1] - a_int_off[b]);
    for (int f = 0; f < 4; ++f) {
      int32_t* ui = u_ids + ((int64_t)f * B + b) * P;
      float* uw = u_wgt + ((int64_t)f * B + b) * P;
      tr_zero(ui, tr_emit_key(d, slot, TK_UIDS + f, ui, P), P);
      tr_zero(uw, tr_emit_key(d, slot, TK_UVALS + f, uw, P), P);
    }
    tr_emit_key(d, slot, TK_Y, y + b, 1);
    __syncwarp();
  }
}

// make_batch of esmm_main (DeepCvrMTL.py:63-105): bags u_cat, u_shop, u_brand, u_int, a_int field-major, a_int's
// weights 1.0
__global__ void __launch_bounds__(TR_THREADS) tr_emit_esmm_kernel(
    const uint8_t* __restrict__ stage, const int64_t* __restrict__ slot_off, const int32_t* __restrict__ slot_len, int B,
    int F, const int32_t* __restrict__ bag_off, int32_t* __restrict__ feat_ids, int32_t* __restrict__ a_ids,
    int32_t* __restrict__ bag_ids, float* __restrict__ bag_wgt, float* __restrict__ y, float* __restrict__ z) {
  __shared__ TrSlot slots[TR_WARPS][TR_KEYS];
  const int wib = threadIdx.x >> 5;
  TrSlot* slot = slots[wib];
  for (int b = blockIdx.x * TR_WARPS + wib; b < B; b += gridDim.x * TR_WARPS) {
    const uint8_t* d = stage + slot_off[b];
    tr_walk(d, slot_len[b], slot, true, false);
    tr_emit_key(d, slot, TK_FEAT, feat_ids + (int64_t)b * F, F);
    for (int j = 0; j < 3; ++j) tr_emit_key(d, slot, TK_ACAT + j, a_ids + (int64_t)j * B + b, 1);
    for (int f = 0; f < 4; ++f) {
      const int o = bag_off[f * B + b], n = bag_off[f * B + b + 1] - o;
      tr_emit_key(d, slot, TK_UIDS + f, bag_ids + o, n);
      tr_emit_key(d, slot, TK_UVALS + f, bag_wgt + o, n);
    }
    const int o = bag_off[4 * B + b], n = bag_off[4 * B + b + 1] - o;
    tr_emit_key(d, slot, TK_AINT, bag_ids + o, n);
    for (int i = tr_lane(); i < n; i += 32) bag_wgt[o + i] = 1.f;
    tr_emit_key(d, slot, TK_Y, y + b, 1);
    tr_emit_key(d, slot, TK_Z, z + b, 1);
    __syncwarp();
  }
}

static unsigned tr_grid(int64_t items) {
  const int64_t want = (items + TR_WARPS - 1) / TR_WARPS, cap = (int64_t)sm_count() * 16;
  return (unsigned)(want < 1 ? 1 : (want < cap ? want : cap));
}

}  // namespace ctr

using namespace ctr;

extern "C" {

int ctr_tfrecord_scan(const void* chunk, size_t len, const int64_t* rec_off, int64_t n_rec, int64_t record_base, int F,
                      int labels_mask, int32_t* lens, uint64_t* err, ctr_stream_t stream) {
  CTR_REQUIRE(n_rec >= 0 && record_base >= 0 && F > 0 && (labels_mask & 1) && err &&
                  (n_rec == 0 || (chunk && rec_off && lens)),
              CTR_ERR_INVALID_ARG, "ctr_tfrecord_scan: bad arguments");
  CTR_REQUIRE(record_base + n_rec < ((int64_t)1 << 47), CTR_ERR_INVALID_ARG, "ctr_tfrecord_scan: record index >= 2^47");
  (void)len;
  if (n_rec == 0) return CTR_OK;
  tr_scan_kernel<<<tr_grid(n_rec), TR_THREADS, 0, as_stream(stream)>>>(
      static_cast<const uint8_t*>(chunk), rec_off, n_rec, record_base, F, labels_mask, lens,
      reinterpret_cast<unsigned long long*>(err));
  CTR_LAUNCHED("ctr_tfrecord_scan");
  return CTR_OK;
}

int ctr_tfrecord_emit_din(const void* stage, const int64_t* slot_off, const int32_t* slot_len, int B, int F, int P,
                          const int32_t* a_int_off, int32_t* feat_ids, int32_t* a_ids, int32_t* a_int_ids,
                          int32_t* u_ids, float* u_wgt, float* y, ctr_stream_t stream) {
  CTR_REQUIRE(stage && slot_off && slot_len && B > 0 && F > 0 && P > 0 && a_int_off && feat_ids && a_ids && u_ids &&
                  u_wgt && y,
              CTR_ERR_INVALID_ARG, "ctr_tfrecord_emit_din: bad arguments");
  tr_emit_din_kernel<<<tr_grid(B), TR_THREADS, 0, as_stream(stream)>>>(
      static_cast<const uint8_t*>(stage), slot_off, slot_len, B, F, P, a_int_off, feat_ids, a_ids, a_int_ids, u_ids,
      u_wgt, y);
  CTR_LAUNCHED("ctr_tfrecord_emit_din");
  return CTR_OK;
}

int ctr_tfrecord_emit_esmm(const void* stage, const int64_t* slot_off, const int32_t* slot_len, int B, int F,
                           const int32_t* bag_off, int32_t* feat_ids, int32_t* a_ids, int32_t* bag_ids, float* bag_wgt,
                           float* y, float* z, ctr_stream_t stream) {
  CTR_REQUIRE(stage && slot_off && slot_len && B > 0 && F > 0 && bag_off && feat_ids && a_ids && y && z,
              CTR_ERR_INVALID_ARG, "ctr_tfrecord_emit_esmm: bad arguments");
  tr_emit_esmm_kernel<<<tr_grid(B), TR_THREADS, 0, as_stream(stream)>>>(
      static_cast<const uint8_t*>(stage), slot_off, slot_len, B, F, bag_off, feat_ids, a_ids, bag_ids, bag_wgt, y, z);
  CTR_LAUNCHED("ctr_tfrecord_emit_esmm");
  return CTR_OK;
}

}  // extern "C"
