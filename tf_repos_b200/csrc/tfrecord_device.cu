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
#include "crc32c.cuh"
#include "example_wire.cuh"   // tr_map_entries, tr_feature_kind and the wire helpers
#include "scan_sort.cuh"      // cta_scan

namespace ctr {

constexpr int TR_KEYS = 15;
constexpr int TR_THREADS = 256, TR_WARPS = TR_THREADS / 32;
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
// ---- CRC-32C (crc32c.cuh): each lane CRCs 1/32 of the record ---------------------------------------------------
__device__ __forceinline__ uint32_t tr_crc32c(const uint8_t* d, int64_t L, const uint32_t* tab, const uint32_t* x8) {
  return crc32c_warp(d, L, tab, x8, CrcLdg{});
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

// a Feature message [s, e) with its values (example_wire.cuh's kind rule).  false = malformed.
__device__ bool tr_feature(const uint8_t* d, int s, int e, TrFeat& r, void* out, int limit, int range_n) {
  r.count = 0; r.range_bad = false;
  return tr_feature_kind(d, s, e, r, [&](int ls, int le) { return tr_list(d, ls, le, r, out, limit, range_n); });
}

// schema key of the map key [s, e): lane k compares key k.  -1 = not a schema key
__device__ int tr_match_key(const uint8_t* d, int s, int e, bool want_z) {
  const int lane = tr_lane(), n = e - s;
  bool hit = false;
  if (lane < TR_KEYS && n == kTrKeyLen[lane] && (lane != TK_Z || want_z)) {
    hit = true;
    for (int i = 0; i < n && hit; ++i) hit = tr_byte(d, s + i) == (uint32_t)(uint8_t)kTrKey[lane][i];
  }
  const unsigned m = __ballot_sync(FULL_MASK, hit);
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

// the map entries of the record [0, L) (example_wire.cuh's walk): slot[k] = the last entry of schema key k.  scan:
// every keyed entry's Feature is parsed (the host parses them all) and slot[k].r holds the counts; emit: only the
// Feature bytes are recorded.  false = malformed.
__device__ bool tr_walk(const uint8_t* d, int L, TrSlot* slot, bool want_z, bool scan) {
  const int lane = tr_lane();
  if (lane < TR_KEYS) slot[lane].fs = -1;
  return tr_map_entries(
      d, L, [&](int ks, int ke) { return tr_match_key(d, ks, ke, want_z); },
      [&](int key, int fs, int fe) {
        TrFeat r{};
        if (scan && !tr_feature(d, fs, fe, r, nullptr, 0, key >= 0 ? tr_range_n(key) : 0)) return false;
        if (key >= 0 && lane == 0) { slot[key].fs = fs; slot[key].fe = fe; slot[key].r = r; }
        return true;
      });
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

// A serving request's batch slot b (DESIGN.md §2.10, §2.14): Example b < n, or Example 0 for b >= n, as make_batch
// pads; its bytes are data[s, s + L).  The walk and checks of tr_scan_kernel without framing, CRC or labels: y and z
// are parsed (they must be well formed) and then dropped, so neither is required nor kind-checked.  -> the check word
// (-1 = accepted); len = on lanes 0-4 the value count of u_catids, u_shopids, u_brandids, u_intids, a_intids (0 when
// rejected), 0 elsewhere.
__device__ __forceinline__ int tr_serve_slot(const uint8_t* data, const int64_t* offsets, int n, int b, int F,
                                             TrSlot* slot, int64_t& s, int& L, int& len) {
  const int lane = tr_lane();
  const int e = b < n ? b : 0;
  s = offsets[e];
  L = (int)(offsets[e + 1] - s);
  int word;
  if (!tr_walk(data + s, L, slot, false, true)) {
    word = TE_MALFORMED << 8;
  } else {
    if (lane == 0) slot[TK_Y].fs = -1;
    __syncwarp();
    word = tr_checks(slot, F, 0);
  }
  len = 0;
  if (word < 0 && lane < 5) {
    const int k = lane < 4 ? TK_UIDS + lane : TK_AINT;
    len = slot[k].fs < 0 ? 0 : slot[k].r.count;
  }
  return word;
}

// DIN serving (DESIGN.md §2.10): one warp per batch slot b of a request slice (tr_serve_slot).  Writes the slot's bytes
// for the emit, its a_int bag length clamped to max_a_int (so the emit stays inside B * max_a_int ids) into
// a_int_off[b] for the scan, and folds the unclamped longest behaviour list / a_int bag of the real Examples into
// maxima[0] / maxima[1].
__global__ void __launch_bounds__(TR_THREADS) tr_din_serve_scan_kernel(
    const uint8_t* __restrict__ data, const int64_t* __restrict__ offsets, int n, int B, int64_t example_base, int F,
    int max_a_int, int64_t* __restrict__ slot_off, int32_t* __restrict__ slot_len, int32_t* __restrict__ a_int_off,
    int32_t* __restrict__ maxima, unsigned long long* __restrict__ err) {
  __shared__ TrSlot slots[TR_WARPS][TR_KEYS];
  const int lane = tr_lane(), wib = threadIdx.x >> 5;
  TrSlot* slot = slots[wib];
  for (int b = blockIdx.x * TR_WARPS + wib; b < B; b += gridDim.x * TR_WARPS) {
    int64_t s;
    int L, len;
    const int word = tr_serve_slot(data, offsets, n, b, F, slot, s, L, len);
    const int u_max = __reduce_max_sync(FULL_MASK, lane < 4 ? len : 0);
    const int a_len = __shfl_sync(FULL_MASK, len, 4);
    if (lane == 0) {
      slot_off[b] = s;
      slot_len[b] = L;
      a_int_off[b] = a_len < max_a_int ? a_len : max_a_int;
      if (b < n) {
        if (u_max) atomicMax(&maxima[0], u_max);
        if (a_len) atomicMax(&maxima[1], a_len);
        if (word >= 0) atomicMin(err, (unsigned long long)(example_base + b) << 16 | (unsigned)word);
      }
    }
    __syncwarp();
  }
}

// ESMM serving (DESIGN.md §2.14): one warp per batch slot b of a request slice (tr_serve_slot).  Writes the slot's
// bytes for the emit and its five bag lengths field-major into bag_off[j * B + b]; slot 0 also zeroes bag_off[5B], so
// that the scan's sum of all 5B + 1 entries is the slice's occurrence total.
__global__ void __launch_bounds__(TR_THREADS) tr_esmm_serve_scan_kernel(
    const uint8_t* __restrict__ data, const int64_t* __restrict__ offsets, int n, int B, int64_t example_base, int F,
    int64_t* __restrict__ slot_off, int32_t* __restrict__ slot_len, int32_t* __restrict__ bag_off,
    unsigned long long* __restrict__ err) {
  __shared__ TrSlot slots[TR_WARPS][TR_KEYS];
  const int lane = tr_lane(), wib = threadIdx.x >> 5;
  TrSlot* slot = slots[wib];
  for (int b = blockIdx.x * TR_WARPS + wib; b < B; b += gridDim.x * TR_WARPS) {
    int64_t s;
    int L, len;
    const int word = tr_serve_slot(data, offsets, n, b, F, slot, s, L, len);
    if (lane < 5) bag_off[(int64_t)lane * B + b] = len;
    if (lane == 0) {
      slot_off[b] = s;
      slot_len[b] = L;
      if (b == 0) bag_off[(int64_t)5 * B] = 0;
      if (b < n && word >= 0) atomicMin(err, (unsigned long long)(example_base + b) << 16 | (unsigned)word);
    }
    __syncwarp();
  }
}

// after the scan: a slice whose occurrence total exceeds the capacity gets empty bags, so the emit writes no
// occurrence (the caller grows its buffers and runs the slice again)
__global__ void __launch_bounds__(1024) tr_esmm_occ_clamp_kernel(int32_t* __restrict__ bag_off, int64_t W,
                                                                  const int64_t* __restrict__ total, int64_t cap) {
  if (*total <= cap) return;
  for (int64_t i = threadIdx.x; i < W; i += blockDim.x) bag_off[i] = 0;
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
  tr_scan_kernel<<<grid_for(n_rec, TR_WARPS, 16), TR_THREADS, 0, as_stream(stream)>>>(
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
  tr_emit_din_kernel<<<grid_for(B, TR_WARPS, 16), TR_THREADS, 0, as_stream(stream)>>>(
      static_cast<const uint8_t*>(stage), slot_off, slot_len, B, F, P, a_int_off, feat_ids, a_ids, a_int_ids, u_ids,
      u_wgt, y);
  CTR_LAUNCHED("ctr_tfrecord_emit_din");
  return CTR_OK;
}

int ctr_din_serve_scan(const void* data, const int64_t* offsets, int64_t n, int64_t example_base, int F, int B,
                       int max_a_int, int64_t* slot_off, int32_t* slot_len, int32_t* a_int_off, int32_t* maxima,
                       uint64_t* err, ctr_stream_t stream) {
  CTR_REQUIRE(data && offsets && n > 0 && n <= B && example_base >= 0 && F > 0 && max_a_int > 0 && slot_off &&
                  slot_len && a_int_off && maxima && err,
              CTR_ERR_INVALID_ARG, "ctr_din_serve_scan: bad arguments");
  CTR_REQUIRE(example_base + n < ((int64_t)1 << 47) && (int64_t)B * max_a_int < ((int64_t)1 << 31),
              CTR_ERR_INVALID_ARG, "ctr_din_serve_scan: example index >= 2^47 or B * max_a_int >= 2^31");
  cudaStream_t st = as_stream(stream);
  tr_din_serve_scan_kernel<<<grid_for(B, TR_WARPS, 16), TR_THREADS, 0, st>>>(
      static_cast<const uint8_t*>(data), offsets, (int)n, B, example_base, F, max_a_int, slot_off, slot_len, a_int_off,
      maxima, reinterpret_cast<unsigned long long*>(err));
  return cta_scan({a_int_off}, {nullptr}, nullptr, (int64_t)B + 1, st, "ctr_din_serve_scan");
}

int ctr_esmm_serve_scan(const void* data, const int64_t* offsets, int64_t n, int64_t example_base, int F, int B,
                        int64_t occ_capacity, int64_t* slot_off, int32_t* slot_len, int32_t* bag_off, int64_t* total,
                        uint64_t* err, ctr_stream_t stream) {
  const char* fn = "ctr_esmm_serve_scan";
  CTR_REQUIRE(data && offsets && n > 0 && n <= B && example_base >= 0 && F > 0 && occ_capacity >= 0 && slot_off &&
                  slot_len && bag_off && total && err,
              CTR_ERR_INVALID_ARG, "%s: bad arguments", fn);
  CTR_REQUIRE(example_base + n < ((int64_t)1 << 47) && occ_capacity < ((int64_t)1 << 31) &&
                  (int64_t)5 * B < ((int64_t)1 << 31),
              CTR_ERR_INVALID_ARG, "%s: example index >= 2^47, occ_capacity >= 2^31 or 5B >= 2^31", fn);
  cudaStream_t st = as_stream(stream);
  const int64_t W = (int64_t)5 * B + 1;
  tr_esmm_serve_scan_kernel<<<grid_for(B, TR_WARPS, 16), TR_THREADS, 0, st>>>(
      static_cast<const uint8_t*>(data), offsets, (int)n, B, example_base, F, slot_off, slot_len, bag_off,
      reinterpret_cast<unsigned long long*>(err));
  CTR_LAUNCHED(fn);
  if (int rc = cta_scan({bag_off}, {total}, nullptr, W, st, fn)) return rc;
  tr_esmm_occ_clamp_kernel<<<1, 1024, 0, st>>>(bag_off, W, total, occ_capacity);
  CTR_LAUNCHED(fn);
  return CTR_OK;
}

int ctr_tfrecord_emit_esmm(const void* stage, const int64_t* slot_off, const int32_t* slot_len, int B, int F,
                           const int32_t* bag_off, int32_t* feat_ids, int32_t* a_ids, int32_t* bag_ids, float* bag_wgt,
                           float* y, float* z, ctr_stream_t stream) {
  CTR_REQUIRE(stage && slot_off && slot_len && B > 0 && F > 0 && bag_off && feat_ids && a_ids && y && z,
              CTR_ERR_INVALID_ARG, "ctr_tfrecord_emit_esmm: bad arguments");
  tr_emit_esmm_kernel<<<grid_for(B, TR_WARPS, 16), TR_THREADS, 0, as_stream(stream)>>>(
      static_cast<const uint8_t*>(stage), slot_off, slot_len, B, F, bag_off, feat_ids, a_ids, bag_ids, bag_wgt, y, z);
  CTR_LAUNCHED("ctr_tfrecord_emit_esmm");
  return CTR_OK;
}

}  // extern "C"
