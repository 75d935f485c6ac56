// aliccp_tfrecord.cu -- joined Ali-CCP samples -> tf.Example TFRecords on the GPU
// (deep_ctr/Feature_pipeline/get_aliccp_tfrecord.py gen_tfrecords, :38-102; DESIGN.md §2.6).
//
// A line is `sample_id,y,z,field:fid:val field:fid:val ...`.  One warp per line, three kernels over a text chunk cut
// at line ends (line starts and the warp splitting from line_starts.cuh):
//   plan      strip, split at ',' (lines without exactly 4 fields are skipped), tokenise the feature list with a ballot
//             over ' ' / ':' separators, classify every triple against the 19 kept field names, fold per-field
//             occurrence counts and id varint bytes, and size the record exactly (16 bytes of framing plus the nested
//             protobuf length prefixes).  Writes the record size, the number of declined numbers (below) and folds one
//             error word per chunk.  Two exclusive scans then give every line its output offset and decline offset.
//   declines  (only when the plan counted any) the (line, start, end) of every declined number, in line order.
//   write     re-tokenises each line and writes its record at the planned offset: the 15 features in sorted key order
//             (packed Int64List / FloatList, as tfrecord.encode_example writes them), the length header and both
//             masked CRC-32Cs (crc32c.cuh).
// Numbers: an id must be [0-9]+ below 2^63 (parse_u63 of decimal.cuh).  A label or value is converted here when it is
// plain decimal with a mantissa <= 2^53 and a decimal exponent of magnitude <= 22, where one fp64 multiply or divide by
// an exact power of ten (decimal.cuh's kPow10) is correctly rounded, i.e. equals Python's float(); it is then rounded
// to float32 as the FloatList does.  Any other number is declined: the host converts it with Python float() and
// uploads the float32 before the write.
// Error word (uint64, ~0 = none): (line << 8) | code, the smallest over the chunk = the first failing line.
#include "common.cuh"
#include "crc32c.cuh"
#include "decimal.cuh"
#include "line_starts.cuh"

namespace ctr {

constexpr int AL_THREADS = 256, AL_WARPS = AL_THREADS / 32;
constexpr int AL_CLASSES = 19, AL_COMMON = 11, AL_UMH = 11, AL_AD = 15, AL_KEYS = 15;
enum { AE_NUL = 1, AE_COUNT = 2, AE_EMPTY = 3, AE_ID = 4 };

__host__ __device__ constexpr uint64_t al_pack(const char* s) {
  uint64_t v = 0;
  int n = 0;
  for (; s[n]; ++n) v |= (uint64_t)(uint8_t)s[n] << (8 * n);
  return v | (uint64_t)n << 56;
}

// Field classes.  0..10: the common fields in the iteration order of the reference's Common_Fileds dict under
// Python 2.7 (DESIGN.md §2.6; oracle/aliccp_tfrecord.py derives it), 11..14: user multi-hot, 15..18: ad.
__constant__ uint64_t kAlField[AL_CLASSES] = {
    al_pack("205"),    al_pack("301"),    al_pack("121"),    al_pack("122"),    al_pack("124"),
    al_pack("125"),    al_pack("126"),    al_pack("127"),    al_pack("128"),    al_pack("129"),
    al_pack("101"),    al_pack("109_14"), al_pack("110_14"), al_pack("127_14"), al_pack("150_14"),
    al_pack("206"),    al_pack("207"),    al_pack("210"),    al_pack("216")};
__constant__ int kAlDefault[AL_CLASSES] = {10, 11, 2, 3, 4, 5, 6, 7, 8, 9, 1, 12, 13, 14, 15, 16, 17, 18, 19};

// Output keys in sorted order; src = the class whose ids / values the key holds (-1: feat_ids, y, z).
__constant__ char kAlKey[AL_KEYS][12] = {"a_brandids", "a_catids",  "a_intids",  "a_shopids",   "feat_ids",
                                         "u_brandids", "u_brandvals", "u_catids", "u_catvals",  "u_intids",
                                         "u_intvals",  "u_shopids", "u_shopvals", "y",          "z"};
__constant__ int kAlKeyLen[AL_KEYS] = {10, 8, 8, 9, 8, 10, 11, 8, 9, 8, 9, 9, 10, 1, 1};
__constant__ int kAlKeySrc[AL_KEYS] = {18, 15, 17, 16, -1, 13, 13, 11, 11, 14, 14, 12, 12, -1, -1};
__constant__ int kAlKeyFloat[AL_KEYS] = {0, 0, 0, 0, 0, 0, 1, 0, 1, 0, 1, 0, 1, 1, 1};
__constant__ int kAlIdKey[AL_CLASSES - AL_UMH] = {7, 11, 5, 9, 1, 3, 2, 0};   // class 11.. -> its ids key
__constant__ int kAlValKey[AL_AD - AL_UMH] = {8, 12, 6, 10};                   // class 11..14 -> its vals key

__device__ __forceinline__ int al_vl(uint64_t v) { return v < 128 ? 1 : (70 - __clzll((long long)v)) / 7; }

// per-warp state in shared memory
struct AlWarp {
  int cnt[AL_CLASSES];        // occurrences of each class in the line
  int bytes[AL_CLASSES];      // varint bytes of its ids
  int run[AL_CLASSES];        // write: occurrences placed so far
  int64_t off[AL_CLASSES];    // write: data-relative position of the class's next id
  int64_t voff[4];            // write: position of each user multi-hot value list
};

struct AlLine {
  int64_t s1, e1, s2, e2, s3, e3;   // fields 1..3 of line.strip().split(',')
  bool nul;
};

// line.strip().split(',') of [p, e) -> false unless it has exactly 4 fields.  Warp-uniform.
__device__ __forceinline__ bool al_fields(const uint8_t* t, int64_t p, int64_t e, AlLine& L) {
  int64_t s, te, c[3] = {0, 0, 0};
  warp_strip(t, p, e, s, te);
  if (warp_seps(t, s, te, ',', c, L.nul) != 3) return false;
  L.s1 = c[0] + 1; L.e1 = c[1];
  L.s2 = c[1] + 1; L.e2 = c[2];
  L.s3 = c[2] + 1; L.e3 = te;
  return true;
}

// Python float() of [s, e) when the text is plain decimal ([+-]?(d+.?d*|.d+)([eE][+-]?d+)?) with mantissa <= 2^53 and
// |decimal exponent| <= 22 (or a zero mantissa), rounded to float32; false = declined.  One lane.
__device__ __forceinline__ bool al_value(const uint8_t* t, int64_t s, int64_t e, float& out) {
  if (e <= s || e - s > 64) return false;
  int64_t p = s;
  uint32_t c = byte_at(t, p);
  const bool neg = c == '-';
  if (c == '+' || c == '-') ++p;
  uint64_t M = 0;
  int nd = 0, frac = 0;
  bool dot = false, big = false;
  for (; p < e; ++p) {
    c = byte_at(t, p);
    if (c >= '0' && c <= '9') {
      ++nd;
      frac += dot;
      if (!big) {
        M = M * 10 + (c - '0');
        big = M > (1ull << 53);
      }
    } else if (c == '.' && !dot) {
      dot = true;
    } else {
      break;
    }
  }
  if (nd == 0) return false;
  int ex = 0;
  if (p < e && (byte_at(t, p) | 0x20) == 'e') {
    ++p;
    bool eneg = false;
    if (p < e && (byte_at(t, p) == '+' || byte_at(t, p) == '-')) eneg = byte_at(t, p++) == '-';
    int ned = 0;
    for (; p < e && byte_at(t, p) >= '0' && byte_at(t, p) <= '9'; ++p, ++ned) {
      ex = ex * 10 + (int)(byte_at(t, p) - '0');
      ex = ex > 10000 ? 10000 : ex;
    }
    if (ned == 0) return false;
    if (eneg) ex = -ex;
  }
  if (p != e || big) return false;
  double d = (double)M;
  const int E = ex - frac;
  if (M != 0) {
    if (E > 22 || E < -22) return false;
    d = E >= 0 ? __dmul_rn(d, kPow10[E]) : __ddiv_rn(d, kPow10[-E]);
  }
  const float f = __double2float_rn(d);
  out = neg ? -f : f;
  return true;
}

// class of the field token [s, e), -1 = a field the reference drops
__device__ __forceinline__ int al_class(const uint8_t* t, int64_t s, int64_t e) {
  const int64_t n = e - s;
  if (n != 3 && n != 6) return -1;
  uint64_t v = (uint64_t)n << 56;
  for (int i = 0; i < n; ++i) v |= (uint64_t)byte_at(t, s + i) << (8 * i);
  for (int c = 0; c < AL_CLASSES; ++c)
    if (kAlField[c] == v) return c;
  return -1;
}

struct AlTok {
  int64_t start, end;   // the token is [start, end); end is a separator or the end of the feature list
  int idx, role, cls;   // token number, idx % 3 (0 field, 1 fid, 2 val), class of its triple's field
};

// re.split('[ :]', fields[3]) by warp_split (line_starts.cuh): visit(sep, tok) once per window (warp-uniform); lanes
// with sep set end a token.  -> number of tokens.
template <class Visit>
__device__ __forceinline__ int al_tokens(const uint8_t* t, int64_t s, int64_t e, Visit&& visit) {
  const int lane = lane_id();
  int count = 0, carry_cls = -1;
  const auto is_sep = [](uint32_t b) { return b == ' ' || b == ':'; };
  warp_split(t, s, e, is_sep, [&](bool sep, int64_t start, int64_t q, unsigned m) {
    AlTok k;
    k.start = start;
    k.end = q;
    k.idx = count + __popc(m & lanemask_lt());
    k.role = k.idx % 3;
    const int cls = sep && k.role == 0 ? al_class(t, k.start, k.end) : -1;
    const unsigned fm = __ballot_sync(FULL_MASK, sep && k.role == 0);
    const unsigned fb = fm & (lanemask_lt() | (1u << lane));   // field tokens at or before this lane
    const int from = __shfl_sync(FULL_MASK, cls, fb ? 31 - __clz(fb) : 0);
    k.cls = fb ? from : carry_cls;
    const int last = __shfl_sync(FULL_MASK, cls, fm ? 31 - __clz(fm) : 0);
    if (fm) carry_cls = last;
    visit(sep, k);
    count += __popc(m);
  });
  return count;
}

__device__ __forceinline__ bool al_is_id(const AlTok& k) { return k.role == 1 && k.cls >= 0 && k.end > k.start; }
__device__ __forceinline__ bool al_is_val(const AlTok& k) {
  return k.role == 2 && k.cls >= AL_UMH && k.cls < AL_AD && k.end > k.start;
}

// smallest token number among the lanes of mask
__device__ __forceinline__ int al_first(unsigned mask, int idx) {
  const int v = __shfl_sync(FULL_MASK, idx, mask ? __ffs(mask) - 1 : 0);
  return mask ? v : 0x7FFFFFFF;
}

struct AlPass1 {
  int code, ndecl;
  bool ys, zs;   // y / z converted here
  float y, z;
};

// Pass 1 over a 4-field line: W.cnt / W.bytes, the error code, the declined numbers (y, z, then user multi-hot values
// in line order; spans != nullptr: their (row, start, end) from spans[3 * span_base] on).
__device__ __forceinline__ void al_pass1(const uint8_t* t, const AlLine& L, AlWarp& W, AlPass1& R, int64_t row, int64_t* spans,
                         int64_t span_base) {
  const int lane = lane_id();
  if (lane < AL_CLASSES) { W.cnt[lane] = 0; W.bytes[lane] = 0; }
  __syncwarp();
  float v = 0.f;
  bool ok = true;
  if (lane < 2) ok = lane == 0 ? al_value(t, L.s1, L.e1, v) : al_value(t, L.s2, L.e2, v);
  R.ys = __shfl_sync(FULL_MASK, ok, 0);
  R.zs = __shfl_sync(FULL_MASK, ok, 1);
  R.y = __shfl_sync(FULL_MASK, v, 0);
  R.z = __shfl_sync(FULL_MASK, v, 1);
  if (spans && lane < 2 && !ok) {
    const int64_t k = span_base + (lane == 1 && !R.ys ? 1 : 0);
    spans[3 * k] = row;
    spans[3 * k + 1] = lane == 0 ? L.s1 : L.s2;
    spans[3 * k + 2] = lane == 0 ? L.e1 : L.e2;
  }
  int ndecl = !R.ys + !R.zs, first_empty = 0x7FFFFFFF, first_bad = 0x7FFFFFFF;
  const int n = al_tokens(t, L.s3, L.e3, [&](bool sep, const AlTok& k) {
    const unsigned em = __ballot_sync(FULL_MASK, sep && k.end == k.start);
    first_empty = min(first_empty, al_first(em, k.idx));
    bool bad = false, decl = false;
    if (sep && al_is_id(k)) {
      uint64_t id;
      bad = !parse_u63(t, k.start, k.end, id);
      if (!bad) {
        atomicAdd(&W.cnt[k.cls], 1);
        atomicAdd(&W.bytes[k.cls], al_vl(id));
      }
    } else if (sep && al_is_val(k)) {
      float f;
      decl = !al_value(t, k.start, k.end, f);
    }
    first_bad = min(first_bad, al_first(__ballot_sync(FULL_MASK, bad), k.idx));
    const unsigned dm = __ballot_sync(FULL_MASK, decl);
    if (spans && decl) {
      const int64_t j = span_base + ndecl + __popc(dm & lanemask_lt());
      spans[3 * j] = row; spans[3 * j + 1] = k.start; spans[3 * j + 2] = k.end;
    }
    ndecl += __popc(dm);
  });
  __syncwarp();
  R.ndecl = ndecl;
  R.code = L.nul                                  ? AE_NUL
           : n % 3                                ? AE_COUNT
           : first_empty < first_bad              ? AE_EMPTY
           : first_bad != 0x7FFFFFFF              ? AE_ID
                                                  : 0;
}

// id bytes of feat_ids' group for common class c (a missing field writes its default id: one byte)
__device__ __forceinline__ int al_group(const AlWarp& W, int c) { return W.cnt[c] ? W.bytes[c] : 1; }

// payload bytes of key k (the packed values)
__device__ __forceinline__ int64_t al_payload(const AlWarp& W, int k) {
  if (k == 4) {
    int64_t P = 0;
    for (int c = 0; c < AL_COMMON; ++c) P += al_group(W, c);
    return P;
  }
  if (k >= 13) return 4;
  const int c = kAlKeySrc[k];
  return kAlKeyFloat[k] ? 4 * (int64_t)max(W.cnt[c], 1) : (int64_t)al_group(W, c);
}

// map entry of key k around a payload of P bytes: entry size, and the offset of the payload inside the entry
__device__ __forceinline__ int64_t al_entry(int k, int64_t P, int64_t& head) {
  const int64_t L1 = 1 + al_vl(P) + P, feat = 1 + al_vl(L1) + L1, E = 2 + kAlKeyLen[k] + 1 + al_vl(feat) + feat;
  head = 1 + al_vl(E) + E - P;
  return 1 + al_vl(E) + E;
}

// size of the framed record from W.cnt / W.bytes (every lane gets it)
__device__ __forceinline__ int64_t al_record_bytes(const AlWarp& W) {
  const int lane = lane_id();
  int64_t x = 0, head;
  if (lane < AL_KEYS) x = al_entry(lane, al_payload(W, lane), head);
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(FULL_MASK, x, o);
  return 16 + 1 + al_vl(x) + x;
}

__device__ __forceinline__ int al_put_varint(uint8_t* o, uint64_t v) {
  int n = 0;
  for (; v >= 128; v >>= 7) o[n++] = (uint8_t)(v | 0x80);
  o[n++] = (uint8_t)v;
  return n;
}
__device__ __forceinline__ void al_put_f32(uint8_t* o, float f) {
  const uint32_t b = __float_as_uint(f);
  o[0] = (uint8_t)b; o[1] = (uint8_t)(b >> 8); o[2] = (uint8_t)(b >> 16); o[3] = (uint8_t)(b >> 24);
}

// per line: rec[row] = framed record bytes (0 = skipped), decl[row] = declined numbers; the chunk's error word
__global__ void __launch_bounds__(AL_THREADS) al_plan_kernel(const uint8_t* __restrict__ t, int64_t len,
                                                            const int64_t* __restrict__ line_start,
                                                            const int64_t* __restrict__ n_newlines, int64_t line_base,
                                                            int64_t* __restrict__ rec, int64_t* __restrict__ decl,
                                                            int64_t* __restrict__ info) {
  __shared__ AlWarp warps[AL_WARPS];
  AlWarp& W = warps[threadIdx.x >> 5];
  const int lane = lane_id();
  const int64_t nn = n_newlines[0], n_lines = chunk_lines(t, len, nn);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    info[0] = n_lines;
    rec[n_lines] = 0;
    decl[n_lines] = 0;
  }
  for (int64_t row = (int64_t)blockIdx.x * AL_WARPS + (threadIdx.x >> 5); row < n_lines;
       row += (int64_t)gridDim.x * AL_WARPS) {
    int64_t p, e;
    line_bounds(line_start, nn, len, row, p, e);
    AlLine L;
    int64_t size = 0, nd = 0;
    if (al_fields(t, p, e, L)) {
      AlPass1 R;
      al_pass1(t, L, W, R, row, nullptr, 0);
      if (R.code && lane == 0)
        atomicMin(reinterpret_cast<unsigned long long*>(&info[1]),
                  (unsigned long long)(line_base + row) << 8 | (unsigned)R.code);
      size = al_record_bytes(W);
      nd = R.ndecl;
    }
    if (lane == 0) { rec[row] = size; decl[row] = nd; }
    __syncwarp();
  }
}

// (row, start, end) of every declined number, at its line's decline offset
__global__ void __launch_bounds__(AL_THREADS) al_declines_kernel(const uint8_t* __restrict__ t, int64_t len,
                                                                const int64_t* __restrict__ line_start,
                                                                const int64_t* __restrict__ n_newlines,
                                                                const int64_t* __restrict__ decl,
                                                                int64_t* __restrict__ spans) {
  __shared__ AlWarp warps[AL_WARPS];
  AlWarp& W = warps[threadIdx.x >> 5];
  const int64_t nn = n_newlines[0], n_lines = chunk_lines(t, len, nn);
  for (int64_t row = (int64_t)blockIdx.x * AL_WARPS + (threadIdx.x >> 5); row < n_lines;
       row += (int64_t)gridDim.x * AL_WARPS) {
    if (decl[row + 1] == decl[row]) continue;
    int64_t p, e;
    line_bounds(line_start, nn, len, row, p, e);
    AlLine L;
    al_fields(t, p, e, L);
    AlPass1 R;
    al_pass1(t, L, W, R, row, spans, decl[row]);
  }
}

// the record of every 4-field line at rec[row]
__global__ void __launch_bounds__(AL_THREADS, 2) al_write_kernel(const uint8_t* __restrict__ t, int64_t len,
                                                             const int64_t* __restrict__ line_start,
                                                             const int64_t* __restrict__ n_newlines,
                                                             const int64_t* __restrict__ rec,
                                                             const int64_t* __restrict__ decl,
                                                             const float* __restrict__ decl_vals,
                                                             uint8_t* __restrict__ out) {
  __shared__ uint32_t tab[256], x8[64];
  __shared__ AlWarp warps[AL_WARPS];
  tr_crc_tables(tab, x8);
  AlWarp& W = warps[threadIdx.x >> 5];
  const int lane = lane_id();
  const int64_t nn = n_newlines[0], n_lines = chunk_lines(t, len, nn);
  for (int64_t row = (int64_t)blockIdx.x * AL_WARPS + (threadIdx.x >> 5); row < n_lines;
       row += (int64_t)gridDim.x * AL_WARPS) {
    if (rec[row + 1] == rec[row]) continue;
    int64_t p, e;
    line_bounds(line_start, nn, len, row, p, e);
    AlLine L;
    al_fields(t, p, e, L);
    AlPass1 R;
    al_pass1(t, L, W, R, row, nullptr, 0);
    if (R.code) continue;   // the host raises on the chunk's first error and never asks for its records
    const int64_t dbase = decl[row];
    uint8_t* const h = out + rec[row];
    uint8_t* const d = h + 12;
    const int64_t total = rec[row + 1] - rec[row], Ld = total - 16;

    // ---- layout: Example tag + length, then one map entry per key ----
    int64_t x = 0, head = 0, P = 0;
    if (lane < AL_KEYS) { P = al_payload(W, lane); x = al_entry(lane, P, head); }
    int64_t entries;
    const int64_t before = warp_scan_excl(x, entries);
    const int64_t eb = 1 + al_vl(entries), at = eb + before;     // this lane's entry
    const int64_t pay = at + head;                               // its payload
    if (lane == 0) { d[0] = 0x0A; al_put_varint(d + 1, entries); }
    if (lane < AL_KEYS) {
      const bool fl = kAlKeyFloat[lane];
      const int kl = kAlKeyLen[lane];
      const int64_t L1 = 1 + al_vl(P) + P, feat = 1 + al_vl(L1) + L1, E = 2 + kl + 1 + al_vl(feat) + feat;
      uint8_t* o = d + at;
      *o++ = 0x0A; o += al_put_varint(o, E);
      *o++ = 0x0A; *o++ = (uint8_t)kl;
      for (int i = 0; i < kl; ++i) *o++ = (uint8_t)kAlKey[lane][i];
      *o++ = 0x12; o += al_put_varint(o, feat);
      *o++ = fl ? 0x12 : 0x1A; o += al_put_varint(o, L1);
      *o++ = 0x0A; o += al_put_varint(o, P);
      if (lane == 13) al_put_f32(o, R.ys ? R.y : decl_vals[dbase]);
      if (lane == 14) al_put_f32(o, R.zs ? R.z : decl_vals[dbase + !R.ys]);
    }
    // class c's first id goes to its key's payload; feat_ids' groups follow each other in class order
    int g_tot;
    const int g_before = warp_scan_excl(lane < AL_COMMON ? al_group(W, lane) : 0, g_tot);
    const bool umh = lane >= AL_UMH && lane < AL_AD;
    const int64_t id_pay = __shfl_sync(FULL_MASK, pay, lane < AL_COMMON ? 4 : lane < AL_CLASSES ? kAlIdKey[lane - AL_UMH] : 0);
    const int64_t val_pay = __shfl_sync(FULL_MASK, pay, umh ? kAlValKey[lane - AL_UMH] : 0);
    if (lane < AL_CLASSES) {
      const int64_t off = lane < AL_COMMON ? id_pay + g_before : id_pay;
      W.off[lane] = off;
      W.run[lane] = 0;
      if (umh) {
        W.voff[lane - AL_UMH] = val_pay;
        if (W.cnt[lane] == 0) al_put_f32(d + val_pay, 1.f);
      }
      if (W.cnt[lane] == 0) d[off] = (uint8_t)kAlDefault[lane];
    }
    __syncwarp();

    // ---- pass 2: every kept id and value at its place, in line order ----
    int nd = !R.ys + !R.zs;
    al_tokens(t, L.s3, L.e3, [&](bool sep, const AlTok& k) {
      const bool id = sep && al_is_id(k), val = sep && al_is_val(k);
      uint64_t v = 0;
      float f = 0.f;
      bool simple = true;
      if (id) parse_u63(t, k.start, k.end, v);
      if (val) simple = al_value(t, k.start, k.end, f);
      const unsigned dm = __ballot_sync(FULL_MASK, val && !simple);
      if (val && !simple) f = decl_vals[dbase + nd + __popc(dm & lanemask_lt())];
      nd += __popc(dm);
      int64_t at = 0;
      unsigned km = __ballot_sync(FULL_MASK, id || val);
      while (km) {   // one kept token at a time, so that each class's values keep their line order
        const int l = __ffs(km) - 1;
        km &= km - 1;
        if (lane == l) {
          if (id) {
            at = W.off[k.cls];
            W.off[k.cls] += al_vl(v);
            W.run[k.cls] += 1;
          } else {
            at = W.voff[k.cls - AL_UMH] + 4 * (int64_t)(W.run[k.cls] - 1);
          }
        }
        __syncwarp();
      }
      if (id) al_put_varint(d + at, v);
      if (val) al_put_f32(d + at, f);
    });
    __syncwarp();

    // ---- framing: length, masked CRC of the length, data, masked CRC of the data ----
    const uint32_t c = crc32c_warp(d, Ld, tab, x8, CrcPlain{});
    if (lane == 0) {
      uint32_t hc = 0xFFFFFFFFu;
      for (int i = 0; i < 8; ++i) {
        const uint8_t b = (uint8_t)((uint64_t)Ld >> (8 * i));
        h[i] = b;
        hc = tab[(hc ^ b) & 0xFF] ^ (hc >> 8);
      }
      const uint32_t mh = crc32c_mask(hc ^ 0xFFFFFFFFu), md = crc32c_mask(c);
      for (int i = 0; i < 4; ++i) { h[8 + i] = (uint8_t)(mh >> (8 * i)); d[Ld + i] = (uint8_t)(md >> (8 * i)); }
    }
    __syncwarp();
  }
}

// workspace: LineStarts (max_rows = len + 1) | rec, decl int64[len + 2]
struct AlWs : LineStarts {
  int64_t *rec, *decl;
  AlWs(void* ws, size_t len) : LineStarts(ws, len, (int64_t)len + 1) {
    uint8_t* b = reinterpret_cast<uint8_t*>(ws);
    size_t o = bytes;
    rec = reinterpret_cast<int64_t*>(b + o); o += align256((len + 2) * 8);
    decl = reinterpret_cast<int64_t*>(b + o); o += align256((len + 2) * 8);
    bytes = o;
  }
};

// chunks the kernels accept: the line-start pass keeps newline counts in int32
constexpr size_t AL_MAX_LEN = (size_t)1 << 31;

}  // namespace ctr

using namespace ctr;

extern "C" {

size_t ctr_aliccp_workspace_bytes(size_t len) { return AlWs(nullptr, len).bytes; }

int ctr_aliccp_plan(const char* text, size_t len, int64_t line_base, int64_t* info, void* ws, size_t ws_bytes,
                    ctr_stream_t stream) {
  CTR_REQUIRE(info && line_base >= 0 && line_base < ((int64_t)1 << 55) && (len == 0 || text), CTR_ERR_INVALID_ARG,
              "ctr_aliccp_plan: bad arguments");
  CTR_REQUIRE(len <= AL_MAX_LEN, CTR_ERR_INVALID_ARG, "ctr_aliccp_plan: chunk too large (len <= 2^31)");
  CTR_REQUIRE(ws && ws_bytes >= ctr_aliccp_workspace_bytes(len), CTR_ERR_WORKSPACE,
              "ctr_aliccp_plan: workspace too small");
  cudaStream_t st = as_stream(stream);
  CTR_REQUIRE(cudaMemsetAsync(info, 0, 4 * sizeof(int64_t), st) == cudaSuccess &&
                  cudaMemsetAsync(info + 1, 0xFF, sizeof(int64_t), st) == cudaSuccess,
              CTR_ERR_CUDA, "ctr_aliccp_plan: memset failed");
  if (len == 0) return CTR_OK;
  const uint8_t* t = reinterpret_cast<const uint8_t*>(text);
  const AlWs A(ws, len);
  if (int rc = A.launch(t, len, st, "ctr_aliccp_plan(lines)")) return rc;
  al_plan_kernel<<<grid_for((int64_t)len + 1, AL_WARPS, 8), AL_THREADS, 0, st>>>(
      t, (int64_t)len, A.line_start, A.n_newlines, line_base, A.rec, A.decl, info);
  CTR_LAUNCHED("ctr_aliccp_plan");
  // rec[0, n] and decl[0, n] become offsets, rec[n] / decl[n] the totals
  return cta_scan({A.rec, A.decl}, {info + 2, info + 3}, info, 1, st, "ctr_aliccp_plan(scan)");
}

int ctr_aliccp_declines(const char* text, size_t len, const void* ws, size_t ws_bytes, int64_t* spans,
                        ctr_stream_t stream) {
  CTR_REQUIRE((len == 0 || (text && spans)), CTR_ERR_INVALID_ARG, "ctr_aliccp_declines: bad arguments");
  CTR_REQUIRE(len <= AL_MAX_LEN, CTR_ERR_INVALID_ARG, "ctr_aliccp_declines: chunk too large (len <= 2^31)");
  CTR_REQUIRE(ws && ws_bytes >= ctr_aliccp_workspace_bytes(len), CTR_ERR_WORKSPACE,
              "ctr_aliccp_declines: workspace too small");
  if (len == 0) return CTR_OK;
  AlWs A(const_cast<void*>(ws), len);
  al_declines_kernel<<<grid_for((int64_t)len + 1, AL_WARPS, 8), AL_THREADS, 0, as_stream(stream)>>>(
      reinterpret_cast<const uint8_t*>(text), (int64_t)len, A.line_start, A.n_newlines, A.decl, spans);
  CTR_LAUNCHED("ctr_aliccp_declines");
  return CTR_OK;
}

int ctr_aliccp_write(const char* text, size_t len, const float* decl_vals, void* out, const void* ws, size_t ws_bytes,
                     ctr_stream_t stream) {
  CTR_REQUIRE((len == 0 || (text && out)), CTR_ERR_INVALID_ARG, "ctr_aliccp_write: bad arguments");
  CTR_REQUIRE(len <= AL_MAX_LEN, CTR_ERR_INVALID_ARG, "ctr_aliccp_write: chunk too large (len <= 2^31)");
  CTR_REQUIRE(ws && ws_bytes >= ctr_aliccp_workspace_bytes(len), CTR_ERR_WORKSPACE,
              "ctr_aliccp_write: workspace too small");
  if (len == 0) return CTR_OK;
  AlWs A(const_cast<void*>(ws), len);
  al_write_kernel<<<grid_for((int64_t)len + 1, AL_WARPS, 8), AL_THREADS, 0, as_stream(stream)>>>(
      reinterpret_cast<const uint8_t*>(text), (int64_t)len, A.line_start, A.n_newlines, A.rec, A.decl, decl_vals,
      static_cast<uint8_t*>(out));
  CTR_LAUNCHED("ctr_aliccp_write");
  return CTR_OK;
}

}  // extern "C"
