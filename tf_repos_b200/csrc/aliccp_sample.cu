// aliccp_sample.cu -- raw Ali-CCP (Tianchi) files -> the joined, remapped, shuffled part files that
// get_aliccp_tfrecord.py reads, on the GPU (DeepMTL/Feature_pipeline/get_join_mapper.py, get_join_reducer.py,
// get_stat_mapper.py, get_stat_reducer.py, get_remap_mapper.py; DESIGN.md §2.7).
//
// A raw line is `md5,feat_num,feat_list` (a common record) or `sample_id,y,z,md5,feat_num,feat_list` (a sample);
// feat_list is `field\x02fid\x03val` tokens joined by \x01.  One warp per line (line starts and the warp splitting from
// line_starts.cuh):
//   classify  strip, the commas by ballot, the y=0/z=1 filter, the \x01 tokens from a ballot of separators (each token
//             then split and checked by the lane that ends it), the restrictions; kept lines insert their md5 into the
//             md5 table (lock-free, CAS on each word; key_table.cuh) and, for train samples, every (field, fid) into
//             the count table.
//             Three one-CTA scans give each common record its arena offset and id, each sample its ordinal.
//   place     common records are copied into the resident arena (the md5's record is the largest id: last wins);
//             samples keep (md5 slot, shuffle key).
//   resolve   slot -> record per sample, the record's multiplicity as an integer histogram.
//   commons   each record's tokens add its multiplicity to the count table (the join is never materialised).
//   vocab     fids with any count >= cutoff, LSD radix sorted and made unique (ids 20, 21, ...); the (field, fid)
//             entries sorted by (field bytes, fid) and rendered as feat_cnts.
//   render    each common record's remapped text, once.
//   emit      per sample line: its exact output size (plan) or its bytes at its offset (write), the offsets coming
//             from a stable sort of (part, r_i) over the samples in line order and an exclusive scan of the sizes.
// Every order comes from a sort or a scan and every reduction is an integer one: two runs give the same bytes.
#include "decimal.cuh"
#include "key_table.cuh"
#include "line_starts.cuh"

namespace ctr {

constexpr int AS_THREADS = 256, AS_WARPS = AS_THREADS / 32;
constexpr int AS_MAX_FIELD = 16, AS_MAX_MD5 = 64, AS_MD5_WORDS = 8;
constexpr int64_t AS_FIRST_ID = 20;
constexpr size_t AS_MAX_LEN = (size_t)1 << 30;

enum { AS_SKIP = 0, AS_COMMON = 1, AS_SAMPLE = 2, AS_FILTERED = 3 };
// info of ctr_aliccp_sample_classify
enum { AI_LINES, AI_ERR, AI_FILTERED, AI_MALFORMED, AI_CNT_DROP, AI_MD5_DROP, AI_COMMONS, AI_CBYTES, AI_SAMPLES, AI_N };

// bytes that no field, val, sample_id, y, z or md5 may hold (restriction): NUL, \x01-\x03, whitespace, ':'
__device__ __forceinline__ bool as_bad(uint32_t c) { return c <= 3 || is_py_space(c) || c == ':'; }

// r_i: the (i+1)-th output of SplitMix64 seeded with `seed`, top 31 bits
__device__ __forceinline__ uint32_t as_shuffle_key(uint64_t seed, uint64_t i) {
  return (uint32_t)(splitmix64_finalize(seed + (i + 1) * 0x9E3779B97F4A7C15ull) >> 33);
}

// ---- tables ----------------------------------------------------------------------------------------------------
// Lock-free open addressing (key_table.cuh): a slot belongs to the key whose words it holds, each word claimed in
// order; every key word is non-zero.

// count table: k0 = fid + 1, k1 / k2 = field bytes 0..7 / 8..15 big-endian zero-padded (k2 = 1 for fields of at most
// 8 bytes: a longer field's byte 8 is above 3), cnt; uint64[4][cap]
struct AsCnt {
  uint64_t *k0, *k1, *k2, *cnt;
  int64_t cap;
  AsCnt() = default;
  __host__ __device__ AsCnt(void* base, int64_t c)
      : k0(reinterpret_cast<uint64_t*>(base)), k1(k0 + c), k2(k0 + 2 * c), cnt(k0 + 3 * c), cap(c) {}
};

// md5 table: tag = length + 1, the md5 packed little-endian into 8 words, rec = the largest record id (-1: none)
struct AsMd5 {
  uint64_t *tag, *w;
  int64_t* rec;
  int64_t cap;
  AsMd5() = default;
  __host__ __device__ AsMd5(void* base, int64_t c)
      : tag(reinterpret_cast<uint64_t*>(base)), w(tag + c), rec(reinterpret_cast<int64_t*>(tag + 9 * c)), cap(c) {}
};

__device__ __forceinline__ void as_pack_field(const uint8_t* t, int64_t s, int64_t e, uint64_t& a, uint64_t& b) {
  a = 0; b = 0;
  for (int i = 0; i < (int)(e - s); ++i) {
    const uint64_t c = byte_at(t, s + i);
    if (i < 8) a |= c << (56 - 8 * i); else b |= c << (56 - 8 * (i - 8));
  }
  if (e - s <= 8) b = 1;
}

__device__ bool as_cnt_add(const AsCnt& T, uint64_t k0, uint64_t k1, uint64_t k2, uint64_t add) {
  const uint64_t h = splitmix64_finalize(k0 ^ splitmix64_finalize(k1 ^ splitmix64_finalize(k2)));
  const int64_t slot = probe(h, T.cap, [&](uint64_t s) {
    return claim(T.k0 + s, k0) == k0 && claim(T.k1 + s, k1) == k1 && claim(T.k2 + s, k2) == k2;
  });
  if (slot >= 0) atomicAdd(reinterpret_cast<unsigned long long*>(T.cnt + slot), (unsigned long long)add);
  return slot >= 0;
}

// slot of the md5 [s, e) (1..64 bytes, no NUL), inserted when missing; -1 = the table is full.  One lane.
__device__ int64_t as_md5_insert(const AsMd5& M, const uint8_t* t, int64_t s, int64_t e) {
  uint64_t w[AS_MD5_WORDS];
  const int n = (int)(e - s), nw = (n + 7) / 8;
  for (int j = 0; j < AS_MD5_WORDS; ++j) w[j] = 0;
  for (int i = 0; i < n; ++i) w[i >> 3] |= (uint64_t)byte_at(t, s + i) << (8 * (i & 7));
  uint64_t h = splitmix64_finalize((uint64_t)n);
  for (int j = 0; j < nw; ++j) h = splitmix64_finalize(h ^ w[j]);
  return probe(h, M.cap, [&](uint64_t slot) {
    bool same = claim(M.tag + slot, (uint64_t)n + 1) == (uint64_t)n + 1;
    for (int j = 0; j < nw && same; ++j) same = claim(M.w + slot * AS_MD5_WORDS + j, w[j]) == w[j];
    return same;
  });
}

// ---- lines and tokens ------------------------------------------------------------------------------------------
struct AsLine {
  int64_t s, te;   // line.strip()
  int nf;          // fields of .split(','); 7 = more than 6
  int64_t c[5];    // the first five commas
  bool nul;
};

// line.strip() of [p, e) and its first five commas (line_starts.cuh); a blank line has one empty field.  Warp-uniform.
__device__ void as_fields(const uint8_t* t, int64_t p, int64_t e, AsLine& L) {
  warp_strip(t, p, e, L.s, L.te);
  L.nf = warp_seps(t, L.s, L.te, ',', L.c, L.nul) + 1;
}

struct AsSpans {
  int64_t md5_s, md5_e, fs, fe;
};

// get_join_mapper.py:15-33: AS_COMMON / AS_SAMPLE / AS_FILTERED by field count and the y=0 / z=1 filter, else AS_SKIP
__device__ __forceinline__ int as_kind(const uint8_t* t, const AsLine& L, AsSpans& S) {
  if (L.nf == 3) {
    S.md5_s = L.s; S.md5_e = L.c[0]; S.fs = L.c[1] + 1; S.fe = L.te;
    return AS_COMMON;
  }
  if (L.nf != 6) return AS_SKIP;
  S.md5_s = L.c[2] + 1; S.md5_e = L.c[3]; S.fs = L.c[4] + 1; S.fe = L.te;
  const bool y0 = L.c[1] - L.c[0] == 2 && byte_at(t, L.c[0] + 1) == '0';
  const bool z1 = L.c[2] - L.c[1] == 2 && byte_at(t, L.c[1] + 1) == '1';
  return y0 && z1 ? AS_FILTERED : AS_SAMPLE;
}

struct AsTok {
  int64_t p2, p3;   // the \x02 and the \x03: field [start, p2), fid (p2, p3), val (p3, end)
  uint64_t fid;
};

// One \x01 token [s, e) (one lane).  0 = field\x02fid\x03val within the restrictions; 1 = a split the mapper's bare
// except skips the line on (not exactly one \x02, or not exactly one \x03 after it); 2 = a restriction.
__device__ int as_token(const uint8_t* t, int64_t s, int64_t e, AsTok& k) {
  int n2 = 0, n3 = 0;
  k.p2 = k.p3 = -1;
  for (int64_t p = s; p < e; ++p)
    if (byte_at(t, p) == 2) { ++n2; k.p2 = p; }
  if (n2 != 1) return 1;
  for (int64_t p = k.p2 + 1; p < e; ++p)
    if (byte_at(t, p) == 3) { ++n3; k.p3 = p; }
  if (n3 != 1) return 1;
  if (k.p2 - s < 1 || k.p2 - s > AS_MAX_FIELD) return 2;
  for (int64_t p = s; p < k.p2; ++p)
    if (as_bad(byte_at(t, p))) return 2;
  // fid: 0 or [1-9][0-9]* below 2^63, so that its text and its number are one key
  if ((byte_at(t, k.p2 + 1) == '0' && k.p3 > k.p2 + 2) || !parse_u63(t, k.p2 + 1, k.p3, k.fid)) return 2;
  for (int64_t p = k.p3 + 1; p < e; ++p)
    if (as_bad(byte_at(t, p))) return 2;
  return 0;
}

// the separator of feat_list.split('\x01'), for warp_split (line_starts.cuh)
struct AsTokEnd {
  __device__ bool operator()(uint32_t b) const { return b == 1; }
};

__device__ __forceinline__ bool as_any_bad(const uint8_t* t, int64_t s, int64_t e) {
  bool bad = false;
  for (int64_t w = s; w < e; w += 32) {
    const int64_t q = w + lane_id();
    bad |= __ballot_sync(FULL_MASK, q < e && as_bad(byte_at(t, q))) != 0;
  }
  return bad;
}

// A common or sample line -> AS_SKIP when a token fails the mapper's split (the line is skipped), else its kind;
// restricted = it breaks a restriction (raised by the host).  Warp-uniform.
__device__ int as_check(const uint8_t* t, const AsLine& L, const AsSpans& S, int kind, bool& restricted) {
  bool malformed = false, bad = false;
  warp_split(t, S.fs, S.fe, AsTokEnd{}, [&](bool end, int64_t s, int64_t q, unsigned) {
    int r = 0;
    if (end) { AsTok k; r = as_token(t, s, q, k); }
    malformed |= __ballot_sync(FULL_MASK, r == 1) != 0;
    bad |= __ballot_sync(FULL_MASK, r == 2) != 0;
  });
  if (malformed) return AS_SKIP;
  bad |= L.nul || S.md5_e - S.md5_s < 1 || S.md5_e - S.md5_s > AS_MAX_MD5 || as_any_bad(t, S.md5_s, S.md5_e);
  if (kind == AS_SAMPLE) bad |= as_any_bad(t, L.s, L.c[2]);   // sample_id, y, z (the commas between them are not bad)
  restricted = bad;
  return kind;
}

// per-line results of classify, scanned in place: cls | slot | fs (feat_list start) | flen (common records) |
// coff (scan of flen) | cord (scan of is-common) | sord (scan of is-sample)
struct AsPerLine {
  uint8_t* cls;
  int32_t *slot, *fs, *flen, *coff, *cord, *sord;
};

__global__ void __launch_bounds__(AS_THREADS) as_classify_kernel(const uint8_t* __restrict__ t, int64_t len,
                                                                const int64_t* __restrict__ line_start,
                                                                const int64_t* __restrict__ nnl, int64_t n_cap,
                                                                int mode, AsCnt C, AsMd5 M, AsPerLine P,
                                                                int64_t* __restrict__ info) {
  const int lane = lane_id();
  const int64_t nn = nnl[0], n_lines = chunk_lines(t, len, nn, n_cap);
  if (blockIdx.x == 0 && threadIdx.x == 0) info[AI_LINES] = n_lines;
  const int64_t warps = (int64_t)gridDim.x * AS_WARPS;
  for (int64_t row = (int64_t)blockIdx.x * AS_WARPS + (threadIdx.x >> 5); row < n_lines; row += warps) {
    int64_t p, e;
    line_bounds(line_start, nn, len, row, p, e);
    AsLine L;
    as_fields(t, p, e, L);
    AsSpans S;
    int kind = as_kind(t, L, S);
    bool restricted = false;
    if (kind == AS_COMMON || kind == AS_SAMPLE) kind = as_check(t, L, S, kind, restricted);
    int64_t slot = -1;
    if (restricted) {
      if (lane == 0) atomicMin(reinterpret_cast<unsigned long long*>(&info[AI_ERR]), (unsigned long long)row);
      kind = AS_SKIP;
    } else if (mode > 0 && (kind == AS_COMMON || kind == AS_SAMPLE)) {
      if (lane == 0) {
        slot = as_md5_insert(M, t, S.md5_s, S.md5_e);
        if (slot < 0) atomicAdd(reinterpret_cast<unsigned long long*>(&info[AI_MD5_DROP]), 1ull);
      }
      slot = __shfl_sync(FULL_MASK, slot, 0);
      if (mode == 2 && kind == AS_SAMPLE) {   // get_stat_mapper.py:17-19 over the sample's own tokens
        warp_split(t, S.fs, S.fe, AsTokEnd{}, [&](bool end, int64_t s, int64_t q, unsigned) {
          if (!end) return;
          AsTok k;
          as_token(t, s, q, k);
          uint64_t a, b;
          as_pack_field(t, s, k.p2, a, b);
          if (!as_cnt_add(C, k.fid + 1, a, b, 1))
            atomicAdd(reinterpret_cast<unsigned long long*>(&info[AI_CNT_DROP]), 1ull);
        });
      }
    }
    if (lane == 0) {
      if (kind == AS_FILTERED) atomicAdd(reinterpret_cast<unsigned long long*>(&info[AI_FILTERED]), 1ull);
      if (kind == AS_SKIP && !restricted) atomicAdd(reinterpret_cast<unsigned long long*>(&info[AI_MALFORMED]), 1ull);
      const int32_t flen = kind == AS_COMMON ? (int32_t)(S.fe - S.fs) : 0;
      P.cls[row] = (uint8_t)kind;
      P.slot[row] = (int32_t)slot;
      P.fs[row] = (kind == AS_COMMON || kind == AS_SAMPLE) ? (int32_t)S.fs : 0;
      P.flen[row] = flen;
      P.coff[row] = flen;
      P.cord[row] = kind == AS_COMMON;
      P.sord[row] = kind == AS_SAMPLE;
    }
  }
}

// common records -> arena + (offset, length, slot), md5 record = the largest id; samples -> (slot, part << 31 | r_i)
__global__ void __launch_bounds__(AS_THREADS) as_place_kernel(const uint8_t* __restrict__ t, const int64_t* __restrict__ info,
                                                             AsPerLine P, int64_t line_base, uint64_t seed, int64_t parts,
                                                             AsMd5 M, uint8_t* __restrict__ arena, int64_t arena_base,
                                                             int64_t* __restrict__ rec_off, int32_t* __restrict__ rec_len,
                                                             int32_t* __restrict__ rec_slot, int64_t rec_base,
                                                             int32_t* __restrict__ s_rec, uint64_t* __restrict__ s_key,
                                                             int64_t sample_base) {
  const int lane = lane_id();
  const int64_t n_lines = info[AI_LINES], warps = (int64_t)gridDim.x * AS_WARPS;
  for (int64_t row = (int64_t)blockIdx.x * AS_WARPS + (threadIdx.x >> 5); row < n_lines; row += warps) {
    const int kind = P.cls[row];
    if (kind == AS_COMMON) {
      const int64_t dst = arena_base + P.coff[row], src = P.fs[row], n = P.flen[row], rid = rec_base + P.cord[row];
      for (int64_t i = lane; i < n; i += 32) arena[dst + i] = t[src + i];
      if (lane == 0) {
        rec_off[rid] = dst;
        rec_len[rid] = (int32_t)n;
        rec_slot[rid] = P.slot[row];
        atomicMax(reinterpret_cast<long long*>(&M.rec[P.slot[row]]), (long long)rid);   // get_join_reducer.py:22
      }
    } else if (kind == AS_SAMPLE && lane == 0) {
      const int64_t k = sample_base + P.sord[row];
      const uint64_t r = as_shuffle_key(seed, (uint64_t)(line_base + row));
      s_rec[k] = P.slot[row];
      s_key[k] = ((r % (uint64_t)parts) << 31) | r;
    }
  }
}

// slot -> record per sample (get_join_reducer.py:26-33); multiplicity histogram; info {no common, superseded}
__global__ void as_resolve_kernel(const AsMd5 M, int32_t* __restrict__ s_rec, int64_t n_samples,
                                  const int32_t* __restrict__ rec_slot, int64_t n_records, uint32_t* __restrict__ mult,
                                  int64_t* __restrict__ info) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n_samples; k += stride) {
    const int64_t r = M.rec[s_rec[k]];
    s_rec[k] = (int32_t)r;
    if (r >= 0) atomicAdd(&mult[r], 1u);
    else atomicAdd(reinterpret_cast<unsigned long long*>(&info[0]), 1ull);
  }
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_records; r += stride)
    if (M.rec[rec_slot[r]] != r) atomicAdd(reinterpret_cast<unsigned long long*>(&info[1]), 1ull);
}

// every token of every record a kept sample resolves to adds that record's multiplicity (get_stat_mapper.py:17-19)
__global__ void __launch_bounds__(AS_THREADS) as_count_commons_kernel(const uint8_t* __restrict__ arena,
                                                                     const int64_t* __restrict__ rec_off,
                                                                     const int32_t* __restrict__ rec_len,
                                                                     const uint32_t* __restrict__ mult, int64_t n_records,
                                                                     AsCnt C, int64_t* __restrict__ info) {
  const int64_t warps = (int64_t)gridDim.x * AS_WARPS;
  for (int64_t r = (int64_t)blockIdx.x * AS_WARPS + (threadIdx.x >> 5); r < n_records; r += warps) {
    const uint32_t m = mult[r];
    if (m == 0) continue;
    const int64_t s0 = rec_off[r];
    warp_split(arena, s0, s0 + rec_len[r], AsTokEnd{}, [&](bool end, int64_t s, int64_t q, unsigned) {
      if (!end) return;
      AsTok k;
      as_token(arena, s, q, k);
      uint64_t a, b;
      as_pack_field(arena, s, k.p2, a, b);
      if (!as_cnt_add(C, k.fid + 1, a, b, m)) atomicAdd(reinterpret_cast<unsigned long long*>(&info[0]), 1ull);
    });
  }
}

// ---- vocabulary ------------------------------------------------------------------------------------------------
// used slots -> entries (k0, k1, k2, cnt); fids of entries with cnt >= cutoff -> kf (k0 = fid + 1).  The compaction's
// order depends on the schedule; everything downstream is sorted by the whole key first.
__global__ void __launch_bounds__(AS_THREADS) as_compact_kernel(AsCnt T, int64_t cutoff, AsCnt E,
                                                               uint64_t* __restrict__ kf, int64_t* __restrict__ counts) {
  const int lane = lane_id();
  const int64_t stride = (int64_t)gridDim.x * AS_THREADS, n_iter = (T.cap + stride - 1) / stride;
  for (int64_t it = 0; it < n_iter; ++it) {   // uniform trip count: the warp-aggregated atomics need whole warps
    const int64_t s = (it * gridDim.x + blockIdx.x) * AS_THREADS + threadIdx.x;
    const bool used = s < T.cap && T.k0[s] != 0;
    const uint64_t c = used ? T.cnt[s] : 0;
    const bool keep = used && (int64_t)c >= cutoff;
    const unsigned bu = __ballot_sync(FULL_MASK, used), bk = __ballot_sync(FULL_MASK, keep);
    unsigned long long eu = 0, ek = 0;
    if (lane == 0 && bu) eu = atomicAdd(reinterpret_cast<unsigned long long*>(&counts[0]), (unsigned long long)__popc(bu));
    if (lane == 0 && bk) ek = atomicAdd(reinterpret_cast<unsigned long long*>(&counts[1]), (unsigned long long)__popc(bk));
    eu = __shfl_sync(FULL_MASK, eu, 0);
    ek = __shfl_sync(FULL_MASK, ek, 0);
    if (used) {
      const int64_t e = (int64_t)eu + __popc(bu & lanemask_lt());
      E.k0[e] = T.k0[s]; E.k1[e] = T.k1[s]; E.k2[e] = T.k2[s]; E.cnt[e] = c;
    }
    if (keep) kf[(int64_t)ek + __popc(bk & lanemask_lt())] = T.k0[s];
  }
}

// sorted kf: run heads
__global__ void as_heads_kernel(const uint64_t* __restrict__ k, const int64_t* __restrict__ n_dev,
                                int32_t* __restrict__ head) {
  const int64_t n = n_dev[0];
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    head[i] = i == 0 || k[i] != k[i - 1];
}

// before the scan of head: head[i] = 1 at run heads; after it, the unique position
__global__ void as_unique_kernel(const uint64_t* __restrict__ k, const int64_t* __restrict__ n_dev,
                                 const int32_t* __restrict__ pos, uint64_t* __restrict__ vocab) {
  const int64_t n = n_dev[0];
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if (i == 0 || k[i] != k[i - 1]) vocab[pos[i]] = k[i] - 1;
}

__device__ __forceinline__ int as_field_len(uint64_t a, uint64_t b) {
  int n = 0;
  while (n < 8 && ((a >> (56 - 8 * n)) & 0xFF)) ++n;
  if (n == 8 && b != 1)
    while (n < 16 && ((b >> (56 - 8 * (n - 8))) & 0xFF)) ++n;
  return n;
}

// feat_cnts line j (get_stat_reducer.py:20-21, in (field bytes, fid) order): `field:fid\tcount\n`
template <bool W>
__global__ void as_feat_cnts_kernel(AsCnt E, const uint32_t* __restrict__ perm, const int64_t* __restrict__ n_dev,
                                    int64_t* __restrict__ off, char* __restrict__ out) {
  const int64_t n = n_dev[0];
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t e = perm[j];
    const uint64_t a = E.k1[e], b = E.k2[e], fid = E.k0[e] - 1, c = E.cnt[e];
    const int fl = as_field_len(a, b), nf = dec_digits(fid), nc = dec_digits(c);
    if (!W) { off[j] = fl + 1 + nf + 1 + nc + 1; continue; }
    char* o = out + off[j];
    for (int i = 0; i < fl; ++i) o[i] = (char)(i < 8 ? (a >> (56 - 8 * i)) : (b >> (56 - 8 * (i - 8))));
    o[fl] = ':';
    put_dec(fid, o + fl + 1, nf);
    o[fl + 1 + nf] = '\t';
    put_dec(c, o + fl + 2 + nf, nc);
    o[fl + 2 + nf + nc] = '\n';
  }
}

// ---- remap -----------------------------------------------------------------------------------------------------
// id of fid: AS_FIRST_ID + its rank among the kept fids, or -1 (dropped)
__device__ __forceinline__ int64_t as_lookup(const uint64_t* __restrict__ vocab, int64_t n, uint64_t fid) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (vocab[mid] < fid) lo = mid + 1; else hi = mid;
  }
  return lo < n && vocab[lo] == fid ? AS_FIRST_ID + lo : -1;
}

// The kept tokens of the \x01 list [s, e) as `field:id:val`, each preceded by ' ' unless it is the first kept one
// (kept counts those already placed): pos += their bytes; W = write them from o + pos.  Warp-uniform; every token
// of the list has passed as_check.
template <bool W>
__device__ void as_remap(const uint8_t* t, int64_t s, int64_t e, const uint64_t* vocab, int64_t n_vocab, char* o,
                         int64_t& pos, int64_t& kept) {
  warp_split(t, s, e, AsTokEnd{}, [&](bool end, int64_t ts, int64_t q, unsigned) {
    AsTok k;
    int64_t id = -1;
    if (end) {
      as_token(t, ts, q, k);
      id = as_lookup(vocab, n_vocab, k.fid);
    }
    const unsigned km = __ballot_sync(FULL_MASK, id >= 0);
    const bool sep = kept + __popc(km & lanemask_lt()) > 0;
    const int nd = id >= 0 ? dec_digits((uint64_t)id) : 0;
    const int64_t L = id >= 0 ? (sep ? 1 : 0) + (k.p2 - ts) + 1 + nd + 1 + (q - k.p3 - 1) : 0;
    int64_t tot;
    const int64_t before = warp_scan_excl(L, tot);
    if (W && id >= 0) {
      char* d = o + pos + before;
      if (sep) *d++ = ' ';
      for (int64_t p = ts; p < k.p2; ++p) *d++ = (char)byte_at(t, p);
      *d++ = ':';
      put_dec((uint64_t)id, d, nd);
      d += nd;
      *d++ = ':';
      for (int64_t p = k.p3 + 1; p < q; ++p) *d++ = (char)byte_at(t, p);
    }
    pos += tot;
    kept += __popc(km);
  });
}

// each record a sample resolves to: its remapped text (plan: rlen[r]; write: the bytes at r_off[r])
template <bool W>
__global__ void __launch_bounds__(AS_THREADS) as_render_kernel(const uint8_t* __restrict__ arena,
                                                              const int64_t* __restrict__ rec_off,
                                                              const int32_t* __restrict__ rec_len,
                                                              const uint32_t* __restrict__ mult, int64_t n_records,
                                                              const uint64_t* __restrict__ vocab, int64_t n_vocab,
                                                              int64_t* __restrict__ r_off, char* __restrict__ out) {
  const int64_t warps = (int64_t)gridDim.x * AS_WARPS;
  for (int64_t r = (int64_t)blockIdx.x * AS_WARPS + (threadIdx.x >> 5); r < n_records; r += warps) {
    int64_t pos = 0, kept = 0;
    if (mult[r]) as_remap<W>(arena, rec_off[r], rec_off[r] + rec_len[r], vocab, n_vocab, W ? out + r_off[r] : nullptr,
                             pos, kept);
    if (!W && lane_id() == 0) r_off[r] = pos;
  }
}

struct AsEmitArgs {
  uint64_t seed;
  int64_t line_base, sample_base;
  const int32_t* s_rec;
  const int64_t* r_off;      // rendered common text: record r is [r_off[r], r_off[r + 1])
  const char* rendered;
  const uint64_t* vocab;
  int64_t n_vocab;
  int64_t* s_val;            // plan: the line's size; write: its offset in the set's output
  int64_t lo, hi;            // write: the group's byte range
  char* out;
  int64_t* info;             // plan: info[0] += lines with an empty feature field
};

// get_remap_mapper.py:28-40 with the documented rule (DESIGN.md §2.7):
//   "%d\t%s,%s,%s,%s\n" % (r_i, sample_id, y, z, ' '.join(kept tokens of the sample, then of its common record))
template <bool W>
__global__ void __launch_bounds__(AS_THREADS) as_emit_kernel(const uint8_t* __restrict__ t, int64_t len,
                                                            const int64_t* __restrict__ line_start,
                                                            const int64_t* __restrict__ nnl,
                                                            const int64_t* __restrict__ info_cls, AsPerLine P,
                                                            AsEmitArgs a) {
  const int lane = lane_id();
  const int64_t nn = nnl[0], n_lines = info_cls[AI_LINES], warps = (int64_t)gridDim.x * AS_WARPS;
  for (int64_t row = (int64_t)blockIdx.x * AS_WARPS + (threadIdx.x >> 5); row < n_lines; row += warps) {
    if (P.cls[row] != AS_SAMPLE) continue;
    const int64_t k = a.sample_base + P.sord[row];
    int64_t base = 0;
    if (W) {
      base = a.s_val[k];
      if (base < a.lo || base >= a.hi) continue;
    }
    int64_t p, e;
    line_bounds(line_start, nn, len, row, p, e);
    AsLine L;
    as_fields(t, p, e, L);
    const uint64_t r = as_shuffle_key(a.seed, (uint64_t)(a.line_base + row));
    const int nr = dec_digits(r);
    char* o = W ? a.out + (base - a.lo) : nullptr;
    int64_t pos = nr + 1 + (L.c[2] - L.s) + 1;
    if (W) {
      for (int64_t i = lane; i < pos; i += 32) {
        char c;
        if (i < nr) { uint64_t v = r; for (int j = nr - 1; j > i; --j) v /= 10; c = (char)('0' + v % 10); }
        else if (i == nr) c = '\t';
        else if (i < pos - 1) c = (char)byte_at(t, L.s + i - nr - 1);
        else c = ',';
        o[i] = c;
      }
    }
    int64_t kept = 0;
    as_remap<W>(t, L.c[4] + 1, L.te, a.vocab, a.n_vocab, o, pos, kept);
    const int32_t rec = a.s_rec[k];
    const int64_t cs = rec >= 0 ? a.r_off[rec] : 0, cl = rec >= 0 ? a.r_off[rec + 1] - cs : 0;
    if (cl > 0) {
      if (kept > 0) {
        if (W && lane == 0) o[pos] = ' ';
        ++pos;
      }
      if (W) for (int64_t i = lane; i < cl; i += 32) o[pos + i] = a.rendered[cs + i];
      pos += cl;
    }
    if (W && lane == 0) o[pos] = '\n';
    ++pos;
    if (!W && lane == 0) {
      a.s_val[k] = pos;
      if (kept == 0 && cl == 0) atomicAdd(reinterpret_cast<unsigned long long*>(&a.info[0]), 1ull);
    }
  }
}

// sorted position p -> size of its sample (scanned into its offset afterwards); per-part byte totals
__global__ void as_sizes_sorted_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ perm,
                                       const int64_t* __restrict__ s_size, int64_t n, int64_t* __restrict__ sz,
                                       int64_t* __restrict__ part_bytes) {
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
    const int64_t v = s_size[perm[p]];
    sz[p] = v;
    atomicAdd(reinterpret_cast<unsigned long long*>(&part_bytes[keys[p] >> 31]), (unsigned long long)v);
  }
}

__global__ void as_offsets_kernel(const uint32_t* __restrict__ perm, const int64_t* __restrict__ off, int64_t n,
                                  int64_t* __restrict__ s_val) {
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x)
    s_val[perm[p]] = off[p];
}

// ---- workspace layouts and launch helpers ------------------------------------------------------------------------
// per chunk: LineStarts (max_rows = n_lines + 1) | info int64[AI_N] | cls uint8[n_lines + 1] |
// slot, fs, flen, coff, cord, sord int32[n_lines + 1]
struct AsChunkWs : LineStarts {
  int64_t* info;
  AsPerLine P;
  AsChunkWs(void* ws, size_t len, int64_t n_lines) : LineStarts(ws, len, n_lines + 1) {
    uint8_t* b = reinterpret_cast<uint8_t*>(ws);
    const size_t n = (size_t)n_lines + 1;
    size_t o = bytes;
    info = reinterpret_cast<int64_t*>(b + o); o += align256(AI_N * 8);
    P.cls = b + o; o += align256(n);
    int32_t** arrs[6] = {&P.slot, &P.fs, &P.flen, &P.coff, &P.cord, &P.sord};
    for (auto a : arrs) { *a = reinterpret_cast<int32_t*>(b + o); o += align256(n * 4); }
    bytes = o;
  }
};

// vocab: counts int64[2] | n_vocab, hist_count, feat_cnts bytes int64 | hist int32[256 * nb] | entries uint64[4][cap] |
// kf, keys, keys2 uint64[cap] | perm, perm2 uint32[cap] | head int32[cap] | lens int64[cap + 1]
struct AsVocabWs {
  int64_t *counts, *n_vocab, *hist_count, *fc_bytes;
  int32_t *hist, *head;
  AsCnt E;
  uint64_t *kf, *keys, *keys2;
  uint32_t *perm, *perm2;
  int64_t* lens;
  size_t bytes;
  AsVocabWs(void* ws, int64_t cap) {
    uint8_t* b = reinterpret_cast<uint8_t*>(ws);
    const size_t c = (size_t)cap, nb = (size_t)ceil_div64(cap, LSD_TILE);
    size_t o = 0;
    counts = reinterpret_cast<int64_t*>(b + o); n_vocab = counts + 2; hist_count = counts + 3; fc_bytes = counts + 4;
    o += align256(5 * 8);
    hist = reinterpret_cast<int32_t*>(b + o); o += align256(256 * nb * 4);
    E = AsCnt(b + o, cap); o += align256(4 * c * 8);
    kf = reinterpret_cast<uint64_t*>(b + o); o += align256(c * 8);
    keys = reinterpret_cast<uint64_t*>(b + o); o += align256(c * 8);
    keys2 = reinterpret_cast<uint64_t*>(b + o); o += align256(c * 8);
    perm = reinterpret_cast<uint32_t*>(b + o); o += align256(c * 4);
    perm2 = reinterpret_cast<uint32_t*>(b + o); o += align256(c * 4);
    head = reinterpret_cast<int32_t*>(b + o); o += align256(c * 4);
    lens = reinterpret_cast<int64_t*>(b + o); o += align256((c + 1) * 8);
    bytes = o;
  }
};

// order: n_dev int64 | hist_count int64 | hist int32[256 * nb] | keys2 uint64[n] | perm, perm2 uint32[n] | sz int64[n]
struct AsOrderWs {
  int64_t *n_dev, *hist_count;
  int32_t* hist;
  uint64_t* keys2;
  uint32_t *perm, *perm2;
  int64_t* sz;
  size_t bytes;
  AsOrderWs(void* ws, int64_t n) {
    uint8_t* b = reinterpret_cast<uint8_t*>(ws);
    const size_t c = (size_t)(n > 0 ? n : 1), nb = (size_t)ceil_div64((int64_t)c, LSD_TILE);
    size_t o = 0;
    n_dev = reinterpret_cast<int64_t*>(b + o); hist_count = n_dev + 1; o += align256(16);
    hist = reinterpret_cast<int32_t*>(b + o); o += align256(256 * nb * 4);
    keys2 = reinterpret_cast<uint64_t*>(b + o); o += align256(c * 8);
    perm = reinterpret_cast<uint32_t*>(b + o); o += align256(c * 4);
    perm2 = reinterpret_cast<uint32_t*>(b + o); o += align256(c * 4);
    sz = reinterpret_cast<int64_t*>(b + o); o += align256((c + 1) * 8);
    bytes = o;
  }
};

static int as_zero(void* p, size_t n, cudaStream_t st, const char* what) {
  CTR_REQUIRE(cudaMemsetAsync(p, 0, n, st) == cudaSuccess, CTR_ERR_CUDA, "%s: memset failed", what);
  return CTR_OK;
}

}  // namespace ctr

using namespace ctr;

extern "C" {

size_t ctr_aliccp_sample_count_table_bytes(int64_t capacity) { return capacity > 0 ? (size_t)capacity * 32 : 0; }

size_t ctr_aliccp_sample_md5_table_bytes(int64_t capacity) { return capacity > 0 ? (size_t)capacity * 80 : 0; }

size_t ctr_aliccp_sample_chunk_workspace_bytes(size_t len, int64_t n_lines) {
  return n_lines >= 0 ? AsChunkWs(nullptr, len, n_lines).bytes : 0;
}

int ctr_aliccp_sample_classify(const char* text, size_t len, int64_t n_lines, int mode, void* count_table,
                               int64_t count_capacity, void* md5_table, int64_t md5_capacity, int64_t* info,
                               void* ws, size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE((len == 0 || text) && n_lines >= 0 && mode >= 0 && mode <= 2 && info, CTR_ERR_INVALID_ARG,
              "ctr_aliccp_sample_classify: bad arguments");
  CTR_REQUIRE(mode == 0 || (md5_table && md5_capacity > 0 && md5_capacity <= KT_MAX_CAP), CTR_ERR_INVALID_ARG,
              "ctr_aliccp_sample_classify: bad md5 table");
  CTR_REQUIRE(mode != 2 || (count_table && count_capacity > 0 && count_capacity <= KT_MAX_CAP), CTR_ERR_INVALID_ARG,
              "ctr_aliccp_sample_classify: bad count table");
  CTR_REQUIRE(len < AS_MAX_LEN, CTR_ERR_INVALID_ARG, "ctr_aliccp_sample_classify: chunk too large (len < 2^30)");
  CTR_REQUIRE(ws && ws_bytes >= ctr_aliccp_sample_chunk_workspace_bytes(len, n_lines), CTR_ERR_WORKSPACE,
              "ctr_aliccp_sample_classify: workspace too small");
  cudaStream_t st = as_stream(stream);
  AsChunkWs W(ws, len, n_lines);
  CTR_REQUIRE(cudaMemsetAsync(W.info, 0, AI_N * 8, st) == cudaSuccess &&
                  cudaMemsetAsync(W.info + AI_ERR, 0xFF, 8, st) == cudaSuccess &&
                  cudaMemsetAsync(W.n_newlines, 0, 16, st) == cudaSuccess,
              CTR_ERR_CUDA, "ctr_aliccp_sample_classify: memset failed");
  const uint8_t* t = reinterpret_cast<const uint8_t*>(text);
  if (len > 0) {
    if (int rc = W.launch(t, len, st, "ctr_aliccp_sample_classify(lines)")) return rc;
    as_classify_kernel<<<grid_for(n_lines, AS_WARPS, 16), AS_THREADS, 0, st>>>(
        t, (int64_t)len, W.line_start, W.n_newlines, n_lines, mode, AsCnt(count_table, count_capacity),
        AsMd5(md5_table, md5_capacity), W.P, W.info);
    CTR_LAUNCHED("ctr_aliccp_sample_classify");
    if (int rc = cta_scan({W.P.coff, W.P.cord, W.P.sord}, {W.info + AI_CBYTES, W.info + AI_COMMONS, W.info + AI_SAMPLES},
                          W.info + AI_LINES, 0, st, "ctr_aliccp_sample_classify(scan)"))
      return rc;
  }
  CTR_REQUIRE(cudaMemcpyAsync(info, W.info, AI_N * 8, cudaMemcpyDeviceToDevice, st) == cudaSuccess, CTR_ERR_CUDA,
              "ctr_aliccp_sample_classify: copy of info failed");
  return CTR_OK;
}

int ctr_aliccp_sample_place(const char* text, size_t len, int64_t n_lines, int64_t line_base, uint64_t seed,
                            int64_t parts, void* md5_table, int64_t md5_capacity, uint8_t* arena, int64_t arena_base,
                            int64_t* rec_off, int32_t* rec_len, int32_t* rec_slot, int64_t rec_base, int32_t* s_rec,
                            uint64_t* s_key, int64_t sample_base, const void* ws, size_t ws_bytes,
                            ctr_stream_t stream) {
  CTR_REQUIRE((len == 0 || text) && n_lines >= 0 && line_base >= 0 && parts >= 1 && parts <= (1 << 20) && md5_table &&
                  md5_capacity > 0 && arena_base >= 0 && rec_base >= 0 && sample_base >= 0,
              CTR_ERR_INVALID_ARG, "ctr_aliccp_sample_place: bad arguments");
  CTR_REQUIRE(ws && ws_bytes >= ctr_aliccp_sample_chunk_workspace_bytes(len, n_lines), CTR_ERR_WORKSPACE,
              "ctr_aliccp_sample_place: workspace too small");
  if (len == 0 || n_lines == 0) return CTR_OK;
  AsChunkWs W(const_cast<void*>(ws), len, n_lines);
  as_place_kernel<<<grid_for(n_lines, AS_WARPS, 16), AS_THREADS, 0, as_stream(stream)>>>(
      reinterpret_cast<const uint8_t*>(text), W.info, W.P, line_base, seed, parts, AsMd5(md5_table, md5_capacity), arena,
      arena_base, rec_off, rec_len, rec_slot, rec_base, s_rec, s_key, sample_base);
  CTR_LAUNCHED("ctr_aliccp_sample_place");
  return CTR_OK;
}

int ctr_aliccp_sample_resolve(const void* md5_table, int64_t md5_capacity, int32_t* s_rec, int64_t n_samples,
                              const int32_t* rec_slot, int64_t n_records, uint32_t* mult, int64_t* info,
                              ctr_stream_t stream) {
  CTR_REQUIRE(md5_table && md5_capacity > 0 && n_samples >= 0 && n_records >= 0 && info &&
                  (n_samples == 0 || (s_rec && mult)) && (n_records == 0 || (rec_slot && mult)),
              CTR_ERR_INVALID_ARG, "ctr_aliccp_sample_resolve: bad arguments");
  cudaStream_t st = as_stream(stream);
  if (int rc = as_zero(info, 16, st, "ctr_aliccp_sample_resolve")) return rc;
  if (n_records)
    if (int rc = as_zero(mult, (size_t)n_records * 4, st, "ctr_aliccp_sample_resolve")) return rc;
  const int64_t n = n_samples > n_records ? n_samples : n_records;
  if (n == 0) return CTR_OK;
  as_resolve_kernel<<<grid_for(n, AS_THREADS, 16), AS_THREADS, 0, st>>>(
      AsMd5(const_cast<void*>(md5_table), md5_capacity), s_rec, n_samples, rec_slot, n_records, mult, info);
  CTR_LAUNCHED("ctr_aliccp_sample_resolve");
  return CTR_OK;
}

int ctr_aliccp_sample_count_commons(const uint8_t* arena, const int64_t* rec_off, const int32_t* rec_len,
                                    const uint32_t* mult, int64_t n_records, void* count_table, int64_t count_capacity,
                                    int64_t* info, ctr_stream_t stream) {
  CTR_REQUIRE(n_records >= 0 && count_table && count_capacity > 0 && count_capacity <= KT_MAX_CAP && info &&
                  (n_records == 0 || (arena && rec_off && rec_len && mult)),
              CTR_ERR_INVALID_ARG, "ctr_aliccp_sample_count_commons: bad arguments");
  cudaStream_t st = as_stream(stream);
  if (int rc = as_zero(info, 8, st, "ctr_aliccp_sample_count_commons")) return rc;
  if (n_records == 0) return CTR_OK;
  as_count_commons_kernel<<<grid_for(n_records, AS_WARPS, 16), AS_THREADS, 0, st>>>(
      arena, rec_off, rec_len, mult, n_records, AsCnt(count_table, count_capacity), info);
  CTR_LAUNCHED("ctr_aliccp_sample_count_commons");
  return CTR_OK;
}

size_t ctr_aliccp_sample_vocab_workspace_bytes(int64_t count_capacity) {
  return count_capacity > 0 ? AsVocabWs(nullptr, count_capacity).bytes : 0;
}

int ctr_aliccp_sample_vocab(const void* count_table, int64_t count_capacity, int64_t cutoff, uint64_t* vocab,
                            int64_t* info, void* ws, size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE(count_table && count_capacity > 0 && count_capacity <= KT_MAX_CAP && vocab && info,
              CTR_ERR_INVALID_ARG, "ctr_aliccp_sample_vocab: bad arguments");
  CTR_REQUIRE(ws && ws_bytes >= ctr_aliccp_sample_vocab_workspace_bytes(count_capacity), CTR_ERR_WORKSPACE,
              "ctr_aliccp_sample_vocab: workspace too small");
  cudaStream_t st = as_stream(stream);
  AsVocabWs V(ws, count_capacity);
  if (int rc = as_zero(V.counts, 5 * 8, st, "ctr_aliccp_sample_vocab")) return rc;
  const int64_t cap = count_capacity;
  const unsigned g = grid_for(cap, AS_THREADS, 16);
  as_compact_kernel<<<g, AS_THREADS, 0, st>>>(AsCnt(const_cast<void*>(count_table), cap), cutoff, V.E, V.kf, V.counts);
  CTR_LAUNCHED("ctr_aliccp_sample_vocab(compact)");
  // kept fids: sorted (8 passes cover k0 < 2^64), unique -> vocab
  uint64_t* sk;
  if (int rc = lsd_sort(V.kf, nullptr, V.keys2, nullptr, V.counts + 1, cap, 8, V.hist, V.hist_count, st,
                        "ctr_aliccp_sample_vocab(sort)", &sk, nullptr))
    return rc;
  as_heads_kernel<<<g, AS_THREADS, 0, st>>>(sk, V.counts + 1, V.head);
  CTR_LAUNCHED("ctr_aliccp_sample_vocab(heads)");
  if (int rc = cta_scan({V.head}, {V.n_vocab}, V.counts + 1, 0, st, "ctr_aliccp_sample_vocab(scan)")) return rc;
  as_unique_kernel<<<g, AS_THREADS, 0, st>>>(sk, V.counts + 1, V.head, vocab);
  CTR_LAUNCHED("ctr_aliccp_sample_vocab(unique)");
  // entries: LSD by fid, then field bytes 8..15, then field bytes 0..7
  lsd_iota_kernel<<<g, AS_THREADS, 0, st>>>(V.perm, V.counts);
  CTR_LAUNCHED("ctr_aliccp_sample_vocab(iota)");
  const uint64_t* words[3] = {V.E.k0, V.E.k2, V.E.k1};
  uint32_t* p = V.perm;
  for (int w = 0; w < 3; ++w) {
    lsd_gather_kernel<<<g, AS_THREADS, 0, st>>>(words[w], p, V.counts, V.keys);
    CTR_LAUNCHED("ctr_aliccp_sample_vocab(gather)");
    uint32_t* other = p == V.perm ? V.perm2 : V.perm;
    if (int rc = lsd_sort(V.keys, p, V.keys2, other, V.counts, cap, 8, V.hist, V.hist_count, st,
                          "ctr_aliccp_sample_vocab(sort)", &sk, &p)) return rc;
  }
  if (p != V.perm) {
    CTR_REQUIRE(cudaMemcpyAsync(V.perm, p, (size_t)cap * 4, cudaMemcpyDeviceToDevice, st) == cudaSuccess, CTR_ERR_CUDA,
                "ctr_aliccp_sample_vocab: copy failed");
  }
  as_feat_cnts_kernel<false><<<g, AS_THREADS, 0, st>>>(V.E, V.perm, V.counts, V.lens, nullptr);
  CTR_LAUNCHED("ctr_aliccp_sample_vocab(feat_cnts)");
  if (int rc = cta_scan({V.lens}, {V.fc_bytes}, V.counts, 0, st, "ctr_aliccp_sample_vocab(scan)")) return rc;
  CTR_REQUIRE(cudaMemcpyAsync(info, V.counts, 5 * 8, cudaMemcpyDeviceToDevice, st) == cudaSuccess, CTR_ERR_CUDA,
              "ctr_aliccp_sample_vocab: copy of info failed");
  return CTR_OK;
}

int ctr_aliccp_sample_feat_cnts(char* out, const void* ws, size_t ws_bytes, int64_t count_capacity,
                                ctr_stream_t stream) {
  CTR_REQUIRE(out && count_capacity > 0 && count_capacity <= KT_MAX_CAP, CTR_ERR_INVALID_ARG,
              "ctr_aliccp_sample_feat_cnts: bad arguments");
  CTR_REQUIRE(ws && ws_bytes >= ctr_aliccp_sample_vocab_workspace_bytes(count_capacity), CTR_ERR_WORKSPACE,
              "ctr_aliccp_sample_feat_cnts: workspace too small");
  AsVocabWs V(const_cast<void*>(ws), count_capacity);
  as_feat_cnts_kernel<true><<<grid_for(count_capacity, AS_THREADS, 16), AS_THREADS, 0, as_stream(stream)>>>(
      V.E, V.perm, V.counts, V.lens, out);
  CTR_LAUNCHED("ctr_aliccp_sample_feat_cnts");
  return CTR_OK;
}

int ctr_aliccp_sample_render(const uint8_t* arena, const int64_t* rec_off, const int32_t* rec_len,
                             const uint32_t* mult, int64_t n_records, const uint64_t* vocab, int64_t n_vocab,
                             int64_t* r_off, char* out, ctr_stream_t stream) {
  CTR_REQUIRE(n_records >= 0 && n_vocab >= 0 && r_off && (n_vocab == 0 || vocab) &&
                  (n_records == 0 || (arena && rec_off && rec_len && mult)),
              CTR_ERR_INVALID_ARG, "ctr_aliccp_sample_render: bad arguments");
  cudaStream_t st = as_stream(stream);
  const unsigned g = grid_for(n_records, AS_WARPS, 16);
  if (!out) {   // plan: r_off[0, n_records] = the exclusive scan of the rendered lengths
    if (int rc = as_zero(r_off + n_records, 8, st, "ctr_aliccp_sample_render")) return rc;
    if (n_records) {
      as_render_kernel<false><<<g, AS_THREADS, 0, st>>>(arena, rec_off, rec_len, mult, n_records, vocab, n_vocab, r_off,
                                                        nullptr);
      CTR_LAUNCHED("ctr_aliccp_sample_render(plan)");
    }
    return cta_scan({r_off}, {nullptr}, nullptr, n_records + 1, st, "ctr_aliccp_sample_render(scan)");
  }
  if (n_records == 0) return CTR_OK;
  as_render_kernel<true><<<g, AS_THREADS, 0, st>>>(arena, rec_off, rec_len, mult, n_records, vocab, n_vocab, r_off, out);
  CTR_LAUNCHED("ctr_aliccp_sample_render(write)");
  return CTR_OK;
}

int ctr_aliccp_sample_emit(const char* text, size_t len, int64_t n_lines, int64_t line_base, uint64_t seed,
                           const int32_t* s_rec, int64_t sample_base, const int64_t* r_off, const char* rendered,
                           const uint64_t* vocab, int64_t n_vocab, int64_t* s_val, int64_t lo, int64_t hi, char* out,
                           int64_t* info, void* ws, size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE((len == 0 || text) && n_lines >= 0 && line_base >= 0 && sample_base >= 0 && s_rec && r_off && s_val &&
                  n_vocab >= 0 && (n_vocab == 0 || vocab) && (out || info) && lo >= 0 && hi >= lo,
              CTR_ERR_INVALID_ARG, "ctr_aliccp_sample_emit: bad arguments");
  CTR_REQUIRE(len < AS_MAX_LEN, CTR_ERR_INVALID_ARG, "ctr_aliccp_sample_emit: chunk too large (len < 2^30)");
  CTR_REQUIRE(ws && ws_bytes >= ctr_aliccp_sample_chunk_workspace_bytes(len, n_lines), CTR_ERR_WORKSPACE,
              "ctr_aliccp_sample_emit: workspace too small");
  cudaStream_t st = as_stream(stream);
  if (!out)
    if (int rc = as_zero(info, 8, st, "ctr_aliccp_sample_emit")) return rc;
  if (len == 0) return CTR_OK;
  AsChunkWs W(ws, len, n_lines);
  const uint8_t* t = reinterpret_cast<const uint8_t*>(text);
  CTR_REQUIRE(cudaMemsetAsync(W.info, 0, AI_N * 8, st) == cudaSuccess &&
                  cudaMemsetAsync(W.info + AI_ERR, 0xFF, 8, st) == cudaSuccess &&
                  cudaMemsetAsync(W.n_newlines, 0, 16, st) == cudaSuccess,
              CTR_ERR_CUDA, "ctr_aliccp_sample_emit: memset failed");
  if (int rc = W.launch(t, len, st, "ctr_aliccp_sample_emit(lines)")) return rc;
  const unsigned g = grid_for(n_lines, AS_WARPS, 16);
  as_classify_kernel<<<g, AS_THREADS, 0, st>>>(t, (int64_t)len, W.line_start, W.n_newlines, n_lines, 0, AsCnt(),
                                               AsMd5(), W.P, W.info);
  CTR_LAUNCHED("ctr_aliccp_sample_emit(classify)");
  if (int rc = cta_scan({W.P.sord}, {nullptr}, W.info + AI_LINES, 0, st, "ctr_aliccp_sample_emit(scan)")) return rc;
  AsEmitArgs a{seed, line_base, sample_base, s_rec, r_off, rendered, vocab, n_vocab, s_val, lo, hi, out, info};
  if (out)
    as_emit_kernel<true><<<g, AS_THREADS, 0, st>>>(t, (int64_t)len, W.line_start, W.n_newlines, W.info, W.P, a);
  else
    as_emit_kernel<false><<<g, AS_THREADS, 0, st>>>(t, (int64_t)len, W.line_start, W.n_newlines, W.info, W.P, a);
  CTR_LAUNCHED("ctr_aliccp_sample_emit");
  return CTR_OK;
}

size_t ctr_aliccp_sample_order_workspace_bytes(int64_t n_samples) {
  return n_samples >= 0 ? AsOrderWs(nullptr, n_samples).bytes : 0;
}

int ctr_aliccp_sample_order(uint64_t* s_key, int64_t* s_val, int64_t n_samples, int64_t parts, int64_t* part_bytes,
                            void* ws, size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE(n_samples >= 0 && n_samples <= INT32_MAX && parts >= 1 && parts <= (1 << 20) && part_bytes &&
                  (n_samples == 0 || (s_key && s_val)),
              CTR_ERR_INVALID_ARG, "ctr_aliccp_sample_order: bad arguments");
  CTR_REQUIRE(ws && ws_bytes >= ctr_aliccp_sample_order_workspace_bytes(n_samples), CTR_ERR_WORKSPACE,
              "ctr_aliccp_sample_order: workspace too small");
  cudaStream_t st = as_stream(stream);
  if (int rc = as_zero(part_bytes, (size_t)parts * 8, st, "ctr_aliccp_sample_order")) return rc;
  if (n_samples == 0) return CTR_OK;
  AsOrderWs O(ws, n_samples);
  CTR_REQUIRE(cudaMemcpyAsync(O.n_dev, &n_samples, 8, cudaMemcpyHostToDevice, st) == cudaSuccess, CTR_ERR_CUDA,
              "ctr_aliccp_sample_order: copy failed");
  int bits = 31;
  while (((int64_t)1 << (bits - 31)) < parts) ++bits;
  const int passes = (bits + 7) / 8;
  const unsigned g = grid_for(n_samples, AS_THREADS, 16);
  lsd_iota_kernel<<<g, AS_THREADS, 0, st>>>(O.perm, O.n_dev);
  CTR_LAUNCHED("ctr_aliccp_sample_order(iota)");
  uint64_t* sk;
  uint32_t* sp;
  if (int rc = lsd_sort(s_key, O.perm, O.keys2, O.perm2, O.n_dev, n_samples, passes, O.hist, O.hist_count, st,
                        "ctr_aliccp_sample_order(sort)", &sk, &sp))
    return rc;
  as_sizes_sorted_kernel<<<g, AS_THREADS, 0, st>>>(sk, sp, s_val, n_samples, O.sz, part_bytes);
  CTR_LAUNCHED("ctr_aliccp_sample_order(sizes)");
  if (int rc = cta_scan({O.sz}, {nullptr}, O.n_dev, 0, st, "ctr_aliccp_sample_order(scan)")) return rc;
  as_offsets_kernel<<<g, AS_THREADS, 0, st>>>(sp, O.sz, n_samples, s_val);
  CTR_LAUNCHED("ctr_aliccp_sample_order(offsets)");
  return CTR_OK;
}

}  // extern "C"
