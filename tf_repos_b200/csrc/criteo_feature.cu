// criteo_feature.cu -- Criteo raw TSV -> libsvm feature pipeline on the GPU (Feature_pipeline/get_criteo_feature.py).
//
// Three passes, each over text chunks cut at line ends (the host reads the files; only the count table and the
// vocabulary stay resident):
//   stats  one thread per train line: the 13 integer columns fold their clipped min/max into int64[26] (shared-memory
//          atomics per CTA, then global atomics: exact and order-free); the 26 categorical values count into an
//          open-addressing table keyed by (field, 8-byte key) (probe policy: key_table.cuh).
//   vocab  keep count >= cutoff, LSD radix sort by (field, -count, key) (13 passes of 8 bits over 104 key bits),
//          write each id back into its table slot.
//   emit   plan: one thread per line computes its output length (and raises what the reference raises); the tile
//          sums are scanned; write: the same thread formats its line at its offset in the tr or va buffer.
// Every order comes from a sort or a scan, every reduction is an integer one: two runs give the same bytes.
//
// Line grammar (get_criteo_feature.py:42,77,135,156): split on '\t' after dropping the '\n'; train lines are
// label, I1..I13, C1..C26; test lines have no label; columns beyond those are ignored.
// Restrictions (DESIGN.md §2.4; each raises): I values match [+-]?[0-9]+ with magnitude <= 2^53; train C values are
// at most 8 bytes, hold no NUL and are not "<unk>", so a value packs big-endian, zero-padded into a uint64 whose
// numeric order is Python's bytewise string order and 0 never is a key.
#include "key_table.cuh"
#include "line_starts.cuh"

namespace ctr {

constexpr int CF_NI = 13, CF_NC = 26, CF_COLS = 1 + CF_NI + CF_NC;
constexpr int CF_THREADS = 256;                       // per-line kernels: one line per thread, one tile per CTA
constexpr uint64_t CF_UNK = 0x3C756E6B3E000000ull;    // "<unk>" packed
constexpr int64_t CF_MAXSIZE = 0x7FFFFFFFFFFFFFFFll;  // Python 2's sys.maxsize on LP64

__constant__ int64_t kClip[CF_NI] = {20, 600, 100, 50, 64000, 500, 100, 50, 500, 10, 10, 10, 50};

// error word: (class << 62) | (line << 16) | (column << 8) | code; the smallest one wins (atomicMin).  class 0 = the
// reference's min/max pass (continuous columns), class 1 = its dictionary pass, so a min/max error anywhere in the
// file comes first, as it does in the reference.
enum { CF_E_COLUMNS = 1, CF_E_NOT_INT = 2, CF_E_RANGE = 3, CF_E_KEY_LONG = 4, CF_E_KEY_NUL = 5, CF_E_KEY_UNK = 6,
       CF_E_ZERO_DIV = 7 };
__device__ __forceinline__ uint64_t cf_err(int cls, int64_t line, int col, int code) {
  return ((uint64_t)cls << 62) | ((uint64_t)line << 16) | ((uint64_t)col << 8) | (uint64_t)code;
}

// ---- count table: keys uint64[cap] | tags uint32[cap] (field + 1, 0 = empty) | vals uint32[cap] ----------------
// vals holds the count after the stats pass and the id (0 = <unk>) after the vocab pass.
struct CfTable {
  uint64_t* keys;
  uint32_t* tags;
  uint32_t* vals;
  int64_t cap;
  CfTable() = default;
  __host__ __device__ CfTable(void* base, int64_t c)
      : keys(reinterpret_cast<uint64_t*>(base)),
        tags(reinterpret_cast<uint32_t*>(reinterpret_cast<uint64_t*>(base) + c)),
        vals(reinterpret_cast<uint32_t*>(reinterpret_cast<uint64_t*>(base) + c) + c),
        cap(c) {}
};

__device__ __forceinline__ uint64_t cf_hash(uint64_t key, int f) {
  return splitmix64_finalize(key ^ ((uint64_t)(f + 1) * 0x9E3779B97F4A7C15ull));
}

// (f, key) owns the slot whose key word is key and whose tag word is f + 1; both are claimed in that order
// (key_table.cuh).
__device__ __forceinline__ bool cf_insert(const CfTable& T, uint64_t key, int f) {
  const uint32_t tag = (uint32_t)f + 1;
  const int64_t slot = probe(cf_hash(key, f), T.cap, [&](uint64_t s) {
    return claim(T.keys + s, key) == key && claim(T.tags + s, tag) == tag;
  });
  if (slot >= 0) atomicAdd(T.vals + slot, 1u);
  return slot >= 0;
}

__device__ __forceinline__ uint32_t cf_lookup(const CfTable& T, uint64_t key, int f) {
  const uint32_t tag = (uint32_t)f + 1;
  uint32_t v = 0;
  probe(cf_hash(key, f), T.cap, [&](uint64_t s) {
    const uint64_t k = T.keys[s];
    const bool hit = k == key && T.tags[s] == tag;
    if (hit) v = T.vals[s];
    return k == 0 || hit;
  });
  return v;
}

// ---- tokens --------------------------------------------------------------------------------------------------
// [+-]?[0-9]+ with magnitude <= 2^53 -> 0 and (neg, mag); CF_E_NOT_INT / CF_E_RANGE otherwise
__device__ __forceinline__ int cf_parse_int(const unsigned char* __restrict__ t, int64_t q, int64_t e, bool& neg,
                                            int64_t& mag) {
  neg = false;
  if (q < e && (t[q] == '+' || t[q] == '-')) { neg = t[q] == '-'; ++q; }
  if (q == e) return CF_E_NOT_INT;
  mag = 0;
  bool big = false;
  for (; q < e; ++q) {
    const unsigned d = (unsigned)t[q] - '0';
    if (d > 9) return CF_E_NOT_INT;
    if (!big) { mag = mag * 10 + d; big = mag > (1ll << 53); }
  }
  return big ? CF_E_RANGE : 0;
}

// value of [q, e) packed big-endian and zero-padded -> 0, or the restriction it breaks
__device__ __forceinline__ int cf_pack_key(const unsigned char* __restrict__ t, int64_t q, int64_t e, uint64_t& key) {
  if (e - q > 8) return CF_E_KEY_LONG;
  key = 0;
  for (int i = 0; q + i < e; ++i) {
    const unsigned c = t[q + i];
    if (c == 0) return CF_E_KEY_NUL;
    key |= (uint64_t)c << (56 - 8 * i);
  }
  return key == CF_UNK ? CF_E_KEY_UNK : 0;
}

__device__ __forceinline__ int64_t cf_col_end(const unsigned char* __restrict__ t, int64_t q, int64_t e) {
  while (q < e && t[q] != '\t') ++q;
  return q;
}

// ---- formatting ----------------------------------------------------------------------------------------------
// "{:.6f}".format(q).rstrip('0').rstrip('.'): the exact binary value of q rounded half-to-even at 1e-6.
// q = m * 2^s; the integer part is m >> -s and the fraction fm / 2^-s is scaled by 10^6 in 128-bit integers.
// In this pipeline |q| < 2^55 (|v - min| <= 2^54, |max - min| >= 1; min = sys.maxsize gives |q| ~ 0.5).
template <bool W>
__device__ __forceinline__ int cf_put_fixed6(double q, char* o) {
  const uint64_t bits = (uint64_t)__double_as_longlong(q);
  const int ex = (int)((bits >> 52) & 0x7FF);
  const uint64_t m = (bits & 0xFFFFFFFFFFFFFull) | (ex ? (1ull << 52) : 0ull);
  const int s = (ex ? ex : 1) - 1075;
  uint64_t ip, fr = 0;
  if (s >= 0) {
    ip = m << s;
  } else {
    const int r = -s;
    uint64_t fm;
    if (r < 64) { ip = m >> r; fm = m & ((1ull << r) - 1); } else { ip = 0; fm = m; }
    if (r < 100) {   // fm * 10^6 < 2^73: from 2^-100 down the scaled fraction is below one half (and no tie)
      const unsigned __int128 F = (unsigned __int128)fm * 1000000u;
      const unsigned __int128 qq = F >> r, rem = F - (qq << r), half = (unsigned __int128)1 << (r - 1);
      fr = (uint64_t)qq;
      if (rem > half || (rem == half && (fr & 1))) ++fr;   // 10^6 is even: the parity of the whole result is fr's
      if (fr == 1000000) { fr = 0; ++ip; }
    }
  }
  int n = 0;
  if (bits >> 63) { if (W) o[n] = '-'; ++n; }
  n += put_dec<W>(ip, o + n);
  if (fr) {
    int nd = 6;
    while (fr % 10 == 0) { fr /= 10; --nd; }
    if (W) {
      o[n] = '.';
      for (int i = nd; i >= 1; --i) { o[n + i] = (char)('0' + fr % 10); fr /= 10; }
    }
    n += 1 + nd;
  }
  return n;
}

struct CfEmitArgs {
  CfTable table;
  const double* num_min;    // [13] float(min_i)
  const double* num_den;    // [13] float(max_i - min_i)
  const int64_t* offsets;   // [26] categorical offsets (offset[0] = 13)
  const char* label;        // test mode: the label every line gets
  int label_len;
  int test;
};

// One output line (get_criteo_feature.py:135-151 train, :156-167 test).  Returns its length; W = write it to o.
// Sets err (plan pass) for what the reference raises on this line: IndexError (too few columns), ValueError (I value
// not an integer; here also the restriction), ZeroDivisionError (max == min and a non-empty I value).
template <bool W>
__device__ int64_t cf_emit_line(const unsigned char* __restrict__ t, int64_t p, int64_t e, const CfEmitArgs& a,
                                int64_t line, uint64_t& err, char* o) {
  int64_t n = 0;
  const int shift = a.test ? 1 : 0, ncols = CF_COLS - shift;
  if (a.test) {
    if (W) for (int i = 0; i < a.label_len; ++i) o[i] = a.label[i];
    n = a.label_len;
  }
  int col = 0;
  int64_t q = p;
  for (;;) {
    const int64_t ce = cf_col_end(t, q, e);
    const int j = col + shift;   // 0 = label, 1..13 = I, 14..39 = C
    if (j == 0) {
      if (W) for (int64_t i = q; i < ce; ++i) o[n + i - q] = (char)t[i];
      n += ce - q;
    } else if (j <= CF_NI) {
      if (W) o[n] = ' ';
      n += 1 + put_dec<W>((uint64_t)j, o + n + 1);
      if (W) o[n] = ':';
      ++n;
      double v = 0.0;
      if (ce > q) {
        bool neg;
        int64_t mag;
        const int code = cf_parse_int(t, q, ce, neg, mag);
        if (code) { err = cf_err(0, line, col, code); return n; }
        const double den = a.num_den[j - 1];
        if (den == 0.0) { err = cf_err(0, line, col, CF_E_ZERO_DIV); return n; }
        const double x = neg ? -(double)mag : (double)mag;   // float("-0") is -0.0
        v = __ddiv_rn(__dsub_rn(x, a.num_min[j - 1]), den);
      }
      n += cf_put_fixed6<W>(v, o + n);
    } else {
      const int f = j - 1 - CF_NI;
      uint64_t key;
      // values the train dictionary cannot hold (empty, > 8 bytes, NUL, "<unk>") are <unk> = 0, as in the reference
      const uint32_t id = (ce > q && cf_pack_key(t, q, ce, key) == 0) ? cf_lookup(a.table, key, f) : 0u;
      if (W) o[n] = ' ';
      n += 1 + put_dec<W>((uint64_t)(a.offsets[f] + id), o + n + 1);
      if (W) { o[n] = ':'; o[n + 1] = '1'; }
      n += 2;
    }
    ++col;
    if (ce >= e || col == ncols) break;
    q = ce + 1;
  }
  if (col < ncols) { err = cf_err(0, line, col, CF_E_COLUMNS); return n; }
  if (W) o[n] = '\n';
  return n + 1;
}

// ---- kernels -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(CF_THREADS) cf_stats_kernel(const unsigned char* __restrict__ t, int64_t len,
                                                             const int64_t* __restrict__ line_start,
                                                             const int64_t* __restrict__ n_newlines, int64_t line_base,
                                                             CfTable table, int64_t* __restrict__ minmax,
                                                             int64_t* __restrict__ info) {
  __shared__ long long smin[CF_NI], smax[CF_NI];
  if (threadIdx.x < CF_NI) { smin[threadIdx.x] = CF_MAXSIZE; smax[threadIdx.x] = -CF_MAXSIZE; }
  __syncthreads();
  const int64_t nn = n_newlines[0], n_lines = chunk_lines(t, len, nn);
  if (blockIdx.x == 0 && threadIdx.x == 0) info[0] = n_lines;
  for (int64_t row = (int64_t)blockIdx.x * CF_THREADS + threadIdx.x; row < n_lines;
       row += (int64_t)gridDim.x * CF_THREADS) {
    int64_t p, e;
    line_bounds(line_start, nn, len, row, p, e);
    const int64_t line = line_base + row;
    uint64_t err = ~0ull;
    int col = 0;
    int64_t q = p;
    for (;;) {
      const int64_t ce = cf_col_end(t, q, e);
      if (col >= 1 && col <= CF_NI) {   // :77-85
        if (ce > q) {
          bool neg;
          int64_t mag;
          const int code = cf_parse_int(t, q, ce, neg, mag);
          if (code) { err = cf_err(0, line, col, code); break; }
          int64_t v = neg ? -mag : mag;
          if (v > kClip[col - 1]) v = kClip[col - 1];
          atomicMin(&smin[col - 1], (long long)v);
          atomicMax(&smax[col - 1], (long long)v);
        }
      } else if (col > CF_NI && ce > q) {   // :42-45
        uint64_t key;
        const int code = cf_pack_key(t, q, ce, key);
        if (code) { err = cf_err(1, line, col, code); break; }
        if (!cf_insert(table, key, col - 1 - CF_NI))
          atomicAdd(reinterpret_cast<unsigned long long*>(&info[2]), 1ull);
      }
      ++col;
      if (ce >= e || col == CF_COLS) break;
      q = ce + 1;
    }
    if (err == ~0ull && col < CF_COLS) err = cf_err(col <= CF_NI ? 0 : 1, line, col, CF_E_COLUMNS);
    if (err != ~0ull) atomicMin(reinterpret_cast<unsigned long long*>(&info[1]), (unsigned long long)err);
  }
  __syncthreads();
  if (threadIdx.x < CF_NI) {
    atomicMin(reinterpret_cast<long long*>(&minmax[threadIdx.x]), smin[threadIdx.x]);
    atomicMax(reinterpret_cast<long long*>(&minmax[CF_NI + threadIdx.x]), smax[threadIdx.x]);
  }
}

// per line: output length; per tile of CF_THREADS lines: tr bytes, va bytes, tr lines
__global__ void __launch_bounds__(CF_THREADS) cf_plan_kernel(const unsigned char* __restrict__ t, int64_t len,
                                                            const int64_t* __restrict__ line_start,
                                                            const int64_t* __restrict__ n_newlines, int64_t line_base,
                                                            const uint8_t* __restrict__ to_train, CfEmitArgs a,
                                                            int32_t* __restrict__ line_len, int64_t* __restrict__ tile_tr,
                                                            int64_t* __restrict__ tile_va, int64_t* __restrict__ tile_trn,
                                                            int64_t* __restrict__ n_tiles, int64_t* __restrict__ info) {
  const int64_t nn = n_newlines[0], n_lines = chunk_lines(t, len, nn);
  if (blockIdx.x == 0 && threadIdx.x == 0) { info[0] = n_lines; n_tiles[0] = (n_lines + CF_THREADS - 1) / CF_THREADS; }
  for (int64_t tile = blockIdx.x; tile * CF_THREADS < n_lines; tile += gridDim.x) {
    const int64_t row = tile * CF_THREADS + threadIdx.x;
    int64_t L = 0;
    bool tr = true;
    if (row < n_lines) {
      int64_t p, e;
      line_bounds(line_start, nn, len, row, p, e);
      uint64_t err = ~0ull;
      L = cf_emit_line<false>(t, p, e, a, line_base + row, err, nullptr);
      if (err != ~0ull) atomicMin(reinterpret_cast<unsigned long long*>(&info[1]), (unsigned long long)err);
      line_len[row] = (int32_t)L;
      tr = a.test || to_train[row];
    }
    int64_t x[2] = {tr ? L : 0, tr ? 0 : L}, s[2];   // tr bytes, va bytes
    block_scan_excl<CF_THREADS>(x, s);
    const int n_tr = __syncthreads_count(row < n_lines && tr);
    if (threadIdx.x == 0) { tile_tr[tile] = s[0]; tile_va[tile] = s[1]; tile_trn[tile] = n_tr; }
  }
}

__global__ void __launch_bounds__(CF_THREADS) cf_write_kernel(const unsigned char* __restrict__ t, int64_t len,
                                                             const int64_t* __restrict__ line_start,
                                                             const int64_t* __restrict__ n_newlines,
                                                             const uint8_t* __restrict__ to_train, CfEmitArgs a,
                                                             const int32_t* __restrict__ line_len,
                                                             const int64_t* __restrict__ tile_tr,
                                                             const int64_t* __restrict__ tile_va, char* __restrict__ out_tr,
                                                             char* __restrict__ out_va) {
  const int64_t nn = n_newlines[0], n_lines = chunk_lines(t, len, nn);
  for (int64_t tile = blockIdx.x; tile * CF_THREADS < n_lines; tile += gridDim.x) {
    const int64_t row = tile * CF_THREADS + threadIdx.x;
    const bool live = row < n_lines, tr = !live || a.test || to_train[row];
    const int64_t L = live ? line_len[row] : 0;
    int64_t x[2] = {tr ? L : 0, tr ? 0 : L}, s[2];   // tr bytes, va bytes
    block_scan_excl<CF_THREADS>(x, s);
    if (live) {
      int64_t p, e;
      line_bounds(line_start, nn, len, row, p, e);
      uint64_t err = ~0ull;
      char* o = tr ? out_tr + tile_tr[tile] + x[0] : out_va + tile_va[tile] + x[1];
      cf_emit_line<true>(t, p, e, a, row, err, o);
    }
  }
}

// ---- vocabulary ----------------------------------------------------------------------------------------------
// kept slots -> (lo = key, hi = field << 32 | ~count, slot); vals are cleared to the <unk> id 0
__global__ void __launch_bounds__(CF_THREADS) vc_compact_kernel(CfTable T, int64_t cutoff, uint64_t* __restrict__ lo,
                                                               uint64_t* __restrict__ hi, uint32_t* __restrict__ sl,
                                                               int64_t* __restrict__ n_kept,
                                                               int64_t* __restrict__ field_counts) {
  __shared__ int cnt[CF_NC];
  if (threadIdx.x < CF_NC) cnt[threadIdx.x] = 0;
  __syncthreads();
  const int64_t stride = (int64_t)gridDim.x * CF_THREADS, n_iter = (T.cap + stride - 1) / stride;
  for (int64_t it = 0; it < n_iter; ++it) {   // uniform trip count: the warp-aggregated atomic below needs whole warps
    const int64_t s = (it * gridDim.x + blockIdx.x) * CF_THREADS + threadIdx.x;
    bool keep = false;
    uint32_t tag = 0, c = 0;
    if (s < T.cap) {
      tag = T.tags[s];
      if (tag) {
        c = T.vals[s];
        T.vals[s] = 0;
        keep = (int64_t)c >= cutoff;
      }
    }
    const uint32_t ballot = __ballot_sync(FULL_MASK, keep);
    unsigned long long base = 0;
    if ((threadIdx.x & 31) == 0 && ballot)
      base = atomicAdd(reinterpret_cast<unsigned long long*>(n_kept), (unsigned long long)__popc(ballot));
    base = __shfl_sync(FULL_MASK, base, 0);
    if (keep) {
      const int64_t pos = (int64_t)base + __popc(ballot & ((1u << (threadIdx.x & 31)) - 1));
      lo[pos] = T.keys[s];
      hi[pos] = ((uint64_t)(tag - 1) << 32) | (uint64_t)(0xFFFFFFFFu - c);
      sl[pos] = (uint32_t)s;
      atomicAdd(&cnt[tag - 1], 1);
    }
  }
  __syncthreads();
  if (threadIdx.x < CF_NC && cnt[threadIdx.x])
    atomicAdd(reinterpret_cast<unsigned long long*>(&field_counts[threadIdx.x]), (unsigned long long)cnt[threadIdx.x]);
}

// The kept items in (hi, lo) order: hi_s = the sorted hi words, lo_s = the lo words sorted alone, order[p] = the
// position in lo_s of sorted item p, by_lo[q] = the compaction index of lo_s[q].  Sorted position p of field f ->
// id p - start(f) + 1, written into the item's slot; its key -> vocab_keys[p]
__global__ void __launch_bounds__(CF_THREADS) vc_assign_kernel(CfTable T, const uint64_t* __restrict__ lo_s,
                                                              const uint64_t* __restrict__ hi_s,
                                                              const uint32_t* __restrict__ sl,
                                                              const uint32_t* __restrict__ by_lo,
                                                              const uint32_t* __restrict__ order,
                                                              const int64_t* __restrict__ n_kept,
                                                              const int64_t* __restrict__ field_counts,
                                                              uint64_t* __restrict__ vocab_keys) {
  __shared__ int64_t start[CF_NC];
  if (threadIdx.x == 0) {
    int64_t s = 0;
    for (int f = 0; f < CF_NC; ++f) { start[f] = s; s += field_counts[f]; }
  }
  __syncthreads();
  const int64_t n = n_kept[0];
  for (int64_t p = (int64_t)blockIdx.x * CF_THREADS + threadIdx.x; p < n; p += (int64_t)gridDim.x * CF_THREADS) {
    const int f = (int)(hi_s[p] >> 32);
    const uint32_t q = order[p];
    T.vals[sl[by_lo[q]]] = (uint32_t)(p - start[f] + 1);
    vocab_keys[p] = lo_s[q];
  }
}

// ---- workspace layouts -----------------------------------------------------------------------------------------
// emit: LineStarts (max_rows = len + 1) | line_len int32[len + 1] | tile_tr, tile_va, tile_trn int64[nt] |
// n_tiles int64[2]
struct CfEmitWs : LineStarts {
  int32_t* line_len;
  int64_t *tile_tr, *tile_va, *tile_trn, *n_tiles;
  CfEmitWs(void* ws, size_t len) : LineStarts(ws, len, (int64_t)len + 1) {
    uint8_t* b = reinterpret_cast<uint8_t*>(ws);
    const size_t nt = (len + 1 + CF_THREADS - 1) / CF_THREADS;
    size_t o = bytes;
    line_len = reinterpret_cast<int32_t*>(b + o); o += align256((len + 1) * 4);
    tile_tr = reinterpret_cast<int64_t*>(b + o); o += align256(nt * 8);
    tile_va = reinterpret_cast<int64_t*>(b + o); o += align256(nt * 8);
    tile_trn = reinterpret_cast<int64_t*>(b + o); o += align256(nt * 8);
    n_tiles = reinterpret_cast<int64_t*>(b + o); o += align256(16);
    bytes = o;
  }
};

// vocab: n_kept, hist_count int64 | hist int32[256 * nb] | lo, hi, keys2 uint64[cap] | sl, by_lo, order, perm2
// uint32[cap] (one aligned block, so that the whole stays within 40 B per slot)
struct CfVocabWs {
  int64_t *n_kept, *hist_count;
  int32_t* hist;
  uint64_t *lo, *hi, *keys2;
  uint32_t *sl, *by_lo, *order, *perm2;
  size_t bytes;
  CfVocabWs(void* ws, int64_t cap) {
    uint8_t* b = reinterpret_cast<uint8_t*>(ws);
    const size_t nb = (size_t)ceil_div64(cap, LSD_TILE), c = (size_t)cap;
    size_t o = 0;
    n_kept = reinterpret_cast<int64_t*>(b + o); hist_count = n_kept + 1; o += align256(16);
    hist = reinterpret_cast<int32_t*>(b + o); o += align256(256 * nb * 4);
    lo = reinterpret_cast<uint64_t*>(b + o); o += align256(c * 8);
    hi = reinterpret_cast<uint64_t*>(b + o); o += align256(c * 8);
    keys2 = reinterpret_cast<uint64_t*>(b + o); o += align256(c * 8);
    sl = reinterpret_cast<uint32_t*>(b + o); by_lo = sl + c; order = by_lo + c; perm2 = order + c;
    o += align256(c * 16);
    bytes = o;
  }
};

// chunk buffers the per-line kernels accept: len < 2^30 keeps block offsets and line lengths in int32
constexpr size_t CF_MAX_LEN = (size_t)1 << 30;

}  // namespace ctr

using namespace ctr;

extern "C" {

size_t ctr_criteo_table_bytes(int64_t capacity) { return capacity > 0 ? (size_t)capacity * 16 : 0; }

size_t ctr_criteo_stats_workspace_bytes(size_t len) { return LineStarts(nullptr, len, (int64_t)len + 1).bytes; }

int ctr_criteo_stats(const char* text, size_t len, int64_t line_base, void* table, int64_t capacity, int64_t* minmax,
                     int64_t* info, void* ws, size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE(info && minmax && table && capacity > 0 && line_base >= 0 && (len == 0 || text), CTR_ERR_INVALID_ARG,
              "ctr_criteo_stats: bad arguments");
  CTR_REQUIRE(capacity <= KT_MAX_CAP, CTR_ERR_INVALID_ARG, "ctr_criteo_stats: capacity > 2^31");
  CTR_REQUIRE(len < CF_MAX_LEN, CTR_ERR_INVALID_ARG, "ctr_criteo_stats: chunk too large (len < 2^30)");
  CTR_REQUIRE(ws && ws_bytes >= ctr_criteo_stats_workspace_bytes(len), CTR_ERR_WORKSPACE,
              "ctr_criteo_stats: workspace too small");
  cudaStream_t st = as_stream(stream);
  CTR_REQUIRE(cudaMemsetAsync(info, 0, 3 * sizeof(int64_t), st) == cudaSuccess &&
                  cudaMemsetAsync(info + 1, 0xFF, sizeof(int64_t), st) == cudaSuccess,
              CTR_ERR_CUDA, "ctr_criteo_stats: memset failed");
  if (len == 0) return CTR_OK;
  const unsigned char* t = reinterpret_cast<const unsigned char*>(text);
  const LineStarts L(ws, len, (int64_t)len + 1);
  if (int rc = L.launch(t, len, st, "ctr_criteo_stats(lines)")) return rc;
  cf_stats_kernel<<<grid_for((int64_t)len + 1, CF_THREADS, 16), CF_THREADS, 0, st>>>(
      t, (int64_t)len, L.line_start, L.n_newlines, line_base, CfTable(table, capacity), minmax, info);
  CTR_LAUNCHED("ctr_criteo_stats");
  return CTR_OK;
}

size_t ctr_criteo_vocab_workspace_bytes(int64_t capacity) {
  return capacity > 0 ? CfVocabWs(nullptr, capacity).bytes : 0;
}

int ctr_criteo_vocab(void* table, int64_t capacity, int64_t cutoff, uint64_t* vocab_keys, int64_t* field_counts,
                     void* ws, size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE(table && capacity > 0 && vocab_keys && field_counts, CTR_ERR_INVALID_ARG, "ctr_criteo_vocab: bad arguments");
  CTR_REQUIRE(capacity <= KT_MAX_CAP, CTR_ERR_INVALID_ARG, "ctr_criteo_vocab: capacity > 2^31");
  CTR_REQUIRE(ws && ws_bytes >= ctr_criteo_vocab_workspace_bytes(capacity), CTR_ERR_WORKSPACE,
              "ctr_criteo_vocab: workspace too small");
  cudaStream_t st = as_stream(stream);
  CfVocabWs V(ws, capacity);
  CfTable T(table, capacity);
  CTR_REQUIRE(cudaMemsetAsync(V.n_kept, 0, 16, st) == cudaSuccess &&
                  cudaMemsetAsync(field_counts, 0, CF_NC * sizeof(int64_t), st) == cudaSuccess,
              CTR_ERR_CUDA, "ctr_criteo_vocab: memset failed");
  const unsigned g = grid_for(capacity, CF_THREADS, 16);
  vc_compact_kernel<<<g, CF_THREADS, 0, st>>>(T, cutoff, V.lo, V.hi, V.sl, V.n_kept, field_counts);
  CTR_LAUNCHED("ctr_criteo_vocab(compact)");
  // (hi, lo) order from two stable sorts over the 13 digits of the 104 key bits: lo in place (8 passes, so the result
  // is back in lo / by_lo) carrying the compaction index, then hi gathered into that order and sorted (5 passes, hi's
  // own buffer as scratch) carrying the lo-sorted position
  lsd_iota_kernel<<<g, CF_THREADS, 0, st>>>(V.by_lo, V.n_kept);
  CTR_LAUNCHED("ctr_criteo_vocab(iota)");
  uint64_t *lo_s, *hi_s;
  uint32_t *by_lo, *order;
  if (int rc = lsd_sort(V.lo, V.by_lo, V.keys2, V.perm2, V.n_kept, capacity, 8, V.hist, V.hist_count, st,
                        "ctr_criteo_vocab(sort)", &lo_s, &by_lo))
    return rc;
  lsd_gather_kernel<<<g, CF_THREADS, 0, st>>>(V.hi, by_lo, V.n_kept, V.keys2);
  CTR_LAUNCHED("ctr_criteo_vocab(gather)");
  lsd_iota_kernel<<<g, CF_THREADS, 0, st>>>(V.order, V.n_kept);
  CTR_LAUNCHED("ctr_criteo_vocab(iota)");
  if (int rc = lsd_sort(V.keys2, V.order, V.hi, V.perm2, V.n_kept, capacity, 5, V.hist, V.hist_count, st,
                        "ctr_criteo_vocab(sort)", &hi_s, &order))
    return rc;
  vc_assign_kernel<<<g, CF_THREADS, 0, st>>>(T, lo_s, hi_s, V.sl, by_lo, order, V.n_kept, field_counts, vocab_keys);
  CTR_LAUNCHED("ctr_criteo_vocab(assign)");
  return CTR_OK;
}

size_t ctr_criteo_emit_workspace_bytes(size_t len) { return CfEmitWs(nullptr, len).bytes; }

static int cf_emit_args(const void* table, int64_t capacity, const double* num_min, const double* num_den,
                        const int64_t* offsets, const char* label, int label_len, int test, CfEmitArgs& a) {
  CTR_REQUIRE(table && capacity > 0 && capacity <= KT_MAX_CAP && num_min && num_den && offsets && label_len >= 0 &&
                  (label_len == 0 || label),
              CTR_ERR_INVALID_ARG, "ctr_criteo_emit: bad arguments");
  a = CfEmitArgs{CfTable(const_cast<void*>(table), capacity), num_min, num_den, offsets, label, label_len, test ? 1 : 0};
  return CTR_OK;
}

int ctr_criteo_emit_plan(const char* text, size_t len, int test, int64_t line_base, const uint8_t* to_train,
                         const void* table, int64_t capacity, const double* num_min, const double* num_den,
                         const int64_t* offsets, const char* label, int label_len, int64_t* info, void* ws,
                         size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE(info && line_base >= 0 && (len == 0 || text) && (test || to_train), CTR_ERR_INVALID_ARG,
              "ctr_criteo_emit_plan: bad arguments");
  CTR_REQUIRE(len < CF_MAX_LEN, CTR_ERR_INVALID_ARG, "ctr_criteo_emit_plan: chunk too large (len < 2^30)");
  CTR_REQUIRE(ws && ws_bytes >= ctr_criteo_emit_workspace_bytes(len), CTR_ERR_WORKSPACE,
              "ctr_criteo_emit_plan: workspace too small");
  CfEmitArgs a;
  if (int rc = cf_emit_args(table, capacity, num_min, num_den, offsets, label, label_len, test, a)) return rc;
  cudaStream_t st = as_stream(stream);
  CTR_REQUIRE(cudaMemsetAsync(info, 0, 5 * sizeof(int64_t), st) == cudaSuccess &&
                  cudaMemsetAsync(info + 1, 0xFF, sizeof(int64_t), st) == cudaSuccess,
              CTR_ERR_CUDA, "ctr_criteo_emit_plan: memset failed");
  if (len == 0) return CTR_OK;
  const unsigned char* t = reinterpret_cast<const unsigned char*>(text);
  const CfEmitWs E(ws, len);
  if (int rc = E.launch(t, len, st, "ctr_criteo_emit_plan(lines)")) return rc;
  cf_plan_kernel<<<grid_for((int64_t)len + 1, CF_THREADS, 16), CF_THREADS, 0, st>>>(
      t, (int64_t)len, E.line_start, E.n_newlines, line_base, to_train, a, E.line_len, E.tile_tr, E.tile_va, E.tile_trn,
      E.n_tiles, info);
  CTR_LAUNCHED("ctr_criteo_emit_plan");
  return cta_scan({E.tile_tr, E.tile_va, E.tile_trn}, {info + 3, info + 4, info + 2}, E.n_tiles, 0, st,
                  "ctr_criteo_emit_plan(scan)");
}

int ctr_criteo_emit_write(const char* text, size_t len, int test, const uint8_t* to_train, const void* table,
                          int64_t capacity, const double* num_min, const double* num_den, const int64_t* offsets,
                          const char* label, int label_len, char* out_tr, char* out_va, const void* ws,
                          size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE((len == 0 || text) && (test || to_train), CTR_ERR_INVALID_ARG, "ctr_criteo_emit_write: bad arguments");
  CTR_REQUIRE(len < CF_MAX_LEN, CTR_ERR_INVALID_ARG, "ctr_criteo_emit_write: chunk too large (len < 2^30)");
  CTR_REQUIRE(ws && ws_bytes >= ctr_criteo_emit_workspace_bytes(len), CTR_ERR_WORKSPACE,
              "ctr_criteo_emit_write: workspace too small");
  CfEmitArgs a;
  if (int rc = cf_emit_args(table, capacity, num_min, num_den, offsets, label, label_len, test, a)) return rc;
  if (len == 0) return CTR_OK;
  CfEmitWs E(const_cast<void*>(ws), len);
  cf_write_kernel<<<grid_for((int64_t)len + 1, CF_THREADS, 16), CF_THREADS, 0, as_stream(stream)>>>(
      reinterpret_cast<const unsigned char*>(text), (int64_t)len, E.line_start, E.n_newlines, to_train, a,
      E.line_len, E.tile_tr, E.tile_va, out_tr, out_va);
  CTR_LAUNCHED("ctr_criteo_emit_write");
  return CTR_OK;
}

}  // extern "C"
