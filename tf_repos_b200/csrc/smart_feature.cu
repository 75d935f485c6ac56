// smart_feature.cu -- the smart and Frappe feature stages on the GPU (deep_ctr/Feature_pipeline/get_smart_feature.py,
// get_frape_feature.py; DESIGN.md §2.12).
//
// smart: a 128-column CSV -> libsvm through a feature_map file of `key fid` lines.
//   map    the feature_map text, resident: one thread per line strips it, splits it on ' ' and classifies its key
//          (categorical `name|value`, or a continuous `name`; keys no lookup can reach are dropped); each kept key is
//          inserted into an open-addressing table (CAS on the slot's first line, full-key comparison against the
//          resident text; probe policy: key_table.cuh), the largest line of a key wins by atomicMax, then a second
//          pass fills each slot's spans.
//   emit   one warp per CSV line: strip (line_starts.cuh) and the commas by ballot; each lane formats the fields it
//          owns (a lookup per categorical field); plan = output bytes per line (a dropped line gives 0), a tiled scan,
//          write = each line at its offset.
//   build  get_feature_map with its NameError fixed: one warp per line inserts every key with the smallest global
//          position (line << 7 | column) by atomicMax of its complement; new keys are copied from the chunk into a
//          resident arena after each chunk; the keys are compacted, radix sorted by position and rendered with fids
//          129, 130, ... in that order.
// Frappe: one warp per line, the label rewrite on the same line-start / plan / scan / write skeleton.
// Every order comes from a sort or a scan and every reduction is an integer one: two runs give the same bytes.
#include "key_table.cuh"
#include "line_starts.cuh"

namespace ctr {

constexpr int SF_THREADS = 256, SF_WARPS = SF_THREADS / 32;
constexpr int SF_COLS = 128, SF_NAMED = 28, SF_CONT_LO = 11, SF_CONT_HI = 27, SF_NCONT = SF_CONT_HI - SF_CONT_LO + 1;
constexpr int SF_MAX_FIELDS = 129;                  // a line of more fields is dropped (CSV_COLUMNS[128] raises)
constexpr size_t SF_MAX_LEN = (size_t)1 << 30;      // chunk and map bytes: line offsets stay in int32
constexpr int SF_SCAN_TILE = 1024;
constexpr uint64_t SF_PENDING = 1ull << 63, SF_OFF_MASK = (1ull << 56) - 1;
constexpr uint32_t SF_CONT_ITEM = 0x80000000u;      // build items: slot number, or this | column for a continuous key

// the 28 named columns of the CSV (the file format); columns 28..127 are xgbf_0 .. xgbf_99
__constant__ char kSfNames[] =
    "is_click" "u_pl" "u_ppvn" "u_de" "u_os" "u_t" "a_m_w" "a_b_w" "c_h" "c_w" "c_al" "u_ctr" "a_a_ctr" "a_t_ctr"
    "c_q_ctr" "c_al_ctr" "c_n_ctr" "c_t_ctr" "c_t_n_ctr" "u_a_city_ctr" "u_a_age_ctr" "u_a_x_ctr" "u_a_g_ctr"
    "u_a_c_ctr" "c_q_a_ctr" "c_q_t_sim" "c_q_adtype_ctr" "c_mw_a_ctr";
__constant__ int kSfNameOff[SF_NAMED + 1] = {0,   8,   12,  18,  22,  26,  29,  34,  39,  42,  45,  49,  54,  61, 68,
                                             75,  83,  90,  97,  106, 118, 129, 138, 147, 156, 165, 174, 188, 198};

__device__ __forceinline__ bool sf_continuous(int c) { return c >= SF_CONT_LO && c <= SF_CONT_HI; }

// column index of the name [s, e), or -1
__device__ int sf_column(const uint8_t* t, int64_t s, int64_t e) {
  const int64_t n = e - s;
  if (n >= 6 && n <= 7 && t[s] == 'x' && t[s + 1] == 'g' && t[s + 2] == 'b' && t[s + 3] == 'f' && t[s + 4] == '_') {
    const unsigned d0 = (unsigned)t[s + 5] - '0', d1 = n == 7 ? (unsigned)t[s + 6] - '0' : 0u;
    if (d0 > 9 || d1 > 9 || (n == 7 && d0 == 0)) return -1;
    return SF_NAMED + (int)(n == 7 ? d0 * 10 + d1 : d0);
  }
  for (int c = 0; c < SF_NAMED; ++c) {
    const int o = kSfNameOff[c], l = kSfNameOff[c + 1] - o;
    if (l != n) continue;
    int i = 0;
    while (i < l && (uint8_t)kSfNames[o + i] == t[s + i]) ++i;
    if (i == l) return c;
  }
  return -1;
}

// CSV_COLUMNS[c] written at o when W; -> its length
template <bool W>
__device__ int sf_put_name(int c, char* o) {
  if (c < SF_NAMED) {
    const int b = kSfNameOff[c], l = kSfNameOff[c + 1] - b;
    if (W) for (int i = 0; i < l; ++i) o[i] = kSfNames[b + i];
    return l;
  }
  if (W) { o[0] = 'x'; o[1] = 'g'; o[2] = 'b'; o[3] = 'f'; o[4] = '_'; }
  return 5 + put_dec<W>((uint64_t)(c - SF_NAMED), o + 5);
}

__device__ __forceinline__ uint64_t sf_hash(int col, const uint8_t* t, int64_t s, int64_t e) {
  uint64_t h = splitmix64_finalize((uint64_t)(col + 1) * 0x9E3779B97F4A7C15ull ^ (uint64_t)(e - s));
  uint64_t w = 0;
  int k = 0;
  for (int64_t q = s; q < e; ++q) {
    w |= (uint64_t)t[q] << (8 * k);
    if (++k == 8) { h = splitmix64_finalize(h ^ w); w = 0; k = 0; }
  }
  return k ? splitmix64_finalize(h ^ w) : h;
}

__device__ __forceinline__ bool sf_same(const uint8_t* a, const uint8_t* b, int64_t n) {
  for (int64_t i = 0; i < n; ++i)
    if (a[i] != b[i]) return false;
  return true;
}

// ---- lines -----------------------------------------------------------------------------------------------------
// the commas of [s, te): the first SF_MAX_FIELDS positions (relative to s) into sc; -> their count (all of them).
// Warp-uniform.
__device__ __forceinline__ int sf_commas(const uint8_t* t, int64_t s, int64_t te, int* sc) {
  const int lane = lane_id();
  int nc = 0;
  for (int64_t w = s; w < te && nc < SF_MAX_FIELDS; w += 32) {
    const int64_t q = w + lane;
    const bool c = q < te && byte_at(t, q) == ',';
    const unsigned m = __ballot_sync(FULL_MASK, c);
    if (c) {
      const int k = nc + __popc(m & lanemask_lt());
      if (k < SF_MAX_FIELDS) sc[k] = (int)(q - s);
    }
    nc += __popc(m);
  }
  __syncwarp();
  return nc;
}

struct SfFields {
  int64_t s, te;
  const int* sc;
  int nc;
  __device__ int64_t fs(int i) const { return i == 0 ? s : s + sc[i - 1] + 1; }
  __device__ int64_t fe(int i) const { return i < nc ? s + sc[i] : te; }
};

// ---- the feature_map table -------------------------------------------------------------------------------------
// ref uint64[cap] (first line + 1, 0 = empty) | win int64[cap] (largest line) | voff, foff int64[cap] | vlen, flen,
// col int32[cap] (+ pad): 48 bytes a slot.  voff / vlen = the key's value bytes in the map text (empty for a
// continuous name), foff / flen = the fid bytes of its winning line.
struct SfMap {
  uint64_t* ref;
  int64_t *win, *voff, *foff;
  int32_t *vlen, *flen, *col;
  int64_t cap;
  SfMap() = default;
  __host__ __device__ SfMap(void* base, int64_t c) : cap(c) {
    ref = reinterpret_cast<uint64_t*>(base);
    win = reinterpret_cast<int64_t*>(ref + c);
    voff = win + c;
    foff = voff + c;
    vlen = reinterpret_cast<int32_t*>(foff + c);
    flen = vlen + c;
    col = flen + c;
  }
};

// per map line: key column (-1: skipped or unreachable), value span, fid span
struct SfMapLines {
  int32_t* col;
  int64_t *vs, *ve, *fs, *fe;
};

__global__ void __launch_bounds__(SF_THREADS) sf_map_parse_kernel(const uint8_t* __restrict__ t, int64_t len,
                                                                 const int64_t* __restrict__ line_start,
                                                                 const int64_t* __restrict__ n_newlines, SfMapLines L,
                                                                 int64_t* __restrict__ info) {
  const int64_t nn = n_newlines[0], n_lines = chunk_lines(t, len, nn);
  if (blockIdx.x == 0 && threadIdx.x == 0) info[0] = n_lines;
  for (int64_t row = (int64_t)blockIdx.x * SF_THREADS + threadIdx.x; row < n_lines;
       row += (int64_t)gridDim.x * SF_THREADS) {
    int64_t p, e;
    line_bounds(line_start, nn, len, row, p, e);
    while (p < e && is_py_space(t[p])) ++p;            // strip()
    while (e > p && is_py_space(t[e - 1])) --e;
    int64_t sp = p;
    while (sp < e && t[sp] != ' ') ++sp;
    int c = -1;
    int64_t vs = sp, ve = sp, fs = 0, fe = 0;
    if (sp < e) {                                      // at least two tokens: map[s[0]] = s[1]
      fs = sp + 1;
      fe = fs;
      while (fe < e && t[fe] != ' ') ++fe;
      int64_t bar = p;
      while (bar < sp && t[bar] != '|') ++bar;
      if (bar < sp) {                                  // name|value: reachable when name is categorical
        c = sf_column(t, p, bar);
        if (c == 0 || sf_continuous(c)) c = -1;
        vs = bar + 1;
      } else {                                         // a bare name: reachable when continuous
        c = sf_column(t, p, sp);
        if (!sf_continuous(c)) c = -1;
      }
    }
    L.col[row] = c;
    L.vs[row] = vs; L.ve[row] = ve; L.fs[row] = fs; L.fe[row] = fe;
  }
}

// info[0] = map lines (from the parse kernel)
__global__ void __launch_bounds__(SF_THREADS) sf_map_insert_kernel(const uint8_t* __restrict__ t, SfMapLines L,
                                                                  SfMap M, int64_t* info) {
  const int64_t n_lines = info[0];
  for (int64_t row = (int64_t)blockIdx.x * SF_THREADS + threadIdx.x; row < n_lines;
       row += (int64_t)gridDim.x * SF_THREADS) {
    const int c = L.col[row];
    if (c < 0) continue;
    const int64_t vs = L.vs[row], ve = L.ve[row];
    const int64_t slot = probe(sf_hash(c, t, vs, ve), M.cap, [&](uint64_t s) {
      const int64_t o = (int64_t)claim(M.ref + s, (uint64_t)(row + 1)) - 1;   // the key's first line
      return L.col[o] == c && L.ve[o] - L.vs[o] == ve - vs && sf_same(t + L.vs[o], t + vs, ve - vs);
    });
    if (slot < 0) {
      atomicAdd(reinterpret_cast<unsigned long long*>(&info[2]), 1ull);
    } else {
      atomicMax(reinterpret_cast<long long*>(M.win + slot), (long long)row);
      atomicAdd(reinterpret_cast<unsigned long long*>(&info[1]), 1ull);
    }
  }
}

__global__ void __launch_bounds__(SF_THREADS) sf_map_fill_kernel(SfMapLines L, SfMap M) {
  for (int64_t s = (int64_t)blockIdx.x * SF_THREADS + threadIdx.x; s < M.cap; s += (int64_t)gridDim.x * SF_THREADS) {
    const uint64_t r = M.ref[s];
    if (r == 0) continue;
    const int64_t o = (int64_t)r - 1, w = M.win[s];
    M.col[s] = L.col[o];
    M.voff[s] = L.vs[o];
    M.vlen[s] = (int32_t)(L.ve[o] - L.vs[o]);
    M.foff[s] = L.fs[w];
    M.flen[s] = (int32_t)(L.fe[w] - L.fs[w]);
  }
}

// fid span of the key (col, v[0, n)) -> (off, len) in the map text; false = absent (the reference's None)
__device__ bool sf_map_find(const SfMap& M, const uint8_t* map_text, int col, const uint8_t* v, int64_t n,
                            int64_t& off, int32_t& flen) {
  bool hit = false;
  probe(sf_hash(col, v, 0, n), M.cap, [&](uint64_t s) {
    if (M.ref[s] == 0) return true;
    hit = M.col[s] == col && M.vlen[s] == n && sf_same(map_text + M.voff[s], v, n);
    if (hit) { off = M.foff[s]; flen = M.flen[s]; }
    return hit;
  });
  return hit;
}

// col_fid int64[2 * 128]: per column the fid span of its bare name (continuous) or of name|UNK (categorical),
// length -1 = absent
__global__ void sf_map_columns_kernel(SfMap M, const uint8_t* __restrict__ map_text, int64_t* __restrict__ col_fid) {
  const int c = threadIdx.x;
  if (c >= SF_COLS) return;
  int64_t off = 0;
  int32_t fl = -1;
  const uint8_t unk[3] = {'U', 'N', 'K'};
  if (!sf_map_find(M, map_text, c, unk, sf_continuous(c) ? 0 : 3, off, fl)) fl = -1;
  col_fid[2 * c] = off;
  col_fid[2 * c + 1] = fl;
}

// ---- emit ------------------------------------------------------------------------------------------------------
struct SfEmitArgs {
  SfMap map;
  const uint8_t* map_text;
  const int64_t* col_fid;
};

// fid bytes (or "None") at o when W; -> its length
template <bool W>
__device__ __forceinline__ int64_t sf_put_fid(const uint8_t* map_text, int64_t off, int32_t fl, char* o) {
  if (fl < 0) {
    if (W) { o[0] = 'N'; o[1] = 'o'; o[2] = 'n'; o[3] = 'e'; }
    return 4;
  }
  if (W) for (int32_t i = 0; i < fl; ++i) o[i] = (char)map_text[off + i];
  return fl;
}

// feature i of the line (get_smart_feature.py:74-84), a space first unless i == 1; -> its length
template <bool W>
__device__ int64_t sf_feature(const uint8_t* t, const SfFields& F, int i, const SfEmitArgs& a, char* o) {
  const int64_t fs = F.fs(i), fe = F.fe(i);
  int64_t n = 0;
  if (i > 1) { if (W) o[0] = ' '; n = 1; }
  int64_t off = a.col_fid[2 * i];
  int32_t fl = (int32_t)a.col_fid[2 * i + 1];
  if (sf_continuous(i)) {
    n += sf_put_fid<W>(a.map_text, off, fl, o + n);
    if (W) { o[n] = ':'; for (int64_t q = fs; q < fe; ++q) o[n + 1 + q - fs] = (char)t[q]; }
    return n + 1 + (fe - fs);
  }
  int64_t off2;
  int32_t fl2;
  if (sf_map_find(a.map, a.map_text, i, t + fs, fe - fs, off2, fl2)) { off = off2; fl = fl2; }
  n += sf_put_fid<W>(a.map_text, off, fl, o + n);
  if (W) { o[n] = ':'; o[n + 1] = '1'; }
  return n + 2;
}

// one warp per line: plan (W = false) writes the output length of each line (0 = dropped) to len_off[row]; write
// (W = true) reads its offset there.  info (plan) = {lines, emitted lines}
template <bool W>
__global__ void __launch_bounds__(SF_THREADS) sf_emit_kernel(const uint8_t* __restrict__ t, int64_t len,
                                                            const int64_t* __restrict__ line_start,
                                                            const int64_t* __restrict__ n_newlines, SfEmitArgs a,
                                                            int64_t* __restrict__ len_off, char* __restrict__ out,
                                                            int64_t* __restrict__ info) {
  __shared__ int sc_s[SF_WARPS][SF_MAX_FIELDS];
  const int lane = lane_id(), warp = threadIdx.x >> 5;
  int* sc = sc_s[warp];
  const int64_t nn = n_newlines[0], n_lines = chunk_lines(t, len, nn), warps = (int64_t)gridDim.x * SF_WARPS;
  if (!W && blockIdx.x == 0 && threadIdx.x == 0) info[0] = n_lines;
  for (int64_t row = (int64_t)blockIdx.x * SF_WARPS + warp; row < n_lines; row += warps) {
    int64_t p, e;
    line_bounds(line_start, nn, len, row, p, e);
    SfFields F;
    warp_strip(t, p, e, F.s, F.te);
    F.sc = sc;
    F.nc = sf_commas(t, F.s, F.te, sc);
    if (F.nc >= SF_MAX_FIELDS) {                       // CSV_COLUMNS[128] raises: the line is dropped
      if (!W && lane == 0) len_off[row] = 0;
      __syncwarp();
      continue;
    }
    const int nf = F.nc + 1;
    const int64_t l0 = F.fe(0) - F.s;
    char* o = W ? out + len_off[row] : nullptr;
    int64_t pos = l0 + 1;                              // s[0] + ' '
    for (int i0 = 1; i0 <= nf - 2; i0 += 32) {
      const int i = i0 + lane;
      const int64_t L = i <= nf - 2 ? sf_feature<false>(t, F, i, a, nullptr) : 0;
      int64_t tot;
      const int64_t x = warp_scan_excl(L, tot);
      if (W && i <= nf - 2) sf_feature<true>(t, F, i, a, o + pos + x);
      pos += tot;
    }
    if (W) {
      for (int64_t q = lane; q < l0; q += 32) o[q] = (char)t[F.s + q];
      if (lane == 0) { o[l0] = ' '; o[pos] = '\n'; }
    } else if (lane == 0) {
      len_off[row] = pos + 1;
      atomicAdd(reinterpret_cast<unsigned long long*>(&info[1]), 1ull);
    }
    __syncwarp();
  }
}

// ---- Frappe (get_frape_feature.py:16-29) -----------------------------------------------------------------------
template <bool W>
__global__ void __launch_bounds__(SF_THREADS) fr_emit_kernel(const uint8_t* __restrict__ t, int64_t len,
                                                            const int64_t* __restrict__ line_start,
                                                            const int64_t* __restrict__ n_newlines,
                                                            int64_t* __restrict__ len_off, char* __restrict__ out,
                                                            int64_t* __restrict__ info) {
  const int lane = lane_id();
  const int64_t nn = n_newlines[0], n_lines = chunk_lines(t, len, nn), warps = (int64_t)gridDim.x * SF_WARPS;
  if (!W && blockIdx.x == 0 && threadIdx.x == 0) info[0] = n_lines;
  for (int64_t row = (int64_t)blockIdx.x * SF_WARPS + (threadIdx.x >> 5); row < n_lines; row += warps) {
    int64_t p, e, s, te;
    line_bounds(line_start, nn, len, row, p, e);
    warp_strip(t, p, e, s, te);
    int64_t sp = te;                                   // the first ' ' of the stripped line
    for (int64_t w = s; w < te; w += 32) {
      const int64_t q = w + lane;
      const unsigned m = __ballot_sync(FULL_MASK, q < te && byte_at(t, q) == ' ');
      if (m) { sp = w + __ffs(m) - 1; break; }
    }
    if (sp == te) {                                    // split(' ', 1) gives one piece: ValueError, skipped
      if (!W && lane == 0) len_off[row] = 0;
      continue;
    }
    const bool relabel = sp - s == 2 && byte_at(t, s) == '-' && byte_at(t, s + 1) == '1';
    const int64_t ll = relabel ? 1 : sp - s, L = ll + (te - sp) + 1;
    if (W) {
      char* o = out + len_off[row];
      if (relabel) { if (lane == 0) o[0] = '0'; }
      else for (int64_t q = lane; q < ll; q += 32) o[q] = (char)byte_at(t, s + q);
      for (int64_t q = lane; q < te - sp; q += 32) o[ll + q] = (char)byte_at(t, sp + q);
      if (lane == 0) o[L - 1] = '\n';
    } else if (lane == 0) {
      len_off[row] = L;
      atomicAdd(reinterpret_cast<unsigned long long*>(&info[1]), 1ull);
    }
  }
}

// ---- line offsets: tiles of SF_SCAN_TILE lengths summed, the sums scanned by one CTA, then each tile scanned ------
__global__ void __launch_bounds__(SF_SCAN_TILE) sf_tile_sum_kernel(const int64_t* __restrict__ a,
                                                                  const int64_t* __restrict__ n_dev,
                                                                  int64_t* __restrict__ tiles,
                                                                  int64_t* __restrict__ n_tiles) {
  const int64_t n = n_dev[0], nt = (n + SF_SCAN_TILE - 1) / SF_SCAN_TILE;
  if (blockIdx.x == 0 && threadIdx.x == 0) n_tiles[0] = nt;
  for (int64_t tile = blockIdx.x; tile < nt; tile += gridDim.x) {
    const int64_t i = tile * SF_SCAN_TILE + threadIdx.x;
    int64_t x[1] = {i < n ? a[i] : 0}, tot[1];
    block_scan_excl<SF_SCAN_TILE>(x, tot);
    if (threadIdx.x == 0) tiles[tile] = tot[0];
  }
}

__global__ void __launch_bounds__(SF_SCAN_TILE) sf_tile_scan_kernel(int64_t* __restrict__ a,
                                                                   const int64_t* __restrict__ n_dev,
                                                                   const int64_t* __restrict__ tiles) {
  const int64_t n = n_dev[0], nt = (n + SF_SCAN_TILE - 1) / SF_SCAN_TILE;
  for (int64_t tile = blockIdx.x; tile < nt; tile += gridDim.x) {
    const int64_t i = tile * SF_SCAN_TILE + threadIdx.x;
    int64_t x[1] = {i < n ? a[i] : 0}, tot[1];
    block_scan_excl<SF_SCAN_TILE>(x, tot);
    if (i < n) a[i] = tiles[tile] + x[0];
  }
}

// lengths a[0, *n_dev) -> exclusive offsets in place, their sum -> *total
static int sf_scan(int64_t* a, const int64_t* n_dev, int64_t max_n, int64_t* tiles, int64_t* n_tiles, int64_t* total,
                   cudaStream_t st, const char* what) {
  const unsigned g = grid_for(max_n, SF_SCAN_TILE, 2);
  sf_tile_sum_kernel<<<g, SF_SCAN_TILE, 0, st>>>(a, n_dev, tiles, n_tiles);
  CTR_LAUNCHED(what);
  if (int rc = cta_scan({tiles}, {total}, n_tiles, 0, st, what)) return rc;
  sf_tile_scan_kernel<<<g, SF_SCAN_TILE, 0, st>>>(a, n_dev, tiles);
  CTR_LAUNCHED(what);
  return CTR_OK;
}

// ---- the feature_map builder (get_smart_feature.py:27-53, CSV_COLUMNS[i] read as fname at :32) -------------------
// table: ref uint64[cap] | npos uint64[cap].  ref = 0 (empty) or column << 56 | offset, with SF_PENDING set while the
// offset is into the current chunk (the key is claimed there); after the chunk its value bytes and a ',' are copied
// to the arena and the offset becomes the arena's.  Every key field is followed by a ',' in its line, so both copies
// of a key end at a ','.  npos = ~(smallest position), position = global line << 7 | column, 0 = none.
// state int64[2 + 17] (zeroed by the caller) = {arena bytes used, arena overflows, ~position of each continuous name}.
struct SfBuild {
  uint64_t *ref, *npos;
  int64_t cap;
  __host__ __device__ SfBuild(void* base, int64_t c)
      : ref(reinterpret_cast<uint64_t*>(base)), npos(reinterpret_cast<uint64_t*>(base) + c), cap(c) {}
};

__device__ __forceinline__ bool sf_key_at(const uint8_t* src, const uint8_t* v, int64_t n) {
  return sf_same(src, v, n) && src[n] == ',';
}

__device__ bool sf_build_insert(const SfBuild& B, const uint8_t* t, const uint8_t* arena, int col, int64_t fs,
                                int64_t fe, uint64_t npos) {
  const uint64_t mine = SF_PENDING | ((uint64_t)col << 56) | (uint64_t)fs;
  const int64_t slot = probe(sf_hash(col, t, fs, fe), B.cap, [&](uint64_t s) {
    const uint64_t r = claim(B.ref + s, mine);   // where the slot's key was first seen
    return (int)((r >> 56) & 0x7F) == col &&
           sf_key_at((r & SF_PENDING ? t : arena) + (r & SF_OFF_MASK), t + fs, fe - fs);
  });
  if (slot >= 0) atomicMax(reinterpret_cast<unsigned long long*>(B.npos + slot), (unsigned long long)npos);
  return slot >= 0;
}

// one warp per line; info = {lines, keys that found no slot}
__global__ void __launch_bounds__(SF_THREADS) sf_build_insert_kernel(const uint8_t* __restrict__ t, int64_t len,
                                                                    const int64_t* __restrict__ line_start,
                                                                    const int64_t* __restrict__ n_newlines,
                                                                    int64_t line_base, SfBuild B,
                                                                    const uint8_t* __restrict__ arena,
                                                                    int64_t* __restrict__ state,
                                                                    int64_t* __restrict__ info) {
  __shared__ int sc_s[SF_WARPS][SF_MAX_FIELDS];
  const int lane = lane_id(), warp = threadIdx.x >> 5;
  int* sc = sc_s[warp];
  const int64_t nn = n_newlines[0], n_lines = chunk_lines(t, len, nn), warps = (int64_t)gridDim.x * SF_WARPS;
  if (blockIdx.x == 0 && threadIdx.x == 0) info[0] = n_lines;
  for (int64_t row = (int64_t)blockIdx.x * SF_WARPS + warp; row < n_lines; row += warps) {
    int64_t p, e;
    line_bounds(line_start, nn, len, row, p, e);
    SfFields F;
    warp_strip(t, p, e, F.s, F.te);
    F.sc = sc;
    F.nc = sf_commas(t, F.s, F.te, sc);
    // columns 1 .. len - 2, and at most 127: a longer line has inserted those when CSV_COLUMNS[128] raises
    const int last = F.nc - 1 < SF_COLS - 1 ? F.nc - 1 : SF_COLS - 1;
    const uint64_t base = (uint64_t)(line_base + row) << 7;
    for (int i = 1 + lane; i <= last; i += 32) {
      const uint64_t npos = ~(base | (uint64_t)i);
      if (sf_continuous(i)) {
        atomicMax(reinterpret_cast<unsigned long long*>(&state[2 + i - SF_CONT_LO]), (unsigned long long)npos);
        continue;
      }
      const int64_t fs = F.fs(i), fe = F.fe(i);
      if (fe - fs == 3 && t[fs] == 'U' && t[fs + 1] == 'N' && t[fs + 2] == 'K') continue;   // the seeded name|UNK
      if (!sf_build_insert(B, t, arena, i, fs, fe, npos))
        atomicAdd(reinterpret_cast<unsigned long long*>(&info[1]), 1ull);
    }
    __syncwarp();
  }
}

// keys claimed in this chunk -> the arena (value bytes and ','); the slot then points there
__global__ void __launch_bounds__(SF_THREADS) sf_build_commit_kernel(const uint8_t* __restrict__ t, SfBuild B,
                                                                    uint8_t* __restrict__ arena, int64_t arena_bytes,
                                                                    int64_t* __restrict__ state) {
  for (int64_t s = (int64_t)blockIdx.x * SF_THREADS + threadIdx.x; s < B.cap; s += (int64_t)gridDim.x * SF_THREADS) {
    const uint64_t r = B.ref[s];
    if (!(r & SF_PENDING)) continue;
    const uint8_t* src = t + (r & SF_OFF_MASK);
    int64_t n = 0;
    while (src[n] != ',') ++n;
    const int64_t at = (int64_t)atomicAdd(reinterpret_cast<unsigned long long*>(&state[0]), (unsigned long long)(n + 1));
    if (at + n + 1 > arena_bytes) {
      atomicAdd(reinterpret_cast<unsigned long long*>(&state[1]), 1ull);
      continue;
    }
    for (int64_t i = 0; i <= n; ++i) arena[at + i] = src[i];
    B.ref[s] = r & ~SF_PENDING & ~SF_OFF_MASK | (uint64_t)at;
  }
}

// every key -> (position, item); item = slot, or SF_CONT_ITEM | column
__global__ void __launch_bounds__(SF_THREADS) sf_build_compact_kernel(SfBuild B, const int64_t* __restrict__ state,
                                                                     uint64_t* __restrict__ keys,
                                                                     uint32_t* __restrict__ items,
                                                                     int64_t* __restrict__ n_keys) {
  const int64_t total = B.cap + SF_NCONT, stride = (int64_t)gridDim.x * SF_THREADS;
  const int64_t n_iter = (total + stride - 1) / stride;
  for (int64_t it = 0; it < n_iter; ++it) {   // uniform trip count: the warp-aggregated atomic needs whole warps
    const int64_t s = (it * gridDim.x + blockIdx.x) * SF_THREADS + threadIdx.x;
    uint64_t np = 0;
    uint32_t item = 0;
    if (s < B.cap) {
      np = B.ref[s] ? B.npos[s] : 0;
      item = (uint32_t)s;
    } else if (s < total) {
      np = (uint64_t)state[2 + s - B.cap];
      item = SF_CONT_ITEM | (uint32_t)(SF_CONT_LO + s - B.cap);
    }
    const bool keep = np != 0;
    const uint32_t ballot = __ballot_sync(FULL_MASK, keep);
    unsigned long long base = 0;
    if ((threadIdx.x & 31) == 0 && ballot)
      base = atomicAdd(reinterpret_cast<unsigned long long*>(n_keys), (unsigned long long)__popc(ballot));
    base = __shfl_sync(FULL_MASK, base, 0);
    if (keep) {
      const int64_t pos = (int64_t)base + __popc(ballot & lanemask_lt());
      keys[pos] = ~np;
      items[pos] = item;
    }
  }
}

// `key fid\n` of sorted key p (fid = 129 + p) at o when W; -> its length
template <bool W>
__device__ int64_t sf_build_line(SfBuild B, const uint8_t* arena, uint32_t item, int64_t p, char* o) {
  int64_t n;
  if (item & SF_CONT_ITEM) {
    n = sf_put_name<W>((int)(item & 0xFF), o);
  } else {
    const uint64_t r = B.ref[item];
    n = sf_put_name<W>((int)((r >> 56) & 0x7F), o);
    const uint8_t* v = arena + (r & SF_OFF_MASK);
    if (W) o[n] = '|';
    ++n;
    int64_t k = 0;
    for (; v[k] != ','; ++k)
      if (W) o[n + k] = (char)v[k];
    n += k;
  }
  if (W) o[n] = ' ';
  n += 1 + put_dec<W>((uint64_t)(SF_COLS + 1 + p), W ? o + n + 1 : nullptr);
  if (W) o[n] = '\n';
  return n + 1;
}

template <bool W>
__global__ void __launch_bounds__(SF_THREADS) sf_build_render_kernel(SfBuild B, const uint8_t* __restrict__ arena,
                                                                    const uint32_t* __restrict__ items,
                                                                    const int64_t* __restrict__ n_keys,
                                                                    int64_t* __restrict__ len_off,
                                                                    char* __restrict__ out) {
  const int64_t n = n_keys[0];
  for (int64_t p = (int64_t)blockIdx.x * SF_THREADS + threadIdx.x; p < n; p += (int64_t)gridDim.x * SF_THREADS) {
    if (W) sf_build_line<true>(B, arena, items[p], p, out + len_off[p]);
    else len_off[p] = sf_build_line<false>(B, arena, items[p], p, nullptr);
  }
}

// ---- workspace layouts -----------------------------------------------------------------------------------------
// lines of a chunk: LineStarts (max_rows = len + 1) | len_off int64[len + 1] | tiles int64[nt] | n_tiles int64[2]
struct SfLinesWs : LineStarts {
  int64_t *len_off, *tiles, *n_tiles;
  SfLinesWs(void* ws, size_t len) : LineStarts(ws, len, (int64_t)len + 1) {
    uint8_t* b = reinterpret_cast<uint8_t*>(ws);
    const size_t nt = (len + 1 + SF_SCAN_TILE - 1) / SF_SCAN_TILE;
    size_t o = bytes;
    len_off = reinterpret_cast<int64_t*>(b + o); o += align256((len + 1) * 8);
    tiles = reinterpret_cast<int64_t*>(b + o); o += align256(nt * 8);
    n_tiles = reinterpret_cast<int64_t*>(b + o); o += align256(16);
    bytes = o;
  }
};

// map: LineStarts (max_rows = len + 1) | col int32[len + 1] | vs, ve, fs, fe int64[len + 1]
struct SfMapWs : LineStarts {
  SfMapLines L;
  SfMapWs(void* ws, size_t len) : LineStarts(ws, len, (int64_t)len + 1) {
    uint8_t* b = reinterpret_cast<uint8_t*>(ws);
    const size_t n = len + 1;
    size_t o = bytes;
    L.col = reinterpret_cast<int32_t*>(b + o); o += align256(n * 4);
    L.vs = reinterpret_cast<int64_t*>(b + o); o += align256(n * 8);
    L.ve = reinterpret_cast<int64_t*>(b + o); o += align256(n * 8);
    L.fs = reinterpret_cast<int64_t*>(b + o); o += align256(n * 8);
    L.fe = reinterpret_cast<int64_t*>(b + o); o += align256(n * 8);
    bytes = o;
  }
};

// build finish / render: n_keys, hist_count int64 | hist int32[256 * nb] | keys, keys2 uint64[N] | items, items2
// uint32[N] | len_off int64[N] | tiles int64[nt] | n_tiles int64[2], N = cap + 17
struct SfBuildWs {
  int64_t *n_keys, *hist_count, *len_off, *tiles, *n_tiles;
  int32_t* hist;
  uint64_t *keys, *keys2;
  uint32_t *items, *items2;
  int64_t n_max;
  size_t bytes;
  SfBuildWs(void* ws, int64_t cap) : n_max(cap + SF_NCONT) {
    uint8_t* b = reinterpret_cast<uint8_t*>(ws);
    const size_t N = (size_t)n_max, nb = (size_t)ceil_div64(n_max, LSD_TILE), nt = (N + SF_SCAN_TILE - 1) / SF_SCAN_TILE;
    size_t o = 0;
    n_keys = reinterpret_cast<int64_t*>(b + o); hist_count = n_keys + 1; o += align256(16);
    hist = reinterpret_cast<int32_t*>(b + o); o += align256(256 * nb * 4);
    keys = reinterpret_cast<uint64_t*>(b + o); o += align256(N * 8);
    keys2 = reinterpret_cast<uint64_t*>(b + o); o += align256(N * 8);
    items = reinterpret_cast<uint32_t*>(b + o); o += align256(N * 4);
    items2 = reinterpret_cast<uint32_t*>(b + o); o += align256(N * 4);
    len_off = reinterpret_cast<int64_t*>(b + o); o += align256(N * 8);
    tiles = reinterpret_cast<int64_t*>(b + o); o += align256(nt * 8);
    n_tiles = reinterpret_cast<int64_t*>(b + o); o += align256(16);
    bytes = o;
  }
};

static int sf_memset_info(int64_t* info, int n, cudaStream_t st, const char* what) {
  CTR_REQUIRE(cudaMemsetAsync(info, 0, n * sizeof(int64_t), st) == cudaSuccess, CTR_ERR_CUDA, "%s: memset failed",
              what);
  return CTR_OK;
}

}  // namespace ctr

using namespace ctr;

extern "C" {

size_t ctr_smart_map_table_bytes(int64_t capacity) { return capacity > 0 ? (size_t)capacity * 48 : 0; }

size_t ctr_smart_map_workspace_bytes(size_t map_len) { return SfMapWs(nullptr, map_len).bytes; }

int ctr_smart_map_build(const char* map_text, size_t map_len, void* table, int64_t capacity, int64_t* col_fid,
                        int64_t* info, void* ws, size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE(table && capacity > 0 && col_fid && info && (map_len == 0 || map_text), CTR_ERR_INVALID_ARG,
              "ctr_smart_map_build: bad arguments");
  CTR_REQUIRE(capacity <= KT_MAX_CAP, CTR_ERR_INVALID_ARG, "ctr_smart_map_build: capacity > 2^31");
  CTR_REQUIRE(map_len < SF_MAX_LEN, CTR_ERR_INVALID_ARG, "ctr_smart_map_build: map too large (len < 2^30)");
  CTR_REQUIRE(ws && ws_bytes >= ctr_smart_map_workspace_bytes(map_len), CTR_ERR_WORKSPACE,
              "ctr_smart_map_build: workspace too small");
  cudaStream_t st = as_stream(stream);
  if (int rc = sf_memset_info(info, 3, st, "ctr_smart_map_build")) return rc;
  const SfMap M(table, capacity);
  const uint8_t* t = reinterpret_cast<const uint8_t*>(map_text);
  if (map_len > 0) {
    const SfMapWs W(ws, map_len);
    if (int rc = W.launch(t, map_len, st, "ctr_smart_map_build(lines)")) return rc;
    const unsigned g = grid_for((int64_t)map_len + 1, SF_THREADS, 16);
    sf_map_parse_kernel<<<g, SF_THREADS, 0, st>>>(t, (int64_t)map_len, W.line_start, W.n_newlines, W.L, info);
    CTR_LAUNCHED("ctr_smart_map_build(parse)");
    sf_map_insert_kernel<<<g, SF_THREADS, 0, st>>>(t, W.L, M, info);
    CTR_LAUNCHED("ctr_smart_map_build(insert)");
    sf_map_fill_kernel<<<grid_for(capacity, SF_THREADS, 16), SF_THREADS, 0, st>>>(W.L, M);
    CTR_LAUNCHED("ctr_smart_map_build(fill)");
  }
  sf_map_columns_kernel<<<1, SF_COLS, 0, st>>>(M, t, col_fid);
  CTR_LAUNCHED("ctr_smart_map_build(columns)");
  return CTR_OK;
}

size_t ctr_smart_emit_workspace_bytes(size_t len) { return SfLinesWs(nullptr, len).bytes; }

static int sf_emit_args(const char* map_text, const void* table, int64_t capacity, const int64_t* col_fid,
                        SfEmitArgs& a) {
  CTR_REQUIRE(table && capacity > 0 && capacity <= KT_MAX_CAP && col_fid, CTR_ERR_INVALID_ARG,
              "ctr_smart_emit: bad arguments");
  a = SfEmitArgs{SfMap(const_cast<void*>(table), capacity), reinterpret_cast<const uint8_t*>(map_text), col_fid};
  return CTR_OK;
}

int ctr_smart_emit_plan(const char* text, size_t len, const char* map_text, const void* table, int64_t capacity,
                        const int64_t* col_fid, int64_t* info, void* ws, size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE(info && (len == 0 || text), CTR_ERR_INVALID_ARG, "ctr_smart_emit_plan: bad arguments");
  CTR_REQUIRE(len < SF_MAX_LEN, CTR_ERR_INVALID_ARG, "ctr_smart_emit_plan: chunk too large (len < 2^30)");
  CTR_REQUIRE(ws && ws_bytes >= ctr_smart_emit_workspace_bytes(len), CTR_ERR_WORKSPACE,
              "ctr_smart_emit_plan: workspace too small");
  SfEmitArgs a;
  if (int rc = sf_emit_args(map_text, table, capacity, col_fid, a)) return rc;
  cudaStream_t st = as_stream(stream);
  if (int rc = sf_memset_info(info, 3, st, "ctr_smart_emit_plan")) return rc;
  if (len == 0) return CTR_OK;
  const uint8_t* t = reinterpret_cast<const uint8_t*>(text);
  const SfLinesWs E(ws, len);
  if (int rc = E.launch(t, len, st, "ctr_smart_emit_plan(lines)")) return rc;
  sf_emit_kernel<false><<<grid_for((int64_t)len + 1, SF_WARPS, 8), SF_THREADS, 0, st>>>(
      t, (int64_t)len, E.line_start, E.n_newlines, a, E.len_off, nullptr, info);
  CTR_LAUNCHED("ctr_smart_emit_plan");
  return sf_scan(E.len_off, info, (int64_t)len + 1, E.tiles, E.n_tiles, info + 2, st, "ctr_smart_emit_plan(scan)");
}

int ctr_smart_emit_write(const char* text, size_t len, const char* map_text, const void* table, int64_t capacity,
                         const int64_t* col_fid, char* out, const void* ws, size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE((len == 0 || (text && out)), CTR_ERR_INVALID_ARG, "ctr_smart_emit_write: bad arguments");
  CTR_REQUIRE(len < SF_MAX_LEN, CTR_ERR_INVALID_ARG, "ctr_smart_emit_write: chunk too large (len < 2^30)");
  CTR_REQUIRE(ws && ws_bytes >= ctr_smart_emit_workspace_bytes(len), CTR_ERR_WORKSPACE,
              "ctr_smart_emit_write: workspace too small");
  SfEmitArgs a;
  if (int rc = sf_emit_args(map_text, table, capacity, col_fid, a)) return rc;
  if (len == 0) return CTR_OK;
  const SfLinesWs E(const_cast<void*>(ws), len);
  sf_emit_kernel<true><<<grid_for((int64_t)len + 1, SF_WARPS, 8), SF_THREADS, 0, as_stream(stream)>>>(
      reinterpret_cast<const uint8_t*>(text), (int64_t)len, E.line_start, E.n_newlines, a, E.len_off, out, nullptr);
  CTR_LAUNCHED("ctr_smart_emit_write");
  return CTR_OK;
}

size_t ctr_smart_build_table_bytes(int64_t capacity) { return capacity > 0 ? (size_t)capacity * 16 : 0; }

size_t ctr_smart_build_insert_workspace_bytes(size_t len) {
  return LineStarts(nullptr, len, (int64_t)len + 1).bytes;
}

int ctr_smart_build_insert(const char* text, size_t len, int64_t line_base, void* table, int64_t capacity,
                           uint8_t* arena, int64_t arena_bytes, int64_t* state, int64_t* info, void* ws,
                           size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE(table && capacity > 0 && arena && arena_bytes > 0 && state && info && line_base >= 0 &&
                  (len == 0 || text),
              CTR_ERR_INVALID_ARG, "ctr_smart_build_insert: bad arguments");
  CTR_REQUIRE(capacity <= KT_MAX_CAP, CTR_ERR_INVALID_ARG, "ctr_smart_build_insert: capacity > 2^31");
  CTR_REQUIRE(len < SF_MAX_LEN, CTR_ERR_INVALID_ARG, "ctr_smart_build_insert: chunk too large (len < 2^30)");
  CTR_REQUIRE(ws && ws_bytes >= ctr_smart_build_insert_workspace_bytes(len), CTR_ERR_WORKSPACE,
              "ctr_smart_build_insert: workspace too small");
  cudaStream_t st = as_stream(stream);
  if (int rc = sf_memset_info(info, 2, st, "ctr_smart_build_insert")) return rc;
  if (len == 0) return CTR_OK;
  const uint8_t* t = reinterpret_cast<const uint8_t*>(text);
  const LineStarts L(ws, len, (int64_t)len + 1);
  if (int rc = L.launch(t, len, st, "ctr_smart_build_insert(lines)")) return rc;
  const SfBuild B(table, capacity);
  sf_build_insert_kernel<<<grid_for((int64_t)len + 1, SF_WARPS, 8), SF_THREADS, 0, st>>>(
      t, (int64_t)len, L.line_start, L.n_newlines, line_base, B, arena, state, info);
  CTR_LAUNCHED("ctr_smart_build_insert");
  sf_build_commit_kernel<<<grid_for(capacity, SF_THREADS, 16), SF_THREADS, 0, st>>>(t, B, arena, arena_bytes, state);
  CTR_LAUNCHED("ctr_smart_build_insert(commit)");
  return CTR_OK;
}

size_t ctr_smart_build_workspace_bytes(int64_t capacity) { return capacity > 0 ? SfBuildWs(nullptr, capacity).bytes : 0; }

int ctr_smart_build_finish(const void* table, int64_t capacity, const uint8_t* arena, const int64_t* state,
                           int64_t* info, void* ws, size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE(table && capacity > 0 && arena && state && info, CTR_ERR_INVALID_ARG,
              "ctr_smart_build_finish: bad arguments");
  CTR_REQUIRE(capacity <= KT_MAX_CAP, CTR_ERR_INVALID_ARG, "ctr_smart_build_finish: capacity > 2^31");
  CTR_REQUIRE(ws && ws_bytes >= ctr_smart_build_workspace_bytes(capacity), CTR_ERR_WORKSPACE,
              "ctr_smart_build_finish: workspace too small");
  cudaStream_t st = as_stream(stream);
  SfBuildWs W(ws, capacity);
  const SfBuild B(const_cast<void*>(table), capacity);
  if (int rc = sf_memset_info(info, 2, st, "ctr_smart_build_finish")) return rc;
  if (int rc = sf_memset_info(W.n_keys, 2, st, "ctr_smart_build_finish")) return rc;
  const unsigned g = grid_for(W.n_max, SF_THREADS, 16);
  sf_build_compact_kernel<<<g, SF_THREADS, 0, st>>>(B, state, W.keys, W.items, W.n_keys);
  CTR_LAUNCHED("ctr_smart_build_finish(compact)");
  // positions are unique, so the sort fixes the fid order; 8 passes over the 64 position bits end back in keys / items
  uint64_t* k;
  uint32_t* v;
  if (int rc = lsd_sort(W.keys, W.items, W.keys2, W.items2, W.n_keys, W.n_max, 8, W.hist, W.hist_count, st,
                        "ctr_smart_build_finish(sort)", &k, &v))
    return rc;
  sf_build_render_kernel<false><<<g, SF_THREADS, 0, st>>>(B, arena, v, W.n_keys, W.len_off, nullptr);
  CTR_LAUNCHED("ctr_smart_build_finish(sizes)");
  CTR_REQUIRE(cudaMemcpyAsync(info, W.n_keys, sizeof(int64_t), cudaMemcpyDeviceToDevice, st) == cudaSuccess,
              CTR_ERR_CUDA, "ctr_smart_build_finish: copy failed");
  return sf_scan(W.len_off, W.n_keys, W.n_max, W.tiles, W.n_tiles, info + 1, st, "ctr_smart_build_finish(scan)");
}

int ctr_smart_build_render(const void* table, int64_t capacity, const uint8_t* arena, char* out, const void* ws,
                           size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE(table && capacity > 0 && capacity <= KT_MAX_CAP && arena && out, CTR_ERR_INVALID_ARG,
              "ctr_smart_build_render: bad arguments");
  CTR_REQUIRE(ws && ws_bytes >= ctr_smart_build_workspace_bytes(capacity), CTR_ERR_WORKSPACE,
              "ctr_smart_build_render: workspace too small");
  SfBuildWs W(const_cast<void*>(ws), capacity);
  const SfBuild B(const_cast<void*>(table), capacity);
  sf_build_render_kernel<true><<<grid_for(W.n_max, SF_THREADS, 16), SF_THREADS, 0, as_stream(stream)>>>(
      B, arena, W.items, W.n_keys, W.len_off, out);
  CTR_LAUNCHED("ctr_smart_build_render");
  return CTR_OK;
}

size_t ctr_frappe_workspace_bytes(size_t len) { return SfLinesWs(nullptr, len).bytes; }

int ctr_frappe_plan(const char* text, size_t len, int64_t* info, void* ws, size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE(info && (len == 0 || text), CTR_ERR_INVALID_ARG, "ctr_frappe_plan: bad arguments");
  CTR_REQUIRE(len < SF_MAX_LEN, CTR_ERR_INVALID_ARG, "ctr_frappe_plan: chunk too large (len < 2^30)");
  CTR_REQUIRE(ws && ws_bytes >= ctr_frappe_workspace_bytes(len), CTR_ERR_WORKSPACE,
              "ctr_frappe_plan: workspace too small");
  cudaStream_t st = as_stream(stream);
  if (int rc = sf_memset_info(info, 3, st, "ctr_frappe_plan")) return rc;
  if (len == 0) return CTR_OK;
  const uint8_t* t = reinterpret_cast<const uint8_t*>(text);
  const SfLinesWs E(ws, len);
  if (int rc = E.launch(t, len, st, "ctr_frappe_plan(lines)")) return rc;
  fr_emit_kernel<false><<<grid_for((int64_t)len + 1, SF_WARPS, 8), SF_THREADS, 0, st>>>(
      t, (int64_t)len, E.line_start, E.n_newlines, E.len_off, nullptr, info);
  CTR_LAUNCHED("ctr_frappe_plan");
  return sf_scan(E.len_off, info, (int64_t)len + 1, E.tiles, E.n_tiles, info + 2, st, "ctr_frappe_plan(scan)");
}

int ctr_frappe_write(const char* text, size_t len, char* out, const void* ws, size_t ws_bytes, ctr_stream_t stream) {
  CTR_REQUIRE(len == 0 || (text && out), CTR_ERR_INVALID_ARG, "ctr_frappe_write: bad arguments");
  CTR_REQUIRE(len < SF_MAX_LEN, CTR_ERR_INVALID_ARG, "ctr_frappe_write: chunk too large (len < 2^30)");
  CTR_REQUIRE(ws && ws_bytes >= ctr_frappe_workspace_bytes(len), CTR_ERR_WORKSPACE,
              "ctr_frappe_write: workspace too small");
  if (len == 0) return CTR_OK;
  const SfLinesWs E(const_cast<void*>(ws), len);
  fr_emit_kernel<true><<<grid_for((int64_t)len + 1, SF_WARPS, 8), SF_THREADS, 0, as_stream(stream)>>>(
      reinterpret_cast<const uint8_t*>(text), (int64_t)len, E.line_start, E.n_newlines, E.len_off, out, nullptr);
  CTR_LAUNCHED("ctr_frappe_write");
  return CTR_OK;
}

}  // extern "C"
