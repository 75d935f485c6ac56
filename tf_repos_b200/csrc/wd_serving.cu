// wd_serving.cu -- the serving input of wide_n_deep's export (wide_n_deep.py:233-242,
// build_parsing_serving_input_receiver_fn(make_parse_example_spec(columns))): the `inputs` tensor of
// wide_n_deep_serving_client.cpp:45-62 is a batch of serialized tf.Examples; one warp per Example parses it and runs
// the feature columns of wide_deep.cu on what it finds (DESIGN.md §2.8).
//
//   I1..I13   FixedLenFeature([1], float32), no default: present with exactly one float
//   C14..C39  VarLenFeature(int64) -> categorical_column_with_identity(10000, default 0): a value outside [0, NB) (all
//             64 bits) becomes 0; embedding_column combiner 'mean' (rows summed in value order, divided by the bag's
//             length), linear_model combiner 'sum'; an empty or missing bag gives a zero row and adds 0
//   any other key is ignored; the last map entry of a key wins; a Feature with no kind set is an empty list
//
// x and lin are wd_input_fwd's outputs, written in its layout and its per-lane order: for a request whose every C key
// holds one value they are bit-identical to ctr_wd_input_fwd on the same ids and numerics.
// Error word (uint64, ~0 = none): (example << 16) | (check << 8) | key, folded with atomicMin; key = 0..12 for
// I1..I13, 13..38 for C14..C39.  Checks of one Example: malformed protobuf first, then keys in that order, each
// missing I key, then several kinds / wrong kind, then an I value count != 1.
#include "common.cuh"
#include "example_wire.cuh"

namespace ctr {

constexpr int WS_NUM = 13, WS_CAT = 26, WS_KEYS = WS_NUM + WS_CAT;
constexpr int WS_THREADS = 256, WS_WARPS = WS_THREADS / 32;
enum { WE_MALFORMED = 1, WE_MISSING = 2, WE_KIND = 3, WE_COUNT = 4 };
enum { WK_NONE = 0, WK_BYTES = 1, WK_FLOAT = 2, WK_INT = 3 };

struct WsSlot {
  int present, kind, count, multi;
  int ls, le;   // payload of the Feature's kind field: the list message
  float val;    // the last float of a FloatList
};

// map key [s, e) -> 0..38 for I1..I13 / C14..C39 (decoded as 'I' or 'C' and a canonical decimal), -1 for any other key
__device__ int ws_key(const uint8_t* d, int s, int e) {
  const int n = e - s;
  if (n < 2 || n > 3) return -1;
  const uint32_t c = tr_byte(d, s), d1 = tr_byte(d, s + 1), d2 = n == 3 ? tr_byte(d, s + 2) : '0';
  if ((c != 'I' && c != 'C') || d1 < '1' || d1 > '9' || d2 < '0' || d2 > '9') return -1;
  const int num = n == 3 ? (int)(d1 - '0') * 10 + (int)(d2 - '0') : (int)(d1 - '0');
  if (c == 'I') return num <= WS_NUM ? num - 1 : -1;
  return num > WS_NUM && num <= WS_KEYS ? num - 1 : -1;
}

// the values of an Int64List [s, e), in order, to add(v); false = malformed (a packed varint unterminated, over 10
// bytes or >= 2^64)
template <class Add>
__device__ __forceinline__ bool ws_ints(const uint8_t* d, int s, int e, Add add) {
  for (int p = s; p < e;) {
    TrField f;
    p = tr_field(d, p, e, f);
    if (p < 0) return false;
    if (f.num != 1) continue;
    if (f.wt == 2) {
      for (int q = f.vs; q < f.ve;) {
        uint64_t v;
        q = tr_varint(d, q, f.ve, v);
        if (q < 0) return false;
        add(v);
      }
    } else if (f.wt == 0) {
      add(f.v);
    }
  }
  return true;
}

// the value count of a BytesList / FloatList / Int64List [s, e) of kind r.kind, appended to r.count, and a FloatList's
// last value; false = malformed
__device__ bool ws_list(const uint8_t* d, int s, int e, WsSlot& r) {
  if (r.kind == WK_INT) return ws_ints(d, s, e, [&](uint64_t) { ++r.count; });
  for (int p = s; p < e;) {
    TrField f;
    p = tr_field(d, p, e, f);
    if (p < 0) return false;
    if (f.num != 1) continue;
    if (r.kind == WK_BYTES) {
      ++r.count;
    } else if (f.wt == 2) {
      if ((f.ve - f.vs) & 3) return false;
      if (f.ve > f.vs) r.val = tr_float(tr_u32(d, f.ve - 4));
      r.count += (f.ve - f.vs) >> 2;
    } else if (f.wt == 5) {
      r.val = tr_float(tr_u32(d, f.vs));
      ++r.count;
    }
  }
  return true;
}

__device__ __forceinline__ int ws_check(const WsSlot& s, int k) {
  const bool num = k < WS_NUM;
  if (!s.present) return num ? (WE_MISSING << 8 | k) : -1;
  if (s.multi || (s.kind != WK_NONE && s.kind != (num ? WK_FLOAT : WK_INT))) return WE_KIND << 8 | k;
  if (num && s.count != 1) return WE_COUNT << 8 | k;
  return -1;
}

// the first failing key in key order -> (check << 8) | key, or -1.  Lane l checks keys l and l + 32.
__device__ int ws_checks(const WsSlot* slot) {
  const int lane = threadIdx.x & 31;
  const int lo = ws_check(slot[lane], lane);
  const int hi = lane + 32 < WS_KEYS ? ws_check(slot[lane + 32], lane + 32) : -1;
  unsigned m = __ballot_sync(FULL_MASK, lo >= 0);
  if (m) return __shfl_sync(FULL_MASK, lo, __ffs(m) - 1);
  m = __ballot_sync(FULL_MASK, hi >= 0);
  return m ? __shfl_sync(FULL_MASK, hi, __ffs(m) - 1) : -1;
}

// one warp per Example b of the request: data[off[b], off[b+1])
__global__ void __launch_bounds__(WS_THREADS)
wd_serve_input_kernel(const uint8_t* __restrict__ data, const int64_t* __restrict__ off, int64_t n, int64_t example_base,
                      const float* __restrict__ emb, const float* __restrict__ wide_cat,
                      const float* __restrict__ wide_num, const float* __restrict__ wide_bias,
                      const int32_t* __restrict__ num_perm, int NB, int K, float* __restrict__ x,
                      float* __restrict__ lin, unsigned long long* __restrict__ err) {
  __shared__ WsSlot slots[WS_WARPS][WS_KEYS];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  WsSlot* slot = slots[wib];
  const int64_t D = (int64_t)WS_CAT * K + WS_NUM;
  const int chunks = emb ? (K + 31) / 32 : (wide_cat ? 1 : 0);
  for (int64_t b = (int64_t)blockIdx.x * WS_WARPS + wib; b < n; b += (int64_t)gridDim.x * WS_WARPS) {
    const int64_t L = off[b + 1] - off[b];
    const uint8_t* d = data + off[b];
    for (int k = lane; k < WS_KEYS; k += 32) slot[k].present = 0;
    // slot[k] = the last entry of key k; every keyed entry's Feature must be well formed
    auto entry = [&](int key, int fs, int fe) {
      WsSlot r{1, WK_NONE, 0, 0, 0, 0, 0.f};
      if (!tr_feature_kind(d, fs, fe, r, [&](int ls, int le) { r.ls = ls; r.le = le; return ws_list(d, ls, le, r); }))
        return false;
      if (key >= 0 && lane == 0) slot[key] = r;
      return true;
    };
    int word = WE_MALFORMED << 8;
    if (L >= 0 && L <= 0x7FFFFFFF &&
        tr_map_entries(d, (int)L, [&](int ks, int ke) { return ws_key(d, ks, ke); }, entry))
      word = ws_checks(slot);
    if (word >= 0) {
      if (lane == 0) atomicMin(err, (unsigned long long)(example_base + b) << 16 | (unsigned)word);
      __syncwarp();
      continue;
    }
    float* xr = emb ? x + b * D : nullptr;
    float acc = 0.f;   // lane f: the linear weights of column f, in value order
    for (int f = 0; f < WS_CAT; ++f) {
      const WsSlot& s = slot[WS_NUM + f];
      const bool bag = s.present && s.kind == WK_INT && s.count > 0;
      for (int c = 0; c < chunks; ++c) {
        const int k = c * 32 + lane;
        const bool row = emb && k < K;
        float sum = 0.f;
        bool first = true;
        auto add = [&](uint64_t v) {
          const int id = v < (uint64_t)NB ? (int)v : 0;
          const int64_t fid = (int64_t)f * NB + id;
          if (row) sum = first ? emb[fid * K + k] : sum + emb[fid * K + k];
          first = false;
          if (c == 0 && lane == f && wide_cat) acc += wide_cat[fid];
        };
        if (bag) ws_ints(d, s.ls, s.le, add);
        if (row) xr[(int64_t)f * K + k] = bag ? sum / (float)s.count : 0.f;
      }
    }
    if (wide_num && lane < WS_NUM) acc += slot[lane].val * wide_num[lane];
    if (lin) {
      acc = warp_sum(acc);
      if (lane == 0) lin[b] = acc + (wide_bias ? wide_bias[0] : 0.f);
    }
    if (emb && lane < WS_NUM) xr[(int64_t)WS_CAT * K + lane] = slot[num_perm[lane]].val;
    __syncwarp();
  }
}

}  // namespace ctr

using namespace ctr;

extern "C" {

int ctr_wd_serve_input(const void* data, const int64_t* offsets, int64_t n, int64_t example_base, const float* emb,
                       const float* wide_cat, const float* wide_num, const float* wide_bias, const int32_t* num_perm,
                       int NB, int K, float* x, float* lin, uint64_t* err, ctr_stream_t stream) {
  CTR_REQUIRE(n >= 0 && example_base >= 0 && NB > 0 && K > 0 && err, CTR_ERR_INVALID_ARG,
              "ctr_wd_serve_input: bad arguments");
  CTR_REQUIRE(example_base + n < ((int64_t)1 << 47), CTR_ERR_INVALID_ARG, "ctr_wd_serve_input: example index >= 2^47");
  CTR_REQUIRE((int64_t)WS_CAT * NB < ((int64_t)1 << 31), CTR_ERR_INVALID_ARG, "ctr_wd_serve_input: 26 * NB >= 2^31");
  if (n == 0) return CTR_OK;
  CTR_REQUIRE(data && offsets, CTR_ERR_INVALID_ARG, "ctr_wd_serve_input: null data/offsets");
  CTR_REQUIRE(!emb || (x && num_perm), CTR_ERR_INVALID_ARG, "ctr_wd_serve_input: emb needs x and num_perm");
  CTR_REQUIRE(!(wide_cat || wide_num) || lin, CTR_ERR_INVALID_ARG, "ctr_wd_serve_input: wide part needs lin");
  const int64_t want = (n + WS_WARPS - 1) / WS_WARPS, cap = (int64_t)sm_count() * 16;
  wd_serve_input_kernel<<<(unsigned)(want < cap ? want : cap), WS_THREADS, 0, as_stream(stream)>>>(
      static_cast<const uint8_t*>(data), offsets, n, example_base, emb, wide_cat, wide_num, wide_bias, num_perm, NB, K,
      x, lin, reinterpret_cast<unsigned long long*>(err));
  CTR_LAUNCHED("ctr_wd_serve_input");
  return CTR_OK;
}

}  // extern "C"
