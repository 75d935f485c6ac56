// epoch.cu -- "exact-deferred" table update: bit-identical to sweeping every row every step
// (optim.cu), at 1/P of the HBM traffic.
//
// Why this is legal: in TensorFlow's semantics (SURVEY.md A.4) a row that no gather touched at step
// t still takes the optimizer step with g = l2*var.  That update is an element-wise recurrence on
// (var, slot0, slot1) that depends on nothing but the row's own state and the scalar lr_t.  So it
// can be *replayed later* -- exactly, in the same fp32 operation order -- the next time the row is
// needed: when a batch gathers it (catch-up), or at the end of an epoch of P steps (epoch sweep),
// where one pass over HBM applies P steps in registers.  A per-row byte `last` counts how many steps
// of the current epoch are already applied to the stored state.
//
// Roofline: the plain sweep moves 24 B/element/step (HBM-bound, 13 ms at config 2); the epoch sweep
// moves 24 B/element per P steps and executes P x ~36 instructions per element, i.e. it turns the
// step from HBM-bound into FP32-issue-bound.
//
// Replaces the same reference lines as optim.cu: optimizer.minimize (DeepFM.py:204-213) with the
// dense l2_loss gradient (DeepFM.py:189-190) [TF-sem].
#include "optim_steps.cuh"

namespace ctr {

// epoch_adam.cu: Adam sweep on the packed fp32 pipe (rows nothing gathered since `from`; the others go to `list`)
// w_*: an optional scalar table [n_rows] that shares `last` and is swept in the same launch.  Returns false if the
// shape does not fit the packed kernels.
bool launch_epoch_sweep_adam(float* var, float* slot0, float* slot1, const uint8_t* last, int64_t n_rows, int K,
                             const float* hyper, const float* lr_table, int from, int upto, double* ss_partials,
                             int n_partials, int32_t* list, int32_t* list_count, int64_t list_cap,
                             int32_t* list_overflow, cudaStream_t st, float* w_var = nullptr,
                             float* w_slot0 = nullptr, float* w_slot1 = nullptr, double* w_ss_partials = nullptr);

__device__ __forceinline__ float sq4(const float4& x) {
  return (x.x * x.x + x.y * x.y) + (x.z * x.z + x.w * x.w);
}

// Rows uniq[0..n_uniq): replay the untouched-row step for steps last[row]..j-1 so that the stored
// state is the state at the START of step j; then (APPLY) take step j with the summed gradient.
// ss[s] (double) accumulates sum(var^2) of the state each replayed/applied step started from.
// second scalar table gathered with the same ids (DeepFM: fm_w next to fm_v): lane 0 of a row carries its element.
// last == nullptr: the two tables share the [N,K] table's `last` bytes (they are always gathered together)
// stage / w_stage (STAGED): per unique row u, the state at the start of step j -- stage[u*3K ..] = var | slot0 | slot1
// of the [N,K] row, w_stage[3u ..] = those of the scalar element
struct RowsW {
  float* var; float* slot0; float* slot1; uint8_t* last; const float* g_uniq; double* ss;
  float* stage = nullptr; float* w_stage = nullptr;
};

// STAGED (WITH_W only): the catch-up and the apply of one step hand the rows over through `stage`, in unique-row
// order, instead of through the tables.  The catch-up (!APPLY) stores the caught-up state in `stage` and writes only
// `var` back (the forward gathers it); slot0 / slot1 and `last` keep their old values until the apply (APPLY) of the
// same step reads `stage`, takes step j and writes the whole row and last = j + 1.  Per row, that replaces two random
// slot writes and a `last` write in the catch-up, and every random read of the apply, with sequential stage traffic.
// Between the two calls the tables hold the caught-up `var` next to the old slots: nothing but the step's forward
// may read them.
template <int OPT, int LPR, int VEC, bool APPLY, bool WITH_W = false, bool STAGED = false>
__global__ void __launch_bounds__(256)
epoch_rows_kernel(float* __restrict__ var, float* __restrict__ slot0, float* __restrict__ slot1,
                  uint8_t* __restrict__ last, const int32_t* __restrict__ uniq,
                  const int32_t* __restrict__ n_uniq, const float* __restrict__ g_uniq, int64_t n_max,
                  const float* __restrict__ hyper, const float* __restrict__ lr_table, int j,
                  double* __restrict__ ss, int set_last, RowsW w = RowsW()) {
  constexpr int K = 4 * LPR * VEC;
  constexpr bool two = OptTraits<OPT>::slots == 2;
  __shared__ float ss_blk[EPOCH_MAX];  // <= 256 rows' worth per CTA: fp32 is plenty; global sums are double
  __shared__ float ssw_blk[EPOCH_MAX];
  if (threadIdx.x < EPOCH_MAX) { ss_blk[threadIdx.x] = 0.f; ssw_blk[threadIdx.x] = 0.f; }
  __syncthreads();
  const int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / LPR;
  const int c = threadIdx.x % LPR;
  const int lane = threadIdx.x & 31;
  const bool active = u < n_max && u < n_uniq[0];
  Hyper h = load_hyper(hyper);
  const AdamConsts ac = adam_consts(h);
  constexpr bool from_stage = STAGED && APPLY;
  const int64_t id = active ? uniq[u] : 0;
  const int l0 = (active && !from_stage) ? last[id] : j;
  const int64_t row = id * K;
  float* const srow = STAGED ? w.stage + u * (3 * K) : nullptr;
  float4 x[VEC], a[VEC], b[VEC];
#pragma unroll
  for (int v = 0; v < VEC; ++v) {
    const int64_t e = row + (c + v * LPR) * 4;
    const int k = (c + v * LPR) * 4;
    if (from_stage) {
      x[v] = active ? *reinterpret_cast<const float4*>(srow + k) : f4_zero();
      a[v] = active ? *reinterpret_cast<const float4*>(srow + K + k) : f4_zero();
      b[v] = (active && two) ? *reinterpret_cast<const float4*>(srow + 2 * K + k) : f4_zero();
    } else {
      x[v] = active ? *reinterpret_cast<const float4*>(var + e) : f4_zero();
      a[v] = active ? *reinterpret_cast<const float4*>(slot0 + e) : f4_zero();
      b[v] = (active && two) ? *reinterpret_cast<const float4*>(slot1 + e) : f4_zero();
    }
  }
  const bool wact = WITH_W && active && c == 0;
  int l0w = j;
  float xw = 0.f, aw = 0.f, bw = 0.f;
  if (wact) {
    if (from_stage) {
      xw = w.w_stage[3 * u]; aw = w.w_stage[3 * u + 1]; bw = two ? w.w_stage[3 * u + 2] : 0.f;
    } else {
      l0w = w.last ? w.last[id] : l0; xw = w.var[id]; aw = w.slot0[id]; bw = two ? w.slot1[id] : 0.f;
    }
  }
  // warp-uniform trip count (the body reduces across the warp); a lane joins at its own row's `last`
  const int lmin = __reduce_min_sync(FULL_MASK, min(l0, l0w));
#pragma unroll 1
  for (int s = lmin; s < j; ++s) {
    h.lr = lr_table[s];
    float q = 0.f;
    if (s >= l0) {
#pragma unroll
      for (int v = 0; v < VEC; ++v) q += sq4(x[v]);
      if (OPT == CTR_OPT_ADAM) {
        adam_untouched<VEC>(x, a, b, h, ac);
      } else {
#pragma unroll
        for (int v = 0; v < VEC; ++v) step_untouched4<OPT>(x[v], a[v], b[v], h);
      }
    }
    q = warp_sum(q);
    if (lane == 0 && q != 0.f) atomicAdd(&ss_blk[s], q);
    if (WITH_W) {
      float qw = 0.f;
      if (wact && s >= l0w) { qw = xw * xw; step_sparse<OPT>(xw, aw, bw, __fmul_rn(h.l2, xw), h); }
      qw = warp_sum(qw);
      if (lane == 0 && qw != 0.f) atomicAdd(&ssw_blk[s], qw);
    }
  }
  if (APPLY) {
    h.lr = lr_table[j];
    float q = 0.f;
    if (active) {
#pragma unroll
      for (int v = 0; v < VEC; ++v) {
        q += sq4(x[v]);
        float4 g = *reinterpret_cast<const float4*>(g_uniq + u * K + (c + v * LPR) * 4);
        g = make_float4(__fadd_rn(g.x, __fmul_rn(h.l2, x[v].x)), __fadd_rn(g.y, __fmul_rn(h.l2, x[v].y)),
                        __fadd_rn(g.z, __fmul_rn(h.l2, x[v].z)), __fadd_rn(g.w, __fmul_rn(h.l2, x[v].w)));
        step_sparse4<OPT>(x[v], a[v], b[v], g, h);
      }
    }
    q = warp_sum(q);
    if (lane == 0 && q != 0.f) atomicAdd(&ss_blk[j], q);
    if (WITH_W) {
      float qw = 0.f;
      if (wact) { qw = xw * xw; step_sparse<OPT>(xw, aw, bw, __fadd_rn(w.g_uniq[u], __fmul_rn(h.l2, xw)), h); }
      qw = warp_sum(qw);
      if (lane == 0 && qw != 0.f) atomicAdd(&ssw_blk[j], qw);
    }
  }
  if (STAGED && !APPLY) {   // hand the caught-up rows to the apply; only `var` goes back to the tables
    if (active) {
#pragma unroll
      for (int v = 0; v < VEC; ++v) {
        const int k = (c + v * LPR) * 4;
        *reinterpret_cast<float4*>(srow + k) = x[v];
        *reinterpret_cast<float4*>(srow + K + k) = a[v];
        if (two) *reinterpret_cast<float4*>(srow + 2 * K + k) = b[v];
        if (l0 < j) *reinterpret_cast<float4*>(var + row + k) = x[v];
      }
    }
    if (wact) {
      w.w_stage[3 * u] = xw; w.w_stage[3 * u + 1] = aw;
      if (two) w.w_stage[3 * u + 2] = bw;
      if (l0w < j) w.var[id] = xw;
    }
  }
  if (STAGED && !APPLY) {
    __syncthreads();
    if (threadIdx.x < EPOCH_MAX && ss_blk[threadIdx.x] != 0.f) atomicAdd(&ss[threadIdx.x], (double)ss_blk[threadIdx.x]);
    if (threadIdx.x < EPOCH_MAX && ssw_blk[threadIdx.x] != 0.f) atomicAdd(&w.ss[threadIdx.x], (double)ssw_blk[threadIdx.x]);
    return;
  }
  if (WITH_W && wact && (APPLY || l0w < j)) {
    w.var[id] = xw; w.slot0[id] = aw;
    if (two) w.slot1[id] = bw;
  }
  if (WITH_W && wact && w.last && (APPLY || l0w < j || set_last >= 0)) w.last[id] = (uint8_t)(set_last >= 0 ? set_last : (APPLY ? j + 1 : j));
  const bool wrote = active && (APPLY || l0 < j);
  const uint8_t new_last = (uint8_t)(set_last >= 0 ? set_last : (APPLY ? j + 1 : j));
  if (wrote) {
#pragma unroll
    for (int v = 0; v < VEC; ++v) {
      const int64_t e = row + (c + v * LPR) * 4;
      *reinterpret_cast<float4*>(var + e) = x[v];
      *reinterpret_cast<float4*>(slot0 + e) = a[v];
      if (two) *reinterpret_cast<float4*>(slot1 + e) = b[v];
    }
  }
  __syncthreads();  // every lane of a row has read `last` before lane 0 of the row rewrites it
  if (active && c == 0 && (wrote || set_last >= 0)) last[id] = new_last;
  if (threadIdx.x < EPOCH_MAX && ss_blk[threadIdx.x] != 0.f) atomicAdd(&ss[threadIdx.x], (double)ss_blk[threadIdx.x]);
  if (WITH_W && threadIdx.x < EPOCH_MAX && ssw_blk[threadIdx.x] != 0.f) atomicAdd(&w.ss[threadIdx.x], (double)ssw_blk[threadIdx.x]);
}

// any K (incl. the scalar first-order table, K = 1): one thread per (row, k).  A CTA holds 256/K whole rows and is
// rounded up to whole warps (the body shuffles with the full mask); the surplus threads own no element.
template <int OPT, bool APPLY>
__global__ void __launch_bounds__(256)
epoch_rows_generic_kernel(float* __restrict__ var, float* __restrict__ slot0, float* __restrict__ slot1,
                          uint8_t* __restrict__ last, const int32_t* __restrict__ uniq,
                          const int32_t* __restrict__ n_uniq, const float* __restrict__ g_uniq,
                          int64_t n_max, int K, const float* __restrict__ hyper,
                          const float* __restrict__ lr_table, int j, double* __restrict__ ss, int set_last) {
  constexpr bool two = OptTraits<OPT>::slots == 2;
  __shared__ float ss_blk[EPOCH_MAX];
  if (threadIdx.x < EPOCH_MAX) ss_blk[threadIdx.x] = 0.f;
  __syncthreads();
  const int rows_per_cta = 256 / K;
  const int64_t u = (int64_t)blockIdx.x * rows_per_cta + threadIdx.x / K;
  const int k = (int)(threadIdx.x % K);
  const int lane = threadIdx.x & 31;
  const bool active = (int)threadIdx.x < rows_per_cta * K && u < n_max && u < n_uniq[0];
  Hyper h = load_hyper(hyper);
  const int64_t id = active ? uniq[u] : 0;
  const int l0 = active ? last[id] : j;
  const int64_t e = id * K + k;
  float x = active ? var[e] : 0.f, a = active ? slot0[e] : 0.f, b = (active && two) ? slot1[e] : 0.f;
  const int lmin = __reduce_min_sync(FULL_MASK, l0);   // warp-uniform trip count, lanes join at their own `last`
#pragma unroll 1
  for (int s = lmin; s < j; ++s) {
    h.lr = lr_table[s];
    float q = 0.f;
    if (s >= l0) {
      q = x * x;
      step_sparse<OPT>(x, a, b, __fmul_rn(h.l2, x), h);
    }
    q = warp_sum(q);
    if (lane == 0 && q != 0.f) atomicAdd(&ss_blk[s], q);
  }
  if (APPLY) {
    h.lr = lr_table[j];
    float q = 0.f;
    if (active) {
      q = x * x;
      step_sparse<OPT>(x, a, b, __fadd_rn(g_uniq[u * K + k], __fmul_rn(h.l2, x)), h);
    }
    q = warp_sum(q);
    if (lane == 0 && q != 0.f) atomicAdd(&ss_blk[j], q);
  }
  if (active && (APPLY || l0 < j)) {
    var[e] = x; slot0[e] = a;
    if (two) slot1[e] = b;
  }
  // the row's `last` byte is written after every k of the row has read it; a CTA holds whole rows, so a row
  // never straddles two CTAs
  __syncthreads();
  if (active && k == 0) last[id] = (uint8_t)(set_last >= 0 ? set_last : (APPLY ? j + 1 : j));
  if (threadIdx.x < EPOCH_MAX && ss_blk[threadIdx.x] != 0.f) atomicAdd(&ss[threadIdx.x], (double)ss_blk[threadIdx.x]);
}

// All rows: replay steps last[row]..upto-1, reset `last` where it was non-zero (reset == true) or
// raise it to `upto` (mid-epoch flush).  ss_partials[s][block] = sum(var^2) of the state step s
// started from, over this block's elements.
// warp w reduces the per-thread accumulators of steps w, w+8, ... (fixed order => deterministic)
__device__ __forceinline__ void sweep_ss_flush(float (*ss_thr)[256], int upto, double* __restrict__ ss_partials,
                                               int n_partials) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int s = warp; s < upto; s += 8) {
    double q = 0.0;
#pragma unroll
    for (int k = 0; k < 8; ++k) q += (double)ss_thr[s][lane + 32 * k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(FULL_MASK, q, o);
    if (lane == 0) ss_partials[(int64_t)s * n_partials + blockIdx.x] = q;
  }
}

// Adagrad / Momentum / Ftrl (Adam has its own sweep, epoch_adam.cu)
template <int OPT>
__global__ void __launch_bounds__(256, 3)
epoch_sweep_kernel(float* __restrict__ var, float* __restrict__ slot0, float* __restrict__ slot1,
                   uint8_t* __restrict__ last, int64_t n4, int K, const float* __restrict__ hyper,
                   const float* __restrict__ lr_table, int upto, int reset,
                   double* __restrict__ ss_partials, int n_partials) {
  constexpr bool two = OptTraits<OPT>::slots == 2;
  constexpr int UNROLL = 2;
  __shared__ float lr_s[EPOCH_MAX];
  // sum(var^2) seen at step s: one fp32 accumulator per thread and step (each takes a few thousand terms of
  // similar size), reduced once at the end; the cross-CTA sum is double (ctr_epoch_reg_loss)
  __shared__ float ss_thr[EPOCH_MAX][256];
  if (threadIdx.x < EPOCH_MAX) lr_s[threadIdx.x] = (threadIdx.x < upto) ? lr_table[threadIdx.x] : 0.f;
  for (int s = 0; s < upto; ++s) ss_thr[s][threadIdx.x] = 0.f;
  __syncthreads();
  Hyper h = load_hyper(hyper);
  float4* v4 = reinterpret_cast<float4*>(var);
  float4* a4 = reinterpret_cast<float4*>(slot0);
  float4* b4 = reinterpret_cast<float4*>(slot1);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int f4_per_row = K >> 2;  // K % 4 == 0 here
  const bool pow2 = (f4_per_row & (f4_per_row - 1)) == 0;
  const int sh = 31 - __clz(f4_per_row);
  auto row_of = [&](int64_t i) { return pow2 ? (i >> sh) : (i / f4_per_row); };
  auto row_head = [&](int64_t i) { return pow2 ? ((i & (f4_per_row - 1)) == 0) : ((i % f4_per_row) == 0); };
  // the loop bound is WARP-UNIFORM (the body contains full-mask shuffles); lanes past n4 are masked
  for (int64_t w0 = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31); w0 < n4; w0 += UNROLL * stride) {
    const int64_t i0 = w0 + (threadIdx.x & 31);
    float4 x[UNROLL], a[UNROLL], b[UNROLL];
    int l0[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const int64_t i = i0 + u * stride;
      if (i < n4) {
        x[u] = ld_stream4(v4 + i);
        a[u] = ld_stream4(a4 + i);
        b[u] = two ? ld_stream4(b4 + i) : f4_zero();
        l0[u] = last[row_of(i)];
      } else {
        x[u] = a[u] = b[u] = f4_zero();
        l0[u] = upto;
      }
    }
#pragma unroll 1
    for (int s = 0; s < upto; ++s) {
      h.lr = lr_s[s];
      float q = 0.f;
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        if (s >= l0[u]) {
          q += sq4(x[u]);
          step_untouched4<OPT>(x[u], a[u], b[u], h);
        }
      }
      ss_thr[s][threadIdx.x] += q;
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const int64_t i = i0 + u * stride;
      if (i < n4 && l0[u] < upto) {
        st_stream4(v4 + i, x[u]);
        st_stream4(a4 + i, a[u]);
        if (two) st_stream4(b4 + i, b[u]);
      }
      if (i < n4 && row_head(i)) {
        const uint8_t nl = reset ? (uint8_t)0 : (uint8_t)(l0[u] < upto ? upto : l0[u]);
        if ((uint8_t)l0[u] != nl) last[row_of(i)] = nl;
      }
    }
  }
  __syncthreads();
  sweep_ss_flush(ss_thr, upto, ss_partials, n_partials);
}

// K == 1 (first-order weights fm_w): a float4 spans 4 rows, each with its own `last` byte.  Adagrad / Momentum / Ftrl.
template <int OPT>
__global__ void __launch_bounds__(256)
epoch_sweep_k1_kernel(float* __restrict__ var, float* __restrict__ slot0, float* __restrict__ slot1,
                      uint8_t* __restrict__ last, int64_t n4, const float* __restrict__ hyper,
                      const float* __restrict__ lr_table, int upto, int reset,
                      double* __restrict__ ss_partials, int n_partials) {
  constexpr bool two = OptTraits<OPT>::slots == 2;
  __shared__ float lr_s[EPOCH_MAX];
  // sum(var^2) seen at step s: one fp32 accumulator per thread and step (each takes a few thousand terms of
  // similar size), reduced once at the end; the cross-CTA sum is double (ctr_epoch_reg_loss)
  __shared__ float ss_thr[EPOCH_MAX][256];
  if (threadIdx.x < EPOCH_MAX) lr_s[threadIdx.x] = (threadIdx.x < upto) ? lr_table[threadIdx.x] : 0.f;
  for (int s = 0; s < upto; ++s) ss_thr[s][threadIdx.x] = 0.f;
  __syncthreads();
  Hyper h = load_hyper(hyper);
  float4* v4 = reinterpret_cast<float4*>(var);
  float4* a4 = reinterpret_cast<float4*>(slot0);
  float4* b4 = reinterpret_cast<float4*>(slot1);
  uint32_t* l4 = reinterpret_cast<uint32_t*>(last);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t w0 = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31); w0 < n4; w0 += stride) {
    const int64_t i = w0 + (threadIdx.x & 31);
    const bool ok = i < n4;
    float4 x = f4_zero(), a = f4_zero(), b = f4_zero();
    uint32_t lw = 0;
    if (ok) {
      x = ld_stream4(v4 + i); a = ld_stream4(a4 + i); b = two ? ld_stream4(b4 + i) : f4_zero();
      lw = l4[i];
    }
    const int l0 = ok ? (int)(lw & 255u) : upto, l1 = ok ? (int)((lw >> 8) & 255u) : upto;
    const int l2_ = ok ? (int)((lw >> 16) & 255u) : upto, l3 = ok ? (int)(lw >> 24) : upto;
#pragma unroll 1
    for (int s = 0; s < upto; ++s) {
      h.lr = lr_s[s];
      float q = 0.f;
      if (s >= l0) { q += x.x * x.x; step_sparse<OPT>(x.x, a.x, b.x, __fmul_rn(h.l2, x.x), h); }
      if (s >= l1) { q += x.y * x.y; step_sparse<OPT>(x.y, a.y, b.y, __fmul_rn(h.l2, x.y), h); }
      if (s >= l2_) { q += x.z * x.z; step_sparse<OPT>(x.z, a.z, b.z, __fmul_rn(h.l2, x.z), h); }
      if (s >= l3) { q += x.w * x.w; step_sparse<OPT>(x.w, a.w, b.w, __fmul_rn(h.l2, x.w), h); }
      ss_thr[s][threadIdx.x] += q;
    }
    if (ok) {
      if (min(min(l0, l1), min(l2_, l3)) < upto) {
        st_stream4(v4 + i, x); st_stream4(a4 + i, a);
        if (two) st_stream4(b4 + i, b);
      }
      uint32_t nl = 0;
      if (!reset) {
        nl = (uint32_t)max(l0, upto) | ((uint32_t)max(l1, upto) << 8) | ((uint32_t)max(l2_, upto) << 16) |
             ((uint32_t)max(l3, upto) << 24);
      }
      if (nl != lw) l4[i] = nl;
    }
  }
  __syncthreads();
  sweep_ss_flush(ss_thr, upto, ss_partials, n_partials);
}

// scalar table / K % 4 != 0: one thread per element
template <int OPT>
__global__ void __launch_bounds__(256)
epoch_sweep_generic_kernel(float* __restrict__ var, float* __restrict__ slot0, float* __restrict__ slot1,
                           uint8_t* __restrict__ last, int64_t n_elem, int K,
                           const float* __restrict__ hyper, const float* __restrict__ lr_table, int upto,
                           int reset, double* __restrict__ ss_partials, int n_partials) {
  constexpr bool two = OptTraits<OPT>::slots == 2;
  __shared__ float lr_s[EPOCH_MAX];
  __shared__ double ss_blk[EPOCH_MAX];
  if (threadIdx.x < EPOCH_MAX) {
    lr_s[threadIdx.x] = (threadIdx.x < upto) ? lr_table[threadIdx.x] : 0.f;
    ss_blk[threadIdx.x] = 0.0;
  }
  __syncthreads();
  Hyper h = load_hyper(hyper);
  float ssq[EPOCH_MAX];
#pragma unroll
  for (int s = 0; s < EPOCH_MAX; ++s) ssq[s] = 0.f;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n_elem; e += stride) {
    const int64_t row = e / K;
    const int l0 = last[row];
    if (l0 < upto) {
      float x = var[e], a = slot0[e], b = two ? slot1[e] : 0.f;
#pragma unroll 1
      for (int s = l0; s < upto; ++s) {
        h.lr = lr_s[s];
        ssq[s] += x * x;
        step_sparse<OPT>(x, a, b, __fmul_rn(h.l2, x), h);
      }
      var[e] = x; slot0[e] = a;
      if (two) slot1[e] = b;
    }
  }
#pragma unroll 1
  for (int s = 0; s < upto; ++s) {
    float q = warp_sum(ssq[s]);
    if ((threadIdx.x & 31) == 0) atomicAdd(&ss_blk[s], (double)q);
  }
  __syncthreads();
  if (threadIdx.x < upto) ss_partials[(int64_t)threadIdx.x * n_partials + blockIdx.x] = ss_blk[threadIdx.x];
}

// `last` of the generic sweep is updated by a separate pass (all k of a row must have read it first)
__global__ void epoch_last_kernel(uint8_t* __restrict__ last, int64_t n_rows, int upto, int reset) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += stride) {
    const uint8_t l0 = last[r];
    const uint8_t nl = reset ? (uint8_t)0 : (uint8_t)(l0 < upto ? upto : l0);
    if (l0 != nl) last[r] = nl;
  }
}

// lr_table[j] = this step's lr_t; Adam: also refresh hyper[8*r] and advance the beta powers
__global__ void epoch_tick_kernel(float* __restrict__ state, float* __restrict__ hyper, int n_hyper,
                                  float* __restrict__ lr_table, int j, int is_adam) {
  float lr_t = state[2];
  if (is_adam) {
    const float b1p = state[0], b2p = state[1];
    lr_t = __fdiv_rn(__fmul_rn(state[2], __fsqrt_rn(__fsub_rn(1.f, b2p))), __fsub_rn(1.f, b1p));
    for (int r = 0; r < n_hyper; ++r) hyper[8 * r] = lr_t;
    state[0] = __fmul_rn(b1p, hyper[1]);
    state[1] = __fmul_rn(b2p, hyper[2]);
  }
  state[3] = state[3] + 1.f;
  lr_table[j] = lr_t;
}

// reg[s] = scale * (ss_rows[s] + sum_b partials[s][b]), s < upto; clears ss_rows for the next epoch
__global__ void epoch_reg_kernel(double* __restrict__ ss_rows, const double* __restrict__ partials,
                                 int n_partials, int upto, float scale, float* __restrict__ reg,
                                 int accumulate) {
  const int s = blockIdx.x;
  __shared__ double sh[256];
  double t = 0.0;
  for (int b = threadIdx.x; b < n_partials; b += 256) t += partials[(int64_t)s * n_partials + b];
  sh[threadIdx.x] = t;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0 && s < upto) {
    const float r = (float)((double)scale * (sh[0] + ss_rows[s]));
    reg[s] = accumulate ? reg[s] + r : r;
    ss_rows[s] = 0.0;
  }
}

}  // namespace ctr

using namespace ctr;

// ---- self-test of the in-range IEEE sqrt / div fast paths (optim_steps.cuh) ------------------------------
__device__ __forceinline__ uint64_t mix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
// a float with exponent uniformly in [e_lo, e_hi] (unbiased) and a mantissa that is random or one of the
// patterns that stress a divider / square root (all ones, all zeros, one bit, just below/above a power of 4)
__device__ __forceinline__ float test_float(uint64_t r, int e_lo, int e_hi) {
  const int e = e_lo + (int)((r >> 40) % (uint64_t)(e_hi - e_lo + 1));
  uint32_t man = (uint32_t)r & 0x7FFFFFu;
  switch ((r >> 32) & 15u) {
    case 0: man = 0x7FFFFFu; break;
    case 1: man = 0u; break;
    case 2: man = 1u; break;
    case 3: man = 0x7FFFFEu; break;
    case 4: man = 1u << ((r >> 36) % 23); break;
    case 5: man = 0x7FFFFFu ^ (1u << ((r >> 36) % 23)); break;
    default: break;
  }
  return __uint_as_float(((uint32_t)(e + 127) << 23) | man);
}
__global__ void __launch_bounds__(256) selftest_divsqrt_kernel(uint64_t seed, int64_t n, unsigned long long* mism) {
  unsigned long long bad_s = 0, bad_d = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t r0 = mix64(seed + 3 * (uint64_t)i), r1 = mix64(seed + 3 * (uint64_t)i + 1), r2 = mix64(seed + 3 * (uint64_t)i + 2);
    const float v = test_float(r0, -101, 39);
    if (__float_as_uint(sqrt_rn_inrange(v)) != __float_as_uint(__fsqrt_rn(v))) ++bad_s;
    // numerators over the whole guarded range [2^-100, 2^60) (half of them in the low decades), denominators over
    // [2^-51, 2^21) and, for a quarter of the cases, of the Adam shape sqrt(v) + eps
    float a = (r1 & 1) ? test_float(r1 >> 1, -100, -56) : test_float(r1 >> 1, -100, 59);
    float b = test_float(r2, -51, 20);
    if (r1 >> 63) a = -a;
    if (((r2 >> 61) & 3) == 0) b = __fadd_rn(__fsqrt_rn(v), 1e-8f);
    if (__float_as_uint(div_rn_inrange(a, b)) != __float_as_uint(__fdiv_rn(a, b))) ++bad_d;
    // a zero numerator: the fast path must give a zero (either sign: see adam_untouched)
    if (div_rn_inrange((r0 >> 62) & 1 ? -0.f : 0.f, b) != 0.f) ++bad_d;
  }
  if (bad_s) atomicAdd(&mism[0], bad_s);
  if (bad_d) atomicAdd(&mism[1], bad_d);
}

extern "C" {

int ctr_selftest_divsqrt(uint64_t seed, int64_t n, int64_t* mismatches, ctr_stream_t stream) {
  CTR_REQUIRE(mismatches && n >= 0, CTR_ERR_INVALID_ARG, "ctr_selftest_divsqrt: bad args");
  cudaStream_t st = as_stream(stream);
  CTR_REQUIRE(cudaMemsetAsync(mismatches, 0, 2 * sizeof(int64_t), st) == cudaSuccess, CTR_ERR_CUDA,
              "ctr_selftest_divsqrt: memset failed");
  if (n == 0) return CTR_OK;
  selftest_divsqrt_kernel<<<sm_count() * 8, 256, 0, st>>>(seed, n, reinterpret_cast<unsigned long long*>(mismatches));
  CTR_LAUNCHED("ctr_selftest_divsqrt");
  return CTR_OK;
}


int ctr_epoch_max_steps(void) { return EPOCH_MAX; }

int ctr_epoch_tick(float* state, float* hyper, int n_hyper, float* lr_table, int j, int is_adam,
                   ctr_stream_t stream) {
  CTR_REQUIRE(state && hyper && lr_table && n_hyper >= 1 && j >= 0 && j < EPOCH_MAX, CTR_ERR_INVALID_ARG,
              "ctr_epoch_tick: bad args (j=%d)", j);
  epoch_tick_kernel<<<1, 1, 0, as_stream(stream)>>>(state, hyper, n_hyper, lr_table, j, is_adam);
  CTR_LAUNCHED("ctr_epoch_tick");
  return CTR_OK;
}

static int launch_epoch_rows(int opt, int apply, float* var, float* slot0, float* slot1, uint8_t* last,
                             const int32_t* uniq, const int32_t* n_uniq, const float* g_uniq, int64_t n_max, int K,
                             const float* hyper, const float* lr_table, int j, double* ss, int set_last,
                             cudaStream_t st) {
  // generic path: a row's K threads sit in one CTA (they synchronise on the row's `last` byte); 256/K rows per CTA,
  // the CTA rounded up to whole warps
  const int gen_rows = K <= 256 ? 256 / K : 0;
  const int gen_block = (gen_rows * K + 31) / 32 * 32;
#define ER_K(OPT, AP, KK, LPR, VEC)                                                                  \
  case KK:                                                                                           \
    epoch_rows_kernel<OPT, LPR, VEC, AP><<<(unsigned)ceil_div64(n_max * LPR, 256), 256, 0, st>>>(    \
        var, slot0, slot1, last, uniq, n_uniq, g_uniq, n_max, hyper, lr_table, j, ss, set_last);     \
    break;
#define ER_AP(OPT, AP)                                                                               \
  switch (K) {                                                                                       \
    ER_K(OPT, AP, 4, 1, 1) ER_K(OPT, AP, 8, 2, 1) ER_K(OPT, AP, 16, 4, 1) ER_K(OPT, AP, 32, 8, 1)    \
    ER_K(OPT, AP, 64, 16, 1) ER_K(OPT, AP, 128, 32, 1) ER_K(OPT, AP, 256, 32, 2)                     \
    default:                                                                                         \
      epoch_rows_generic_kernel<OPT, AP><<<(unsigned)ceil_div64(n_max, gen_rows), gen_block, 0, st>>>(   \
          var, slot0, slot1, last, uniq, n_uniq, g_uniq, n_max, K, hyper, lr_table, j, ss, set_last); \
  }
#define ER_CALL(OPT)                     \
  if (apply) { ER_AP(OPT, true) } else { ER_AP(OPT, false) }
  CTR_OPT_SWITCH(opt, ER_CALL)
#undef ER_CALL
#undef ER_AP
#undef ER_K
  CTR_LAUNCHED("ctr_epoch_rows");
  return CTR_OK;
}

static bool epoch_rows2_supported(int K) {
  return K == 4 || K == 8 || K == 16 || K == 32 || K == 64 || K == 128 || K == 256;
}

static bool epoch_rows_supported(int K) {
  return K >= 1 && K <= 256;
}

int ctr_epoch_rows(int opt, int apply, float* var, float* slot0, float* slot1, uint8_t* last,
                   const int32_t* uniq, const int32_t* n_uniq, const float* g_uniq, int64_t n_max, int K,
                   const float* hyper, const float* lr_table, int j, double* ss, ctr_stream_t stream) {
  CTR_REQUIRE(n_max >= 0 && K > 0 && j >= 0 && j < EPOCH_MAX, CTR_ERR_INVALID_ARG,
              "ctr_epoch_rows: bad n_max/K/j");
  if (n_max == 0) return CTR_OK;
  CTR_REQUIRE(var && slot0 && last && uniq && n_uniq && hyper && lr_table && ss, CTR_ERR_INVALID_ARG,
              "ctr_epoch_rows: null buffer");
  CTR_REQUIRE(!apply || g_uniq, CTR_ERR_INVALID_ARG, "ctr_epoch_rows: g_uniq required when apply != 0");
  CTR_REQUIRE(n_slots_of(opt) == 1 || slot1, CTR_ERR_INVALID_ARG, "ctr_epoch_rows: slot1 required");
  CTR_REQUIRE(epoch_rows_supported(K), CTR_ERR_UNSUPPORTED, "ctr_epoch_rows: K=%d must be <= 256", K);
  return launch_epoch_rows(opt, apply, var, slot0, slot1, last, uniq, n_uniq, g_uniq, n_max, K, hyper, lr_table, j,
                           ss, -1, as_stream(stream));
}

// The [N,K] table and a scalar table [N] gathered with the same ids (fm_v + fm_w), in ONE launch: lane 0 of every row
// carries the scalar table's element.  Same arithmetic as two ctr_epoch_rows calls.
static int launch_epoch_rows2(int opt, int apply, float* var, float* slot0, float* slot1, uint8_t* last,
                              const RowsW& w, const int32_t* uniq, const int32_t* n_uniq, const float* g_uniq,
                              int64_t n_max, int K, const float* hyper, const float* lr_table, int j, double* ss,
                              int set_last, cudaStream_t st) {
  const bool staged = w.stage != nullptr;
#define ER2_K(OPT, AP, KK, LPR, VEC)                                                                       \
  case KK:                                                                                                 \
    if (staged)                                                                                            \
      epoch_rows_kernel<OPT, LPR, VEC, AP, true, true><<<(unsigned)ceil_div64(n_max * LPR, 256), 256, 0, st>>>( \
          var, slot0, slot1, last, uniq, n_uniq, g_uniq, n_max, hyper, lr_table, j, ss, set_last, w);      \
    else                                                                                                   \
      epoch_rows_kernel<OPT, LPR, VEC, AP, true><<<(unsigned)ceil_div64(n_max * LPR, 256), 256, 0, st>>>(  \
          var, slot0, slot1, last, uniq, n_uniq, g_uniq, n_max, hyper, lr_table, j, ss, set_last, w);      \
    break;
#define ER2_AP(OPT, AP)                                                                                    \
  switch (K) {                                                                                             \
    ER2_K(OPT, AP, 4, 1, 1) ER2_K(OPT, AP, 8, 2, 1) ER2_K(OPT, AP, 16, 4, 1) ER2_K(OPT, AP, 32, 8, 1)      \
    ER2_K(OPT, AP, 64, 16, 1) ER2_K(OPT, AP, 128, 32, 1) ER2_K(OPT, AP, 256, 32, 2)                        \
  }
#define ER2_CALL(OPT) if (apply) { ER2_AP(OPT, true) } else { ER2_AP(OPT, false) }
  CTR_OPT_SWITCH(opt, ER2_CALL)
#undef ER2_CALL
#undef ER2_AP
#undef ER2_K
  CTR_LAUNCHED("ctr_epoch_rows2");
  return CTR_OK;
}

// w_last == last: the tables share one `last` byte per row (ctr_epoch_sweep with a scalar table).  stage / w_stage:
// both NULL, or both given (the staged hand-over of the catch-up and the apply of one step, epoch_rows_kernel STAGED).
int ctr_epoch_rows2(int opt, int apply, float* var, float* slot0, float* slot1, uint8_t* last, float* w_var, float* w_slot0,
                    float* w_slot1, uint8_t* w_last, const int32_t* uniq, const int32_t* n_uniq, const float* g_uniq,
                    const float* gw_uniq, int64_t n_max, int K, const float* hyper, const float* lr_table, int j, double* ss,
                    double* ss_w, float* stage, float* w_stage, ctr_stream_t stream) {
  CTR_REQUIRE(n_max >= 0 && j >= 0 && j < EPOCH_MAX, CTR_ERR_INVALID_ARG, "ctr_epoch_rows2: bad n_max/j");
  CTR_REQUIRE(epoch_rows2_supported(K), CTR_ERR_UNSUPPORTED, "ctr_epoch_rows2: K=%d (supported: 4..256 powers of two)", K);
  CTR_REQUIRE(!stage == !w_stage, CTR_ERR_INVALID_ARG, "ctr_epoch_rows2: stage and w_stage must both be given or both NULL");
  if (n_max == 0) return CTR_OK;
  CTR_REQUIRE(var && slot0 && last && w_var && w_slot0 && w_last && uniq && n_uniq && hyper && lr_table && ss && ss_w,
              CTR_ERR_INVALID_ARG, "ctr_epoch_rows2: null buffer");
  CTR_REQUIRE(!apply || (g_uniq && gw_uniq), CTR_ERR_INVALID_ARG, "ctr_epoch_rows2: gradients required when apply != 0");
  CTR_REQUIRE(n_slots_of(opt) == 1 || (slot1 && w_slot1), CTR_ERR_INVALID_ARG, "ctr_epoch_rows2: slot1 required");
  RowsW w;
  w.var = w_var; w.slot0 = w_slot0; w.slot1 = w_slot1; w.last = (w_last == last) ? nullptr : w_last; w.g_uniq = gw_uniq;
  w.ss = ss_w; w.stage = stage; w.w_stage = w_stage;
  return launch_epoch_rows2(opt, apply, var, slot0, slot1, last, w, uniq, n_uniq, g_uniq, n_max, K, hyper, lr_table, j,
                            ss, -1, as_stream(stream));
}

int ctr_epoch_shared_last_supported(int opt, int64_t n_rows, int K) {
  return opt == CTR_OPT_ADAM && epoch_rows2_supported(K) && n_rows > 0 && n_rows % 4 == 0;
}

// the sweep kernels of Adagrad, Momentum and Ftrl (Adam takes the packed sweep of epoch_adam.cu)
#define EPOCH_NON_ADAM_SWITCH(opt, CALL)                                 \
  switch (opt) {                                                         \
    case CTR_OPT_ADAGRAD: { CALL(CTR_OPT_ADAGRAD) } break;               \
    case CTR_OPT_MOMENTUM: { CALL(CTR_OPT_MOMENTUM) } break;             \
    case CTR_OPT_FTRL: { CALL(CTR_OPT_FTRL) } break;                     \
    default:                                                             \
      ::ctr::set_error("unknown optimizer %d", opt);                     \
      return CTR_ERR_INVALID_ARG;                                        \
  }

int ctr_epoch_sweep(int opt, float* var, float* slot0, float* slot1, float* w_var, float* w_slot0, float* w_slot1,
                    uint8_t* last, int64_t n_rows, int K, const float* hyper, const float* lr_table, int from, int upto,
                    int reset, double* ss_partials, double* w_ss_partials, int* n_partials_host, int32_t* list,
                    int64_t list_cap, int32_t* list_count, double* ss_rows, double* w_ss_rows, int32_t* list_overflow,
                    ctr_stream_t stream) {
  CTR_REQUIRE(n_rows >= 0 && K > 0 && from >= 0 && from <= upto && upto <= EPOCH_MAX, CTR_ERR_INVALID_ARG,
              "ctr_epoch_sweep: bad n_rows/K/from/upto");
  // the scalar table that shares `last` (fm_w next to fm_v): all of its buffers or none
  const bool with_w = w_var != nullptr;
  CTR_REQUIRE(with_w ? (w_slot0 && w_slot1 && w_ss_partials && w_ss_rows)
                     : !(w_slot0 || w_slot1 || w_ss_partials || w_ss_rows),
              CTR_ERR_INVALID_ARG, "ctr_epoch_sweep: w_var, w_slot0, w_slot1, w_ss_partials, w_ss_rows: all or none");
  CTR_REQUIRE(!with_w || ctr_epoch_shared_last_supported(opt, n_rows, K), CTR_ERR_UNSUPPORTED,
              "ctr_epoch_sweep: a shared `last` needs Adam, K in {4..256} powers of two and n_rows %% 4 == 0 "
              "(K=%d, n_rows=%lld)", K, (long long)n_rows);
  const int grid = sm_count() * 3;
  const int n_partials = sm_count() * 6;     // row length of ss_partials (>= every grid used here)
  if (n_partials_host) *n_partials_host = n_partials;
  if (n_rows == 0 || upto == 0) return CTR_OK;
  CTR_REQUIRE(var && slot0 && last && hyper && lr_table && ss_partials, CTR_ERR_INVALID_ARG,
              "ctr_epoch_sweep: null buffer");
  CTR_REQUIRE(n_slots_of(opt) == 1 || slot1, CTR_ERR_INVALID_ARG, "ctr_epoch_sweep: slot1 required");
  const bool last_aligned = ((uintptr_t)last & 3) == 0;
  CTR_REQUIRE(!with_w || last_aligned, CTR_ERR_INVALID_ARG, "ctr_epoch_sweep: a shared `last` must be 4-byte aligned");
  cudaStream_t st = as_stream(stream);
  const int64_t n_elem = n_rows * K;
  const int f4 = K / 4;
  const bool row_in_warp = K % 4 == 0 && (f4 & (f4 - 1)) == 0 && f4 <= 32;
  const bool k1_packed = K == 1 && n_rows % 4 == 0 && last_aligned;   // a float4 holds 4 rows, a uint32 their `last`

  if (opt == CTR_OPT_ADAM) {
    CTR_REQUIRE(list && list_count && ss_rows && list_cap > 0, CTR_ERR_INVALID_ARG,
                "ctr_epoch_sweep: Adam needs list, list_count, ss_rows and list_cap > 0");
    if ((K % 4 == 0 && epoch_rows_supported(K)) || k1_packed) {
      // ---- the packed pipe (epoch_adam.cu): untouched rows here, gathered rows through `list` ----------------
      if (from == upto) {   // nothing to replay (a flush reached upto already): no step's partials, `last` -> 0 on reset
        const size_t bytes = (size_t)upto * n_partials * sizeof(double);
        CTR_REQUIRE(cudaMemsetAsync(ss_partials, 0, bytes, st) == cudaSuccess &&
                    (!with_w || cudaMemsetAsync(w_ss_partials, 0, bytes, st) == cudaSuccess), CTR_ERR_CUDA,
                    "ctr_epoch_sweep: memset failed");
        if (reset) {
          epoch_last_kernel<<<grid, 256, 0, st>>>(last, n_rows, upto, reset);
          CTR_LAUNCHED("ctr_epoch_sweep(last)");
        }
        return CTR_OK;
      }
      CTR_REQUIRE(cudaMemsetAsync(list_count, 0, sizeof(int32_t), st) == cudaSuccess, CTR_ERR_CUDA,
                  "ctr_epoch_sweep: memset failed");
      const bool ok = launch_epoch_sweep_adam(var, slot0, slot1, last, n_rows, K, hyper, lr_table, from, upto,
                                              ss_partials, n_partials, list, list_count, list_cap, list_overflow, st,
                                              w_var, w_slot0, w_slot1, w_ss_partials);
      CTR_REQUIRE(ok, CTR_ERR_UNSUPPORTED, "ctr_epoch_sweep: packed path refused K=%d", K);
      CTR_LAUNCHED("ctr_epoch_sweep(adam)");
      // rows gathered since `from` (both tables): catch up from their own `last` to upto; they get their final `last` here
      int rc;
      if (with_w) {
        RowsW w;
        w.var = w_var; w.slot0 = w_slot0; w.slot1 = w_slot1; w.last = nullptr; w.g_uniq = nullptr; w.ss = w_ss_rows;
        rc = launch_epoch_rows2(opt, 0, var, slot0, slot1, last, w, list, list_count, nullptr, list_cap, K, hyper,
                                lr_table, upto, ss_rows, reset ? 0 : upto, st);
      } else {
        rc = launch_epoch_rows(opt, 0, var, slot0, slot1, last, list, list_count, nullptr, list_cap, K, hyper, lr_table,
                               upto, ss_rows, reset ? 0 : upto, st);
      }
      if (rc != CTR_OK) return rc;
      if (!(reset && from == 0)) {   // untouched rows hold `from`: rewrite (an epoch-end sweep leaves their 0 alone)
        epoch_last_kernel<<<grid, 256, 0, st>>>(last, n_rows, upto, reset);
        CTR_LAUNCHED("ctr_epoch_sweep(last)");
      }
      return CTR_OK;
    }
  } else if (row_in_warp) {   // a row's float4s sit in one warp: `last` can be rewritten in place
#define ES_CALL(OPT)                                                                           \
  epoch_sweep_kernel<OPT><<<grid, 256, 0, st>>>(var, slot0, slot1, last, n_elem / 4, K, hyper, \
                                                lr_table, upto, reset, ss_partials, n_partials);
    EPOCH_NON_ADAM_SWITCH(opt, ES_CALL)
#undef ES_CALL
    CTR_LAUNCHED("ctr_epoch_sweep");
    return CTR_OK;
  } else if (k1_packed) {
#define ES1_CALL(OPT)                                                                                \
  epoch_sweep_k1_kernel<OPT><<<grid, 256, 0, st>>>(var, slot0, slot1, last, n_rows / 4, hyper, lr_table, \
                                                   upto, reset, ss_partials, n_partials);
    EPOCH_NON_ADAM_SWITCH(opt, ES1_CALL)
#undef ES1_CALL
    CTR_LAUNCHED("ctr_epoch_sweep(k1)");
    return CTR_OK;
  }
  // rows that span warps / CTAs (K/4 not a power of two <= 32, Adam: K > 256) or K % 4 != 0: one thread per element,
  // `last` rewritten by a separate pass once every element of the row has read it
#define ESG_CALL(OPT)                                                                                \
  epoch_sweep_generic_kernel<OPT><<<grid, 256, 0, st>>>(var, slot0, slot1, last, n_elem, K, hyper,   \
                                                        lr_table, upto, reset, ss_partials, n_partials);
  CTR_OPT_SWITCH(opt, ESG_CALL)
#undef ESG_CALL
  CTR_LAUNCHED("ctr_epoch_sweep(generic)");
  epoch_last_kernel<<<grid, 256, 0, st>>>(last, n_rows, upto, reset);
  CTR_LAUNCHED("ctr_epoch_sweep(last)");
  return CTR_OK;
}
#undef EPOCH_NON_ADAM_SWITCH

int ctr_epoch_reg_loss(double* ss_rows, const double* ss_partials, int n_partials, int upto, float scale,
                       float* reg, int accumulate, ctr_stream_t stream) {
  CTR_REQUIRE(ss_rows && ss_partials && reg && n_partials >= 0 && upto >= 0 && upto <= EPOCH_MAX,
              CTR_ERR_INVALID_ARG, "ctr_epoch_reg_loss: bad args");
  if (upto == 0) return CTR_OK;
  epoch_reg_kernel<<<upto, 256, 0, as_stream(stream)>>>(ss_rows, ss_partials, n_partials, upto, scale, reg,
                                                        accumulate);
  CTR_LAUNCHED("ctr_epoch_reg_loss");
  return CTR_OK;
}

}  // extern "C"
