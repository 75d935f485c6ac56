/*
 * ctr_b200.h -- C ABI of libctr_b200.so, the H100 (sm_90a) CTR feature-interaction engine.
 *
 * This is the drop-in boundary for the hot path of lambdaji/tf_repos'
 * deep_ctr/Model_pipeline/*.py `model_fn`s.  The reference has no FFI of its own (it is
 * TensorFlow-1.4 Python); each entry point below replaces the cluster of TF ops cited next to
 * it (file:line relative to the reference checkout).  INTEGRATION.md shows the ctypes binding a
 * maintainer of the reference would add.
 *
 * Conventions
 *  - every pointer is a DEVICE pointer owned by the caller unless the name ends in `_host`;
 *    tensors are contiguous row-major fp32 / int32 (ids may be int32 or int64, see id_bits);
 *  - no allocation inside the library: scratch is caller-provided, sized by *_workspace_bytes();
 *  - every call enqueues work on `stream` and returns immediately (no host sync, graph-capturable);
 *  - return value: 0 = CTR_OK, <0 = ctr_status; text via ctr_last_error() (thread-local);
 *  - no C++ exception crosses the ABI; no global mutable state except the launch counter.
 */
#ifndef CTR_B200_H_
#define CTR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* ctr_stream_t; /* a cudaStream_t / CUstream */

enum ctr_status {
  CTR_OK = 0,
  CTR_ERR_INVALID_ARG = -1,
  CTR_ERR_UNSUPPORTED = -2,
  CTR_ERR_CUDA = -3,
  CTR_ERR_WORKSPACE = -4
};

/* interaction modes of the embedding kernels */
enum ctr_fm_mode {
  CTR_FM_DEEPFM = 0, /* y_v[B] = 0.5*sum_k((sum_f e)^2 - sum_f e^2)        DeepFM.py:129-135 */
  CTR_FM_NFM = 1,    /* bi[B,K] = 0.5*((sum_f e)^2 - sum_f e^2)            NFM.py:122-128    */
  CTR_FM_PLAIN = 2   /* gather+scale only                                  DCN.py:135-138, PNN.py:134-136, AFM.py:128-130 */
};

enum ctr_optimizer {
  CTR_OPT_ADAM = 0,     /* tf.train.AdamOptimizer      DeepFM.py:205 */
  CTR_OPT_ADAGRAD = 1,  /* tf.train.AdagradOptimizer   DeepFM.py:207 */
  CTR_OPT_MOMENTUM = 2, /* tf.train.MomentumOptimizer  DeepFM.py:209 */
  CTR_OPT_FTRL = 3      /* tf.train.FtrlOptimizer      DeepFM.py:211 */
};

/* ---- library ------------------------------------------------------------------------------- */
int ctr_abi_version(void);
const char* ctr_last_error(void);
/* number of kernels this library has launched in this process (bench.py's gpu_launches) */
int64_t ctr_launch_count(void);
/* number of SMs the library sized its persistent grids for (132 on H100 SXM); <0 on error */
int ctr_device_sm_count(void);

/* ---- K1: gather + scale + FM first/second order + emit x ------------------------------------
 * Replaces tf.nn.embedding_lookup(FM_W/FM_V) + multiply + reduce_sum/square chain,
 * DeepFM.py:125-135,151 (NFM.py:118-128; plain gather DCN.py:135-138).
 *   ids   [B,F]  int32 (id_bits=32) or int64 (id_bits=64); vals [B,F] f32
 *   V     [N,K]  f32;   W [N] f32 or NULL (no first-order term)
 *   x     [B,F*K] = V[ids]*vals            (NULL to skip; NFM does not need it)
 *   y_w   [B]     = sum_f W[ids]*vals      (NULL iff W NULL)
 *   y2    mode DEEPFM: [B]; mode NFM: [B,K]; mode PLAIN: ignored (may be NULL)
 *   S     [B,K]   = sum_f e  (saved for the backward; NULL in PLAIN mode)
 *   oob   optional int32[2] device word: {count, first bad id}; TF raises InvalidArgument for ids
 *         outside [0,N) on CPU -- here such an occurrence contributes 0 and is counted.
 */
int ctr_fm_embed_fwd(const void* ids, int id_bits, const float* vals, const float* V, const float* W,
                     int64_t N, int B, int F, int K, int mode, float* x, float* y_w, float* y2,
                     float* S, int32_t* oob, ctr_stream_t stream);

/* ---- K2: backward of K1 w.r.t. the gathered rows ---------------------------------------------
 * Replaces the autodiff of DeepFM.py:125-135,151 that optimizer.minimize (DeepFM.py:213) builds:
 * per-occurrence IndexedSlices values for FM_V and FM_W.
 *   x   [B,F*K] the scaled embeddings saved by the forward;  S [B,K] saved by the forward
 *   dX  [B,F*K] upstream grad of x (NULL = 0);  dy2: DEEPFM [B] upstream of y_v, NFM [B,K] of bi
 *   dyw [B] upstream of y_w (NULL iff g_w NULL)
 *   g_rows [B*F,K] = (dy2*(S-e) + dX) * val ;  g_w [B*F] = dyw*val
 */
int ctr_fm_embed_bwd(const float* vals, const float* x, const float* S, const float* dX,
                     const float* dy2, const float* dyw, int B, int F, int K, int mode,
                     float* g_rows, float* g_w, ctr_stream_t stream);

/* ---- K3: de-duplication of IndexedSlices ------------------------------------------------------
 * Replaces optimizer._deduplicate_indexed_slices = tf.unique + unsorted_segment_sum that
 * optimizer.minimize applies to the embedding gradients (DeepFM.py:213, [TF-sem]).
 * Stable LSD radix sort of (id, position), then run-length encoding.  Integer outputs are
 * bit-exact w.r.t. numpy.unique(return_inverse=True) + a stable argsort:
 *   perm        [n]  positions 0..n-1 sorted by (id, position)
 *   uniq        [n]  ascending distinct ids (first *n_uniq valid)
 *   inverse     [n]  inverse[p] = index into uniq of ids[p]
 *   seg_offsets [n+1] run starts in the sorted order; seg_offsets[*n_uniq] = n
 *   n_uniq      int32[1] device scalar
 *   long_list   int32[n+1] scratch-out: [0] = number of runs longer than CTR_LONG_SEG, then their
 *               uniq indices (consumed by ctr_segment_sum_rows)
 */
#define CTR_LONG_SEG 128
size_t ctr_unique_segment_workspace_bytes(int64_t n, int64_t N);
int ctr_unique_segment(const int32_t* ids, int64_t n, int64_t N, int32_t* perm, int32_t* uniq,
                       int32_t* inverse, int32_t* seg_offsets, int32_t* n_uniq, int32_t* long_list,
                       void* ws, size_t ws_bytes, ctr_stream_t stream);

/* g_uniq[u,:] = sum over the run u of g_rows[perm[i],:]  (fixed-shape trees: deterministic).
 * g_w / gw_uniq are the optional scalar column of the first-order table (NULL to skip). */
int ctr_segment_sum_rows(const float* g_rows, const float* g_w, const int32_t* perm,
                         const int32_t* seg_offsets, const int32_t* n_uniq,
                         const int32_t* long_list, int64_t n, int K, float* g_uniq, float* gw_uniq,
                         void* ws /* optional scratch (e.g. the ctr_unique_segment workspace, free by now): runs longer than
                         CTR_LONG_SEG are cut into 1024-occurrence chunks summed by separate CTAs and added in chunk order
                         (as many runs as the scratch has partial rows for); NULL = one CTA per long run */,
                         size_t ws_bytes, ctr_stream_t stream);

/* ---- K4: optimizer apply on table rows ---------------------------------------------------------
 * TF-1.x arithmetic, [TF-sem] (see oracle/tf_semantics.py for the restatement and its sources).
 * `hyper` is a DEVICE float[8]: {lr_t, beta1, beta2, eps, l2_reg, aux0, aux1, aux2} so that a
 * captured CUDA graph can be replayed while the step counter advances.
 *   Adam:     lr_t = lr*sqrt(1-b2^t)/(1-b1^t) precomputed (ctr_adam_tick);
 *   Adagrad:  lr_t = lr;            slot0 = accumulator
 *   Momentum: lr_t = lr; aux0 = momentum; slot0 = accumulator
 *   Ftrl:     lr_t = lr; aux0 = lr_power, aux1 = l1, aux2 = l2(ftrl);  slot0 = accum, slot1 = linear
 *
 * sparse apply: rows uniq[0..*n_uniq) get g = g_uniq + l2_reg*var and the optimizer's *sparse*
 * update.  If stage != NULL the new (var, slot0, slot1) rows are written to stage[3][n][K]
 * instead of in place (exact mode: the dense sweep runs next, then ctr_opt_patch_rows).
 */
int ctr_opt_sparse_rows(int opt, float* var, float* slot0, float* slot1, const int32_t* uniq,
                        const int32_t* n_uniq, const float* g_uniq, int64_t n_max, int K,
                        const float* hyper, float* stage, ctr_stream_t stream);
/* dense sweep: every one of the n_elem elements takes the step with g = l2_reg*var (what TF does
 * to rows no gather touched, because l2_loss densifies the gradient and sparse Adam decays every
 * row).  Also accumulates sum(var_old^2) into sumsq_partials[grid] (for tf.nn.l2_loss in the
 * loss, DeepFM.py:189-190) when non-NULL; *n_partials returns the number written. */
int ctr_opt_dense_sweep(int opt, float* var, float* slot0, float* slot1, int64_t n_elem,
                        const float* hyper, float* sumsq_partials, int* n_partials_host,
                        ctr_stream_t stream);
int ctr_opt_patch_rows(float* var, float* slot0, float* slot1, const int32_t* uniq,
                       const int32_t* n_uniq, const float* stage, int64_t n_max, int K, int n_slots,
                       ctr_stream_t stream);
/* dense variables with an explicit gradient (MLP weights, biases, fm_bias, cross_w/b):
 * TF's fused ApplyAdam/ApplyAdagrad/ApplyMomentum/ApplyFtrl kernels; g += l2_reg*var first when
 * l2_reg (hyper[4]) != 0. */
int ctr_opt_dense_grad(int opt, float* var, float* slot0, float* slot1, const float* grad,
                       int64_t n_elem, const float* hyper, ctr_stream_t stream);
/* Called once at the start of a step: lr_t = lr*sqrt(1-b2p)/(1-b1p) from the CURRENT beta powers is
 * written to hyper[8*r] for r < n_hyper (consecutive hyper records: tables, dense variables ...),
 * then the powers advance the way AdamOptimizer._finish does (fp32 running products) and the step
 * counter increments.  state = device float[4] {beta1_power, beta2_power, lr, global_step}. */
int ctr_adam_tick(float* state, float* hyper, int n_hyper, ctr_stream_t stream);
/* deterministic sum of n floats -> out[0] (two-level fixed tree) ; scale applied at the end */
int ctr_reduce_sum(const float* in, int64_t n, float scale, float* out, float* ws, size_t ws_bytes,
                   ctr_stream_t stream);
/* 0.5*sum(t^2) (tf.nn.l2_loss) of a whole tensor, deterministic */
size_t ctr_l2_loss_workspace_bytes(int64_t n);
/* out[0] = scale * 0.5 * sum(t^2) */
int ctr_l2_loss(const float* t, int64_t n, float scale, float* out, void* ws, size_t ws_bytes, ctr_stream_t stream);

/* ---- K4': exact-deferred ("epoch") table update ---------------------------------------------------
 * Same results, bit for bit, as ctr_opt_sparse_rows(stage) + ctr_opt_dense_sweep + ctr_opt_patch_rows
 * every step, at 1/P of the HBM traffic: the update TF gives a row that nothing gathered
 * (g = l2_reg*var, DeepFM.py:189-190 + non-lazy sparse Adam, [TF-sem]) is an element-wise recurrence,
 * so it is replayed lazily -- when a batch gathers the row (ctr_epoch_rows) or once per epoch of P
 * steps for all rows in one pass over HBM (ctr_epoch_sweep).
 *   last      uint8[N] per row: steps of the current epoch already applied to the stored state
 *   lr_table  device float[ctr_epoch_max_steps()]: lr_t of every step of the current epoch
 *   ss        device double[ctr_epoch_max_steps()]: sum(var^2) seen by the row kernels, per step
 * Step j of an epoch:  ctr_epoch_tick(j) ; ctr_unique_segment(ids) ;
 *   ctr_epoch_rows(apply=0, j)  -> gathered rows hold the state at the start of step j
 *   forward / backward / ctr_segment_sum_rows ;  ctr_epoch_rows(apply=1, j) ;
 *   after the last step (or to flush mid-epoch): ctr_epoch_sweep(upto, reset) ; ctr_epoch_reg_loss.
 */
int ctr_epoch_max_steps(void);
int ctr_epoch_tick(float* state, float* hyper, int n_hyper, float* lr_table, int j, int is_adam,
                   ctr_stream_t stream);
int ctr_epoch_rows(int opt, int apply, float* var, float* slot0, float* slot1, uint8_t* last,
                   const int32_t* uniq, const int32_t* n_uniq, const float* g_uniq, int64_t n_max, int K,
                   const float* hyper, const float* lr_table, int j, double* ss, ctr_stream_t stream);
/* ctr_epoch_rows for the [N,K] table AND a scalar table [N] gathered with the same ids (fm_v + fm_w, DeepFM.py:115-116)
 * in one launch; K in {4, 8, 16, 32, 64, 128, 256}.  Same arithmetic as two ctr_epoch_rows calls.  w_last == last: the
 * tables share one `last` byte per row (see ctr_epoch_sweep).
 * stage / w_stage: both NULL, or both given (device float[n_max * 3K] and float[n_max * 3], indexed by unique row).
 * Given, the catch-up (apply=0) and the apply (apply=1) of the same step j hand the rows over through them: the catch-up
 * writes the caught-up var | slot0 | slot1 there and only var back to the tables; the apply reads them from there and
 * writes every row, slot and `last` byte.  Same results as without a stage.  Both calls of a step must then use the same
 * uniq / n_uniq and stage, and between them only var of the gathered rows may be read (the slots and `last` are stale). */
int ctr_epoch_rows2(int opt, int apply, float* var, float* slot0, float* slot1, uint8_t* last, float* w_var, float* w_slot0,
                    float* w_slot1, uint8_t* w_last, const int32_t* uniq, const int32_t* n_uniq, const float* g_uniq,
                    const float* gw_uniq, int64_t n_max, int K, const float* hyper, const float* lr_table, int j, double* ss,
                    double* ss_w, float* stage, float* w_stage, ctr_stream_t stream);
/* All rows -> state after `upto` steps of this epoch.  Rows whose `last` byte equals `from` (nothing gathered
 * them since the previous sweep; from = 0 after an epoch-end sweep) replay steps from..upto-1; the others replay
 * last..upto-1.  reset != 0: epoch end, every `last` byte returns to 0; reset == 0: mid-epoch flush, `last` = upto.
 * ss_partials: device double[ctr_epoch_max_steps()][*n_partials_host] (*n_partials_host is always
 * 6 * ctr_device_sm_count(), so it can be sized before the first call), ZERO-INITIALISED ONCE by the caller: a call
 * rewrites, for every step < upto, one entry per CTA it launches (fewer than *n_partials_host) and ctr_epoch_reg_loss
 * sums whole rows, so the entries no CTA owns must hold 0.
 * list / list_cap / list_count / ss_rows: required for Adam (CTR_ERR_INVALID_ARG if one is missing or list_cap is 0),
 * unused otherwise: device int32[list_cap], a device int32 counter, and the row kernels' per-step sum(var^2)
 * accumulator (the `ss` of ctr_epoch_rows).  Adam with K % 4 == 0 and K <= 256, or K == 1 with n_rows % 4 == 0 and a
 * 4-byte aligned `last`, takes the packed-pipe sweep (csrc/epoch_adam.cu): it lists the rows gathered since `from`
 * and catches them up in a second pass.
 * CAPACITY: the list receives every row whose `last` byte exceeds `from`, i.e. every row a ctr_epoch_rows call
 * gathered since the previous sweep.  With at most n_ids distinct ids per step that is at most
 * min(n_rows, n_ids * (upto - from)) <= min(n_rows, n_ids * ctr_epoch_max_steps()) rows; list_cap must be at least
 * that.  *list_count returns the number of gathered rows found.  If it exceeds list_cap, the rows beyond list_cap
 * were NOT caught up although their `last` byte is rewritten: the table is wrong.
 * list_overflow (nullable): device int32 counter to which the packed sweep ADDS the number of gathered rows it found
 * beyond list_cap (it is not cleared here).  Non-zero after a call means the capacity rule above was broken and the
 * table no longer holds the every-step state; the models' check_ids() raises on it.
 * w_var, w_slot0, w_slot1, w_ss_partials, w_ss_rows: all NULL (one table), or all given: a scalar table [n_rows]
 * gathered with the same ids as the [N,K] table (fm_v + fm_w) that shares its `last` bytes (pass the same `last` to
 * ctr_epoch_rows2 as both last and w_last).  One launch then sweeps both tables, rows gathered since `from` go to one
 * list, and its catch-up steps both tables; w_ss_partials / w_ss_rows are the scalar table's ss_partials / ss_rows.
 * The list holds each gathered ROW once (not once per table), so the same list_cap covers both.  Needs
 * ctr_epoch_shared_last_supported (Adam, K in {4, 8, ..., 256}, n_rows % 4 == 0) and a 4-byte aligned `last`;
 * otherwise keep one `last` array per table and sweep each on its own. */
int ctr_epoch_shared_last_supported(int opt, int64_t n_rows, int K);
int ctr_epoch_sweep(int opt, float* var, float* slot0, float* slot1, float* w_var, float* w_slot0, float* w_slot1,
                    uint8_t* last, int64_t n_rows, int K, const float* hyper, const float* lr_table, int from, int upto,
                    int reset, double* ss_partials, double* w_ss_partials, int* n_partials_host, int32_t* list,
                    int64_t list_cap, int32_t* list_count, double* ss_rows, double* w_ss_rows, int32_t* list_overflow,
                    ctr_stream_t stream);
/* reg[s] (+)= scale*(ss_rows[s] + sum_b ss_partials[s][b]) for s < upto; clears ss_rows[s] */
int ctr_epoch_reg_loss(double* ss_rows, const double* ss_partials, int n_partials, int upto, float scale,
                       float* reg, int accumulate, ctr_stream_t stream);
/* Diagnostics: the epoch sweeps evaluate sqrt/div through hand-scheduled IEEE fast paths with one range
 * check per four elements (optim_steps.cuh).  This compares them, bit for bit, with the compiler's
 * sqrt.rn / div.rn on n pseudo-random in-range operands (seeded; uniform mantissas, hard mantissa
 * patterns mixed in).  mismatches: device int64[2] = {sqrt mismatches, div mismatches} (overwritten). */
int ctr_selftest_divsqrt(uint64_t seed, int64_t n, int64_t* mismatches, ctr_stream_t stream);
/* The packed (FMUL2/FADD2/FFMA2) untouched-row Adam loops of the epoch sweep (csrc/adam_packed.cuh) against the
 * scalar step, bit for bit, on n random 8-element states of a regime (0: normal range; 1: tiny / denormal / zero
 * first moments; 2: also denormal / zero second moments), `steps` (1..4) steps each.
 * out3: device int64[3] = {elements whose (var, m, v) bits differ, trajectories the validity check rejected, total}. */
int ctr_selftest_adam_packed(int regime, uint64_t seed, int64_t n, int steps, float lr, float l2, int64_t* out3,
                             ctr_stream_t stream);

/* ---- loss head -----------------------------------------------------------------------------------
 * y = ((bias + y_a) + y_b) + y_c (NULL terms skipped; DeepFM.py:172-175), pred = sigmoid(y)
 * (:176), loss_ce = sum(max(y,0) - y*t + log1p(exp(-|y|)))/B_total (:188), dy = (pred - t)/B_total,
 * dbias = sum(dy).  B_total = B on one GPU; 1 = summed loss (canned estimators); the global batch under data parallelism (the per-rank
 * loss_ce / dbias / gradients then SUM to the global mean).  labels NULL => inference (y, pred only).
 */
int ctr_logit_loss(const float* bias, const float* y_a, const float* y_b, const float* y_c,
                   const float* labels, int B, int B_total, float* y, float* pred, float* loss_ce,
                   float* dy, float* dbias, ctr_stream_t stream);

/* ---- dense layers: wgmma 3xTF32 GEMMs with fused epilogues -----------------------------------------
 * tf.contrib.layers.fully_connected (DeepFM.py:156,165) + tf.nn.dropout (:162) and their autodiff.
 *   fwd: out[M,Nd] = dropout(act(in[M,Kd] @ Wt[Kd,Nd] + b)),  act 0 = identity, 1 = relu;
 *        drop_mask = binary keep mask [M,Nd] (NULL = no dropout): out = x / keep_prob * mask.
 *   bwd: dOut is overwritten with dZ = (dOut*mask/keep) * (out > 0);  db = colsum(dZ);
 *        dW = in^T @ dZ (split over M, deterministic);  dIn = dZ @ Wt^T (NULL to skip).
 * fc1: the N = 1 output layer over the concatenation [in_a | in_b] (in_b NULL/Kb = 0 for DeepFM's
 *      deep_out; DCN's out_layer takes [x_L, x_deep], DCN.py:178-181).
 * Accumulation order is fixed => bit-reproducible. */
int ctr_fc_fwd(const float* in, const float* Wt, const float* b, const float* drop_mask, float keep_prob,
               int M, int Kd, int Nd, int act, float* out, ctr_stream_t stream);
/* same, plus a per-row-group bias: out = act(in@Wt + b + group_bias[row / group_P]) -- DIN's attention
 * layer, where the ad-embedding part of [e, e-a, a] @ W is one row per sample (DIN.py:161-164) */
int ctr_fc_fwd_grouped(const float* in, const float* Wt, const float* b, const float* group_bias, int group_P,
                       const float* drop_mask, float keep_prob, int M, int Kd, int Nd, int act, float* out,
                       ctr_stream_t stream);
size_t ctr_fc_bwd_workspace_bytes(int M, int Kd, int Nd);
/* accumulate_din != 0: dIn += dZ @ Wt^T (instead of =) */
int ctr_fc_bwd(const float* in, const float* Wt, const float* out, const float* drop_mask, float keep_prob,
               float* dOut, int M, int Kd, int Nd, int act, float* dIn, int accumulate_din, float* dW, float* db,
               void* ws, size_t ws_bytes, ctr_stream_t stream);
int ctr_fc1_fwd(const float* in_a, int Ka, const float* in_b, int Kb, const float* w, const float* b, int M,
                float* y, ctr_stream_t stream);
size_t ctr_fc1_bwd_workspace_bytes(int M, int Ka, int Kb);
int ctr_fc1_bwd(const float* in_a, int Ka, const float* in_b, int Kb, const float* w, const float* dy, int M,
                float* d_a, float* d_b, float* dw, float* db, void* ws, size_t ws_bytes, ctr_stream_t stream);
/* binary keep mask: mask[i] = (hash(seed, *step_dev, i) < keep_prob) -- tf.nn.dropout's
 * floor(keep_prob + uniform); step_dev = device float holding the global step (NULL = 0) so that a
 * captured graph draws a fresh mask every replay.  Not TF's Philox stream. */
int ctr_dropout_mask(float* mask, int64_t n, float keep_prob, uint64_t seed, const float* step_dev,
                     ctr_stream_t stream);

/* ---- batch normalisation after the relu of a hidden layer ------------------------------------------
 * Replaces batch_norm_layer (DeepFM.py:159-160,231-235; DCN.py:171,241-247; PNN.py:181; NFM.py:143; DIN.py:206):
 * tf.contrib.layers.batch_norm(decay, center=True, scale=True, updates_collections=None), epsilon 0.001 [TF-sem],
 * followed by the layer's dropout (drop_mask NULL = none).  x, out: [n, H] row-major.
 * train != 0: batch moments (biased variance) -> save_mean / save_var [H]; moving_mean / moving_var are updated in
 * place (moving -= (moving - batch)*(1 - decay)).  train == 0: moving statistics, no dropout, nothing written but out.
 * ctr_bn_bwd: gradients through the batch moments; d_x [n,H], d_gamma / d_beta [H] (overwritten). */
size_t ctr_bn_workspace_bytes(int H);   /* scratch for the chunked column reductions (TRAIN forward and backward) */
int ctr_bn_fwd(const float* x, int n, int H, const float* gamma, const float* beta, float* moving_mean,
               float* moving_var, int train, float decay, float eps, const float* drop_mask, float keep_prob, float* out,
               float* save_mean, float* save_var, void* ws, size_t ws_bytes, ctr_stream_t stream);
int ctr_bn_bwd(const float* d_out, const float* x, int n, int H, const float* save_mean, const float* save_var,
               const float* gamma, float eps, const float* drop_mask, float keep_prob, float* d_x, float* d_gamma,
               float* d_beta, void* ws, size_t ws_bytes, ctr_stream_t stream);

/* ---- K5: DCN cross network (DCN.py:140-145) ------------------------------------------------------
 * x_{l+1} = x0 * (x_l . w_l) + x_l + b_l,  l = 0..L-1;  w,b: [L,D];  x0: [B,D], D = F*K (D%4==0, <=2048)
 * fwd saves the L scalars s[b,l] = x_l . w_l;  bwd recomputes x_l from x0 and s.
 * bwd: dx0 = dx_in (NULL = 0) + dL/dx0 through the cross network;  dw, db: [L,D] (deterministic).
 * Limits (CTR_ERR_UNSUPPORTED, checked before anything else, so a call with B = 0 and NULL buffers probes them):
 *   both: D % 4 == 0, D <= 2048, L <= 32;  fwd: L >= 0 (L = 0 copies x0);  bwd: L >= 1 and the per-warp slab
 *   2*L*D floats must fit 200 KB (8*L*D <= 204800 bytes: D = 2048 allows L <= 12).  B = 0 launches nothing. */
int ctr_cross_fwd(const float* x0, const float* w, const float* b, int B, int D, int L, float* xL, float* s,
                  ctr_stream_t stream);
size_t ctr_cross_bwd_workspace_bytes(int B, int D, int L);
int ctr_cross_bwd(const float* x0, const float* w, const float* b, const float* s, const float* dxL,
                  const float* dx_in, int B, int D, int L, float* dx0, float* dw, float* db, void* ws,
                  size_t ws_bytes, ctr_stream_t stream);

/* ---- DeepMVM multi-view product (DeepMVM.py:144-150) ----------------------------------------------
 * a = x + mvm_b (broadcast over the batch);  x_mvm[b,k] = (((a[b,0,k] * a[b,1,k]) * a[b,2,k]) * ... ) * a[b,F-1,k]
 * x: [B, F*K] (K1 CTR_FM_PLAIN output), mvm_b: [F,K], x_mvm: [B,K].  Every op is one IEEE-rounded fp32 op in field
 * order, with gradual underflow (bit-identical to a sequential fp32 restatement).  F <= 64, K <= 256.
 * bwd (TF autodiff of the chain, no division): with g = d_xmvm and P_i = a_0*...*a_i as the forward rounds it,
 * for i = F-1..1 { da_i = g*P_{i-1}; g = g*a_i }, da_0 = g;  d_e = da + dX (dX NULL = 0), d_e: [B, F*K];
 * d_mvm_b[f,k] = sum_b da[b,f,k] (overwritten; per-CTA partials in ws, fixed-order merge: deterministic). */
int ctr_mvm_fwd(const float* x, const float* mvm_b, int B, int F, int K, float* x_mvm, ctr_stream_t stream);
size_t ctr_mvm_bwd_workspace_bytes(int B, int F, int K);
int ctr_mvm_bwd(const float* x, const float* mvm_b, const float* d_xmvm, const float* dX, int B, int F, int K,
                float* d_e, float* d_mvm_b, void* ws, size_t ws_bytes, ctr_stream_t stream);

/* ---- ESMM shared embedding layer and multi-task head (DeepMTL/Model_pipeline/DeepCvrMTL.py) --------------------
 * embed_fwd (:153-164): x [B, (F'+8)K] = [common F'K | u_cat | u_shop | u_brand | u_int | a_cat | a_shop | a_brand |
 *     a_int] from feat_ids [B,F'], a_ids [3,B] (a_cat, a_shop, a_brand) and one CSR over 5B bags: bag j*B+b (j = u_cat,
 *     u_shop, u_brand, u_int, a_int) is occurrences [bag_off[j*B+b], bag_off[j*B+b+1]) of bag_ids / bag_wgt.
 *     bag sum = ((0 + e_0*w_0) + e_1*w_1) + ... in occurrence order, each * and + one IEEE-rounded op (no FMA); a_int is
 *     unweighted (its bag_wgt entries are not read).  Empty bag -> +0 row.  Ids outside [0,N) are counted into
 *     oob[0] (oob[1] = first) like ctr_gather_scale_rows and contribute zero rows.  K in {4,8,16,32,64,128,256}.
 * embed_bwd: g_rows [n_rows, K] in the order [common (row b*F'+f) | a_cat B | a_shop B | a_brand B | occurrences
 *     bag_off[5B] | zero rows up to n_rows]: the dx slice of each lookup, times w (one rounded multiply) for u_* bags.
 * head (:205-223), one CTA, fixed-order reductions (deterministic); labels y, z NULL => inference:
 *     pctr = sigmoid(y_ctr), pcvr = sigmoid(y_cvr), pctcvr = pctr*pcvr;
 *     losses[0] = sum_{i<n} CE(y_ctr_i, y_i) / n;  losses[1] = sum_{i<n} -(z*log(p+eps)) - ((1-z)*log((1-p)+eps)) / n,
 *     eps = 1e-7 (tf.losses.log_loss, SUM_BY_NONZERO_WEIGHTS);
 *     with g_ctr = w_ctr/n, g_cvr = w_cvr/n (w_ctr, w_cvr: the fp32 constants w and 1-w):
 *       dp = ((-g_cvr*z) * rcp(p+eps)) + -((-g_cvr*(1-z)) * rcp((1-p)+eps))
 *       d_cvr = ((dp*pctr)*pcvr)*(1-pcvr)
 *       d_ctr = (pctr - y)*g_ctr + ((dp*pcvr)*pctr)*(1-pctr)
 *     rows n..B-1 get d = +0. */
int ctr_esmm_embed_fwd(const int32_t* feat_ids, const int32_t* a_ids, const int32_t* bag_ids, const float* bag_wgt,
                       const int32_t* bag_off, const float* V, int64_t N, int B, int Fp, int K, float* x, int32_t* oob,
                       ctr_stream_t stream);
int ctr_esmm_embed_bwd(const float* dx, const float* bag_wgt, const int32_t* bag_off, int B, int Fp, int K,
                       int64_t n_rows, float* g_rows, ctr_stream_t stream);
int ctr_esmm_head(const float* y_ctr, const float* y_cvr, const float* y, const float* z, int B, int n, float w_ctr,
                  float w_cvr, float* pctr, float* pcvr, float* pctcvr, float* losses, float* d_ctr, float* d_cvr,
                  ctr_stream_t stream);

/* ---- K6/K9: DIN embedding + field-wise pooling layers (DIN.py:143-183) ---------------------------
 * gather_scale_rows: out[(i/G)*ld_group + (i%G)*K + k] = V[ids[i]][k] * (wgt ? wgt[i] : 1)
 *     (tf.nn.embedding_lookup of feat_ids / a_catids / padded behaviour ids, DIN.py:143-147,155-156;
 *      G, ld_group let the rows land directly inside the concatenated MLP input, DIN.py:199)
 * bag_sum: tf.nn.embedding_lookup_sparse(combiner="sum") over CSR bags (a_intids, DIN.py:148; the
 *     non-attention pooling branch :180-183) and its gradient g_rows[i] = d_out[bag(i)] * w_i.
 *     An id outside [0,N) adds nothing; bag_sum_fwd_oob also counts it into oob[0] (oob[1] = first) like
 *     ctr_gather_scale_rows (TF raises InvalidArgumentError); oob may be NULL.
 * din_pool: att = sigmoid(z); u[b] = sum_p (ids[b,p] > 0) * att[b,p] * E[b,p,:]   (DIN.py:169-172)
 *     bwd: dE = mask*att*du (written, not accumulated); dz = mask*att*(1-att)*(E . du)
 * scale_rows: out[i,:] = (x[(i/G)*ld_group + (i%G)*K : +K] + add[i,:]) * w[i]  (add, w optional)
 * axpby: out = alpha*a + beta*b */
int ctr_gather_scale_rows(const int32_t* ids, const float* wgt, const float* V, int64_t N, int64_t n, int K,
                          int G, int64_t ld_group, float* out, int32_t* oob, ctr_stream_t stream);
int ctr_bag_sum_fwd_oob(const int32_t* ids, const float* wgt, const int32_t* offsets, const float* V, int64_t N,
                        int B, int K, int64_t ld, float* out, int32_t* oob, ctr_stream_t stream);
int ctr_bag_sum_bwd(const float* d_out, int64_t ld, const float* wgt, const int32_t* offsets, int B, int K,
                    float* g_rows, ctr_stream_t stream);
int ctr_scale_rows(const float* x, const float* add, const float* w, int64_t n, int K, int G, int64_t ld_group,
                   float* out, ctr_stream_t stream);
int ctr_din_pool_fwd(const float* E, const float* z, const int32_t* ids, int B, int P, int K, float* att, float* u,
                     int64_t ld_u, ctr_stream_t stream);
int ctr_din_pool_bwd(const float* E, const float* att, const int32_t* ids, const float* du, int64_t ld_u, int B,
                     int P, int K, float* dE, float* dz, ctr_stream_t stream);
/* Attention unit backward through the N=1 output and the hidden layer's relu/dropout in ONE pass over the [B*P, H] hidden
 * activations Hh (autodiff of DIN.py:164-169): dZ[r][c] = dz[r]*w2[c] (*mask/keep) where Hh > 0; dU[b][c] = sum_p dZ
 * (the group-bias gradient; colsum(dU) is the layer's bias gradient); gw2_part[b][c] = sum_p dz*Hh (colsum = the output
 * layer's weight gradient).  Then ctr_fc_bwd(act = 2) takes dZ as is. */
int ctr_din_att_dz(const float* Hh, const float* drop_mask, float keep_prob, const float* dz, const float* w2, int B, int P,
                   int H, float* dZ, float* dU, float* gw2_part, ctr_stream_t stream);
/* out[k] = sum_r part[r*ld + k], k < ncols: deterministic column sums of many rows (fixed order) */
int ctr_colsum_rows(const float* part, int rows, int ld, int ncols, float* out, ctr_stream_t stream);
int ctr_axpby(const float* a, float alpha, const float* b, float beta, int64_t n, float* out, ctr_stream_t stream);

/* ---- K7/K8: all-pairs interactions (pair order i < j row-major; P = F(F-1)/2) -----------------------
 * pnn_product: z[b] = [x[b] (F*K) | inner (P)]            (outer = 0; PNN.py:148-153)
 *              z[b] = [x[b] (F*K) | outer (P*K*K)]        (outer = 1; PNN.py:164-167, "NOT ready yet")
 *   bwd: dX = dz[:, :F*K] + product-rule terms of the tail.
 * afm_pairs:  pw[b,p,:] = e_i * e_j (AFM.py:132-138);  bwd: dX[b,f,:] = sum_o dpw[b,pair(f,o),:] * e_o
 * afm_pool:   att = softmax_p(logit) (AFM.py:151), w = dropout(att) (:152-153), y_emb = sum_p w_p pw_p (:156);
 *   bwd: dpw = w * dy_emb (written), dlogit = softmax backward.
 * dropout_apply: out = x / keep * mask  (NFM's dropout on the bi-interaction vector, NFM.py:136-137;
 *   AFM's on y_emb, AFM.py:157-158)
 * Limits (CTR_ERR_UNSUPPORTED, checked before anything else, so a call with B = 0 and NULL buffers probes them):
 *   pnn_product_fwd: 16*F*(K+1) <= 204800 bytes of shared memory (F = 39: K <= 327);
 *   pnn_product_bwd: 32*F*(K+1) <= 204800 (F = 39: K <= 163);  afm_pool_*: P <= 10240 (F <= 143). */
int ctr_pnn_product_fwd(const float* x, int B, int F, int K, int outer, float* z, ctr_stream_t stream);
int ctr_pnn_product_bwd(const float* x, const float* dz, int B, int F, int K, int outer, float* dX,
                        ctr_stream_t stream);
int ctr_afm_pairs_fwd(const float* x, int B, int F, int K, float* pw, ctr_stream_t stream);
int ctr_afm_pairs_bwd(const float* x, const float* dpw, int B, int F, int K, float* dX, ctr_stream_t stream);
int ctr_afm_pool_fwd(const float* pw, const float* logit, const float* mask, float keep, int B, int P, int K,
                     float* att, float* y_emb, ctr_stream_t stream);
int ctr_afm_pool_bwd(const float* pw, const float* att, const float* mask, float keep, const float* dy_emb, int B,
                     int P, int K, float* dpw, float* dlogit, ctr_stream_t stream);
int ctr_dropout_apply(const float* x, const float* mask, float keep, int64_t n, float* out, ctr_stream_t stream);

/* ---- row-sharded table routing (not in the reference; SURVEY.md 8e) ---------------------------------
 * owner(id) = id % G, local row = id / G.  gather_scalar: out[i] = W[ids[i]].
 * Routing keys (tf_repos_b200/sharded.py): key(id) = (id % G) * ceil(N/G) + id / G, so that ONE
 * ctr_unique_segment of the keys yields the unique ids in bucket order (owner-major, ascending id inside an owner),
 * `inverse` = the occurrence's position in the received row cache, and perm / seg_offsets = the gradient segments in
 * cache order.  ids outside [0, N) are counted in oob (may be NULL) and routed to row 0.
 * shard_split: counts[o] = unique ids owned by rank o, local_ids[u] = local row of the u-th unique key. */
int ctr_shard_keys(const int32_t* ids, int64_t n, int64_t N, int G, int32_t* keys, int32_t* oob, ctr_stream_t stream);
int ctr_shard_split(const int32_t* uniq_keys, const int32_t* n_uniq, int64_t n_max, int64_t N, int G, int32_t* counts,
                    int32_t* local_ids, ctr_stream_t stream);
int ctr_gather_scalar(const int32_t* ids, const float* W, int64_t N, int64_t n, float* out, ctr_stream_t stream);

/* ---- wide_n_deep feature columns (wide_n_deep.py:92-107; SURVEY.md 8f-2) ------------------------------------
 * categorical_column_with_identity(num_buckets=NB, default_value=0) + embedding_column(K) per categorical
 * column, numeric columns appended in the name-sorted order (num_perm), and the linear_model over the same
 * columns.  The Fc per-column tables are stacked: column f owns rows [f*NB, (f+1)*NB) of emb [Fc*NB, K] and
 * wide_cat [Fc*NB]; flat_ids[b,f] = f*NB + (0 <= id < NB ? id : 0).
 *   x   [B, Fc*K + Fd] = [emb rows of columns 0..Fc-1 | dense[b, num_perm[0..Fd-1]]]      (emb != NULL)
 *   lin [B] = sum_f wide_cat[flat_ids[b,f]] + sum_j dense[b,j]*wide_num[j] + wide_bias     (wide_* != NULL)
 * bwd: g_rows[b*Fc+f,:] = dX[b, f*K:(f+1)*K], g_cat[b*Fc+f] = dy[b], g_num[j] = sum_b dy[b]*dense[b,j],
 *      g_bias = sum_b dy[b]  (fixed reduction trees: deterministic).  NULL outputs are skipped. */
int ctr_wd_input_fwd(const int32_t* ids, const float* dense, const float* emb, const float* wide_cat,
                     const float* wide_num, const float* wide_bias, const int32_t* num_perm, int B, int Fc, int Fd,
                     int NB, int K, int32_t* flat_ids, float* x, float* lin, ctr_stream_t stream);
int ctr_wd_input_bwd(const float* dX, const float* dy, const float* dense, int B, int Fc, int Fd, int K, float* g_rows,
                     float* g_cat, float* g_num, float* g_bias, ctr_stream_t stream);

/* ---- wide_n_deep serving input (wide_n_deep.py:233-242, wide_n_deep_serving_client.cpp:45-62; DESIGN.md §2.8) -----
 * The export's serving_default parses the request's `inputs` tensor -- n serialized tf.Examples -- with
 * make_parse_example_spec(columns): I1..I13 FixedLenFeature([1], float32) without default, C14..C39
 * VarLenFeature(int64), other keys ignored, the last map entry of a key wins.  Example b is data[offsets[b],
 * offsets[b+1]) (device bytes, offsets int64 [n+1], each Example < 2^31 bytes).  One warp per Example parses it
 * (packed and unpacked lists) and writes what ctr_wd_input_fwd writes with Fc = 26, Fd = 13:
 *   x   [n, 26*K + 13] = [mean of the bag's emb rows per column C14..C39 (zero row for an empty or missing bag) |
 *                         I values in num_perm order]                                            (emb != NULL)
 *   lin [n] = sum of the bags' wide_cat weights + sum_j I(j+1)*wide_num[j] + wide_bias           (wide_* != NULL)
 * An int64 value outside [0, NB) (all 64 bits) becomes 0.  With one value per C key, x and lin are bit-identical to
 * ctr_wd_input_fwd.  err (device uint64, set to ~0 by the caller) is min-folded with (example_base + b) << 16 |
 * check << 8 | key; check 1 = malformed protobuf (key 0), 2 = I key missing, 3 = several kinds in one Feature or a
 * wrong kind (not FloatList under I, not Int64List under C), 4 = I key without exactly one value; key 0..12 = I1..I13,
 * 13..38 = C14..C39.  The rows of a rejected Example are not written. */
int ctr_wd_serve_input(const void* data, const int64_t* offsets, int64_t n, int64_t example_base, const float* emb,
                       const float* wide_cat, const float* wide_num, const float* wide_bias, const int32_t* num_perm,
                       int NB, int K, float* x, float* lin, uint64_t* err, ctr_stream_t stream);

/* ---- libsvm input (HOST buffers) -------------------------------------------------------------------
 * decode_libsvm of input_fn (DeepFM.py:65-81): "<label> <id>:<val> ..." lines -> ids int32 [rows,F],
 * vals f32 [rows,F], labels f32 [rows].  Parses complete lines of buf_host[0,len) up to max_rows;
 * returns rows parsed (or <0), *consumed_host = bytes consumed.  All pointers are HOST pointers. */
int64_t ctr_parse_libsvm(const char* buf_host, size_t len, int F, int64_t max_rows, int final_chunk,
                         int32_t* ids_host, float* vals_host, float* labels_host, size_t* consumed_host);
int ctr_libsvm_count_fields(const char* buf_host, size_t len);

/* ---- libsvm input (DEVICE buffers; SURVEY.md 8f-1) -----------------------------------------------------
 * The same decode_libsvm (DeepFM.py:65-81) for text that is already in device memory: the first max_rows
 * complete lines of text[0,len) (plus an unterminated last line when final_chunk != 0) are tokenised by one
 * thread each.  Every value this path emits has exactly the bits ctr_parse_libsvm (strtof/strtol) gives;
 * whatever it cannot guarantee is only COUNTED and the caller re-parses the chunk with the host entry point:
 *   info (device int64[5]) = { rows, bytes consumed, blank lines, malformed lines (bad token / pair count != F),
 *                             lines holding a number for the host (inf/nan/hex, > 15 digits, |exp10| > 22,
 *                             fp32 subnormal/overflow, or within one double-ulp of an fp32 rounding boundary) }
 * ids/vals/labels rows are valid iff info[2] == info[3] == info[4] == 0.  len < 2^32. */
size_t ctr_parse_libsvm_device_workspace_bytes(size_t len, int64_t max_rows);
int ctr_parse_libsvm_device(const char* text, size_t len, int F, int64_t max_rows, int final_chunk, int32_t* ids,
                            float* vals, float* labels, int64_t* info, void* ws, size_t ws_bytes, ctr_stream_t stream);

/* ---- wide_n_deep CSV input (DEVICE buffers; DESIGN.md §2.9) ------------------------------------------------
 * The tf.decode_csv of input_fn (wide_n_deep.py:55-73; record_defaults [[0.0]] + 13*[[0.0]] + 26*[[0]]) for text that
 * is already in device memory: the first max_rows complete lines of text[0,len) (plus an unterminated last line when
 * final_chunk != 0) are split on ',' by one thread each into n_float float columns then n_int int columns; an empty
 * field takes its default (0.0 / 0).  Column 0 = label, then n_float-1 dense, then n_int:
 *   labels f32 [rows], dense f32 [rows, n_float-1], cat int32 [rows, n_int], row-major; ids are not clamped.
 * Every value this path emits has exactly the bits wide_deep_main.decode_csv_file (Python float() / int(), NumPy cast)
 * gives; whatever it cannot guarantee is only COUNTED and the caller re-parses the piece with the host decoder:
 *   info (device int64[5]) = { rows, bytes consumed, blank lines, malformed lines (field count != n_float + n_int, or
 *                             a '"', blank or tab in the line), lines holding a number for the host (a float outside
 *                             the fast decimal path of ctr_parse_libsvm_device or not ending at its field's end; an
 *                             int that is not [+-]?[0-9]{1,9}) }
 * labels/dense/cat rows are valid iff info[2] == info[3] == info[4] == 0.  len < 2^32.  No allocation and no
 * synchronisation inside. */
size_t ctr_parse_csv_device_workspace_bytes(size_t len, int64_t max_rows);
int ctr_parse_csv_device(const char* text, size_t len, int n_float, int n_int, int64_t max_rows, int final_chunk,
                         float* labels, float* dense, int32_t* cat, int64_t* info, void* ws, size_t ws_bytes,
                         ctr_stream_t stream);

/* ---- Criteo feature pipeline (deep_ctr/Feature_pipeline/get_criteo_feature.py; DESIGN.md §2.4) ----------------
 * Raw Criteo TSV -> tr/va/te.libsvm + feature_map, byte for byte.  `text` is a chunk of whole lines (a last line
 * without '\n' counts), len < 2^30; line_base = index of its first line in the file (error positions are file lines).
 * Error word (device int64, ~0 = none; the smallest over the file is the one the reference raises first):
 *   (class << 62) | (line << 16) | (column << 8) | code; class 0 = min/max pass, 1 = dictionary pass; column =
 *   index into the line's '\t' split; code 1 = too few columns (IndexError), 2 = I value not [+-]?[0-9]+ (ValueError /
 *   restriction), 3 = |I value| > 2^53, 4 = C value > 8 bytes, 5 = C value holds NUL, 6 = C value is "<unk>"
 *   (restrictions), 7 = max == min and a non-empty I value (ZeroDivisionError).
 * table: ctr_criteo_table_bytes(capacity) bytes, zeroed by the caller; open addressing on (field, value), capacity
 *   slots (<= 2^31).
 * stats (:74-85 min/max, :39-45 counts; train lines): minmax int64[26] = {min[13], max[13]}, initialised by the caller
 *   to {sys.maxsize..., -sys.maxsize...} and folded into; info int64[3] = {lines, error word, values dropped because
 *   no slot was found within min(capacity, 32768) probes -- non-zero means capacity is too small}.
 * vocab (:46-51): count >= cutoff kept, sorted by (field, -count, value), ids 1..n per field written into the table
 *   (all other values -> 0 = <unk>).  vocab_keys uint64[capacity]: the kept values field-major in id order, packed
 *   big-endian and zero-padded; field_counts int64[26].  Run once, after the last stats call.
 * emit (:127-167): plan then write, over the same text and ws.  test = 0: train lines, to_train uint8[lines] = the
 *   split decision of each line (:148), column 0 is the label; test = 1: columns shifted by one, every line gets
 *   label[0, label_len) (the last train line's label, :167).  num_min / num_den double[13] = float(min), float(max -
 *   min); offsets int64[26] (:119-123).  plan: info int64[5] = {lines, error word, tr lines, tr bytes, va bytes};
 *   write (only after a plan without error): lines to out_tr (or out_va when to_train is 0), each in input order. */
size_t ctr_criteo_table_bytes(int64_t capacity);
size_t ctr_criteo_stats_workspace_bytes(size_t len);
int ctr_criteo_stats(const char* text, size_t len, int64_t line_base, void* table, int64_t capacity, int64_t* minmax,
                     int64_t* info, void* ws, size_t ws_bytes, ctr_stream_t stream);
size_t ctr_criteo_vocab_workspace_bytes(int64_t capacity);
int ctr_criteo_vocab(void* table, int64_t capacity, int64_t cutoff, uint64_t* vocab_keys, int64_t* field_counts,
                     void* ws, size_t ws_bytes, ctr_stream_t stream);
size_t ctr_criteo_emit_workspace_bytes(size_t len);
int ctr_criteo_emit_plan(const char* text, size_t len, int test, int64_t line_base, const uint8_t* to_train,
                         const void* table, int64_t capacity, const double* num_min, const double* num_den,
                         const int64_t* offsets, const char* label, int label_len, int64_t* info, void* ws,
                         size_t ws_bytes, ctr_stream_t stream);
int ctr_criteo_emit_write(const char* text, size_t len, int test, const uint8_t* to_train, const void* table,
                          int64_t capacity, const double* num_min, const double* num_den, const int64_t* offsets,
                          const char* label, int label_len, char* out_tr, char* out_va, const void* ws,
                          size_t ws_bytes, ctr_stream_t stream);

/* ---- TFRecord input of DIN / ESMM (DIN.py:57-99, DeepCvrMTL.py:63-105; DESIGN.md §2.5) ------------------------
 * frame (HOST buffers): walks the records of buf_host[0, len) -- uint64 length | uint32 masked CRC-32C of the length |
 *   data | uint32 masked CRC-32C of the data -- checking every header CRC, up to max_records.  rec_off[i] = byte offset
 *   of record i's header.  info (host int64[5]) = { records, bytes consumed (whole records only), error class, error
 *   offset, bytes the next record needs }; class 0 = none, 1 = truncated header, 2 = header CRC mismatch, 3 = truncated
 *   record, 4 = record longer than 2^31 - 17 bytes.  A tail too short for the next record is an error only when
 *   final_chunk != 0 (otherwise it is left unconsumed).
 * scan (device): one warp per framed record of chunk (records from ctr_tfrecord_frame over the same bytes): the data
 *   CRC, the protobuf walk and decode_tfrecord_files' checks.  labels_mask: bit 0 = y required (always), bit 1 = z
 *   (ESMM).  lens int32 [n_rec][5] = value counts of u_catids, u_shopids, u_brandids, u_intids, a_intids.  err (device
 *   uint64, set to ~0 by the caller once) is min-folded with (record_base + i) << 16 | check << 8 | arg; check 0 = data
 *   CRC, 1 = malformed protobuf, 2 = required key missing or empty (arg = key: 0 y, 1 z, 2 feat_ids, 3 a_catids,
 *   4 a_shopids, 5 a_brandids), 3 = feat_ids count != F, 4 = u_*ids / u_*vals lengths differ (arg = 0 cat, 1 shop,
 *   2 brand, 3 int), 5 = wrong or several Feature kinds, 6 = id outside [0, 2^31) (arg = schema key: 0 y, 1 z,
 *   2 feat_ids, 3-5 a_cat/shop/brandids, 6 a_intids, 7-10 u_cat/shop/brand/intids, 11-14 u_cat/shop/brand/intvals).
 * emit (device): one batch of B slots; slot b's record data is stage[slot_off[b], + slot_len[b]) and must have passed
 *   the scan.  Writes din_main.make_batch's tensors (feat_ids [B,F], a_ids [3,B], a_int_ids, u_ids [4,B,P] and u_wgt
 *   [4,B,P] zero-padded, y [B]) at the caller's a_int_off [B+1], or esmm_main.make_batch's (feat_ids, a_ids, bag_ids,
 *   bag_wgt, y, z) at the caller's bag_off [5B+1]. */
enum { CTR_TFR_OK = 0, CTR_TFR_TRUNCATED_HEADER = 1, CTR_TFR_CORRUPTED_LENGTH = 2, CTR_TFR_TRUNCATED_RECORD = 3,
       CTR_TFR_TOO_LARGE = 4 };
int ctr_tfrecord_frame(const void* buf_host, size_t len, int final_chunk, int64_t* rec_off, int64_t max_records,
                       int64_t* info);
int ctr_tfrecord_scan(const void* chunk, size_t len, const int64_t* rec_off, int64_t n_rec, int64_t record_base, int F,
                      int labels_mask, int32_t* lens, uint64_t* err, ctr_stream_t stream);
int ctr_tfrecord_emit_din(const void* stage, const int64_t* slot_off, const int32_t* slot_len, int B, int F, int P,
                          const int32_t* a_int_off, int32_t* feat_ids, int32_t* a_ids, int32_t* a_int_ids,
                          int32_t* u_ids, float* u_wgt, float* y, ctr_stream_t stream);
int ctr_tfrecord_emit_esmm(const void* stage, const int64_t* slot_off, const int32_t* slot_len, int B, int F,
                           const int32_t* bag_off, int32_t* feat_ids, int32_t* a_ids, int32_t* bag_ids, float* bag_wgt,
                           float* y, float* z, ctr_stream_t stream);

/* ---- DIN serving input (DIN.py:60-77 without labels, DIN.py:385-397; DESIGN.md §2.10) ----------------------------
 * One slice of a serving request: n serialized tf.Examples, Example b = data[offsets[b], offsets[b+1]) (device bytes,
 * offsets int64 [n+1], each Example < 2^31 bytes), 1 <= n <= B.  One warp per batch slot b < B walks its Example (slot
 * b >= n repeats Example 0, as din_main.make_batch pads) with the scan's walk and checks, minus the CRC and the labels:
 * y and z must be well formed but are neither required nor kind-checked.  Writes
 *   slot_off int64 [B], slot_len int32 [B]   the slot's bytes, for ctr_tfrecord_emit_din(data, slot_off, slot_len, ...)
 *   a_int_off int32 [B+1]                    exclusive scan (one CTA, on the device) of the a_intids bag lengths, each
 *                                            clamped to max_a_int, so the emit writes at most B * max_a_int ids
 *   maxima int32 [2]                         atomicMax-folded (set to 0 by the caller): the longest u_*ids list and the
 *                                            longest a_intids bag of the n Examples, unclamped; a longer value than the
 *                                            emit's P / max_a_int means the slice must be run again with larger buffers
 *   err                                      min-folded as ctr_tfrecord_scan's with (example_base + b) << 16, b < n;
 *                                            checks 1-6 (no CRC), arg as there (check 2: keys 2-5 only)
 * A rejected Example's lengths are 0.  No allocation and no synchronisation inside. */
int ctr_din_serve_scan(const void* data, const int64_t* offsets, int64_t n, int64_t example_base, int F, int B,
                       int max_a_int, int64_t* slot_off, int32_t* slot_len, int32_t* a_int_off, int32_t* maxima,
                       uint64_t* err, ctr_stream_t stream);

/* ---- Ali-CCP TFRecord writer (deep_ctr/Feature_pipeline/get_aliccp_tfrecord.py; DESIGN.md §2.6) ----------------
 * Joined Ali-CCP lines `id,y,z,field:fid:val ...` -> framed tf.Example records, byte-identical to
 * tfrecord.write_records(path, [tfrecord.encode_example(features) ...]) of the features gen_tfrecords builds.  `text` is
 * a chunk of whole lines (a last line without '\n' counts), len <= 2^31; line_base = index of its first line in the
 * file.  plan, declines and write share one workspace of ctr_aliccp_workspace_bytes(len) bytes and run over the same
 * text, in that order.
 * plan (replaces :42-94, the per-line parse): info int64[4] = {lines, error word, output bytes, declined numbers}.
 *   Error word (~0 = none) = the smallest (line_base + line) << 8 | code; code 1 = NUL byte in the line, 2 = token
 *   count not a multiple of 3 (the reference's reshape raises), 3 = empty token, 4 = kept field's fid not [0-9]+ below
 *   2^63 (restrictions; a non-integer fid also raises in the reference).
 * declines (only when info[3] > 0): spans int64[info[3]][3] = (line in the chunk, start, end) of every y, z and user
 *   multi-hot value the device does not convert (anything but plain decimal with mantissa <= 2^53 and |exponent| <=
 *   22), in line order.
 * write (replaces :48-98, the Example and the TFRecordWriter; only after a plan without error): decl_vals float[info[3]]
 *   = float32(float(token)) of every declined span (null when there are none); out[info[2]] = the records of the
 *   chunk's 4-field lines, in line order. */
size_t ctr_aliccp_workspace_bytes(size_t len);
int ctr_aliccp_plan(const char* text, size_t len, int64_t line_base, int64_t* info, void* ws, size_t ws_bytes,
                    ctr_stream_t stream);
int ctr_aliccp_declines(const char* text, size_t len, const void* ws, size_t ws_bytes, int64_t* spans,
                        ctr_stream_t stream);
int ctr_aliccp_write(const char* text, size_t len, const float* decl_vals, void* out, const void* ws, size_t ws_bytes,
                     ctr_stream_t stream);

/* ---- Ali-CCP sample stage (DeepMTL/Feature_pipeline/get_join_*.py, get_stat_*.py, get_remap_mapper.py; DESIGN.md
 * §2.7) --------------------------------------------------------------------------------------------------------------
 * Raw Tianchi lines -> `r_i\tsample_id,y,z,field:id:val ...` part files and feat_cnts.  Tables: the count table
 * (ctr_aliccp_sample_count_table_bytes(cap), zeroed) keys (field, fid) of the train set; the md5 table
 * (ctr_aliccp_sample_md5_table_bytes(cap): its first 72 * cap bytes zeroed, the last 8 * cap set to 0xFF) keys the md5s
 * of one set.  Chunks are whole lines (a last line without '\n' counts), len < 2^30, n_lines = the chunk's line count.
 * classify (replaces get_join_mapper.py:15-40 and, mode 2, get_stat_mapper.py:16-19 over each sample's own tokens;
 *   mode 0 = classify only, 1 = insert md5s, 2 = also count): info int64[9] = {lines, first restricted line in the chunk
 *   (~0 = none), y=0/z=1 samples, skipped lines, count-table overflows, md5-table overflows, common records, their
 *   feat_list bytes, kept samples}.  The workspace (ctr_aliccp_sample_chunk_workspace_bytes) then feeds place.
 * place (get_join_reducer.py:18-22): common records' feat_lists -> arena[arena_base ...], rec_off / rec_len / rec_slot
 *   from rec_base on, each md5's record = its last one; samples -> s_rec (md5 slot), s_key (part << 31 | r_i).
 * resolve (get_join_reducer.py:26-33): s_rec := the slot's record (-1: none); mult[r] = samples joined to record r;
 *   info int64[2] = {samples without a record, superseded records}.
 * count_commons (get_stat_mapper.py:17-19 over the joined common tokens): each token of record r adds mult[r];
 *   info[0] = count-table overflows.
 * vocab (get_stat_reducer.py, get_remap_mapper.py:10-21 under DESIGN.md §2.7's rule): vocab uint64[cap] = the fids
 *   with a (field, fid) count >= cutoff, ascending (id = 20 + index); info int64[5] = {entries, kept (field, fid),
 *   kept fids, -, feat_cnts bytes}.  feat_cnts (after vocab, same workspace): the feat_cnts text.
 * render: out == null: r_off int64[n + 1] = exclusive scan of each record's remapped text length (0 unless mult > 0);
 *   else the texts at r_off.
 * emit (get_remap_mapper.py:28-40): out == null: s_val[k] = the output line size of sample k, info[0] = lines with an
 *   empty feature field; else every sample with lo <= s_val[k] < hi (s_val = offsets from order) written at
 *   out + s_val[k] - lo.
 * order: s_key sorted stably (so ties keep line order), s_val sizes -> offsets in (part, r_i, line) order,
 *   part_bytes int64[parts]. */
size_t ctr_aliccp_sample_count_table_bytes(int64_t capacity);
size_t ctr_aliccp_sample_md5_table_bytes(int64_t capacity);
size_t ctr_aliccp_sample_chunk_workspace_bytes(size_t len, int64_t n_lines);
int ctr_aliccp_sample_classify(const char* text, size_t len, int64_t n_lines, int mode, void* count_table,
                               int64_t count_capacity, void* md5_table, int64_t md5_capacity, int64_t* info,
                               void* ws, size_t ws_bytes, ctr_stream_t stream);
int ctr_aliccp_sample_place(const char* text, size_t len, int64_t n_lines, int64_t line_base, uint64_t seed,
                            int64_t parts, void* md5_table, int64_t md5_capacity, uint8_t* arena, int64_t arena_base,
                            int64_t* rec_off, int32_t* rec_len, int32_t* rec_slot, int64_t rec_base, int32_t* s_rec,
                            uint64_t* s_key, int64_t sample_base, const void* ws, size_t ws_bytes,
                            ctr_stream_t stream);
int ctr_aliccp_sample_resolve(const void* md5_table, int64_t md5_capacity, int32_t* s_rec, int64_t n_samples,
                              const int32_t* rec_slot, int64_t n_records, uint32_t* mult, int64_t* info,
                              ctr_stream_t stream);
int ctr_aliccp_sample_count_commons(const uint8_t* arena, const int64_t* rec_off, const int32_t* rec_len,
                                    const uint32_t* mult, int64_t n_records, void* count_table, int64_t count_capacity,
                                    int64_t* info, ctr_stream_t stream);
size_t ctr_aliccp_sample_vocab_workspace_bytes(int64_t count_capacity);
int ctr_aliccp_sample_vocab(const void* count_table, int64_t count_capacity, int64_t cutoff, uint64_t* vocab,
                            int64_t* info, void* ws, size_t ws_bytes, ctr_stream_t stream);
int ctr_aliccp_sample_feat_cnts(char* out, const void* ws, size_t ws_bytes, int64_t count_capacity,
                                ctr_stream_t stream);
int ctr_aliccp_sample_render(const uint8_t* arena, const int64_t* rec_off, const int32_t* rec_len,
                             const uint32_t* mult, int64_t n_records, const uint64_t* vocab, int64_t n_vocab,
                             int64_t* r_off, char* out, ctr_stream_t stream);
int ctr_aliccp_sample_emit(const char* text, size_t len, int64_t n_lines, int64_t line_base, uint64_t seed,
                           const int32_t* s_rec, int64_t sample_base, const int64_t* r_off, const char* rendered,
                           const uint64_t* vocab, int64_t n_vocab, int64_t* s_val, int64_t lo, int64_t hi, char* out,
                           int64_t* info, void* ws, size_t ws_bytes, ctr_stream_t stream);
size_t ctr_aliccp_sample_order_workspace_bytes(int64_t n_samples);
int ctr_aliccp_sample_order(uint64_t* s_key, int64_t* s_val, int64_t n_samples, int64_t parts, int64_t* part_bytes,
                            void* ws, size_t ws_bytes, ctr_stream_t stream);

/* ---- smart and Frappe feature stages (deep_ctr/Feature_pipeline/get_smart_feature.py, get_frape_feature.py; DESIGN.md
 * §2.12) --------------------------------------------------------------------------------------------------------------
 * `text` is a chunk of whole lines (a last line without '\n' counts), len < 2^30.  Lines end at '\n' only and are
 * strip()ped with Python 2's whitespace (' ', \t, \n, \r, \x0b, \x0c).
 * map (replaces :56-63, the feature_map load): map_text[0, map_len) = the whole feature_map file, resident while the
 *   table is used; table = ctr_smart_map_table_bytes(capacity) bytes, zeroed by the caller, capacity slots (<= 2^31).
 *   Each line with two or more ' ' tokens maps s[0] -> s[1]; a key some lookup can reach (categorical `name|value` or a
 *   continuous `name`) is inserted, the later line of a repeated key wins.  col_fid int64[2 * 128] = per column the
 *   (offset, length) in map_text of the fid of its bare name (continuous columns) or of name|UNK (categorical), length
 *   -1 = absent.  info int64[3] = {map lines, keys inserted, keys that found no slot within min(capacity, 32768) probes
 *   -- non-zero means capacity is too small}.
 * emit (:68-89): plan then write, over the same text and ws.  plan: info int64[3] = {lines, emitted lines, output
 *   bytes}; a line of 130 or more fields is dropped.  write: the emitted lines to out[0, info[2]), in input order; a
 *   fid absent from the map prints as None.
 * build (get_feature_map, :27-53, with CSV_COLUMNS[i] at :32 read as fname): table = ctr_smart_build_table_bytes(
 *   capacity) bytes and state int64[19], both zeroed by the caller; arena = arena_bytes bytes that hold each distinct
 *   categorical value once, plus one byte.  insert, once per chunk of the `tr` files in order (line_base = lines before
 *   the chunk over all of them): info int64[2] = {lines, keys that found no slot}; state[1] = keys the arena could not
 *   hold.  Either non-zero leaves the table unusable.  finish: the keys in order of their first (line, column), info
 *   int64[2] = {keys, map bytes}; render (after finish, same ws): out[0, info[1]) = `key fid\n` for fids 129, 130, ...
 * frappe (get_frape_feature.py:16-29): plan: info int64[3] = {lines, kept lines, output bytes}; write: the kept lines,
 *   label -1 rewritten to 0, to out[0, info[2]).
 * No allocation and no synchronisation inside. */
size_t ctr_smart_map_table_bytes(int64_t capacity);
size_t ctr_smart_map_workspace_bytes(size_t map_len);
int ctr_smart_map_build(const char* map_text, size_t map_len, void* table, int64_t capacity, int64_t* col_fid,
                        int64_t* info, void* ws, size_t ws_bytes, ctr_stream_t stream);
size_t ctr_smart_emit_workspace_bytes(size_t len);
int ctr_smart_emit_plan(const char* text, size_t len, const char* map_text, const void* table, int64_t capacity,
                        const int64_t* col_fid, int64_t* info, void* ws, size_t ws_bytes, ctr_stream_t stream);
int ctr_smart_emit_write(const char* text, size_t len, const char* map_text, const void* table, int64_t capacity,
                         const int64_t* col_fid, char* out, const void* ws, size_t ws_bytes, ctr_stream_t stream);
size_t ctr_smart_build_table_bytes(int64_t capacity);
size_t ctr_smart_build_insert_workspace_bytes(size_t len);
int ctr_smart_build_insert(const char* text, size_t len, int64_t line_base, void* table, int64_t capacity,
                           uint8_t* arena, int64_t arena_bytes, int64_t* state, int64_t* info, void* ws,
                           size_t ws_bytes, ctr_stream_t stream);
size_t ctr_smart_build_workspace_bytes(int64_t capacity);
int ctr_smart_build_finish(const void* table, int64_t capacity, const uint8_t* arena, const int64_t* state,
                           int64_t* info, void* ws, size_t ws_bytes, ctr_stream_t stream);
int ctr_smart_build_render(const void* table, int64_t capacity, const uint8_t* arena, char* out, const void* ws,
                           size_t ws_bytes, ctr_stream_t stream);
size_t ctr_frappe_workspace_bytes(size_t len);
int ctr_frappe_plan(const char* text, size_t len, int64_t* info, void* ws, size_t ws_bytes, ctr_stream_t stream);
int ctr_frappe_write(const char* text, size_t len, char* out, const void* ws, size_t ws_bytes, ctr_stream_t stream);

/* ---- CRC-32C of whole tensors (TensorFlow checkpoint bundles; DESIGN.md §2.11) ---------------------------------------
 * ranges: device int64 [n][2] = {address, length in bytes}.  An address needs only 4-byte alignment; a length may be 0
 * or exceed 2^32.  total_bytes >= the sum of the lengths (it sizes the grid and the workspace of
 * ctr_crc32c_workspace_bytes(n, total_bytes) bytes).  crc[r] = the standard CRC-32C of range r (initial value and
 * final XOR 0xFFFFFFFF, what tfrecord.crc32c returns); masked[r] = ((crc >> 15) | (crc << 17)) + 0xA282EAD8 (mod 2^32),
 * the value a bundle's BundleEntryProto.crc32c holds.  Either output may be NULL, not both.  Deterministic. */
size_t ctr_crc32c_workspace_bytes(int n, int64_t total_bytes);
int ctr_crc32c_ranges(const int64_t* ranges, int n, int64_t total_bytes, uint32_t* crc, uint32_t* masked, void* ws,
                      size_t ws_bytes, ctr_stream_t stream);

/* ---- eval / infer scoring (DESIGN.md §2.13) --------------------------------------------------------------------------
 * auc_counts (tf.metrics.auc's 200-threshold confusion counts, DeepFM.py:194, DeepCvrMTL.py:229-233): pred, label f32
 *   [n], n < 2^40; thresholds f32 [200] ascending.  counts int64 [2][201] += per class (row 0: label == 0, row 1:
 *   label != 0, a NaN label included) the histogram of k = #{t : t < pred}; a NaN pred has k = 200, and a pred equal to
 *   a threshold is not above it.  Suffix sums of row 1 (row 0) from k = i + 1 are tf's tp (fp) at threshold i.  Exact
 *   and independent of order; the caller zeroes counts once and accumulates over calls.
 * format_preds (pred.txt, DeepFM.py:351-353): appends row r's "%f\n" % a[r] (b NULL) or "%f\t%f\n" % (a[r], b[r]) for
 *   r < n at out[*offset, ...), the bytes of Python's "%f" % float(x) for every float32 (nan, inf, -inf, -0.000000,
 *   subnormals, FLT_MAX), and advances *offset (device int64) by the bytes of the rows.  A row is at most 48 bytes
 *   per column.  Bytes at or past out_bytes are not written (*offset still advances: *offset > out_bytes after the call
 *   means the buffer was too small).  ws = ctr_format_preds_workspace_bytes(n) bytes.
 * n = 0 is a no-op; no allocation and no synchronisation inside. */
int ctr_auc_counts(const float* pred, const float* label, int64_t n, const float* thresholds, int64_t* counts,
                   ctr_stream_t stream);
size_t ctr_format_preds_workspace_bytes(int64_t n);
int ctr_format_preds(const float* a, const float* b, int64_t n, char* out, int64_t out_bytes, int64_t* offset,
                     void* ws, size_t ws_bytes, ctr_stream_t stream);

/* ---- table initialisation (glorot_normal_initializer, DeepFM.py:115-116; truncated at 2 sigma) --- */
int ctr_init_trunc_normal(float* t, int64_t n, float stddev, uint64_t seed, ctr_stream_t stream);
int ctr_fill(float* t, int64_t n, float value, ctr_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* CTR_B200_H_ */
