"""DeepFM's FM kernels (csrc/fm_embed.cu: K1 forward in its LDG, TMA-staged and generic-K forms, K2 backward), the
batch-norm layer (csrc/batch_norm.cu) and NFM's bi dropout, against fp64 references or exact fp32 restatements across
their dispatch space; then DeepFM (DeepFM.py flags: K=32, deep_layers=256,128,64, dropout=0.5 x 3, Adam 5e-4,
l2 1e-4, batch 64), DeepFM at the benchmark's shape (K=16, B=8192) and NFM (NFM.py flags: K=64, deep_layers=128,64,
dropout=0.5,0.8,0.8, Adam 0.05, l2 1e-3, batch 128) with injected dropout masks against the oracle.

Error bounds (U = 2^-24, gam(n) = nU / (1 - nU): n rounded fp32 operations along one path, relative to the sum of the
|terms| they combine).  Every kernel bound is elementwise or per sample.
  K1, per sample b and column k, with e_fk = V[id_f, k] * val_f and A_k = sum_f |e_fk| (fp64, exact products):
    x      one multiply: bit-exact against fp32 V[id] * val.
    S      each e is rounded once, then at most F - 1 adds on any path (per-slot sequential sums, then the slot
           butterfly): |S - S64| <= gam(F + 1) A_k.  The generic kernel sums fields in order: bit-exact against the
           sequential fp32 sum of x.
    y_w    per lane fmaf over its fields, then a 5-level butterfly: gam(F + 1) sum_f |W val|.
    d_k    = fl(fl(S*S) - q) with q = sum_f e^2 (fmaf chain + butterfly): |s*s - S^2| <= |s - S| |s + S| gives
           2 gam(F + 1) A_k^2 to first order, q is within gam(F + 3) A_k^2 (sum e^2 <= A_k^2), the product and the
           subtraction add U each of a value <= A_k^2.  Together (gam is superadditive): |d_k - D_k| <= gam(3F + 8) A_k^2.
    bi     (NFM) 0.5 d_k, exact halving: 0.5 gam(3F + 8) A_k^2 per element.
    y2     (DeepFM) |D_k| <= A_k^2 (S^2 and sum e^2 both lie in [0, A_k^2]); the K-sum has depth <= K + 5 (generic:
           K/32 lane terms + 5 butterfly levels), so 0.5 gam(3F + K + 16) sum_k A_k^2 per sample.
  K2, from the same fp32 inputs (S, x, dX, dy2): g = fl(fl(w2 * fl(S - x) + dX) * val) has three roundings: within
    gam(3) (|w2| (|S| + |x|) + |dX|) |val| of (w2 (S - x) + dX) val (|S - x| <= |S| + |x| also covers fl(S - x));
    g_w = dyw * val and PLAIN's dX * val are one multiply: bit-exact.
  Batch norm, per column (n_c rows in chunk c of 32; the chunk sums run n_c/8 rows per thread, then 8 partials):
    mean   chunk mean within Ec = gam(n_c/8 + 12) mean_c|x|; the merge (n_c * mean_c, 32 adds, / n) leaves the batch mean
           within E = gam(n/256 + 48) sum|x|/n.
    var    with D_c = |mean_c - mean| and e_c = Ec + E, the chunked two-pass sum and Chan's merge compute, in exact
           arithmetic on the rounded means, the true M2 plus at most sum n_c (2 D_c e_c + 2 e_c^2) (first order in the
           chunk means' errors, since sum n_c (mean_c - mean) = 0); their own roundings add
           gam(n/256 + 80) (var + sum n_c ((D_c + e_c)^2 + e_c^2) / n).
    y      inv = (1/sqrtf(var + eps)) gamma: relative error rho = 0.5 Evar / (var + eps) + 4U; y = x inv + (beta - mean inv)
           cancels, so its bound is (rho + 3U) (|x inv| + |mean inv| + |beta|) + |inv| E; dropout /keep adds U of |y|/keep.
    moving moving -= (moving - batch) (1 - decay): (1 - decay) times the statistic's bound + gam(3) (|moving| + |batch|).
    d_beta, d_gamma  n-term sums along the same chunking (depth n/256 + 44): gam(n/256 + 45) sum|dY| and
           (gam(n/256 + 48) + rho') sum|dY xhat| + rstd E sum|dY|, rho' = 0.5 Evar / (var + eps) + 3U.
    d_x    gamma rstd (dY - d_beta/n - xhat d_gamma/n): (rho' + 8U) |gamma| rstd (|dY| + |d_beta|/n + |xhat| |d_gamma|/n)
           plus |gamma| rstd times (err(d_beta) + |xhat| err(d_gamma) + (|xhat| (rho' + 2U) + rstd E) |d_gamma|) / n.
Model-level bounds follow the pin of DIN (tests/test_gpu_din_attention.py): the sum of the stage bounds along the path,
scaled by each gradient tensor's largest magnitude (per sample for the per-occurrence rows), because the oracle does not
expose the magnitudes of the terms each gradient sums.
"""
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.test_gpu_din_attention import U, _bits_equal, _pick_split, _within, gemm_rel

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INT32_MAX = 2 ** 31 - 1
SPECIALISED_K = (4, 8, 16, 32, 64, 128, 256)


def gam(n):
    return n * U / (1 - n * U)


def _dev():
    return torch.device("cuda:0")


# ---------------------------------------------------------------------------------------------------------------------
# K1: fm_embed_fwd
# ---------------------------------------------------------------------------------------------------------------------
def _fm_inputs(B, F, N, K, seed, regime="random"):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, N, (B, F), generator=g)
    ids.view(-1)[0] = 0
    ids.view(-1)[-1] = N - 1
    vals = torch.rand(B, F, generator=g) * 2 - 0.5
    V = torch.randn(N, K, generator=g) * 0.3
    W = torch.randn(N, generator=g) * 0.3
    if regime == "single":            # one active field per sample: S == e, so y2 and bi are exactly 0
        keep = torch.zeros(B, F)
        keep[torch.arange(B), torch.randint(0, F, (B,), generator=g)] = 1.0
        vals = vals * keep
    elif regime == "cancel":          # field pairs (id, v), (id, -v): S ~ 0 while sum e^2 is large
        for f in range(0, F - 1, 2):
            ids[:, f + 1] = ids[:, f]
            vals[:, f + 1] = -vals[:, f]
    elif regime == "scale":           # |val| near 1e3 on even samples, near 1e-3 on odd ones
        mag = torch.where(torch.arange(B)[:, None] % 2 == 0, torch.tensor(1e3), torch.tensor(1e-3))
        vals = mag * (0.5 + torch.rand(B, F, generator=g)) * torch.sign(vals + 0.25)
    elif regime == "edges":           # only the first and last row of the table
        ids = torch.where(torch.rand(B, F, generator=g) < 0.5, torch.tensor(0), torch.tensor(N - 1))
    return ids, vals.float(), V.float(), W.float()


def _fm_ref(ids, vals, V, W):
    idl = ids.long()
    e32 = V[idl] * vals[..., None]                                  # [B, F, K] fp32, one rounding each
    e = V.double()[idl] * vals.double()[..., None]                  # exact products
    A = e.abs().sum(1)                                              # [B, K]
    S = e.sum(1)
    Q = (e * e).sum(1)
    D = S * S - Q
    wv = W.double()[idl] * vals.double()
    F, K = ids.shape[1], V.shape[1]
    return dict(x=e32.reshape(ids.shape[0], -1), e32=e32, S=S, S_bound=gam(F + 1) * A,
                y_w=wv.sum(1), y_w_bound=gam(F + 1) * wv.abs().sum(1),
                bi=0.5 * D, bi_bound=0.5 * gam(3 * F + 8) * A * A,
                y2=0.5 * D.sum(1), y2_bound=0.5 * gam(3 * F + K + 16) * (A * A).sum(1))


def _fm_run(ids, vals, V, W, mode, want_x=True, oob=False):
    from tf_repos_b200 import ops
    d = _dev()
    B, F = ids.shape
    K = V.shape[1]
    nan = float("nan")
    out = {}
    x = torch.full((B, F * K), nan, device=d) if want_x else None
    yw = torch.full((B,), nan, device=d) if W is not None else None
    y2 = S = None
    if mode != ops.FM_PLAIN:
        y2 = torch.full((B, K) if mode == ops.FM_NFM else (B,), nan, device=d)
        S = torch.full((B, K), nan, device=d)
    cnt = torch.zeros(2, dtype=torch.int32, device=d) if oob else None
    ops.fm_embed_fwd(ids.to(d), vals.to(d), V.to(d), W.to(d) if W is not None else None, mode, x=x, y_w=yw, y2=y2,
                     S=S, oob=cnt)
    for k, t in (("x", x), ("y_w", yw), ("y2", y2), ("S", S), ("oob", cnt)):
        if t is not None:
            out[k] = t.cpu()
    return out


def _check_fwd(ids, vals, V, W, what, generic):
    """all three modes at these inputs; x / W given and absent across them"""
    from tf_repos_b200 import ops
    ref = _fm_ref(ids, vals, V, W)
    F = ids.shape[1]
    runs = [(ops.FM_DEEPFM, True, W), (ops.FM_NFM, False, W), (ops.FM_PLAIN, True, None), (ops.FM_DEEPFM, False, None)]
    for mode, want_x, w in runs:
        tag = f"{what} mode={mode} x={want_x} W={w is not None}"
        o = _fm_run(ids, vals, V, w, mode, want_x)
        if want_x:
            _bits_equal(o["x"], ref["x"], f"{tag}: x = V[id]*val (one multiply)")
        if w is not None:
            _within(o["y_w"], ref["y_w"], ref["y_w_bound"], f"{tag}: y_w")
        if mode == ops.FM_PLAIN:
            continue
        _within(o["S"], ref["S"], ref["S_bound"], f"{tag}: S")
        if generic:
            s = torch.zeros(ids.shape[0], V.shape[1])
            for f in range(F):
                s = s + ref["e32"][:, f]
            _bits_equal(o["S"], s, f"{tag}: generic S = sequential fp32 sum over fields")
        if mode == ops.FM_NFM:
            _within(o["y2"], ref["bi"], ref["bi_bound"], f"{tag}: bi")
        else:
            _within(o["y2"], ref["y2"], ref["y2_bound"], f"{tag}: y2")
    return ref


# (K, F, B): every specialised K and generic K in {1, 3, 10, 33, 100}, with every kernel instance reached at F > 32;
# F crosses the 32-field chunk boundary and TMA's F <= 64 limit; B leaves a partial 4-warp CTA
FWD_CASES = [
    (4, 65, 4097), (4, 1, 3), (8, 33, 5), (8, 2, 1), (16, 39, 4097), (16, 31, 3), (32, 64, 5), (32, 32, 1),
    (64, 65, 3), (64, 33, 4097), (128, 1, 5), (128, 31, 3), (128, 32, 1), (128, 33, 4097), (128, 64, 5),
    (128, 65, 3), (256, 39, 5), (256, 2, 3), (1, 39, 4097), (3, 65, 5), (10, 33, 3), (33, 39, 5), (100, 64, 1),
    (100, 2, 4097),
]


@pytest.mark.parametrize("K,F,B", FWD_CASES)
def test_fm_embed_fwd_dispatch_space_against_fp64(K, F, B):
    N = 1000
    for bits, idt in ((32, torch.int32), (64, torch.int64)):
        ids, vals, V, W = _fm_inputs(B, F, N, K, seed=K * 1000 + F * 10 + bits)
        _check_fwd(ids.to(idt), vals, V, W, f"K={K} F={F} B={B} int{bits}", K not in SPECIALISED_K)


@pytest.mark.parametrize("regime", ["single", "cancel", "scale", "edges"])
@pytest.mark.parametrize("K,F", [(4, 33), (16, 39), (128, 33), (256, 33), (10, 39), (100, 65)])
def test_fm_embed_fwd_value_regimes(K, F, regime):
    from tf_repos_b200 import ops
    B, N = 37, 500
    ids, vals, V, W = _fm_inputs(B, F, N, K, seed=K + F, regime=regime)
    _check_fwd(ids.to(torch.int32), vals, V, W, f"K={K} F={F} {regime}", K not in SPECIALISED_K)
    if regime == "single":
        # the separately rounded fl(S*S) - q is exactly 0 when one field is active, as tf.square - tf.reduce_sum is
        for mode in (ops.FM_DEEPFM, ops.FM_NFM):
            o = _fm_run(ids.to(torch.int64), vals, V, W, mode)
            assert torch.all(o["y2"] == 0), f"K={K} F={F} mode={mode}: y2 / bi must be exactly 0 with one active field"


@pytest.mark.parametrize("K,F", [(16, 39), (256, 33), (128, 33), (128, 64), (10, 33), (33, 65)])
def test_fm_embed_fwd_out_of_range_ids_count_once_and_add_zero(K, F):
    """LDG (16, 256), TMA (128 at F <= 64), generic (10, 33)"""
    from tf_repos_b200 import ops
    B, N = 9, 300
    ids, vals, V, W = _fm_inputs(B, F, N, K, seed=7 * K + F)
    for idt, bad in ((torch.int32, [-1, N, INT32_MAX]), (torch.int64, [-1, N, INT32_MAX, 2 ** 31 + 5])):
        bi = ids.clone().to(idt)
        where = []
        for j, v in enumerate(bad):
            b, f = (2 * j + 1) % B, (5 * j + 31) % F          # fields on both sides of the 32-field chunk boundary
            where.append((b, f)); bi[b, f] = v
        b, f = 4, F - 1                                       # a second bad field in one sample
        where.append((b, f)); bi[b, f] = bad[0]
        # the same batch with the bad fields made harmless by hand: a valid id (0) and val 0
        good_ids, good_vals = bi.clone(), vals.clone()
        for b, f in where:
            good_ids[b, f] = 0; good_vals[b, f] = 0.0
        for mode in (ops.FM_DEEPFM, ops.FM_NFM, ops.FM_PLAIN):
            w = W if mode != ops.FM_PLAIN else None
            o = _fm_run(bi, vals, V, w, mode, oob=True)
            r = _fm_run(good_ids, good_vals, V, w, mode)
            tag = f"K={K} F={F} {idt} mode={mode}"
            assert o["oob"][0].item() == len(where), f"{tag}: each bad occurrence counts once: {o['oob'].tolist()}"
            assert o["oob"][1].item() in {int(np.int64(v).astype(np.int32)) for v in bad}, f"{tag}: {o['oob'].tolist()}"
            for k in r:                                        # each bad field adds exactly zero; the rest is unchanged
                assert torch.equal(o[k], r[k]), f"{tag}: {k} differs from the batch with the bad fields zeroed"
            xr = o["x"].view(B, F, K)
            assert torch.all(xr[[b for b, _ in where], [f for _, f in where]] == 0), f"{tag}: x of a bad field"
            mask = torch.ones(B, F, dtype=torch.bool)
            for b, f in where:
                mask[b, f] = False
            want = (V[good_ids.long()] * vals[..., None])[mask]
            _bits_equal(xr[mask], want, f"{tag}: x of the good fields")


@pytest.mark.parametrize("F", [1, 31, 32, 33, 64, 65])
def test_fm_embed_fwd_k128_tma_default_and_its_fallback(F):
    """K = 128 takes the TMA-staged kernel by default at F <= 64 and falls back to the LDG kernel at F = 65"""
    B, N = 37, 400
    for idt in (torch.int32, torch.int64):
        ids, vals, V, W = _fm_inputs(B, F, N, 128, seed=F)
        _check_fwd(ids.to(idt), vals, V, W, f"K=128 F={F} {idt}", False)


TMA_CHILD = r"""
import hashlib, json, sys
import torch
sys.path.insert(0, %(root)r)
from tf_repos_b200 import ops
out = {}
for K in (16, 32, 64, 128):
    for F in (1, 31, 33, 64):
        B, N = 37, 700
        g = torch.Generator().manual_seed(K * 100 + F)
        ids = torch.randint(0, N, (B, F), generator=g); ids[0, 0] = N - 1
        vals = (torch.rand(B, F, generator=g) * 2 - 0.5).cuda()
        V = (torch.randn(N, K, generator=g) * 0.3).cuda(); W = (torch.randn(N, generator=g) * 0.3).cuda()
        for idt in (torch.int32, torch.int64):
            for mode in (ops.FM_DEEPFM, ops.FM_NFM, ops.FM_PLAIN):
                x = torch.empty(B, F * K, device="cuda"); yw = torch.empty(B, device="cuda")
                y2 = torch.empty((B, K) if mode == ops.FM_NFM else (B,), device="cuda"); S = torch.empty(B, K, device="cuda")
                if mode == ops.FM_PLAIN:
                    y2 = S = None
                ops.fm_embed_fwd(ids.to(idt).cuda(), vals, V, W, mode, x=x, y_w=yw, y2=y2, S=S)
                h = hashlib.sha256()
                for t in (x, yw, y2, S):
                    if t is not None:
                        h.update(t.cpu().numpy().tobytes())
                out[f"K={K} F={F} {idt} mode={mode}"] = h.hexdigest()
print("RESULT " + json.dumps(out))
"""


def _tma_child(setting):
    env = dict(os.environ, CTR_FM_EMBED_TMA=setting)
    r = subprocess.run([sys.executable, "-c", TMA_CHILD % {"root": ROOT}], capture_output=True, text=True, timeout=600,
                       env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1]
    return json.loads(line[len("RESULT "):])


def test_fm_embed_fwd_tma_and_ldg_give_the_same_bits():
    """fm_embed_fwd_tma_kernel keeps fm_embed_fwd_kernel's mapping and arithmetic order: one process per setting"""
    tma, ldg = _tma_child("1"), _tma_child("0")
    assert tma.keys() == ldg.keys() and len(tma) == 4 * 4 * 2 * 3
    diff = [k for k in tma if tma[k] != ldg[k]]
    assert not diff, f"TMA and LDG outputs differ for {diff}"


# ---------------------------------------------------------------------------------------------------------------------
# K2: fm_embed_bwd
# ---------------------------------------------------------------------------------------------------------------------
def _bwd_inputs(B, F, N, K, seed, single=False):
    ids, vals, V, _ = _fm_inputs(B, F, N, K, seed, regime="single" if single else "random")
    g = torch.Generator().manual_seed(seed + 1)
    e32 = V[ids.long()] * vals[..., None]
    x = e32.reshape(B, F * K)
    S = e32.sum(1)                                              # any fp32 S: K2's bound is relative to its inputs
    dX = torch.randn(B, F * K, generator=g) * 0.1
    dy_s = torch.randn(B, generator=g)
    dy_k = torch.randn(B, K, generator=g)
    dyw = torch.randn(B, generator=g)
    return vals, x, S, dX, dy_s, dy_k, dyw


def _bwd_run(vals, x, S, dX, dy2, dyw, K, mode):
    from tf_repos_b200 import ops
    d = _dev()
    B, F = vals.shape
    g_rows = torch.full((B * F, K), float("nan"), device=d)
    g_w = torch.full((B * F,), float("nan"), device=d) if dyw is not None else None
    c = lambda t: t.to(d).contiguous() if t is not None else None
    ops.fm_embed_bwd(c(vals), c(x), c(S), c(dX), c(dy2), c(dyw), K, mode, g_rows, g_w)
    return g_rows.cpu(), (g_w.cpu() if g_w is not None else None)


@pytest.mark.parametrize("K", list(SPECIALISED_K) + [1, 10, 33])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_fm_embed_bwd_against_fp64_from_the_same_inputs(K, mode):
    B, F, N = 37, 39, 300
    vals, x, S, dX, dy_s, dy_k, dyw = _bwd_inputs(B, F, N, K, seed=K * 10 + mode)
    dy2 = None if mode == 2 else (dy_s if mode == 0 else dy_k)
    for use_dx in ((True,) if mode == 2 else (True, False)):
        for use_w in (True, False):
            tag = f"K={K} mode={mode} dX={use_dx} g_w={use_w}"
            g_rows, g_w = _bwd_run(vals, x, S, dX if use_dx else None, dy2, dyw if use_w else None, K, mode)
            v64 = vals.double().reshape(B, F, 1)
            dX64 = dX.double().reshape(B, F, K) if use_dx else torch.zeros(B, F, K, dtype=torch.float64)
            if mode == 2:
                _bits_equal(g_rows, (dX.reshape(B, F, K) * vals[..., None]).reshape(B * F, K),
                            f"{tag}: PLAIN g_rows = dX*val (one multiply)")
            else:
                w2 = dy2.double().reshape(B, 1, 1) if mode == 0 else dy2.double().reshape(B, 1, K)
                S64, x64 = S.double().reshape(B, 1, K), x.double().reshape(B, F, K)
                ref = (w2 * (S64 - x64) + dX64) * v64
                bound = gam(3) * (w2.abs() * (S64.abs() + x64.abs()) + dX64.abs()) * v64.abs()
                _within(g_rows.reshape(B, F, K), ref, bound, f"{tag}: g_rows")
            if use_w:
                _bits_equal(g_w, (dyw[:, None] * vals).reshape(-1), f"{tag}: g_w = dyw*val (one multiply)")


@pytest.mark.parametrize("K", list(SPECIALISED_K) + [1, 10, 33])
def test_fm_embed_bwd_single_active_field(K):
    """with one field active S - x is exactly 0 for it: g_rows = fl(dX * val); the inactive fields (val 0) give 0"""
    B, F, N = 5, 33, 200
    vals, x, S, dX, dy_s, dy_k, dyw = _bwd_inputs(B, F, N, K, seed=K, single=True)
    active = (vals != 0).reshape(B * F)
    for mode, dy2 in ((0, dy_s), (1, dy_k)):
        g_rows, _ = _bwd_run(vals, x, S, dX, dy2, None, K, mode)
        want = (dX.reshape(B, F, K) * vals[..., None]).reshape(B * F, K)
        _bits_equal(g_rows[active], want[active], f"K={K} mode={mode}: active field")
        assert torch.all(g_rows[~active] == 0), f"K={K} mode={mode}: inactive fields must give 0"


# ---------------------------------------------------------------------------------------------------------------------
# batch norm: ctr_bn_fwd (train / eval), ctr_bn_bwd
# ---------------------------------------------------------------------------------------------------------------------
EPS = 1e-3
DECAY = float(np.float32(0.9))
CHUNKS = 32


def _bn_x(n, H, g):
    """column c takes regime c % 6: relu(N(0,1)); dead (0); constant 0.75; 1e3 + 1e-2 N(0,1); one nonzero row;
    relu(N(0,1)) scaled by 1e-3 .. 1e2"""
    x = torch.relu(torch.randn(n, H, generator=g))
    for c in range(H):
        r = c % 6
        if r == 1:
            x[:, c] = 0.0
        elif r == 2:
            x[:, c] = 0.75
        elif r == 3:
            x[:, c] = 1e3 + 1e-2 * torch.randn(n, generator=g)
        elif r == 4:
            x[:, c] = 0.0
            x[(7 * c) % n, c] = 3.0 * float(torch.randn(1, generator=g)) + 0.5
        elif r == 5:
            x[:, c] *= 10.0 ** (-3 + (c // 6) % 6)
    return x.float()


def _bn_ref(x, gamma, beta, mm0, mv0, mask, keep, d_out):
    """fp64, batch_norm.cu's header formulas: tf.nn.moments (biased), x*inv + (beta - mean*inv), the in-place moving
    average, autodiff; plus the per-element bounds of the module docstring"""
    n, H = x.shape
    x64 = x.double().requires_grad_(True)
    g64 = gamma.double().requires_grad_(True)
    b64 = beta.double().requires_grad_(True)
    mean = x64.mean(0)
    var = ((x64 - mean) ** 2).mean(0)
    inv = torch.rsqrt(var + EPS) * g64
    y = x64 * inv + (b64 - mean * inv)
    if mask is not None:
        y = y / keep * mask.double()
    y.backward(d_out.double())
    X = x.double().numpy()
    m, v = mean.detach().numpy(), var.detach().numpy()
    absx = np.abs(X)
    E = gam(n // 256 + 48) * absx.mean(0)
    acc, pen = np.zeros(H), np.zeros(H)
    for ch in range(CHUNKS):
        r0, r1 = n * ch // CHUNKS, n * (ch + 1) // CHUNKS
        nc = r1 - r0
        if nc == 0:
            continue
        mc = X[r0:r1].mean(0)
        e = gam(nc // 8 + 12) * absx[r0:r1].mean(0) + E
        D = np.abs(mc - m)
        acc += nc * ((D + e) ** 2 + e ** 2)
        pen += nc * (2 * D * e + 2 * e * e)
    Evar = gam(n // 256 + 80) * (v + acc / n) + pen / n
    rstd = 1.0 / np.sqrt(v + EPS)
    G, Bt = gamma.double().numpy(), beta.double().numpy()
    invn = rstd * G
    rho = 0.5 * Evar / (v + EPS) + 4 * U
    yb = (rho + 3 * U) * (absx * np.abs(invn) + np.abs(m * invn) + np.abs(Bt)) + np.abs(invn) * E
    y64 = y.detach().numpy()
    if mask is not None:
        M = mask.double().numpy()
        yb = (yb / keep + U * np.abs(y64)) * M
        dY = d_out.double().numpy() / keep * M
    else:
        dY = d_out.double().numpy()
    omd = 1.0 - DECAY
    mm = mm0.double().numpy() - (mm0.double().numpy() - m) * omd
    mv = mv0.double().numpy() - (mv0.double().numpy() - v) * omd
    mmb = omd * E + gam(3) * (np.abs(mm0.double().numpy()) + np.abs(m))
    mvb = omd * Evar + gam(3) * (np.abs(mv0.double().numpy()) + np.abs(v))
    xhat = (X - m) * rstd
    rho2 = 0.5 * Evar / (v + EPS) + 3 * U
    depth = n // 256 + 44
    db, dg = b64.grad.numpy(), g64.grad.numpy()
    db_b = gam(depth + 1) * np.abs(dY).sum(0)
    dg_b = (gam(depth + 4) + rho2) * np.abs(dY * xhat).sum(0) + rstd * E * np.abs(dY).sum(0)
    gr = np.abs(G) * rstd
    dx_b = gr * ((rho2 + 8 * U) * (np.abs(dY) + np.abs(db) / n + np.abs(xhat) * np.abs(dg) / n)
                 + (db_b + np.abs(xhat) * dg_b + (np.abs(xhat) * (rho2 + 2 * U) + rstd * E) * np.abs(dg)) / n)
    return dict(mean=m, mean_b=E, var=v, var_b=Evar, y=y64, y_b=yb, mm=mm, mm_b=mmb, mv=mv, mv_b=mvb,
                dx=x64.grad.numpy(), dx_b=dx_b, dg=dg, dg_b=dg_b, db=db, db_b=db_b, rstd=rstd, dY=dY)


def _bn_data(n, H, keep, seed):
    g = torch.Generator().manual_seed(seed)
    x = _bn_x(n, H, g)
    gamma = 1.0 + 0.3 * torch.randn(H, generator=g)
    beta = 0.2 * torch.randn(H, generator=g)
    mm0 = torch.randn(H, generator=g) * 0.1
    mv0 = 1.0 + 0.1 * torch.rand(H, generator=g)
    mask = (torch.rand(n, H, generator=g) < keep).float() if keep < 1.0 else None
    d_out = torch.randn(n, H, generator=g)
    return x, gamma, beta, mm0, mv0, mask, d_out


def _bn_gpu(x, gamma, beta, mm0, mv0, mask, keep, d_out):
    from tf_repos_b200 import ops
    d = _dev()
    n, H = x.shape
    nan = float("nan")
    xd, gd, bd = x.to(d), gamma.to(d), beta.to(d)
    mm, mv = mm0.to(d).clone(), mv0.to(d).clone()
    md = mask.to(d) if mask is not None else None
    out = torch.full((n, H), nan, device=d)
    sm, sv = torch.full((H,), nan, device=d), torch.full((H,), nan, device=d)
    ops.bn_fwd(xd, gd, bd, mm, mv, True, DECAY, md, keep, out, sm, sv)
    dx = torch.full((n, H), nan, device=d)
    dg, db = torch.full((H,), nan, device=d), torch.full((H,), nan, device=d)
    ops.bn_bwd(d_out.to(d), xd, sm, sv, gd, md, keep, dx, dg, db)
    return {k: t.cpu() for k, t in dict(out=out, mean=sm, var=sv, mm=mm, mv=mv, dx=dx, dg=dg, db=db).items()}


BN_CASES = [(1, 16, 1.0), (2, 33, 0.8), (5, 300, 0.5), (31, 64, 1.0), (32, 1, 0.8), (33, 256, 0.5), (64, 31, 1.0),
            (1000, 300, 0.8), (8192, 256, 0.5), (65537, 16, 1.0)]


@pytest.mark.parametrize("n,H,keep", BN_CASES)
def test_bn_train_and_backward_against_fp64(n, H, keep):
    x, gamma, beta, mm0, mv0, mask, d_out = _bn_data(n, H, keep, seed=n * 7 + H)
    r = _bn_ref(x, gamma, beta, mm0, mv0, mask, keep, d_out)
    o = _bn_gpu(x, gamma, beta, mm0, mv0, mask, keep, d_out)
    tag = f"n={n} H={H} keep={keep}"
    _within(o["mean"], r["mean"], r["mean_b"], f"{tag}: save_mean")
    _within(o["var"], r["var"], r["var_b"], f"{tag}: save_var")
    _within(o["out"], r["y"], r["y_b"], f"{tag}: out")
    _within(o["mm"], r["mm"], r["mm_b"], f"{tag}: moving_mean")
    _within(o["mv"], r["mv"], r["mv_b"], f"{tag}: moving_variance")
    _within(o["db"], r["db"], r["db_b"], f"{tag}: d_beta")
    _within(o["dg"], r["dg"], r["dg_b"], f"{tag}: d_gamma")
    _within(o["dx"], r["dx"], r["dx_b"], f"{tag}: d_x")
    # exact columns: a dead unit has mean and var exactly 0, a constant 0.75 exactly (0.75, 0) (every partial sum of
    # 0.75s below 2^22 is exact); the dead unit's d_x is gamma rstd (dY - d_beta/n)
    dead = [c for c in range(H) if c % 6 == 1]
    const = [c for c in range(H) if c % 6 == 2]
    if dead:
        assert torch.all(o["mean"][dead] == 0) and torch.all(o["var"][dead] == 0), f"{tag}: dead unit's moments"
        rs = 1.0 / np.sqrt(EPS)
        want = gamma.double().numpy()[dead] * rs * (r["dY"][:, dead] - r["db"][dead] / n)
        _within(o["dx"][:, dead], want, r["dx_b"][:, dead], f"{tag}: dead unit's d_x")
    if const:
        assert torch.all(o["mean"][const] == 0.75) and torch.all(o["var"][const] == 0), f"{tag}: constant column"


@pytest.mark.parametrize("n,H", [(5, 300), (1000, 64), (33, 33)])
def test_bn_eval_uses_moving_statistics_and_writes_only_out(n, H):
    from tf_repos_b200 import ops
    d = _dev()
    x, gamma, beta, mm0, mv0, mask, _ = _bn_data(n, H, 0.5, seed=n + H)
    mm, mv = mm0.to(d), mv0.to(d)
    sm, sv = torch.full((H,), 7.0, device=d), torch.full((H,), 7.0, device=d)
    out = torch.full((n, H), float("nan"), device=d)
    ops.bn_fwd(x.to(d), gamma.to(d), beta.to(d), mm, mv, False, DECAY, mask.to(d), 0.5, out, sm, sv)
    assert torch.equal(mm.cpu(), mm0) and torch.equal(mv.cpu(), mv0), "eval must not move the moving statistics"
    assert torch.all(sm == 7.0) and torch.all(sv == 7.0), "eval must not write save_mean / save_var"
    inv = torch.rsqrt(mv0.double() + EPS) * gamma.double()
    ref = x.double() * inv + (beta.double() - mm0.double() * inv)         # no dropout in eval
    bound = 8 * U * (x.double().abs() * inv.abs() + (mm0.double() * inv).abs() + beta.double().abs())
    _within(out, ref, bound, f"eval n={n} H={H}")


def test_bn_is_bit_reproducible():
    args = _bn_data(8192, 300, 0.8, seed=11)
    x, gamma, beta, mm0, mv0, mask, d_out = args
    a = _bn_gpu(x, gamma, beta, mm0, mv0, mask, 0.8, d_out)
    b = _bn_gpu(x, gamma, beta, mm0, mv0, mask, 0.8, d_out)
    for k in a:
        _bits_equal(b[k], a[k], f"second call: {k}")


def test_bn_empty_batch_writes_nothing():
    from tf_repos_b200 import _lib, ops
    d = _dev()
    H = 33
    mm, mv = torch.full((H,), 3.0, device=d), torch.full((H,), 4.0, device=d)
    sm, sv = torch.full((H,), 5.0, device=d), torch.full((H,), 6.0, device=d)
    x = torch.empty(0, H, device=d)
    gd, bd = torch.ones(H, device=d), torch.zeros(H, device=d)
    g_, b_ = torch.full((H,), 8.0, device=d), torch.full((H,), 9.0, device=d)
    n0 = _lib.launch_count()
    ops.bn_fwd(x, gd, bd, mm, mv, True, DECAY, None, 1.0, torch.empty(0, H, device=d), sm, sv)
    ops.bn_bwd(torch.empty(0, H, device=d), x, sm, sv, gd, None, 1.0, torch.empty(0, H, device=d), g_, b_)
    assert _lib.launch_count() == n0
    for t, v in ((mm, 3.0), (mv, 4.0), (sm, 5.0), (sv, 6.0), (g_, 8.0), (b_, 9.0)):
        assert torch.all(t == v)


def test_bn_requires_raise_before_any_launch():
    from tf_repos_b200 import _lib
    from tf_repos_b200._lib import CtrError
    L = _lib.raw()
    d = _dev()
    n, H = 40, 33
    t = lambda *s: torch.full(s, 2.0, device=d)
    x, out, dx, mask = t(n, H), t(n, H), t(n, H), t(n, H)
    gamma, beta, mm, mv, sm, sv, dg, db = (t(H) for _ in range(8))
    need = int(L.ctr_bn_workspace_bytes(H))
    assert need == 2 * CHUNKS * H * 4
    ws = torch.empty(need, dtype=torch.uint8, device=d)
    p = lambda a: a.data_ptr()
    st = torch.cuda.current_stream().cuda_stream
    cases = [
        ("ctr_bn_fwd", "workspace too small",
         lambda: L.ctr_bn_fwd(p(x), n, H, p(gamma), p(beta), p(mm), p(mv), 1, DECAY, EPS, None, 1.0, p(out), p(sm),
                              p(sv), p(ws), need - 4, st)),
        ("ctr_bn_fwd", "save_mean/save_var required in TRAIN mode",
         lambda: L.ctr_bn_fwd(p(x), n, H, p(gamma), p(beta), p(mm), p(mv), 1, DECAY, EPS, None, 1.0, p(out), None,
                              p(sv), p(ws), need, st)),
        ("ctr_bn_fwd", "keep must be > 0 with a mask",
         lambda: L.ctr_bn_fwd(p(x), n, H, p(gamma), p(beta), p(mm), p(mv), 1, DECAY, EPS, p(mask), 0.0, p(out), p(sm),
                              p(sv), p(ws), need, st)),
        ("ctr_bn_bwd", "workspace too small",
         lambda: L.ctr_bn_bwd(p(out), p(x), n, H, p(sm), p(sv), p(gamma), EPS, None, 1.0, p(dx), p(dg), p(db), p(ws),
                              need - 4, st)),
        ("ctr_bn_bwd", "keep must be > 0 with a mask",
         lambda: L.ctr_bn_bwd(p(out), p(x), n, H, p(sm), p(sv), p(gamma), EPS, p(mask), -1.0, p(dx), p(dg), p(db),
                              p(ws), need, st)),
    ]
    for name, msg, call in cases:
        n0 = _lib.launch_count()
        with pytest.raises(CtrError, match=msg):
            _lib.check(call(), name)
        assert _lib.launch_count() == n0, f"{name} ({msg}) launched a kernel"
    torch.cuda.synchronize()
    for a in (x, out, dx, mm, mv, sm, sv, dg, db):
        assert torch.all(a == 2.0), "a refused call wrote a buffer"


def test_dropout_apply_matches_fp32_bit_for_bit():
    """NFM's bi dropout: fp32 x / keep * mask at an odd n"""
    from tf_repos_b200 import ops
    d = _dev()
    g = torch.Generator().manual_seed(3)
    n = 128 * 64 + 77
    for keep in (0.5, 0.8, 0.3):
        x = torch.randn(n, generator=g) * 10.0 ** torch.randint(-3, 4, (n,), generator=g)
        mask = (torch.rand(n, generator=g) < keep).float()
        out = torch.full((n,), float("nan"), device=d)
        ops.dropout_apply(x.to(d), mask.to(d), keep, out)
        k32 = torch.tensor(keep, dtype=torch.float32)
        _bits_equal(out, x / k32 * mask, f"dropout_apply keep={keep}")


# ---------------------------------------------------------------------------------------------------------------------
# DeepFM and NFM at the reference's default configurations, with injected dropout masks, against the oracle
# ---------------------------------------------------------------------------------------------------------------------
F39 = 39
DFM = dict(deep_layers="256,128,64", dropout="0.5,0.5,0.5", l2_reg=1e-4, learning_rate=5e-4, optimizer="Adam")
NFM_DEF = dict(deep_layers="128,64", dropout="0.5,0.8,0.8", l2_reg=1e-3, learning_rate=0.05, optimizer="Adam")
CONFIGS = {   # name: (model, K, B, N, flags)
    "deepfm": ("DeepFM", 32, 64, 20_000, DFM),
    "nfm": ("NFM", 64, 128, 20_000, NFM_DEF),
}


def _oracle_model(model, K, N, kw, batch_norm, dtype):
    from oracle import models as om
    cls = om.DeepFM if model == "DeepFM" else om.NFM
    ref = cls(F39, N, K, seed=4, dtype=dtype, batch_norm=batch_norm, batch_norm_decay=0.9, **kw)
    g = torch.Generator().manual_seed(1)
    tab, lin = ("fm_v", "fm_w") if model == "DeepFM" else ("emb", "linear")
    ref.params[tab].copy_(torch.randn(N, K, generator=g) * 0.1)
    ref.params[lin].copy_(torch.randn(N, generator=g) * 0.1)
    for name, p in ref.params.items():      # non-trivial batch-norm gamma / beta
        if name.endswith("/gamma"):
            p.copy_(1.0 + 0.2 * torch.randn(p.shape, generator=g))
        elif name.endswith("/beta"):
            p.copy_(0.1 * torch.randn(p.shape, generator=g))
    for p in ref.params.values():
        p.copy_(p.float().to(dtype))          # both sides start from the same fp32 values
    return ref


def _gpu_model(model, K, B, N, kw, batch_norm, mode="exact", epoch_steps=8):
    from tf_repos_b200.deepfm import DeepFM
    from tf_repos_b200.nfm import NFM
    cls = DeepFM if model == "DeepFM" else NFM
    return cls(F39, N, K, B, update_mode=mode, epoch_steps=epoch_steps, device="cuda:0", batch_norm=batch_norm,
               batch_norm_decay=0.9, **kw)


def _model_masks(model, B, K, kw, step):
    g = torch.Generator().manual_seed(700 + step)
    widths = [int(w) for w in kw["deep_layers"].split(",")]
    keep = [float(k) for k in kw["dropout"].split(",")]
    mlp = [(torch.rand(B, w, generator=g) < keep[i]).float() for i, w in enumerate(widths)]
    if model == "DeepFM":
        return mlp, [m.cuda() for m in mlp]
    bi = (torch.rand(B, K, generator=g) < keep[0]).float()
    return {"bi": bi, "mlp": mlp}, {"bi": bi.cuda(), "mlp": [m.cuda() for m in mlp]}


def _criteo(B, N, step):
    from tf_repos_b200 import synth
    ids, vals, labels = synth.criteo_batch(B, N, F39, seed=500 + step)
    return ids, vals, labels, {"feat_ids": ids.long(), "feat_vals": vals}


def _tol_grad(model, K, B, batch_norm):
    """the stage bounds along one step's path (module docstring; gemm_rel as in DIN's pin).  DeepFM forward: K1
    (gam(3F + K + 16)), the MLP GEMMs (R = F*K, 256, 128; one bias add each), the output dot (R = 64, + bias) and the
    logit / sigmoid-CE stages (8U); backward: the same GEMMs' dIn (R = 64, 128, 256), the dW products over B rows in
    fc.cu's split-R chunks (+ their partial adds), fc1's dW (B + 64 adds) and K2 (gam(3)).  NFM: K1's bi
    (gam(3F + 8)) feeds a 64 -> 128 -> 64 MLP, and the bi dropout and its backward add 2U each.  Batch norm adds per layer, forward and backward, its
    moment and d_gamma / d_beta sums over B rows: gam(B/256 + 100) twice."""
    if model == "DeepFM":
        widths, din = (256, 128, 64), F39 * K
        k1 = gam(3 * F39 + K + 16)
    else:
        widths, din = (128, 64), K
        k1 = gam(3 * F39 + 8) + 4 * U
    fwd, bwd, d = k1, gam(3), din
    for w in widths:
        fwd += gemm_rel(d, 1)
        bwd += gemm_rel(w) + gemm_rel(B, adds=_pick_split(d, w, B) + 1)
        d = w
    fwd += gam(widths[-1] + 1) + 8 * U
    bwd += gam(B + 64)
    bn = 2 * len(widths) * gam(B // 256 + 100) if batch_norm else 0.0
    return fwd + bwd + bn


def _one_step_against_fp64(model, K, B, N, kw, batch_norm):
    ref = _oracle_model(model, K, N, kw, batch_norm, torch.float64)
    gpu = _gpu_model(model, K, B, N, kw, batch_norm)
    gpu.load_variables(ref.params)
    ids, vals, labels, batch = _criteo(B, N, 0)
    mc, mg = _model_masks(model, B, K, kw, 0)
    _, out, _, dgrads = ref.gradients(batch, labels, mc)
    gpu.train_step(ids.cuda(), vals.cuda(), labels.cuda(), masks=mg)
    gpu.check_ids()
    torch.cuda.synchronize()
    tol = _tol_grad(model, K, B, batch_norm)
    tag = f"{model} K={K} B={B} batch_norm={batch_norm}"
    # logits of the step (train-mode forward with the masks), before the update; per sample, the FM / linear terms'
    # magnitudes plus the batch's largest deep term
    y = out["y"]
    vals64 = vals.double()
    lin = ref.params["fm_w" if model == "DeepFM" else "linear"][ids.long()].double()
    scale = (lin * vals64).abs().sum(1) + y.abs().max()
    if model == "DeepFM":
        scale = scale + 0.5 * (out["S"].abs() ** 2).sum(1) + out["y_v"].abs().max()
    _within(gpu.y[:B], y, tol * scale, f"{tag}: logits")
    assert set(dgrads) == set(gpu.dense.grads), (sorted(dgrads), sorted(gpu.dense.grads))
    for name, gref in dgrads.items():
        got = gpu.dense.grads[name].cpu()
        _within(got, gref.reshape(got.shape), tol * gref.abs().max(), f"{tag}: {name}")
    per = out["per_occurrence"]
    gv = per["v"].reshape(B, F39 * K)
    rows_scale = gv.abs().amax(1, keepdim=True)
    _within(gpu.g_rows[: B * F39].cpu().reshape(B, F39 * K), gv, tol * rows_scale, f"{tag}: per-occurrence g_rows")
    gw = per["w"].reshape(B, F39)
    _within(gpu.g_w[: B * F39].cpu().reshape(B, F39), gw, tol * gw.abs().amax(1, keepdim=True),
            f"{tag}: per-occurrence g_w")


@pytest.mark.parametrize("batch_norm", [False, True])
@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_default_config_one_step_against_fp64(cfg, batch_norm):
    model, K, B, N, kw = CONFIGS[cfg]
    _one_step_against_fp64(model, K, B, N, kw, batch_norm)


def test_deepfm_benchmark_shape_one_step_against_fp64():
    """bench.py's shape: K = 16, B = 8192 (the fp64 oracle runs on the CPU)"""
    _one_step_against_fp64("DeepFM", 16, 8192, 100_000, DFM, False)


def _full_state(m):
    m.flush()
    out = [t.var for t in m.tables] + [s for t in m.tables for s in t.slots] + [m.dense.flat] + list(m.dense.slots)
    out += list(m.mlp.bn_state.values())
    return [t.clone() for t in out]


# Variables that need more than 2e-5 against the fp32 oracle, at twice the largest ratio measured over three steps in
# both update modes (H100 SXM, 700 W).  Adam's first steps move an element by about lr * g / |g| whatever its size, so
# an element whose gradient nearly cancels (sums over the dropout-masked batch, batch norm's d_x) moves by up to lr in a
# direction set by the last bits of g, which the two fp32 implementations round differently.  The fp64 one-step test
# above pins those gradients themselves.  Measured: DeepFM mlp1/weights 2.3e-5; DeepFM with batch norm mlp0/weights
# 5.1e-4, fm_v 4.4e-5, mlp1/weights 4.4e-5, bn_0/moving_mean 2.3e-5; NFM emb 1.5e-4, mlp0/weights 4.9e-5, mlp1/weights
# 4.8e-5; NFM with batch norm emb 1.2e-3, mlp1/weights 8.4e-4, mlp0/weights 7.6e-5, deep_out/weights 7.1e-5,
# mlp1/biases 3.7e-5.
FP32_DEVIATIONS = {
    ("deepfm", False): {"Deep-part/mlp1/weights": 5e-5},
    ("deepfm", True): {"Deep-part/mlp0/weights": 1.1e-3, "fm_v": 9e-5, "Deep-part/mlp1/weights": 9e-5,
                       "Deep-part/bn_0/moving_mean": 5e-5},
    ("nfm", False): {"emb": 3.1e-4, "Deep-part/mlp0/weights": 1e-4, "Deep-part/mlp1/weights": 1e-4},
    ("nfm", True): {"emb": 2.4e-3, "Deep-part/mlp1/weights": 1.7e-3, "Deep-part/mlp0/weights": 1.6e-4,
                    "Deep-part/deep_out/weights": 1.5e-4, "Deep-part/mlp1/biases": 8e-5},
}


@pytest.mark.parametrize("mode", ["exact", "exact_deferred"])
@pytest.mark.parametrize("batch_norm", [False, True])
@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_default_config_three_steps_match_the_fp32_oracle(cfg, batch_norm, mode):
    model, K, B, N, kw = CONFIGS[cfg]
    ref = _oracle_model(model, K, N, kw, batch_norm, torch.float32)
    gpu = _gpu_model(model, K, B, N, kw, batch_norm, mode, epoch_steps=2)
    gpu.load_variables(ref.params)
    worst = {}
    for step in range(3):
        ids, vals, labels, batch = _criteo(B, N, step)
        mc, mg = _model_masks(model, B, K, kw, step)
        ref.train_step(batch, labels, mc)
        gpu.train_step(ids.cuda(), vals.cuda(), labels.cuda(), masks=mg)
        gpu.check_ids()
        vs = gpu.variables()
        for name, want in list(ref.params.items()) + list(ref.bn_state.items()):
            got, want = vs[name].cpu().double().numpy().reshape(want.shape), want.double().numpy()
            worst[name] = max(worst.get(name, 0.0), _excess(got, want))
    if batch_norm:   # PREDICT normalises with the moving statistics checked above
        ids, vals, _, batch = _criteo(B, N, 9)
        prob = gpu.predict(ids.cuda(), vals.cuda())
        want = ref.predict(batch)
        for got, w, what in ((gpu.y[:B], want["y"], "predict logits"), (prob, want["prob"], "predict prob")):
            worst[what] = _excess(got.cpu().double().numpy(), w.double().numpy())
    # test_gpu_deepfm.py's tolerance, |got - want| <= 2e-5 (|want| + the variable's scale), except where FP32_DEVIATIONS
    # states more
    tol = {**{k: 2e-5 for k in worst}, **FP32_DEVIATIONS.get((cfg, batch_norm), {})}
    bad = {k: v for k, v in worst.items() if v > tol[k]}
    assert not bad, f"{model} ({mode}, batch_norm={batch_norm}): {bad}; all: {worst}"


def _excess(got, want):
    """the smallest t with |got - want| <= t (|want| + max|want|)"""
    return float(np.max(np.abs(got - want) / (np.abs(want) + max(np.abs(want).max(), 1e-30))))


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_default_config_with_masks_and_batch_norm_is_bit_reproducible(cfg):
    model, K, B, N, kw = CONFIGS[cfg]
    ref = _oracle_model(model, K, N, kw, True, torch.float32)
    states = []
    for _ in range(2):
        m = _gpu_model(model, K, B, N, kw, True)
        m.load_variables(ref.params)
        for step in range(3):
            ids, vals, labels, _ = _criteo(B, N, 20 + step)
            _, mg = _model_masks(model, B, K, kw, 20 + step)
            m.train_step(ids.cuda(), vals.cuda(), labels.cuda(), masks=mg)
        states.append(_full_state(m) + [m.g_rows.clone(), m.g_w.clone(), m.dense.grad.clone()])
    for x, y in zip(*states):
        _bits_equal(y, x, f"{model}: two fresh models")
