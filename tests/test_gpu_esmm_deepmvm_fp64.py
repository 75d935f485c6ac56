"""The shared logit / sigmoid-CE kernel (csrc/loss.cu), ctr_l2_loss (csrc/optim.cu) and ESMM's multi-task head
(csrc/esmm.cu) against fp64 references or exact fp32 restatements, per element or per sample; then ESMM
(DeepCvrMTL.py flags: K=32, deep_layers=256,128,64, dropout=0.5 x 3, batch 64, ctr_task_wgt 0.5, Adam 5e-4, l2 1e-4;
the README's run line: K=16, 256,128, dropout 0.8,0.5, batch 1024, ctr_task_wgt 0.3, Adam 1e-4, l2 5e-3; F' = 11 in
both) and DeepMVM (DeepMVM.py flags: K=32, F=39, 256,128,64, dropout 0.5 x 3, batch 64, Adam 5e-4, l2 1e-4; run.sh:
K=32, batch 256, 256,128, dropout 0.8,0.8, Adam 1e-4, l2 1e-4) with injected dropout masks against the oracle.

Error bounds (U = 2^-24, gam(n) = nU / (1 - nU): n rounded fp32 operations along one path, relative to the sum of the
|terms| they combine; (1 + U)^a (1 + U)^b <= 1 + gam(a + b)).  Library functions are not assumed to round correctly:
the CUDA Programming Guide bounds expf by 2 ulp, logf and log1pf by 1 ulp; one ulp of a normal result is at most
2U of it, of a subnormal one 2^-149.  TINY = 2^-126 is the smallest normal fp32.
  sigmoid  p = fl(1 / fl(1 + expf(-y))): expf's 2 ulp are a factor (1 + 4U) <= (1 + U)^4 on e = exp(-y), and 1 + e
           then carries at most 4U e / (1 + e) <= 4U; the add and the division round once each, so |p - P| <= gam(6) P,
           plus 2^-150 (half an ulp) where the quotient is subnormal.  Where expf(-y) overflows (y < -88.72) p = 0;
           that is accepted only where P < TINY (it is, since P < e^-88.72 < 2^-126 = e^-87.34).  Where fl(P) = 1,
           P >= 1 - 2^-25, so e <= 2^-25 (1 + 4U) < 2^-24 and fl(1 + e) = 1: p must be exactly 1.
  ctr_logit_loss (one CTA of 1024 threads; thread i takes samples i, i + 1024, ...):
    y      bias + y_a + y_b + y_c left to right with __fadd_rn (+0 when the bias is absent): bit-exact.
    dy     fl(fl(p - t) * fl(1 / B_total)), correctly rounded ops from the kernel's own p: bit-exact.
    dbias  ceil(B/1024) sequential adds per thread, then two 5-level warp trees: d = ceil(B/1024) + 10 levels,
           |dbias - sum dy| <= gam(d) sum |dy| (sum over the kernel's dy in fp64).
    loss   term T = max(y, 0) - y t + log1p(exp(-|y|)); with A = max(y, 0) + |y t| and L = log1p(exp(-|y|)):
           fmaxf is exact and fl(max - y t) rounds at most twice (once if contracted to an FMA) -> gam(2) A.  expf's 4U
           moves log1p by at most 4U e <= 8U L (log1p(e) >= e/2 for e <= 1), log1pf adds 2U: gam(11) L.  The last add
           rounds once: per term gam(12) (A + L), plus 2^-147 where exp(-|y|) is subnormal.  Then the d-level sum and
           the two roundings of l * fl(1 / B_total): |loss - sum T / B_total| <= gam(d + 14) sum (A + L) / B_total.
  ctr_l2_loss: grid G = reduce_grid(n) = clamp(ceil(n / 2048), 1, 1024) CTAs of 256 threads; each thread sums
    m = ceil(n / 256G) squares in sequence (each v*v + s at most two roundings), then 5 warp levels and 8 sequential
    adds; one CTA sums the G partials (ceil(G/256) per thread, 5 + 8 levels), then one multiply by 0.5f * scale
    (exact halving).  depth = m + ceil(G/256) + 28, |out - scale sum t^2 / 2| <= gam(depth) scale sum t^2 / 2;
    n = 0 gives exactly +0.
  ctr_esmm_head: pctr, pcvr as the sigmoid above; pctcvr = fl(pt * pv) and every gradient op after the sigmoids is
    __f*_rn / __frcp_rn: d_ctr and d_cvr are bit-exact against the fp32 chain of esmm_oracle.head_reference fed the
    kernel's own pt and pv, including rows where q1 or q2 is the log epsilon.  ctr_loss terms as ctr_logit_loss's
    (gam(12) each); cvr_loss terms fl(fl(-z logf(q1)) - fl((1 - z) logf(q2))) from the kernel's own q1 = fl(p + eps),
    q2 = fl(fl(1 - p) + eps): logf's 2U and two roundings, gam(4) (z |log q1| + (1 - z) |log q2|).  Both sums run
    over the n real rows only, d = ceil(B/1024) + 10 levels, then one __fdiv_rn by n: gam(d + 13) and gam(d + 5).
    Rows >= n get d_ctr = d_cvr = +0.
  The dense sweep's l2 term (the table's l2 * l2_loss in exact mode): each thread sums m = ceil(n / (4 * 256 * 2 SMs))
    float4s of squares (3 roundings per float4, one add each), plus the scalar tail; 5 + 8 levels per CTA; the
    8 * SMs partials through ctr_reduce_sum (5 + 5 + 8 and 1 + 5 + 8 levels); fl(0.5 l2) and the multiply: m + 51.
Model-level bounds follow the pins of DIN and DeepFM (tests/test_gpu_fm_batch_norm.py): the sum of the stage bounds
along the path (_tol_esmm, _tol_mvm), scaled by each tensor's largest magnitude (per sample for the per-occurrence rows),
because the oracle does not expose the magnitudes of the terms each gradient sums.  DeepMVM's product
x_mvm = prod_f (e_f + b_f) rounds e, each add and each multiply: with M_f = |e_f| + |b_f|, |x_mvm - X| <= gam(3F) prod M
(no cancellation in a product); a multiply whose result is below TINY errs by up to 2^-150 instead, which the
trailing factors then scale: 2^-150 sum_{f >= 1} prod_{g > f} M_g (1 + gam(3F)).  At the reference's glorot
initialisation most x_mvm elements are subnormal, so the pin also runs factors of +-[0.9, 1.1].
"""
import math

import numpy as np
import pytest
import torch

from tests import esmm_oracle as eo
from tests.deepmvm_oracle import DeepMVM as OracleDeepMVM
from tests.test_gpu_din_attention import U, _bits_equal, _np, _pick_split, _within, gemm_rel
from tests.test_gpu_fm_batch_norm import _excess, gam

pytestmark = pytest.mark.gpu

TINY = 2.0 ** -126
HALF_SUB = 2.0 ** -150          # half an ulp of a subnormal result
NAN = float("nan")


def _dev():
    return torch.device("cuda:0")


def _nan(*shape):
    return torch.full(shape, NAN, device=_dev())


def _all_nan(t, what):
    assert torch.all(torch.isnan(t)), f"{what}: a buffer the call must not write was written"


def _check_sigmoid(got, y, what):
    """per element against the fp64 sigmoid of the fp32 logits y (module docstring)"""
    p, y64 = _np(got), y.double().cpu().numpy()
    P = 1.0 / (1.0 + np.exp(-y64))
    zero_ok = (p == 0) & (P < TINY)
    keep = ~zero_ok
    _within(p[keep], P[keep], gam(6) * P[keep] + HALF_SUB, f"{what}: sigmoid")
    ones = P.astype(np.float32) == 1.0
    assert np.all(p[ones] == 1.0), f"{what}: sigmoid must be exactly 1 where fp32 rounds it to 1"
    return P


def _ce_terms(y64, t64):
    """T, A, L of the sigmoid-CE term (module docstring), fp64"""
    m = np.maximum(y64, 0.0)
    L = np.log1p(np.exp(-np.abs(y64)))
    return m - y64 * t64 + L, m + np.abs(y64 * t64), L


def _sub_exp(y64):
    """2^-147 per term where exp(-|y|) is subnormal"""
    return np.where(np.exp(-np.abs(y64)) < TINY, 2.0 ** -147, 0.0)


# ---------------------------------------------------------------------------------------------------------------------
# 1. ctr_logit_loss
# ---------------------------------------------------------------------------------------------------------------------
LOSS_B = [1, 31, 1023, 1024, 1025, 8192, 10000]
BIAS = -0.375


def _logit_inputs(B, seed):
    """sample i takes regime i % 5: |y| <= 4; +-[15, 17] (p rounds to 1 above ~16.6); [-104, -88] (expf(-y) overflows
    below -88.72, p is subnormal above it); exactly 0 (with the bias); N(0, 2)"""
    g = torch.Generator().manual_seed(seed)
    r = torch.arange(B) % 5
    tgt = torch.rand(B, generator=g) * 8 - 4
    sign = torch.where(torch.rand(B, generator=g) < 0.5, -1.0, 1.0)
    tgt = torch.where(r == 1, sign * (15 + 2 * torch.rand(B, generator=g)), tgt)
    tgt = torch.where(r == 2, -(88 + 16 * torch.rand(B, generator=g)), tgt)
    tgt = torch.where(r == 4, 2 * torch.randn(B, generator=g), tgt)
    y_b = (torch.randn(B, generator=g) * 0.25).float()
    y_c = (torch.randn(B, generator=g) * 0.25).float()
    fixed = {1: 17.0, 2: -88.2, 3: 0.0, 7: -100.0}             # p = 1, subnormal p, y = 0, expf(-y) = inf
    for i, v in fixed.items():
        if i < B:
            tgt[i], y_b[i], y_c[i] = v, 0.0, 0.0
    y_a = (tgt - BIAS - y_b - y_c).float()
    zero = r == 3
    y_a[zero], y_b[zero], y_c[zero] = -BIAS, 0.0, 0.0          # fl(BIAS + -BIAS) + 0 + 0 = 0
    labels = (torch.rand(B, generator=g) < 0.5).float()
    return [y_a, y_b, y_c], labels


def _logit_run(bias, terms, labels, B, B_total, outputs=True):
    from tf_repos_b200 import ops
    d = _dev()
    o = dict(y=_nan(B), pred=_nan(B), loss_ce=_nan(1), dy=_nan(B), dbias=_nan(1))
    c = lambda t: t.to(d) if t is not None else None
    ops.logit_loss(c(bias), *[c(t) for t in terms], c(labels), B, B_total=B_total, **o)
    return {k: v.cpu() for k, v in o.items()}


@pytest.mark.parametrize("bt", ["B", "4B", "1"])
@pytest.mark.parametrize("B", LOSS_B)
def test_logit_loss_against_fp64_per_element(B, bt):
    B_total = {"B": B, "4B": 4 * B, "1": 1}[bt]
    terms, labels = _logit_inputs(B, seed=B * 3 + len(bt))
    t64 = labels.double().numpy()
    inv32 = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(B_total), dtype=torch.float32)
    depth = math.ceil(B / 1024) + 10
    for sub in range(1, 8):                                   # every non-empty subset of (y_a, y_b, y_c)
        use = [terms[j] if sub >> j & 1 else None for j in range(3)]
        for with_bias in (False, True):
            bias = torch.tensor([BIAS]) if with_bias else None
            tag = f"B={B} B_total={B_total} terms={sub:03b} bias={with_bias}"
            o = _logit_run(bias, use, labels, B, B_total)
            want = torch.full((B,), BIAS if with_bias else 0.0)
            for t in use:
                if t is not None:
                    want = want + t
            _bits_equal(o["y"], want, f"{tag}: y = left-to-right fp32 sum")
            _check_sigmoid(o["pred"], o["y"], f"{tag}: pred")
            _bits_equal(o["dy"], (o["pred"] - labels) * inv32, f"{tag}: dy = fl(fl(p - t) * fl(1/B_total))")
            dy = o["dy"].double().numpy()
            _within(o["dbias"], [dy.sum()], [gam(depth) * np.abs(dy).sum()], f"{tag}: dbias")
            y64 = o["y"].double().numpy()
            T, A, L = _ce_terms(y64, t64)
            bound = (gam(depth + 14) * (A + L).sum() + _sub_exp(y64).sum()) / B_total
            _within(o["loss_ce"], [T.sum() / B_total], [bound], f"{tag}: loss_ce")
            if sub == 7 and with_bias and B >= 8:               # every regime is reached
                y, p = o["y"], o["pred"]
                assert torch.any(y == 0) and torch.any(p == 0) and torch.any(p == 1), tag
                assert torch.any((p > 0) & (p < TINY)), f"{tag}: no subnormal pred"
                assert torch.any((y.abs() <= 4) & (y != 0)), tag


@pytest.mark.parametrize("B", [1, 1025, 8192])
def test_logit_loss_predict_only_writes_y_and_pred(B):
    terms, labels = _logit_inputs(B, seed=B)
    bias = torch.tensor([BIAS])
    train = _logit_run(bias, terms, labels, B, B)
    o = _logit_run(bias, terms, None, B, B)
    for k in ("loss_ce", "dy", "dbias"):
        _all_nan(o[k], f"predict-only B={B}: {k}")
    _bits_equal(o["y"], train["y"], f"predict-only B={B}: y")
    _bits_equal(o["pred"], train["pred"], f"predict-only B={B}: pred")


# ---------------------------------------------------------------------------------------------------------------------
# 2. ctr_l2_loss
# ---------------------------------------------------------------------------------------------------------------------
def _reduce_grid(n):
    return min(max(-(-n // 2048), 1), 1024)


def _l2_depth(n):
    G = _reduce_grid(n)
    return -(-max(n, 1) // (256 * G)) + -(-G // 256) + 28


@pytest.mark.parametrize("n", [0, 1, 255, 257, 1023, 1025, 1_000_003])
def test_l2_loss_against_fp64(n):
    from tf_repos_b200 import ops
    d = _dev()
    g = torch.Generator().manual_seed(n + 1)
    t = (torch.randn(n, generator=g) * 10.0 ** (6 * torch.rand(n, generator=g) - 3)).float()
    ws = torch.empty(1024, dtype=torch.float32, device=d)
    for scale in (3.7e-3, 2.5, 5e-3):
        out = _nan(1)
        ops.l2_loss(t.to(d), out, ws, scale=scale)
        if n == 0:
            _bits_equal(out, torch.zeros(1), f"n=0 scale={scale}: +0")
            continue
        s32 = float(np.float32(scale))
        ref = s32 * (t.double() ** 2).sum().item() / 2
        _within(out, [ref], [gam(_l2_depth(n)) * ref], f"n={n} scale={scale}")


# ---------------------------------------------------------------------------------------------------------------------
# 3. ESMM head: ctr_esmm_head
# ---------------------------------------------------------------------------------------------------------------------
# (y_ctr, y_cvr, y, z): p rounds to 1 with z = 0 (q2 = eps); p = 0 with z = 1 (q1 = eps); pt or pv saturated at 1, at
# 0 (expf overflow) or subnormal; y = 0; z = 1 with y = 0; logits exactly 0
HEAD_ROWS = [(30.0, 30.0, 1.0, 0.0), (0.0, -110.0, 1.0, 1.0), (30.0, 2.0, 1.0, 0.0), (-95.0, 3.0, 1.0, 1.0),
             (16.0, 16.5, 1.0, 1.0), (-88.3, 1.0, 0.0, 0.0), (2.0, -100.0, 0.0, 0.0), (0.0, 0.0, 0.0, 0.0),
             (1.5, -0.5, 0.0, 1.0), (-15.5, 15.5, 0.0, 1.0), (30.0, 30.0, 0.0, 0.0), (-60.0, -60.0, 1.0, 1.0),
             (17.0, -16.0, 1.0, 0.0), (-87.5, -88.0, 0.0, 1.0)]


def _head_inputs(B, seed):
    g = torch.Generator().manual_seed(seed)
    a, c = torch.randn(B, generator=g) * 4, torch.randn(B, generator=g) * 4
    y = (torch.rand(B, generator=g) < 0.4).float()
    z = y * (torch.rand(B, generator=g) < 0.5).float()
    for i in range(0, B, 3):                                  # every third row is a special row, cyclically
        a[i], c[i], y[i], z[i] = HEAD_ROWS[(i // 3) % len(HEAD_ROWS)]
    return a.float(), c.float(), y, z


def _head_run(a, c, y, z, n, w, grads=True, losses=True):
    from tf_repos_b200 import ops
    d = _dev()
    B = a.numel()
    o = dict(pctr=_nan(B), pcvr=_nan(B), pctcvr=_nan(B), losses=_nan(2), d_ctr=_nan(B), d_cvr=_nan(B))
    c_ = lambda t: t.to(d) if t is not None else None
    ops.esmm_head(c_(a), c_(c), c_(y), c_(z), n, w, 1.0 - w, o["pctr"], o["pcvr"], o["pctcvr"],
                  o["losses"] if losses else None, o["d_ctr"] if grads else None, o["d_cvr"] if grads else None)
    return {k: v.cpu() for k, v in o.items()}


HEAD_B = [1, 64, 1023, 1024, 1025, 3000, 8192]


@pytest.mark.parametrize("w", [0.0, 0.3, 0.5, 1.0])
@pytest.mark.parametrize("B", HEAD_B)
def test_esmm_head_against_fp64_and_its_fp32_chain(B, w):
    a, c, y, z = _head_inputs(B, seed=B + int(w * 10))
    eps32 = torch.tensor(eo.LOG_EPS, dtype=torch.float32)
    one = torch.ones((), dtype=torch.float32)
    depth = math.ceil(B / 1024) + 10
    for n in sorted({1, B - 3, B} - {-2, -1, 0}):
        tag = f"B={B} n={n} w={w}"
        o = _head_run(a, c, y, z, n, w)
        pt, pv, p = o["pctr"], o["pcvr"], o["pctcvr"]
        _check_sigmoid(pt, a, f"{tag}: pctr")
        _check_sigmoid(pv, c, f"{tag}: pcvr")
        _bits_equal(p, pt * pv, f"{tag}: pctcvr = fl(pt * pv)")
        ref = eo.head_reference(a[:n], c[:n], y[:n], z[:n], w, 1.0 - w, pt=pt[:n], pv=pv[:n])
        _bits_equal(o["d_ctr"][:n], ref[5], f"{tag}: d_ctr against the fp32 chain")
        _bits_equal(o["d_cvr"][:n], ref[6], f"{tag}: d_cvr against the fp32 chain")
        _bits_equal(o["d_ctr"][n:], torch.zeros(B - n), f"{tag}: d_ctr of rows >= n is +0")
        _bits_equal(o["d_cvr"][n:], torch.zeros(B - n), f"{tag}: d_cvr of rows >= n is +0")
        a64, t64, z64 = a[:n].double().numpy(), y[:n].double().numpy(), z[:n].double().numpy()
        T, A, L = _ce_terms(a64, t64)
        _within(o["losses"][0:1], [T.sum() / n], [(gam(depth + 13) * (A + L).sum() + _sub_exp(a64).sum()) / n],
                f"{tag}: ctr_loss")
        q1 = (p[:n] + eps32).double().numpy()
        q2 = ((one - p[:n]) + eps32).double().numpy()
        l1, l2 = z64 * np.log(q1), (1 - z64) * np.log(q2)
        _within(o["losses"][1:2], [(-l1 - l2).sum() / n], [gam(depth + 5) * (np.abs(l1) + np.abs(l2)).sum() / n],
                f"{tag}: cvr_loss")
    # the regimes are reached (B >= 40 holds every special row below n = B - 3)
    if B >= 64:
        o = _head_run(a, c, y, z, B, w)
        pt, pv, p = o["pctr"], o["pcvr"], o["pctcvr"]
        assert torch.any((p == 1) & (z == 0)) and torch.any((p == 0) & (z == 1))
        assert torch.any(pt == 1) and torch.any(pt == 0) and torch.any(pv == 0) and torch.any((pt > 0) & (pt < TINY))
        assert torch.any(y == 0) and torch.any((z == 1) & (y == 0))


@pytest.mark.parametrize("B", [1, 1025, 3000])
def test_esmm_head_eval_and_inference_write_only_their_outputs(B):
    a, c, y, z = _head_inputs(B, seed=7 * B)
    n = max(B - 3, 1)
    train = _head_run(a, c, y, z, n, 0.3)
    ev = _head_run(a, c, y, z, n, 0.3, grads=False)            # eval: labels, no d_*
    for k in ("pctr", "pcvr", "pctcvr", "losses"):
        _bits_equal(ev[k], train[k], f"eval B={B}: {k}")
    inf = _head_run(a, c, None, None, 0, 0.3)                   # inference: sentinels in losses and d_*
    for k in ("losses", "d_ctr", "d_cvr"):
        _all_nan(inf[k], f"inference B={B}: {k}")
    for k in ("pctr", "pcvr", "pctcvr"):
        _bits_equal(inf[k], train[k], f"inference B={B}: {k}")


# ---------------------------------------------------------------------------------------------------------------------
# 4. ESMM at the reference's configurations: one step against the fp64 oracle
# ---------------------------------------------------------------------------------------------------------------------
FP = 11                 # the README's field count (the flag's default is 0)
N_ESMM = 40_000
LONG_BAG = 517
ESMM_CFGS = {   # name: (K, B, deep_layers, dropout, ctr_task_wgt, learning_rate, l2_reg)
    "flags": (32, 64, "256,128,64", "0.5,0.5,0.5", 0.5, 5e-4, 1e-4),
    "readme": (16, 1024, "256,128", "0.8,0.5", 0.3, 1e-4, 5e-3),
}


def _esmm_batch(B, N, seed):
    """Ali-CCP-like CSR bags: empty bags at the first, a middle and the last sample, bags of length 1, one of
    length 517 with duplicate ids, zero and negative weights; ids 0 and N - 1 in every kind of lookup"""
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(0, 7, (5, B), generator=g)
    lens[1] = torch.randint(0, 30, (B,), generator=g)
    lens[:, 0] = 0; lens[:, B // 2] = 0; lens[:, B - 1] = 0
    lens[0, 1] = 1; lens[4, 3] = 1; lens[1, 2] = LONG_BAG
    off = torch.zeros(5 * B + 1, dtype=torch.int32)
    off[1:] = torch.cumsum(lens.reshape(-1), 0).to(torch.int32)
    nnz = int(off[-1])
    ids = torch.randint(0, N, (nnz,), generator=g, dtype=torch.int32)
    ids[::7] = 0
    ids[3::13] = N - 1
    ids[1::11] = 5                                            # duplicates inside the long bag and others
    wgt = torch.rand(nnz, generator=g) * 3
    wgt[::5] = 0.0
    wgt[2::9] *= -1.0
    feat = torch.randint(0, N, (B, FP), generator=g, dtype=torch.int32)
    feat[0, 0], feat[B - 1, FP - 1] = 0, N - 1
    a_ids = torch.randint(0, N, (3, B), generator=g, dtype=torch.int32)
    a_ids[0, 0], a_ids[2, B - 1] = N - 1, 0
    y = (torch.rand(B, generator=g) < 0.4).float()
    z = y * (torch.rand(B, generator=g) < 0.5).float()
    return {"feat_ids": feat, "a_ids": a_ids, "bag_ids": ids, "bag_wgt": wgt, "bag_off": off}, (y, z)


def _long(batch):
    return {k: (v.long() if k.endswith("ids") else v) for k, v in batch.items()}


def _cuda(batch):
    return {k: v.cuda() for k, v in batch.items()}


def _esmm_masks(cfg, step):
    """independent binary keep masks per tower and layer"""
    K, B, layers, dropout = ESMM_CFGS[cfg][:4]
    g = torch.Generator().manual_seed(900 + step)
    widths, keep = [int(x) for x in layers.split(",")], [float(x) for x in dropout.split(",")]
    cpu = {t: [(torch.rand(B, wd, generator=g) < k).float() for wd, k in zip(widths, keep)] for t in eo.TOWERS}
    return cpu, {t: [m.cuda() for m in ms] for t, ms in cpu.items()}


def _round_to_fp32(params):
    for p in params.values():
        p.copy_(p.float().to(p.dtype))


def _bn_params(ref, g):
    for name, p in ref.params.items():
        if name.endswith("/gamma"):
            p.copy_(1.0 + 0.2 * torch.randn(p.shape, generator=g))
        elif name.endswith("/beta"):
            p.copy_(0.1 * torch.randn(p.shape, generator=g))


def _esmm_oracle(cfg, bn, dtype, mode="exact"):
    K, B, layers, dropout, w, lr, l2 = ESMM_CFGS[cfg]
    ref = eo.ESMM(FP, N_ESMM, K, deep_layers=layers, dropout=dropout, ctr_task_wgt=w, batch_norm=bn,
                  batch_norm_decay=0.9, seed=4, dtype=dtype, l2_reg=l2, learning_rate=lr, optimizer="Adam",
                  update_mode=mode)
    g = torch.Generator().manual_seed(1)
    ref.params["embeddings"].copy_(torch.randn(N_ESMM, K, generator=g) * 0.1)
    _bn_params(ref, g)
    _round_to_fp32(ref.params)
    return ref


def _esmm_gpu(cfg, bn, cap, mode="exact", epoch_steps=8):
    from tf_repos_b200.esmm import ESMM
    K, B, layers, dropout, w, lr, l2 = ESMM_CFGS[cfg]
    return ESMM(FP, N_ESMM, K, B, cap, deep_layers=layers, dropout=dropout, ctr_task_wgt=w, l2_reg=l2,
                learning_rate=lr, optimizer="Adam", update_mode=mode, epoch_steps=epoch_steps, device="cuda:0",
                batch_norm=bn, batch_norm_decay=0.9)


def _tower_tol(din, widths, keep, B, bn):
    """one MLP tower, forward and backward: the GEMMs (R = din, widths; one bias add each), the dropout's /keep (one
    rounding each way where keep is not a power of two), the output dot (+ bias), the dIn products (R = widths), the
    dW products over B rows in fc.cu's split-R chunks (+ their partial adds), fc1's dW (B + 64 adds) and its dIn
    multiply; batch norm's moment and d_gamma / d_beta sums over B rows, gam(B/256 + 100) each way per layer"""
    fwd, bwd, d = 0.0, U, din
    for wd, k in zip(widths, keep):
        rk = 0.0 if math.log2(k).is_integer() else U
        fwd += gemm_rel(d, 1) + rk
        bwd += gemm_rel(wd) + gemm_rel(B, adds=_pick_split(d, wd, B) + 1) + rk
        d = wd
    fwd += gam(d + 1)
    bwd += gam(B + 64)
    bnt = 2 * len(widths) * gam(B // 256 + 100) if bn else 0.0
    return fwd + bwd + bnt


def _tol_esmm(cfg, bn):
    """the bag sums (one multiply and up to LONG_BAG sequential adds), both towers at R = (F'+8)K, the head (two
    sigmoids, gam(6) each, and at most 14 rounded ops of the gradient chain), the one-rounding AddN of the two towers'
    dx and the one-multiply backward of the bag rows"""
    K, B, layers, dropout = ESMM_CFGS[cfg][:4]
    widths, keep = [int(x) for x in layers.split(",")], [float(x) for x in dropout.split(",")]
    return gam(LONG_BAG + 1) + _tower_tol((FP + 8) * K, widths, keep, B, bn) + gam(26) + 2 * U


def _sweep_depth(n):
    from tf_repos_b200 import ops
    sm = ops.sweep_partials_count() // 8
    return -(-n // (4 * 256 * 2 * sm)) + 51


@pytest.mark.parametrize("bn", [False, True])
@pytest.mark.parametrize("cfg", list(ESMM_CFGS))
def test_esmm_reference_config_one_step_against_fp64(cfg, bn):
    K, B, layers, dropout, w, lr, l2 = ESMM_CFGS[cfg]
    ref = _esmm_oracle(cfg, bn, torch.float64)
    batch, labels = _esmm_batch(B, N_ESMM, seed=11)
    nnz = batch["bag_ids"].numel()
    gpu = _esmm_gpu(cfg, bn, nnz + 13)
    gpu.load_variables({**ref.params, **ref.bn_state})
    mc, mg = _esmm_masks(cfg, 0)
    reg = float(ref.reg_loss())
    _, out, _, dgrads = ref.gradients(_long(batch), labels, mc)
    parts = gpu.train_step(_cuda(batch), tuple(l.cuda() for l in labels), masks=mg).cpu()
    gpu.check_ids()
    torch.cuda.synchronize()
    tol = _tol_esmm(cfg, bn)
    tag = f"ESMM {cfg} batch_norm={bn}"
    # logits, probabilities and losses of the step (train-mode forward with the masks, before the update)
    E = {}
    for t in eo.TOWERS:
        yr = out[f"y_{t}"]
        E[t] = tol * float(yr.abs().max())
        _within(gpu.towers[t].y[:B], yr, E[t], f"{tag}: {t} logits")
    pt, pv, P = out["pctr"].numpy(), out["pcvr"].numpy(), out["pctcvr"].numpy()
    dpt, dpv = E["ctr"] / 4 + gam(6) * pt + HALF_SUB, E["cvr"] / 4 + gam(6) * pv + HALF_SUB
    dP = dpt * pv + pt * dpv + dpt * dpv + U * P
    _within(gpu.pctr, pt, dpt, f"{tag}: pctr")
    _within(gpu.pcvr, pv, dpv, f"{tag}: pcvr")
    _within(gpu.pctcvr, P, dP, f"{tag}: pctcvr")
    y64, z64 = labels[0].double().numpy(), labels[1].double().numpy()
    depth = math.ceil(B / 1024) + 10
    T, A, L = _ce_terms(out["y_ctr"].numpy(), y64)
    _within(parts[0:1], [T.mean()], [E["ctr"] + gam(depth + 13) * (A + L).mean()], f"{tag}: ctr_loss")
    # cvr_loss: d log(q)/dp = 1/q, with q = p + eps (z = 1) or 1 - p + eps (z = 0); the kernel's fp32 eps and the
    # rounding of q add |eps32 - eps| and gam(2) q.  Where q <= 2 dP (p within the logit bound of 1 or 0), the
    # kernel's q lies in [eps32 (1 - U), q + dP + eps_err + gam(2)], and log over that interval bounds the term
    q = np.where(z64 == 1, P + eo.LOG_EPS, 1 - P + eo.LOG_EPS)
    lt = -np.log(q)
    eps_err = abs(float(np.float32(eo.LOG_EPS)) - eo.LOG_EPS)
    near = q <= 2 * dP
    wide = np.log((q + dP + eps_err + gam(2)) / (float(np.float32(eo.LOG_EPS)) * (1 - U)))
    per_sample = np.where(near, wide, (dP + eps_err + gam(2) * q) / np.where(near, 1.0, q - dP)) + gam(4) * np.abs(lt)
    _within(parts[1:2], [lt.mean()], [per_sample.mean() + gam(depth + 5) * np.abs(lt).mean()], f"{tag}: cvr_loss")
    _within(parts[2:3], [reg], [gam(_sweep_depth(N_ESMM * K)) * reg], f"{tag}: l2 * l2_loss(embeddings)")
    # every dense gradient
    assert set(dgrads) == set(gpu.dense.grads), (sorted(dgrads), sorted(gpu.dense.grads))
    for name, gref in dgrads.items():
        got = gpu.dense.grads[name].cpu()
        _within(got, gref.reshape(got.shape), tol * gref.abs().max(), f"{tag}: {name}")
    # every per-occurrence row of g_all, scaled per sample by the largest |d x| slice the sample's rows reveal
    per = out["per_occurrence"]
    common, a_rows, occ = per["common"], per["a"], per["occ"]
    off = batch["bag_off"].long()
    bag_of = torch.repeat_interleave(torch.arange(5 * B), off[1:] - off[:-1])
    sample, kind = bag_of % B, bag_of // B
    wgt = torch.where(kind < 4, batch["bag_wgt"].double(), torch.ones(nnz, dtype=torch.float64))
    slice_mag = occ.abs().amax(1) / torch.where(wgt != 0, wgt.abs(), torch.ones_like(wgt))
    S = torch.maximum(common.abs().amax((1, 2)), a_rows.abs().amax((0, 2)))
    S = S.scatter_reduce(0, sample, slice_mag, reduce="amax")
    g_all = gpu.g_all.cpu()
    nf = B * FP + 3 * B
    _within(g_all[:B * FP].reshape(B, FP, K), common, tol * S[:, None, None], f"{tag}: common rows")
    _within(g_all[B * FP:nf].reshape(3, B, K), a_rows, tol * S[None, :, None], f"{tag}: a_* rows")
    _within(g_all[nf:nf + nnz], occ, tol * (S[sample] * wgt.abs())[:, None], f"{tag}: bag occurrence rows")
    assert torch.all(occ[wgt == 0] == 0)
    _bits_equal(g_all[nf + nnz:], torch.zeros(gpu.n_total - nf - nnz, K), f"{tag}: capacity slots past nnz")


# ---------------------------------------------------------------------------------------------------------------------
# 5. DeepMVM at the reference's configurations: one step against the fp64 oracle
# ---------------------------------------------------------------------------------------------------------------------
F39 = 39
N_MVM = 20_000
MVM_CFGS = {   # name: (K, B, deep_layers, dropout, learning_rate, l2_reg)
    "flags": (32, 64, "256,128,64", "0.5,0.5,0.5", 5e-4, 1e-4),
    "run_sh": (32, 256, "256,128", "0.8,0.8", 1e-4, 1e-4),
}


def _mvm_oracle(cfg, init, dtype, mode="exact", bn=False):
    K, B, layers, dropout, lr, l2 = MVM_CFGS[cfg]
    ref = OracleDeepMVM(F39, N_MVM, K, deep_layers=layers, dropout=dropout, batch_norm=bn, batch_norm_decay=0.9,
                        seed=5, dtype=dtype, l2_reg=l2, learning_rate=lr, optimizer="Adam", update_mode=mode)
    g = torch.Generator().manual_seed(9)
    if init == "o1":            # factors +-[0.9, 1.1]: the product term is not negligible
        sign = torch.where(torch.rand(F39, K, generator=g) < 0.5, -1.0, 1.0)
        ref.params["mvm_b"].copy_(sign * (0.9 + 0.2 * torch.rand(F39, K, generator=g)))
        ref.params["mvm_w"].copy_(torch.randn(N_MVM, K, generator=g) * 0.02)
    _bn_params(ref, g)
    _round_to_fp32(ref.params)
    return ref


def _mvm_gpu(cfg, mode="exact", epoch_steps=8, bn=False):
    from tf_repos_b200.deepmvm import DeepMVM
    K, B, layers, dropout, lr, l2 = MVM_CFGS[cfg]
    return DeepMVM(F39, N_MVM, K, B, deep_layers=layers, dropout=dropout, l2_reg=l2, learning_rate=lr,
                   optimizer="Adam", update_mode=mode, epoch_steps=epoch_steps, device="cuda:0", batch_norm=bn,
                   batch_norm_decay=0.9)


def _mvm_batch(cfg, step):
    from tf_repos_b200 import synth
    K, B = MVM_CFGS[cfg][:2]
    ids, vals, labels = synth.criteo_batch(B, N_MVM, F39, seed=600 + step)
    ids[0, F39 - 1], ids[B - 1, F39 - 1] = 0, N_MVM - 1
    return ids, vals, labels


def _mvm_masks(cfg, step):
    K, B, layers, dropout = MVM_CFGS[cfg][:4]
    g = torch.Generator().manual_seed(800 + step)
    cpu = [(torch.rand(B, int(wd), generator=g) < float(k)).float()
           for wd, k in zip(layers.split(","), dropout.split(","))]
    return cpu, [m.cuda() for m in cpu]


def _tol_mvm(cfg):
    """K1's one multiply, the product and its backward (gam(3F) each), the deep part as one tower at R = FK with the
    output dot over [x_mvm, h] (K more terms), the logit / sigmoid-CE stages (8U), d_e = da + dX and g_rows = d_e * val
    (one rounding each), and mvm_b's batch sum of da (per-thread rows, the CTA's rows and the CTAs: B + 16 adds)"""
    K, B, layers, dropout = MVM_CFGS[cfg][:4]
    widths, keep = [int(x) for x in layers.split(",")], [float(x) for x in dropout.split(",")]
    return (U + 2 * gam(3 * F39) + _tower_tol(F39 * K, widths, keep, B, False) + gam(K) + 8 * U + 2 * U
            + gam(B + 16))


@pytest.mark.parametrize("init", ["glorot", "o1"])
@pytest.mark.parametrize("cfg", list(MVM_CFGS))
def test_deepmvm_reference_config_one_step_against_fp64(cfg, init):
    K, B, layers, dropout, lr, l2 = MVM_CFGS[cfg]
    ref = _mvm_oracle(cfg, init, torch.float64)
    gpu = _mvm_gpu(cfg)
    gpu.load_variables(ref.params)
    ids, vals, labels = _mvm_batch(cfg, 0)
    mc, mg = _mvm_masks(cfg, 0)
    wv, bv = ref.params["mvm_w"], ref.params["mvm_b"]
    reg_w, reg_b = l2 * float((wv ** 2).sum()) / 2, l2 * float((bv ** 2).sum()) / 2
    ref.l2_reg = 0.0               # the oracle then returns mvm_b's data gradient alone, as dense.grads holds it
    _, out, _, dgrads = ref.gradients({"feat_ids": ids.long(), "feat_vals": vals}, labels, mc)
    parts = gpu.train_step(ids.cuda(), vals.cuda(), labels.cuda(), masks=mg).cpu()
    gpu.check_ids()
    torch.cuda.synchronize()
    tol = _tol_mvm(cfg)
    tag = f"DeepMVM {cfg} init={init}"
    xm = out["x_mvm"]
    if init == "o1":
        assert xm.abs().median() > 1e-3, f"{tag}: the product term is negligible"
    # x_mvm per element: gam(3F) prod M plus the subnormal products' 2^-150 times their trailing factors
    e = wv[ids.long()] * vals.double()[..., None]
    M = e.abs() + bv.abs()                                        # [B, F, K]
    suffix = torch.flip(torch.cumprod(torch.flip(M[:, 1:], [1]), 1), [1])   # prod_{g >= f} M_g, f = 1..F-1
    uf = HALF_SUB * (torch.cat([suffix[:, 1:], torch.ones(B, 1, K, dtype=M.dtype)], 1)).sum(1) * (1 + gam(3 * F39))
    _within(gpu.x_mvm[:B], xm, gam(3 * F39) * M.prod(1) + uf, f"{tag}: x_mvm")
    # logits: per sample, the product term's magnitude through deep_out plus the batch's largest logit
    w_out = ref.params["DeepMVM-out/deep_out/weights"][:K, 0].abs()
    y = out["y"]
    E_y = tol * ((M.prod(1) * w_out).sum(1) + y.abs().max()) + (uf * w_out).sum(1)
    _within(gpu.y[:B], y, E_y, f"{tag}: logits")
    depth = math.ceil(B / 1024) + 10
    T, A, L = _ce_terms(y.numpy(), labels.double().numpy())
    _within(parts[0:1], [T.mean()], [E_y.mean().item() + gam(depth + 14) * (A + L).mean()], f"{tag}: CE")
    _within(parts[1:2], [reg_w], [gam(_sweep_depth(N_MVM * K)) * reg_w], f"{tag}: l2 * l2_loss(mvm_w)")
    _within(parts[2:3], [reg_b], [gam(_l2_depth(F39 * K) + 1) * reg_b], f"{tag}: l2 * l2_loss(mvm_b)")
    # every dense gradient; mvm_b's batch sum of da adds each subnormal product's 2^-150 times at most
    # C = max(1, max M)^F max(1, max |deep_out weights|) per rounding, 2F roundings per sample
    assert set(dgrads) == set(gpu.dense.grads), (sorted(dgrads), sorted(gpu.dense.grads))
    C = max(1.0, float(M.max())) ** F39 * max(1.0, float(w_out.max()))
    for name, gref in dgrads.items():
        got = gpu.dense.grads[name].cpu()
        extra = B * 2 * F39 * HALF_SUB * C if name == "mvm_b" else 0.0
        _within(got, gref.reshape(got.shape), tol * gref.abs().max() + extra, f"{tag}: {name}")
    gv = out["per_occurrence"]["emb"].reshape(B, F39 * K)
    _within(gpu.g_rows[:B * F39].cpu().reshape(B, F39 * K), gv, tol * gv.abs().amax(1, keepdim=True),
            f"{tag}: per-occurrence g_rows")


# ---------------------------------------------------------------------------------------------------------------------
# 6. Three steps against the fp32 oracle, and bit reproducibility
# ---------------------------------------------------------------------------------------------------------------------
# Variables that need more than 2e-5 against the fp32 oracle, at twice the largest ratio measured over three steps
# in every update mode of the test (H100 SXM, 700 W).  As in test_gpu_fm_batch_norm.py: Adam's first steps move an
# element by about lr * g / |g| whatever its size, so an element whose gradient nearly cancels (sums over the
# dropout-masked batch, batch norm's d_x, the first layer's bias summed over B = 1024 rows) moves by up to lr in a
# direction set by the last bits of g, which the two fp32 implementations round differently; the biases start at 0,
# so that step is a large part of their scale after three steps.  The fp64 one-step tests above pin those gradients
# themselves.  Measured: ESMM flags with batch norm ctr_mlp1/weights 1.03e-4, cvr_mlp0/weights 5.6e-5,
# ctr_mlp0/weights 4.6e-5, embeddings 3.9e-5 (lazy), ctr_mlp2/weights 3.1e-5; ESMM readme cvr_mlp0/biases 6.8e-4,
# embeddings 1.5e-4, cvr_mlp0/weights 8.3e-5 (all three lazy); ESMM readme with batch norm cvr_mlp0/biases 9.5e-4,
# cvr_mlp1/biases 7.6e-5; DeepMVM flags at the glorot initialisation mvm_w 2.2e-5.
FP32_DEVIATIONS = {
    ("esmm", "flags", True): {"ctr_mlp1/weights": 2.1e-4, "cvr_mlp0/weights": 1.2e-4, "ctr_mlp0/weights": 1e-4,
                              "embeddings": 8e-5, "ctr_mlp2/weights": 7e-5},
    ("esmm", "readme", False): {"cvr_mlp0/biases": 1.4e-3, "embeddings": 3.1e-4, "cvr_mlp0/weights": 1.7e-4},
    ("esmm", "readme", True): {"cvr_mlp0/biases": 1.9e-3, "cvr_mlp1/biases": 1.6e-4},
    ("deepmvm", "flags", "glorot"): {"mvm_w": 4.5e-5},
}


def _fp32_worst(ref, gpu, worst):
    vs = gpu.variables()
    for name, want in list(ref.params.items()) + list(ref.bn_state.items()):
        got, want = vs[name].cpu().double().numpy().reshape(want.shape), want.double().numpy()
        worst[name] = max(worst.get(name, 0.0), _excess(got, want))


def _assert_fp32(worst, key, what):
    tol = {**{k: 2e-5 for k in worst}, **FP32_DEVIATIONS.get(key, {})}
    bad = {k: v for k, v in worst.items() if v > tol[k]}
    assert not bad, f"{what}: {bad}; all: {worst}"


@pytest.mark.parametrize("mode", ["exact", "exact_deferred", "lazy"])
@pytest.mark.parametrize("bn", [False, True])
@pytest.mark.parametrize("cfg", list(ESMM_CFGS))
def test_esmm_reference_config_three_steps_match_the_fp32_oracle(cfg, bn, mode):
    B = ESMM_CFGS[cfg][1]
    ref = _esmm_oracle(cfg, bn, torch.float32, mode="lazy" if mode == "lazy" else "exact")
    batches = [_esmm_batch(B, N_ESMM, seed=30 + s) for s in range(3)]
    gpu = _esmm_gpu(cfg, bn, max(b["bag_ids"].numel() for b, _ in batches), mode, epoch_steps=2)
    gpu.load_variables({**ref.params, **ref.bn_state})
    worst = {}
    for step, (batch, labels) in enumerate(batches):
        mc, mg = _esmm_masks(cfg, step)
        ref.train_step(_long(batch), labels, mc)
        gpu.train_step(_cuda(batch), tuple(l.cuda() for l in labels), masks=mg)
        gpu.check_ids()
        _fp32_worst(ref, gpu, worst)
    _assert_fp32(worst, ("esmm", cfg, bn), f"ESMM {cfg} ({mode}, batch_norm={bn})")


@pytest.mark.parametrize("mode", ["exact", "exact_deferred"])
@pytest.mark.parametrize("init", ["glorot", "o1"])
@pytest.mark.parametrize("cfg", list(MVM_CFGS))
def test_deepmvm_reference_config_three_steps_match_the_fp32_oracle(cfg, init, mode):
    ref = _mvm_oracle(cfg, init, torch.float32)
    gpu = _mvm_gpu(cfg, mode, epoch_steps=2)
    gpu.load_variables(ref.params)
    worst = {}
    for step in range(3):
        ids, vals, labels = _mvm_batch(cfg, 10 + step)
        mc, mg = _mvm_masks(cfg, 10 + step)
        ref.train_step({"feat_ids": ids.long(), "feat_vals": vals}, labels, mc)
        gpu.train_step(ids.cuda(), vals.cuda(), labels.cuda(), masks=mg)
        gpu.check_ids()
        _fp32_worst(ref, gpu, worst)
    _assert_fp32(worst, ("deepmvm", cfg, init), f"DeepMVM {cfg} init={init} ({mode})")


def _state(m, rows):
    m.flush()
    out = [m.V.var] + list(m.V.slots) + [m.dense.flat] + list(m.dense.slots) + [m.dense.grad, rows]
    return [t.clone() for t in out] + [v.clone() for v in m.variables().values()]


@pytest.mark.parametrize("cfg", list(ESMM_CFGS))
def test_esmm_with_masks_and_batch_norm_is_bit_reproducible(cfg):
    B = ESMM_CFGS[cfg][1]
    ref = _esmm_oracle(cfg, True, torch.float32)
    batches = [_esmm_batch(B, N_ESMM, seed=50 + s) for s in range(3)]
    cap = max(b["bag_ids"].numel() for b, _ in batches)
    states = []
    for _ in range(2):
        m = _esmm_gpu(cfg, True, cap)
        m.load_variables({**ref.params, **ref.bn_state})
        for step, (batch, labels) in enumerate(batches):
            m.train_step(_cuda(batch), tuple(l.cuda() for l in labels), masks=_esmm_masks(cfg, 20 + step)[1])
        states.append(_state(m, m.g_all))
    for x, y in zip(*states):
        _bits_equal(y, x, f"ESMM {cfg}: two fresh models")


@pytest.mark.parametrize("cfg", list(MVM_CFGS))
def test_deepmvm_with_masks_and_batch_norm_is_bit_reproducible(cfg):
    ref = _mvm_oracle(cfg, "o1", torch.float32, bn=True)
    states = []
    for _ in range(2):
        m = _mvm_gpu(cfg, bn=True)
        m.load_variables(ref.params)
        for step in range(3):
            ids, vals, labels = _mvm_batch(cfg, 20 + step)
            m.train_step(ids.cuda(), vals.cuda(), labels.cuda(), masks=_mvm_masks(cfg, 20 + step)[1])
        states.append(_state(m, m.g_rows))
    for x, y in zip(*states):
        _bits_equal(y, x, f"DeepMVM {cfg}: two fresh models")
