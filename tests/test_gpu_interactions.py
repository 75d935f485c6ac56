"""PNN's product, AFM's pairwise-attention and DCN's cross kernels (csrc/pairwise.cu, csrc/cross.cu) and the N = 1 output
layer (fc1) against fp64 references or exact fp32 restatements, at the reference's default shapes and across their
dispatch space; then AFM, PNN (Inner) and DCN at the reference's default configurations against the oracle.

Defaults (F = 39 Criteo fields): AFM K=256, attention_layers=256, dropout=1.0,0.5, l2_reg=1.0, Adam lr 0.1, B=128, so
P = 741 pairs and B*P = 94,848 attention rows; PNN Inner K=32, deep_layers=256,128,64, dropout 0.5, B=64 (MLP input
39*32 + 741 = 1989); DCN K=32 (D = 1248), cross_layers=3, deep_layers=256,128,64, dropout 0.5, B=64.

Error bounds (each comparison states which one and why):
  U          = 2^-24: unit roundoff of one round-to-nearest fp32 operation.
  gam(n)     = n*U / (1 - n*U): the classic bound for a chain of n rounded fp32 operations (adds or fmaf) whose partial
               sums are each bounded by sum|terms|; the bound is gam(n) * sum|terms| (a magnitude the test computes in
               fp64 per element).  fmaf(0, 0, s) is exact, so padded lanes add no rounding.
  pnn inner  z tail: one fmaf chain of K products from 0 -> gam(K) * sum_k |e_i e_j|.
  pnn dX     inner: F-1 fmafs then the add of dz -> gam(F) * (sum_o |dz_p e_o| + |dz_x|);
             outer: (F-1)*K fmafs then the add -> gam((F-1)*K + 1) * (sum |d e| + |dz_x|).
  afm dX     F-1 fmafs from 0 -> gam(F-1) * sum_o |dpw e_o|.
  softmax    m = max is exact; arg = fl(lg - m) has a relative error U, i.e. e^arg moves by a factor e^(U|arg|);
             CUDA expf is within 2 ulp (4U relative) -> eps_p = 4U + U|arg_p| (+ first-order products).  The sum runs
             ceil(P/256) per-thread adds then an 8-level tree: rel. eps_s = max_p eps_p + gam(ceil(P/256) + 8);
             att = ex/s rounds once more: |att - a| <= a (eps_p + eps_s + U) (x 1.01 for the second-order terms),
             plus 2^-126 absolute where e^arg is below the normal range (flushed or denormal; s >= 1).
  SUB        = 2^-149: below 2^-126 (where tiny attention weights put w*pw, da*att and att*(da - s)) the relative
             bound no longer holds; each rounding there errs by at most SUB/2 absolute, so those bounds add SUB per
             rounding (P for y_emb, ceil(P/256) + 8 for s, 3 for dlogit).
  y_emb      from the GPU's own att: w = fl(fl(att/keep) * mask) restated exactly, then P fmafs -> gam(P) sum|w pw|.
  dlogit     from the GPU's own att: dot = pw.dy is K fmafs (gam(K) S, S = sum|pw dy|), da = fl(dot*mask/keep) one
             more U; s = sum da*att is ceil(P/256) + 8 chained roundings; dlogit = att*(da - s) two roundings.  It
             cancels, so it is bounded relative to att*(|da| + |s|), never relative to |dlogit|.
  cross      x_L is restated exactly with the kernel's own s; s_l is a per-lane fmaf chain of 4*NV products plus 5
             shuffle adds -> gam(4 NV + 5) sum|x_l w_l|.  The backward is recomputed in fp64 along the same recursion
             (g_L = dxL; ds = g.x0; db_l += g; dw_l += ds x_l; dx0 += g s_l; g += ds w_l) with a running first-order
             absolute error bound eg / eds carried alongside; dw/db accumulate m = ceil(B/n_warps) samples per warp
             slab and then n_warps partials in order -> gam(m + n_warps); dx0 = L fmafs + 2 adds -> gam(L + 2).
  fc1        y: ceil(Ka/32) + ceil(Kb/32) fmafs, 5 shuffle adds, + b -> gam(n + 6); dw/db: a chain of <= 64 rows per
             chunk, then colsum_rows (ceil(chunks/8) adds per row group, 8 more) -> gam(64 + ceil(chunks/8) + 8).
  gemm_rel   as in test_gpu_din_attention.py: a 3xTF32 product over a reduction of length R, then
             `adds` rounded fp32 additions, relative to |A|@|B| + |addends|.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TRUNC = 2.0 ** -23
SPLIT = 3 * 2.0 ** -21
TINY = 2.0 ** -126
SUB = 2.0 ** -149    # the subnormal spacing: a rounding whose result is below 2^-126 errs by up to SUB/2


def gam(n):
    return n * U / (1 - n * U)


def gemm_rel(R, adds=0):
    return SPLIT + (9 / 8 * R * (1 + 2.0 ** -9) + adds + 1) * TRUNC


def _dev():
    return torch.device("cuda:0")


def _np(t):
    return t.detach().cpu().double().numpy() if torch.is_tensor(t) else np.asarray(t, dtype=np.float64)


def _within(got, ref, bound, what):
    """|got - ref| <= bound elementwise (bound already holds the derivation's scale)."""
    got, ref, bound = _np(got), _np(ref), np.broadcast_to(_np(bound), np.shape(_np(ref)))
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert np.all(np.isfinite(got)), f"{what}: non-finite output"
    err = np.abs(got - ref)
    bad = err > bound
    if bad.any():
        i = np.unravel_index(np.argmax(np.where(bad, err / np.maximum(bound, 1e-300), 0)), err.shape)
        raise AssertionError(f"{what}: {int(bad.sum())} of {err.size} elements outside the bound; worst at {i}: "
                             f"got {got[i]!r} ref {ref[i]!r} err {err[i]:.3e} bound {bound[i]:.3e}")


def _bits_equal(a, b, what):
    a = a.detach().cpu().contiguous().view(torch.int32)
    b = b.detach().cpu().contiguous().view(torch.int32)
    if not torch.equal(a, b):
        n = int((a != b).sum())
        raise AssertionError(f"{what}: {n} of {a.numel()} elements differ in their bits")


def _sm_count():
    from tf_repos_b200 import _lib
    return int(_lib.raw().ctr_device_sm_count())


def _pairs(F):
    row, col = [], []
    for i in range(F - 1):                  # PNN.py:144-147, AFM.py:134-136: i < j, row-major
        for j in range(i + 1, F):
            row.append(i); col.append(j)
    return torch.tensor(row, dtype=torch.long), torch.tensor(col, dtype=torch.long)


def _rejected(call, outs, what):
    """call() raises CtrError, launches nothing and leaves the sentinel-filled outputs as they were."""
    from tf_repos_b200 import _lib
    from tf_repos_b200._lib import CtrError
    before = [o.clone() for o in outs]
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    with pytest.raises(CtrError):
        call()
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0, f"{what}: a rejected call launched a kernel"
    for o, b in zip(outs, before):
        _bits_equal(o, b, f"{what}: a rejected call wrote an output")


# ---------------------------------------------------------------------------------------------------------------------
# pnn_product_fwd / _bwd: z = [x | inner (P) or outer (P*K*K)] and dX (PNN.py:141-167)
# ---------------------------------------------------------------------------------------------------------------------
PNN_B = (1, 3, 5, 64, 4097)         # only 64 is a multiple of the 4 warps (samples) per CTA
OUTER_TAIL_MAX = 1 << 16            # outer runs where P*K*K stays small


def _pnn_case(B, F, K, outer, g):
    from tf_repos_b200 import ops
    d = _dev()
    P = F * (F - 1) // 2
    FK = F * K
    row, col = _pairs(F)
    x = torch.randn(B, F, K, generator=g) * torch.exp(torch.randn(B, F, 1, generator=g))
    x = x.reshape(B, FK).contiguous()
    ld = FK + (P * K * K if outer else P)
    z = torch.full((B, ld), float("nan"), device=d)
    xd = x.to(d)
    ops.pnn_product_fwd(xd, B, F, K, outer, z)
    zc = z.cpu()
    what = f"B={B} F={F} K={K} outer={outer}"
    _bits_equal(zc[:, :FK], x, f"pnn fwd copy of x {what}")
    e = x.view(B, F, K)
    e64 = e.double()
    if outer:
        # e_i[a] * e_j[c]: one rounded fp32 multiply per element
        _bits_equal(zc[:, FK:], (e[:, row, :, None] * e[:, col, None, :]).reshape(B, -1), f"pnn outer tail {what}")
    else:
        G = e64 @ e64.transpose(1, 2)
        Ga = e64.abs() @ e64.abs().transpose(1, 2)
        _within(zc[:, FK:], G[:, row, col], gam(K) * Ga[:, row, col], f"pnn inner tail {what}")
    dz = torch.randn(B, ld, generator=g)
    dX = torch.full((B, FK), float("nan"), device=d)
    ops.pnn_product_bwd(xd, dz.to(d), B, F, K, outer, dX)
    dz64 = dz.double()
    dzx = dz64[:, :FK].view(B, F, K)
    if outer:
        dt = dz64[:, FK:].view(B, P, K, K)                 # dt[a, c] multiplies e_i[a] * e_j[c]
        gi = torch.einsum("bpac,bpc->bpa", dt, e64[:, col])
        gj = torch.einsum("bpac,bpa->bpc", dt, e64[:, row])
        mi = torch.einsum("bpac,bpc->bpa", dt.abs(), e64[:, col].abs())
        mj = torch.einsum("bpac,bpa->bpc", dt.abs(), e64[:, row].abs())
        ref = dzx.clone().index_add_(1, row, gi).index_add_(1, col, gj)
        mag = dzx.abs().index_add_(1, row, mi).index_add_(1, col, mj)
        bound = gam((F - 1) * K + 1) * mag
    else:
        Dm = torch.zeros(B, F, F, dtype=torch.float64)
        Dm[:, row, col] = dz64[:, FK:]
        Dm[:, col, row] = dz64[:, FK:]
        ref = dzx + Dm @ e64
        bound = gam(F) * (dzx.abs() + Dm.abs() @ e64.abs())
    _within(dX.cpu().view(B, F, K), ref, bound, f"pnn dX {what}")


@pytest.mark.parametrize("K", [1, 3, 4, 10, 16, 32, 64, 128])
@pytest.mark.parametrize("F", [2, 3, 13, 39])
def test_pnn_product_fwd_bwd(F, K):
    """Inner at every B; outer where its tail is small.  F=39 with K=64 and 128 puts the bwd kernel's
    2 * 4 * F * (K+1) floats above 48 KB, on the opt-in shared-memory path."""
    g = torch.Generator().manual_seed(F * 1000 + K)
    P = F * (F - 1) // 2
    for B in PNN_B:
        _pnn_case(B, F, K, False, g)
    if P * K * K <= OUTER_TAIL_MAX:
        for B in PNN_B:
            if B * P * K * K <= 1 << 24:
                _pnn_case(B, F, K, True, g)


def test_pnn_product_shared_memory_limits():
    """fwd stages 4 warps x F x (K+1) floats, bwd twice that, up to 200 KB: at F = 39 fwd takes K <= 327 and bwd
    K <= 163.  The largest accepted K computes correctly; the smallest rejected one raises and launches nothing."""
    from tf_repos_b200 import ops
    F, B = 39, 5
    kf = 200 * 1024 // (4 * F * 4) - 1
    kb = 200 * 1024 // (2 * 4 * F * 4) - 1
    assert (kf, kb) == (327, 163)
    g = torch.Generator().manual_seed(7)
    d = _dev()
    P = F * (F - 1) // 2
    for K in (kb, kf):                       # fwd at both (bwd at kb): checked against fp64
        x = torch.randn(B, F * K, generator=g)
        z = torch.full((B, F * K + P), float("nan"), device=d)
        ops.pnn_product_fwd(x.to(d), B, F, K, False, z)
        e64 = x.double().view(B, F, K)
        row, col = _pairs(F)
        G = e64 @ e64.transpose(1, 2)
        Ga = e64.abs() @ e64.abs().transpose(1, 2)
        _within(z.cpu()[:, F * K:], G[:, row, col], gam(K) * Ga[:, row, col], f"pnn fwd at K={K}")
    _pnn_case(B, F, kb, False, g)
    ops.pnn_product_check(F, kb, False)
    for K, which in ((kf + 1, "fwd"), (kb + 1, "bwd")):
        x = torch.randn(B, F * K, device=d)
        ld = F * K + P
        if which == "fwd":
            z = torch.full((B, ld), 3.0, device=d)
            _rejected(lambda: ops.pnn_product_fwd(x, B, F, K, False, z), [z], f"pnn fwd K={K}")
        else:
            dz = torch.randn(B, ld, device=d)
            dX = torch.full((B, F * K), 3.0, device=d)
            _rejected(lambda: ops.pnn_product_bwd(x, dz, B, F, K, False, dX), [dX], f"pnn bwd K={K}")
    # fwd alone still takes K = kb + 1 .. kf
    z = torch.full((B, F * (kb + 1) + P), float("nan"), device=d)
    ops.pnn_product_fwd(torch.randn(B, F * (kb + 1), device=d), B, F, kb + 1, False, z)
    assert torch.isfinite(z).all()


# ---------------------------------------------------------------------------------------------------------------------
# afm_pairs_fwd / _bwd: pw[b,p,:] = e_i * e_j (AFM.py:132-138) and dX
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,F,K", [(128, 39, 256), (1000, 10, 64), (3, 2, 1), (7, 13, 5)])
def test_afm_pairs_fwd_bwd(B, F, K):
    from tf_repos_b200 import ops
    d = _dev()
    P = F * (F - 1) // 2
    threads = _sm_count() * 16 * 256        # ew_grid's cap: sm_count * 16 CTAs of 256 threads
    if B >= 128:                            # these two shapes run both grid-stride loops more than once per thread
        assert B * P * K > threads and B * F * K > threads
    g = torch.Generator().manual_seed(B + F + K)
    x = torch.randn(B, F * K, generator=g)
    xd = x.to(d)
    pw = torch.full((B * P, K), float("nan"), device=d)
    ops.afm_pairs_fwd(xd, B, F, K, pw)
    row, col = _pairs(F)
    e = x.view(B, F, K)
    _bits_equal(pw, (e[:, row] * e[:, col]).reshape(B * P, K), f"pw B={B} F={F} K={K}")
    dpw = torch.randn(B * P, K, generator=g)
    dX = torch.full((B, F * K), float("nan"), device=d)
    ops.afm_pairs_bwd(xd, dpw.to(d), B, F, K, dX)
    dXc = dX.cpu().view(B, F, K)
    for b0 in range(0, B, 32):              # fp64 reference in slices of samples (the default shape is 24 M products)
        e64 = e[b0:b0 + 32].double()
        d3 = dpw.view(B, P, K)[b0:b0 + 32].double()
        ref = torch.zeros_like(e64).index_add_(1, row, d3 * e64[:, col]).index_add_(1, col, d3 * e64[:, row])
        mag = torch.zeros_like(e64).index_add_(1, row, (d3 * e64[:, col]).abs()).index_add_(1, col, (d3 * e64[:, row]).abs())
        _within(dXc[b0:b0 + 32], ref, gam(F - 1) * mag, f"afm dX B={B} F={F} K={K} from sample {b0}")


# ---------------------------------------------------------------------------------------------------------------------
# afm_pool_fwd / _bwd: att = softmax_p(logit), w = dropout(att), y_emb = sum_p w_p pw_p (AFM.py:151-156) and backward
# ---------------------------------------------------------------------------------------------------------------------
def _pool_logits(P, g):
    """sample 0: N(0,1); 1: N(0,1)*30; 2: one logit 100 above the rest; 3: all equal; 4: N(0,1) (zero mask)"""
    lg = torch.randn(5, P, generator=g)
    lg[1] *= 30
    lg[2, P // 3] = lg[2].max() + 100
    lg[3] = 0.37
    return lg


@pytest.mark.parametrize("K", [1, 4, 255, 256, 257, 512])
@pytest.mark.parametrize("P", [1, 2, 255, 256, 257, 741, 10240])
def test_afm_pool_fwd_bwd(P, K):
    from tf_repos_b200 import ops
    d = _dev()
    B = 5
    g = torch.Generator().manual_seed(P * 7 + K)
    lg = _pool_logits(P, g)
    pw = torch.randn(B, P, K, generator=g)
    dy = torch.randn(B, K, generator=g)
    pwd, lgd, dyd = pw.to(d), lg.reshape(-1).to(d), dy.to(d)
    # att against the fp64 softmax of the same fp32 logits
    l64 = lg.double()
    arg = l64 - l64.max(1, keepdim=True).values
    ex = torch.exp(arg)
    a_ref = ex / ex.sum(1, keepdim=True)
    eps_p = 4 * U + U * arg.abs()
    eps_s = eps_p.max(1, keepdim=True).values + gam(-(-P // 256) + 8)
    att_bound = a_ref * (eps_p + eps_s + U) * 1.01 + TINY
    n_s = -(-P // 256) + 8
    one_over_p = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(P), dtype=torch.float32)
    results = {}
    for keep in (0.5, 0.8, 1.0):
        masks = [None] if keep == 1.0 else []
        mask = (torch.rand(B, P, generator=g) < keep).float()
        mask[4] = 0.0                                        # sample 4: every weight dropped
        masks.append(torch.ones(B, P) if keep == 1.0 else mask)
        for mk in masks:
            what = f"P={P} K={K} keep={keep} mask={'none' if mk is None else 'ones' if keep == 1.0 else 'random'}"
            att = torch.full((B * P,), float("nan"), device=d)
            y = torch.full((B, K), float("nan"), device=d)
            mkd = mk.reshape(-1).to(d) if mk is not None else None
            ops.afm_pool_fwd(pwd, lgd, mkd, keep, B, P, K, att, y)
            ac = att.cpu().view(B, P)
            _within(ac, a_ref, att_bound, f"att {what}")
            assert torch.all(ac[3] == one_over_p), f"att with all logits equal must be fl(1/P) ({what})"
            # y_emb from the GPU's own att: w restated exactly, then P fmafs
            w = ac if mk is None else (ac / keep) * mk
            w64 = w.double()
            y_ref = torch.bmm(w64.unsqueeze(1), pw.double()).squeeze(1)
            y_mag = torch.bmm(w64.abs().unsqueeze(1), pw.double().abs()).squeeze(1)
            yc = y.cpu()
            _within(yc, y_ref, gam(P) * y_mag + P * SUB, f"y_emb {what}")
            # backward
            dpw = torch.full((B * P, K), float("nan"), device=d)
            dlg = torch.full((B * P,), float("nan"), device=d)
            ops.afm_pool_bwd(pwd, att, mkd, keep, dyd, B, P, K, dpw, dlg)
            _bits_equal(dpw.cpu().view(B, P, K), w.unsqueeze(2) * dy.unsqueeze(1), f"dpw {what}")
            a = ac.double()
            dot = torch.bmm(pw.double(), dy.double().unsqueeze(2)).squeeze(2)
            S = torch.bmm(pw.double().abs(), dy.double().abs().unsqueeze(2)).squeeze(2)
            if mk is None:
                da, eda = dot, gam(K) * S
            else:
                m64 = mk.double()
                da = dot * m64 / keep
                eda = gam(K) * S * m64 / keep + U * da.abs()
            s = (da * a).sum(1, keepdim=True)
            es = (a * eda).sum(1, keepdim=True) + gam(n_s) * (a * (da.abs() + eda)).sum(1, keepdim=True) + n_s * SUB
            dl_ref = a * (da - s)
            dl_bound = (a * (eda + es) + 2 * U * a * (da.abs() + s.abs())) * 1.01 + 3 * SUB
            dlc = dlg.cpu().view(B, P)
            _within(dlc, dl_ref, dl_bound, f"dlogit {what}")
            if mk is not None and keep < 1.0:
                assert torch.all(yc[4] == 0) and torch.all(dpw.cpu().view(B, P, K)[4] == 0) and torch.all(dlc[4] == 0), \
                    f"an all-zero mask must give y_emb = 0, dpw = 0, dlogit = 0 ({what})"
            if keep == 1.0:
                results.setdefault("k1", []).append((att.cpu(), yc, dpw.cpu(), dlc))
    none, ones = results["k1"]
    for u, v, nm in zip(none, ones, ("att", "y_emb", "dpw", "dlogit")):
        _bits_equal(v, u, f"{nm}: mask=None vs an all-ones mask at keep=1 (P={P} K={K})")


def test_afm_pool_pair_limit():
    """P <= 10240 (the [P] weights live in 40 KB of dynamic shared memory); P = 10241 is rejected before any launch."""
    from tf_repos_b200 import ops
    d = _dev()
    B, K = 2, 4
    ops.afm_pool_check(10240, K)
    P = 10241
    pw = torch.randn(B * P, K, device=d)
    lg = torch.randn(B * P, device=d)
    att = torch.full((B * P,), 3.0, device=d)
    y = torch.full((B, K), 3.0, device=d)
    _rejected(lambda: ops.afm_pool_fwd(pw, lg, None, 1.0, B, P, K, att, y), [att, y], "afm_pool_fwd P=10241")
    dpw = torch.full((B * P, K), 3.0, device=d)
    dlg = torch.full((B * P,), 3.0, device=d)
    _rejected(lambda: ops.afm_pool_bwd(pw, att, None, 1.0, y, B, P, K, dpw, dlg), [dpw, dlg], "afm_pool_bwd P=10241")


# ---------------------------------------------------------------------------------------------------------------------
# cross_fwd / cross_bwd: x_{l+1} = x0 * (x_l . w_l) + x_l + b_l (DCN.py:140-145) and its backward
# ---------------------------------------------------------------------------------------------------------------------
def _nv(D):
    return -(-(D // 4) // 32)


def _wpc(D, L):
    """cross.cu bwd_warps_per_cta: per-warp slab of 2*L*D floats within 200 KB, at most 4 warps"""
    return min(4, 200 * 1024 // (2 * L * D * 4))


# every NV instance: nv = 1..16, with 7, 9, 11, 13, 14 and 15 running a larger instance with idle lanes
CROSS_D = (4, 256, 384, 388, 512, 640, 768, 772, 1024, 1028, 1248, 1284, 1536, 1540, 1700, 1920, 2048)
CROSS_CASES = ([(D, 3) for D in CROSS_D]
               + [(4, 1), (772, 1), (2048, 1), (388, 6), (1248, 6), (4, 32), (256, 32), (772, 32)]
               + [(2048, 4), (2048, 6), (2048, 12)])          # wpc = 3, 2, 1
assert {_nv(D) for D in CROSS_D} == set(range(1, 17))
assert {_wpc(D, L) for D, L in CROSS_CASES} == {1, 2, 3, 4}


@pytest.mark.parametrize("D,L", CROSS_CASES)
def test_cross_fwd_bwd(D, L):
    from tf_repos_b200 import ops
    d = _dev()
    wpc = _wpc(D, L)
    n_warps = _sm_count() * wpc
    assert ops.cross_bwd_workspace_bytes(1, D, L) == n_warps * 2 * L * D * 4
    nv = _nv(D)
    g = torch.Generator().manual_seed(D * 40 + L)
    w = torch.randn(L, D, generator=g) / D ** 0.5
    b = torch.randn(L, D, generator=g) * 0.1
    wd, bd = w.to(d), b.to(d)
    ws = torch.empty(ops.cross_bwd_workspace_bytes(1, D, L), dtype=torch.uint8, device=d)
    for i, B in enumerate((1, n_warps - 1, n_warps, n_warps + 1, 4 * n_warps + 3)):
        what = f"D={D} L={L} (nv={nv} wpc={wpc}) B={B}"
        x0 = torch.randn(B, D, generator=g) * 0.5
        x0d = x0.to(d)
        xL = torch.full((B, D), float("nan"), device=d)
        s = torch.full((B, L), float("nan"), device=d)
        ops.cross_fwd(x0d, wd, bd, xL, s)
        sc = s.cpu()
        # x_L: ((x0 * s_l) + x_l) + b_l restated in fp32 with the kernel's own s
        x = x0.clone()
        xs = []
        for l in range(L):
            xs.append(x)
            x = ((x0 * sc[:, l:l + 1]) + x) + b[l]
        _bits_equal(xL, x, f"x_L {what}")
        for l in range(L):
            t = xs[l].double() * w[l].double()
            _within(sc[:, l], t.sum(1), gam(4 * nv + 5) * t.abs().sum(1), f"s_{l} {what}")
        # backward
        dxL = torch.randn(B, D, generator=g)
        dx_in = torch.randn(B, D, generator=g) if i % 2 == 0 else None
        dx0 = torch.full((B, D), float("nan"), device=d)
        dw = torch.full((L, D), float("nan"), device=d)
        db = torch.full((L, D), float("nan"), device=d)
        ops.cross_bwd(x0d, wd, bd, s, dxL.to(d), dx_in.to(d) if dx_in is not None else None, dx0, dw, db, ws)
        X0, S, W = x0.double(), sc.double(), w.double()
        gr = dxL.double()
        eg = torch.zeros_like(gr)
        acc = torch.zeros_like(gr); acc_mag = torch.zeros_like(gr); acc_err = torch.zeros_like(gr)
        dw_ref, dw_mag, dw_err = (torch.zeros(L, D, dtype=torch.float64) for _ in range(3))
        db_ref, db_mag, db_err = (torch.zeros(L, D, dtype=torch.float64) for _ in range(3))
        for l in reversed(range(L)):
            xl = xs[l].double()
            G = gr.abs() + eg
            ds = (gr * X0).sum(1, keepdim=True)
            eds = (eg * X0.abs()).sum(1, keepdim=True) + gam(4 * nv + 5) * (G * X0.abs()).sum(1, keepdim=True)
            DS = ds.abs() + eds
            db_ref[l], db_mag[l], db_err[l] = gr.sum(0), G.sum(0), eg.sum(0)
            dw_ref[l], dw_mag[l], dw_err[l] = (ds * xl).sum(0), (DS * xl.abs()).sum(0), (eds * xl.abs()).sum(0)
            sl = S[:, l:l + 1]
            acc = acc + gr * sl
            acc_mag = acc_mag + G * sl.abs()
            acc_err = acc_err + eg * sl.abs()
            eg = eg + eds * W[l].abs() + U * (G + DS * W[l].abs())
            gr = gr + ds * W[l]
        G = gr.abs() + eg
        din = dx_in.double() if dx_in is not None else torch.zeros_like(gr)
        _within(dx0, acc + gr + din, (acc_err + eg + gam(L + 2) * (acc_mag + G + din.abs())) * 1.01, f"dx0 {what}")
        chain = -(-B // n_warps) + n_warps
        _within(dw, dw_ref, (dw_err + gam(chain) * dw_mag) * 1.01, f"dw {what}")
        _within(db, db_ref, (db_err + gam(chain) * db_mag) * 1.01, f"db {what}")
        dw2 = torch.full_like(dw, float("nan"))
        db2 = torch.full_like(db, float("nan"))
        ops.cross_bwd(x0d, wd, bd, s, dxL.to(d), None, dx0, dw2, db2, ws)
        _bits_equal(dw2, dw, f"dw on a second run {what}")
        _bits_equal(db2, db, f"db on a second run {what}")


@pytest.mark.parametrize("D", [4, 772, 2048])
def test_cross_fwd_with_no_layer_copies_x0(D):
    from tf_repos_b200 import ops
    d = _dev()
    x0 = torch.randn(37, D, device=d)
    xL = torch.full_like(x0, float("nan"))
    ops.cross_fwd(x0, torch.empty(0, D, device=d), torch.empty(0, D, device=d), xL, torch.empty(37, 0, device=d))
    _bits_equal(xL, x0, f"L=0 x_L D={D}")


def test_cross_rejections_launch_nothing():
    from tf_repos_b200 import ops
    d = _dev()
    B = 9
    for D, L, fwd_ok in ((6, 1, False), (2052, 1, False), (4, 33, False), (2048, 13, True)):
        x0 = torch.randn(B, D, device=d)
        w = torch.randn(L, D, device=d) * 0.01
        b = torch.randn(L, D, device=d)
        xL = torch.full((B, D), 3.0, device=d)
        s = torch.full((B, L), 3.0, device=d)
        if fwd_ok:                                               # fwd has no slab: D = 2048, L = 13 runs
            ops.cross_fwd(x0, w, b, xL, s)
            assert torch.isfinite(xL).all()
        else:
            _rejected(lambda: ops.cross_fwd(x0, w, b, xL, s), [xL, s], f"cross_fwd D={D} L={L}")
        if fwd_ok:
            assert ops.cross_bwd_workspace_bytes(B, D, L) == 0, "no warp fits the slab"
        ws = torch.empty(1 << 20, dtype=torch.uint8, device=d)
        dx0 = torch.full((B, D), 3.0, device=d)
        dw = torch.full((L, D), 3.0, device=d)
        db = torch.full((L, D), 3.0, device=d)
        _rejected(lambda: ops.cross_bwd(x0, w, b, s, xL, None, dx0, dw, db, ws), [dx0, dw, db], f"cross_bwd D={D} L={L}")


# ---------------------------------------------------------------------------------------------------------------------
# fc1 at these models' shapes: AFM's attention_out (M = B*P rows) and deep_out, DCN's out_layer over [x_L | x_deep]
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,Ka,Kb", [(94_848, 256, 0), (128, 256, 0), (64, 1248, 64), (65, 1248, 64)])
def test_fc1_at_model_shapes(M, Ka, Kb):
    from tf_repos_b200 import ops
    d = _dev()
    g = torch.Generator().manual_seed(M + Ka + Kb)
    A = torch.randn(M, Ka, generator=g)
    Bm = torch.randn(M, Kb, generator=g) if Kb else None
    w = torch.randn(Ka + Kb, generator=g) / (Ka + Kb) ** 0.5
    bias = torch.randn(1, generator=g)
    Ad, Bd, wd = A.to(d), (Bm.to(d) if Kb else None), w.to(d)
    y = torch.full((M,), float("nan"), device=d)
    ops.fc1_fwd(Ad, Bd, wd, bias.to(d), y)
    A64, w64 = A.double(), w.double()
    ref = A64 @ w64[:Ka] + bias.double()
    mag = A64.abs() @ w64[:Ka].abs() + bias.double().abs()
    if Kb:
        ref = ref + Bm.double() @ w64[Ka:]
        mag = mag + Bm.double().abs() @ w64[Ka:].abs()
    _within(y, ref, gam(-(-Ka // 32) + -(-Kb // 32) + 6) * mag, f"fc1 y M={M}")
    dy = torch.randn(M, generator=g) * (torch.rand(M, generator=g) < 0.7)
    chunks = -(-M // 64)
    if M == 94_848:
        assert chunks == 1482
    ws = torch.empty(max(ops.fc1_bwd_workspace_bytes(M, Ka, Kb), 16), dtype=torch.uint8, device=d)

    def run():
        d_a = torch.full((M, Ka), float("nan"), device=d)
        d_b = torch.full((M, Kb), float("nan"), device=d) if Kb else None
        dw = torch.full((Ka + Kb,), float("nan"), device=d)
        db = torch.full((1,), float("nan"), device=d)
        ops.fc1_bwd(Ad, Bd, wd, dy.to(d), d_a, d_b, dw, db, ws)
        return d_a, d_b, dw, db

    d_a, d_b, dw, db = run()
    _bits_equal(d_a, dy[:, None] * w[None, :Ka], f"fc1 d_a M={M}")
    if Kb:
        _bits_equal(d_b, dy[:, None] * w[None, Ka:], f"fc1 d_b M={M}")
    IN = torch.cat([A64, Bm.double()], 1) if Kb else A64
    dy64 = dy.double()
    chain = 64 + -(-chunks // 8) + 8
    _within(dw, IN.T @ dy64, gam(chain) * (IN.abs().T @ dy64.abs()), f"fc1 dw M={M}")
    _within(db, dy64.sum().reshape(1), gam(chain) * dy64.abs().sum().reshape(1), f"fc1 db M={M}")
    _, _, dw2, db2 = run()
    _bits_equal(dw2, dw, "fc1 dw on a second run")
    _bits_equal(db2, db, "fc1 db on a second run")


# ---------------------------------------------------------------------------------------------------------------------
# construction rejects shapes the kernels reject (before: the first predict or train step failed)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model,kw,flag", [
    ("PNN", dict(field_size=39, embedding_size=164, model_type="Inner"), "--embedding_size"),
    ("PNN", dict(field_size=39, embedding_size=256, model_type="Inner"), "--embedding_size"),
    ("AFM", dict(field_size=144, embedding_size=4), "--field_size"),
    ("DCN", dict(field_size=39, embedding_size=64), "--embedding_size"),
    ("DCN", dict(field_size=39, embedding_size=10), "--embedding_size"),
    ("DCN", dict(field_size=13, embedding_size=32, cross_layers=33), "--cross_layers"),
    ("DCN", dict(field_size=64, embedding_size=32, cross_layers=13), "--cross_layers"),
])
def test_unsupported_shapes_raise_at_construction(model, kw, flag):
    from tf_repos_b200 import _lib
    from tf_repos_b200.afm import AFM
    from tf_repos_b200.dcn import DCN
    from tf_repos_b200.pnn import PNN
    cls = {"PNN": PNN, "AFM": AFM, "DCN": DCN}[model]
    F, K = kw.pop("field_size"), kw.pop("embedding_size")
    n0 = _lib.launch_count()
    with pytest.raises(ValueError, match=flag):
        cls(F, 1000, K, 8, device="cuda:0", **kw)
    assert _lib.launch_count() == n0


def test_largest_supported_shapes_construct():
    from tf_repos_b200.afm import AFM
    from tf_repos_b200.dcn import DCN
    from tf_repos_b200.pnn import PNN
    PNN(39, 100, 163, 4, model_type="Inner", deep_layers="8", dropout="1.0", device="cuda:0")
    AFM(143, 100, 4, 2, attention_layers="8", device="cuda:0")
    DCN(39, 100, 52, 4, deep_layers="8", dropout="1.0", cross_layers=6, device="cuda:0")       # D = 2028
    DCN(64, 100, 32, 4, deep_layers="8", dropout="1.0", cross_layers=12, device="cuda:0")      # D = 2048, wpc = 1


# ---------------------------------------------------------------------------------------------------------------------
# AFM, PNN (Inner) and DCN at the reference's default configurations (AFM.py:44-53, PNN.py:44-61, DCN.py:43-53)
# ---------------------------------------------------------------------------------------------------------------------
DF, DN = 39, 10_000
MODELS = {
    "AFM": dict(B=128, K=256, kw=dict(attention_layers="256", dropout="1.0,0.5", l2_reg=1.0, learning_rate=0.1,
                                      optimizer="Adam")),
    "PNN": dict(B=64, K=32, kw=dict(model_type="Inner", deep_layers="256,128,64", dropout="0.5,0.5,0.5", l2_reg=1e-4,
                                    learning_rate=5e-4, optimizer="Adam")),
    "DCN": dict(B=64, K=32, kw=dict(deep_layers="256,128,64", cross_layers=3, dropout="0.5,0.5,0.5", l2_reg=1e-4,
                                    learning_rate=5e-4, optimizer="Adam")),
}
NAMES = list(MODELS)


def _pick_split(M, N, R):
    """fc.cu pick_split: the number of split-R chunks of a dW product"""
    t = 128
    tiles = ((M + t - 1) // t) * ((N + t - 1) // t)
    s = max((2 * _sm_count() + tiles - 1) // tiles, 1)
    return max(min(s, (R + 255) // 256, 64), 1)


def _dw_rel(Kd, Nd, M):
    S = _pick_split(Kd, Nd, M)
    return gemm_rel(-(-M // S), adds=S)


def _tol(name, B):
    """One step's gradients pass through these rounded stages, each within its bound of the magnitude of the terms it
    sums; to first order the gradient error is their sum.  It is applied to the largest magnitude of each gradient,
    which bounds the magnitude of its summed terms up to their cancellation (as in test_gpu_din_attention.py)."""
    head = 16 * U                                         # logit sum, sigmoid CE and dy
    if name == "AFM":
        P, K, A = 741, 256, 256
        M = B * P
        chunks = -(-M // 64)
        fwd = U + gemm_rel(K, 1) + gam(8 + 6) + 300 * U + gam(P) + 2 * U + gam(8 + 6)
        bwd = (U + 2 * U + gam(64 + 8 + 8) + U + gam(K) + gam(-(-P // 256) + 8) + 4 * U + U
               + gam(64 + -(-chunks // 8) + 8) + gemm_rel(A, 1) + _dw_rel(K, A, M) + gam(DF - 1) + U)
    elif name == "PNN":
        K, Dz = 32, 39 * 32 + 741
        fwd = gam(K) + gemm_rel(Dz, 1) + gemm_rel(256, 1) + gemm_rel(128, 1) + 6 * U + gam(2 + 6)
        bwd = (U + gam(64 + 9) + gemm_rel(64) + gemm_rel(128) + gemm_rel(256) + _dw_rel(Dz, 256, B)
               + _dw_rel(256, 128, B) + _dw_rel(128, 64, B) + 6 * U + gam(DF) + U)
    else:
        D, L = 1248, 3
        n_warps = _sm_count() * _wpc(D, L)
        fwd = L * (gam(4 * 10 + 5) + 3 * U) + gemm_rel(D, 1) + gemm_rel(256, 1) + gemm_rel(128, 1) + 6 * U + gam(41 + 6)
        bwd = (U + gam(64 + 9) + gemm_rel(64) + gemm_rel(128) + gemm_rel(256, 1) + _dw_rel(D, 256, B)
               + _dw_rel(256, 128, B) + _dw_rel(128, 64, B) + 6 * U
               + L * (gam(4 * 10 + 5) + 2 * U) + gam(-(-B // n_warps) + n_warps) + gam(L + 2) + U)
    return head + fwd + bwd


def _oracle(name, dtype):
    from oracle import models as om
    c = MODELS[name]
    ref = getattr(om, name)(DF, DN, c["K"], seed=4, dtype=dtype, **c["kw"])
    g = torch.Generator().manual_seed(1)
    ref.params["emb"].copy_(torch.randn(DN, c["K"], generator=g) * 0.1)
    if "linear" in ref.params:
        ref.params["linear"].copy_(torch.randn(DN, generator=g) * 0.1)
    for p in ref.params.values():
        p.copy_(p.float().to(dtype))                        # both sides start from the same fp32 values
    return ref


def _gpu(name, mode="exact", epoch_steps=8, B=None):
    from tf_repos_b200.afm import AFM
    from tf_repos_b200.dcn import DCN
    from tf_repos_b200.pnn import PNN
    c = MODELS[name]
    cls = {"AFM": AFM, "PNN": PNN, "DCN": DCN}[name]
    return cls(DF, DN, c["K"], B or c["B"], update_mode=mode, epoch_steps=epoch_steps, device="cuda:0", **c["kw"])


def _masks(name, B, step):
    """injected dropout masks: AFM's dropout[1] on y_emb (dropout[0] = 1.0 is the identity); the MLP's three layers"""
    g = torch.Generator().manual_seed(900 + step)
    if name == "AFM":
        m = (torch.rand(B, MODELS[name]["K"], generator=g) < 0.5).float()
        return {"pool": m}, {"pool": m.cuda()}
    lst = [(torch.rand(B, w, generator=g) < 0.5).float() for w in (256, 128, 64)]
    if name == "PNN":
        return {"mlp": lst}, {"mlp": [m.cuda() for m in lst]}
    return lst, [m.cuda() for m in lst]


def _batch(B, step):
    from tf_repos_b200 import synth
    ids, vals, labels = synth.criteo_batch(B, DN, DF, seed=300 + step)
    return ids, vals, labels, {"feat_ids": ids.long(), "feat_vals": vals}


def _one_step(name, B):
    ref = _oracle(name, torch.float64)
    gpu = _gpu(name, B=B)
    gpu.load_variables(ref.params)
    ids, vals, labels, batch = _batch(B, 0)
    mc, mg = _masks(name, B, 0)
    _, out, _, dgrads = ref.gradients(batch, labels, mc)
    gpu.train_step(ids.cuda(), vals.cuda(), labels.cuda(), mg)
    gpu.check_ids()
    torch.cuda.synchronize()
    tol = _tol(name, B)
    K = MODELS[name]["K"]
    scale = {}
    if name == "AFM":
        # attention_out/biases is the sum of the softmax backward over all B*P rows, exactly 0 in exact arithmetic:
        # its bound scales with the magnitude of those rows, sum att * (|da| + |sum_p da att|) (the GPU's own values)
        P = DF * (DF - 1) // 2
        a = gpu.att[:B * P].double().view(B, P)
        da = torch.bmm(gpu.pw[:B * P].double().view(B, P, K), gpu.d_emb2[:B].double().view(B, K, 1)).squeeze(2)
        s = (a * da).sum(1, keepdim=True)
        scale["Attention-part/attention_out/biases"] = float((a * (da.abs() + s.abs())).sum())
    assert set(dgrads) == set(gpu.dense.grads), (sorted(dgrads), sorted(gpu.dense.grads))
    for n, gref in dgrads.items():
        if n in ref.l2_vars:                                # the GPU adds l2 * var inside the optimizer kernel
            gref = gref - torch.tensor(ref.l2_reg, dtype=torch.float64) * ref.params[n]
        got = gpu.dense.grads[n].cpu()
        _within(got, gref.reshape(got.shape), tol * scale.get(n, gref.abs().max()), f"{name} {n} (B={B})")
    per = out["per_occurrence"]
    site = "emb" if name == "DCN" else "v"
    r = per[site].reshape(B * DF, K)
    _within(gpu.g_rows[:B * DF].cpu(), r, tol * r.abs().max(), f"{name} per-occurrence emb rows (B={B})")
    if name != "DCN":
        r = per["w"].reshape(B * DF)
        _within(gpu.g_w[:B * DF].cpu(), r, tol * r.abs().max(), f"{name} per-occurrence linear (B={B})")


@pytest.mark.parametrize("name", NAMES)
def test_default_config_one_step_gradients_match_fp64(name):
    _one_step(name, MODELS[name]["B"])


def test_dcn_default_config_one_step_with_several_samples_per_cross_warp():
    """B = 4 n_warps + 3: the model path gives every cross_bwd warp four or five samples"""
    n_warps = _sm_count() * _wpc(1248, 3)
    _one_step("DCN", 4 * n_warps + 3)


def _gpu_state_views(gpu, name):
    """(var, [slots]) views of the GPU model's state by TF name (tables, then dense variables in the flat buffer)"""
    out = {t.name: (t.var, list(t.slots)) for t in gpu.tables}
    flat = gpu.dense.flat
    for n, v in gpu.dense.views.items():
        off = (v.data_ptr() - flat.data_ptr()) // 4
        out[n] = (v, [s[off:off + v.numel()].view(v.shape) for s in gpu.dense.slots])
    return out


@pytest.mark.parametrize("mode", ["exact", "exact_deferred"])
@pytest.mark.parametrize("name", NAMES)
def test_default_config_three_steps_match_the_fp32_oracle(name, mode):
    """Parameters after each of three steps, at the tolerance test_gpu_din.py holds models to.  Adam's first steps
    move an element by about lr * sign(g).  The GPU's gradient and the fp32 oracle's are each within the one-step bound
    of the exact one, so they may differ by delta = twice that bound.  Where the oracle's gradient lies within delta of
    zero the sign is legitimately either, which at AFM's lr = 0.1 is a 0.2 difference.  Near zero the step is also
    sensitive through eps: a gradient error delta moves u = lr_t m / (sqrt(v) + eps) by up to
    lr_t delta ((1 - b1) + sqrt(1 - b2) |m| / (sqrt(v) + eps)) / (sqrt(v) + eps).  Only elements where that exceeds
    the tolerance may differ; they must be few, and they are reset to the oracle's state so the difference does not
    spread."""
    B = MODELS[name]["B"]
    ref = _oracle(name, torch.float32)
    gpu = _gpu(name, mode, epoch_steps=2)
    gpu.load_variables(ref.params)
    tol = _tol(name, B)
    l2 = ref.l2_reg
    n_excluded = 0
    for step in range(3):
        ids, vals, labels, batch = _batch(B, step)
        mc, mg = _masks(name, B, step)
        before = {n: p.clone() for n, p in ref.params.items()}
        _, _, tgrads, dgrads = ref.gradients(batch, labels, mc)
        ref.apply_gradients(tgrads, dgrads)
        gpu.train_step(ids.cuda(), vals.cuda(), labels.cuda(), mg)
        gpu.check_ids()
        # the gradient each element's update saw, and how close to zero it may legitimately be
        b1, b2, eps = float(ref.adam.b1), float(ref.adam.b2), float(ref.adam.eps)
        t = step + 1
        lr_t = float(ref.learning_rate) * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)
        delta = {}
        for n, gd in dgrads.items():
            data = gd - l2 * before[n] if n in ref.l2_vars else gd
            delta[n] = (gd, 2 * tol * data.abs().max().item())
        for n, (summed, uniq) in tgrads.items():
            gt = (l2 * before[n]).clone() if n in ref.l2_vars else torch.zeros_like(before[n])
            gt[uniq] += summed.reshape((-1,) + tuple(gt.shape[1:]))
            delta[n] = (gt, 2 * tol * summed.abs().max().item())
        vs = gpu.variables()
        views = _gpu_state_views(gpu, name)
        for n, want in ref.params.items():
            got = vs[n].cpu().reshape(want.shape)
            err = (got.double() - want.double()).abs()
            allowed = 2e-5 * want.double().abs() + 2e-5 * max(want.double().abs().max().item(), 1e-30)
            off = err > allowed
            gn, dn = delta[n]
            m, v = (sl.double() for sl in ref.slots[n])
            den = v.sqrt() + eps
            sens = lr_t * dn * ((1 - b1) + math.sqrt(1 - b2) * m.abs() / den) / den
            ambiguous = (gn.double().abs() <= dn) | (sens > allowed / 2)
            stray = off & ~ambiguous
            assert not stray.any(), (f"{name} {n} after step {step} ({mode}): {int(stray.sum())} elements outside the "
                                     f"tolerance, worst {err[stray].max().item():.3e}")
            k = int(off.sum())
            if k:
                n_excluded += k
                var, slots = views[n]
                idx = off.reshape(-1).nonzero().reshape(-1).to(var.device)
                var.view(-1)[idx] = want.reshape(-1).to(var.device)[idx]
                for s_gpu, s_ref in zip(slots, ref.slots[n]):
                    s_gpu.reshape(-1)[idx] = s_ref.reshape(-1).to(var.device)[idx]
    n_total = sum(p.numel() for p in ref.params.values())
    assert n_excluded <= max(16, n_total // 10_000), f"{name}: {n_excluded} elements had a near-zero gradient"


def _state(m):
    m.flush()
    out = []
    for t in m.tables:
        out += [t.var] + list(t.slots)
    out += [m.dense.flat] + list(m.dense.slots)
    return [t.clone() for t in out]


@pytest.mark.parametrize("name", NAMES)
def test_default_config_deferred_equals_exact_bit_for_bit(name):
    B = MODELS[name]["B"]
    ref = _oracle(name, torch.float32)
    a = _gpu(name, "exact")
    b = _gpu(name, "exact_deferred", epoch_steps=4)
    a.load_variables(ref.params); b.load_variables(ref.params)
    for step in range(8):                                   # two epochs
        ids, vals, labels, _ = _batch(B, 10 + step)
        _, mg = _masks(name, B, 10 + step)
        la = a.train_step(ids.cuda(), vals.cuda(), labels.cuda(), mg)
        lb = b.train_step(ids.cuda(), vals.cuda(), labels.cuda(), mg)
        assert torch.equal(la[0], lb[0]), f"{name}: CE differs at step {step}"
        if step in (1, 5):                                  # mid-epoch flushes
            for x, y in zip(_state(a), _state(b)):
                _bits_equal(y, x, f"{name}: exact_deferred vs exact after step {step}")
    for x, y in zip(_state(a), _state(b)):
        _bits_equal(y, x, f"{name}: exact_deferred vs exact after two epochs")


@pytest.mark.parametrize("name", NAMES)
def test_default_config_is_bit_reproducible(name):
    B = MODELS[name]["B"]
    ref = _oracle(name, torch.float32)
    states = []
    for _ in range(2):
        m = _gpu(name, "exact")
        m.load_variables(ref.params)
        for step in range(3):
            ids, vals, labels, _ = _batch(B, 20 + step)
            _, mg = _masks(name, B, 20 + step)
            m.train_step(ids.cuda(), vals.cuda(), labels.cuda(), mg)
        states.append(_state(m) + [m.g_rows.clone(), m.dense.grad.clone()])
    for x, y in zip(*states):
        _bits_equal(y, x, f"{name}: two fresh models")
