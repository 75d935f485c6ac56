"""DIN's attention unit and pooling kernels at the reference's default shape and its edges, against fp64 references or
exact fp32 restatements, and DIN at the reference's default configuration (DIN.py:35-46: K=32, deep_layers=256,128,64,
dropout=0.5,0.5,0.5, attention pooling; the attention hidden width is deep_layers[0] = 256, quirk Q5) against the oracle.

Error bounds used below (each comparison states which one and why):
  U        = 2^-24: unit roundoff of one round-to-nearest fp32 operation.
  TRUNC    = 2^-23: relative error of one fp32 addition the tensor core truncates instead of rounding.
  SPLIT    = 3*2^-21: 3xTF32 (csrc/tc_gemm.cu:4-8).  hi = rna_tf32(a) is within 2^-11 of a; lo = a - hi is exact but the MMA
             reads it truncated to tf32 (2^-10 of lo = 2^-21 of a); a_lo*b_lo (2^-22) is dropped.  Per product that is
             2^-21 + 2^-21 + 2^-22 (+ O(2^-32)) <= 3*2^-21 of |a||b|; tf32 x tf32 products are exact in fp32.
  gemm_rel(R, adds): a product over a reduction of length R, then `adds` rounded fp32 additions (split-R partial sums,
             bias, group bias, C += acc), relative to |A|@|B| + |addends|.  One wgmma k8 step aligns its 8 products and the
             accumulator and truncates each: <= 9 truncations per 8 reduction indices, 9/8*R*TRUNC; the cross-term accumulator
             (2^-10 of the main one) adds at most 2^-9 of that; acc + acc2 is one more rounding.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TRUNC = 2.0 ** -23
SPLIT = 3 * 2.0 ** -21
DIN_K = (4, 8, 16, 32, 64, 128, 256)


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


def _pick_split(M, N, R):
    """fc.cu pick_split: the number of split-R chunks of a dW product (needed for its error bound)."""
    t = 128
    tiles = ((M + t - 1) // t) * ((N + t - 1) // t)
    s = max((2 * _sm_count() + tiles - 1) // tiles, 1)
    return max(min(s, (R + 255) // 256, 64), 1)


# ---------------------------------------------------------------------------------------------------------------------
# fc_fwd_grouped: Hh = relu(E @ Wc + b + U[i // P]) (/keep * mask), the attention unit's hidden layer (DIN.py:164-168)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [16, 40, 250, 256, 300])
@pytest.mark.parametrize("P", [1, 3, 100, 128, 129])
def test_fc_fwd_grouped(P, H):
    from tf_repos_b200 import ops
    d = _dev()
    B = 37                                   # M = 37*P: not a multiple of 128 except at P = 128
    M = B * P
    g = torch.Generator().manual_seed(P * 1000 + H)
    keep = 0.5
    for j, K in enumerate((4, 8, 32, 64, 128)):
        E = torch.randn(M, K, generator=g)
        Wc = torch.randn(K, H, generator=g) / K ** 0.5
        Ug = torch.randn(B, H, generator=g) * 0.5
        b = torch.randn(H, generator=g) * 0.1 if j % 2 else None
        mask = (torch.rand(M, H, generator=g) < keep).float() if j % 2 == 0 else None
        out = torch.full((M, H), float("nan"), device=d)
        ops.fc_fwd_grouped(E.to(d), Wc.to(d), b.to(d) if b is not None else None, Ug.to(d), P,
                           mask.to(d) if mask is not None else None, keep, 1, out)
        gid = torch.arange(M) // P
        pre = E.double() @ Wc.double() + Ug.double()[gid] + (b.double() if b is not None else 0.0)
        mag = E.double().abs() @ Wc.double().abs() + Ug.double().abs()[gid] + (b.double().abs() if b is not None else 0.0)
        # relu is 1-Lipschitz, so a pre-activation within the bound of 0 cannot leave it whichever side it lands on;
        # /0.5 doubles the error exactly, *mask (0/1) is exact.  Adds: bias, group bias.
        bound = gemm_rel(K, adds=2) * mag
        ref = pre.clamp_min(0.0)
        if mask is not None:
            ref, bound = ref / keep * mask.double(), bound / keep * mask.double()
        _within(out, ref, bound, f"fc_fwd_grouped P={P} H={H} K={K} bias={b is not None} mask={mask is not None}")


# ---------------------------------------------------------------------------------------------------------------------
# fc_bwd(act=2, accumulate_din): dE += dZ @ Wc^T and dWc = E^T @ dZ, as DIN's attention backward calls it
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,K,H", [
    (50_001, 32, 256),    # the reference's default unit (K <= 64, H >= 128: transposed dW); S = 64 ragged chunks of 782
    (12_807, 64, 128),    # transposed dW at its edge
    (50_001, 128, 256),   # plain dW path, S = 64
    (4_773, 8, 300),      # transposed dW with a ragged second column tile
    (1_000, 4, 16),       # narrow layer: plain dW path
])
def test_fc_bwd_act2_accumulate(M, K, H):
    from tf_repos_b200 import ops
    d = _dev()
    g = torch.Generator().manual_seed(M + K + H)
    E = torch.randn(M, K, generator=g)
    Wc = torch.randn(K, H, generator=g) / K ** 0.5
    dZ = torch.randn(M, H, generator=g) * (torch.rand(M, H, generator=g) < 0.6)   # relu/dropout zeros, as din_att_dz leaves
    dE_old = torch.randn(M, K, generator=g)
    ws = torch.empty(ops.fc_bwd_workspace_bytes(M, K, H), dtype=torch.uint8, device=d)

    def run():
        dE = dE_old.to(d).clone()
        dW = torch.full((K, H), float("nan"), device=d)
        dZd = dZ.to(d)
        ops.fc_bwd(E.to(d), Wc.to(d), None, None, 1.0, dZd, 2, dE, dW, None, ws, accumulate_din=True)
        assert torch.equal(dZd.cpu(), dZ), "act=2 must leave dZ as it is"
        return dE, dW

    dE, dW = run()
    E64, W64, dZ64 = E.double(), Wc.double(), dZ.double()
    # dE: one product over H, then C += acc (one rounded add), relative to |dZ|@|Wc|^T + |dE_old|
    _within(dE, dE_old.double() + dZ64 @ W64.T, gemm_rel(H, adds=1) * (dZ64.abs() @ W64.abs().T + dE_old.double().abs()),
            f"dE += dZ Wc^T (M={M} K={K} H={H})")
    # dW: S split-R chunks of ceil(M/S) rows each on the GEMM, then S - 1 fixed-order fp32 adds
    transposed = K <= 64 and H >= 128
    S = _pick_split(H, K, M) if transposed else _pick_split(K, H, M)
    _within(dW, E64.T @ dZ64, gemm_rel(-(-M // S), adds=S) * (E64.abs().T @ dZ64.abs()),
            f"dW (M={M} K={K} H={H} S={S} transposed={transposed})")
    dE2, dW2 = run()
    _bits_equal(dE2, dE, "dE on a second call")
    _bits_equal(dW2, dW, "dW on a second call")


# ---------------------------------------------------------------------------------------------------------------------
# din_att_dz: the attention unit's output layer + relu + dropout backward and per-sample sums in one pass
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("P", [1, 100])
@pytest.mark.parametrize("H", [16, 256, 300])
def test_din_att_dz(H, P, masked):
    from tf_repos_b200 import ops
    d = _dev()
    B = 48
    rng = np.random.default_rng(H * 7 + P + masked)
    keep = np.float32(0.7)                          # not a power of two: the division has to round
    Hh = (np.maximum(rng.standard_normal((B * P, H)), 0) * (rng.random((B * P, H)) < 0.7)).astype(np.float32)
    dz = rng.standard_normal(B * P).astype(np.float32)
    w2 = rng.standard_normal(H).astype(np.float32)
    mask = (rng.random((B * P, H)) < keep).astype(np.float32) if masked else None
    t = lambda a: torch.from_numpy(a).to(d)
    dZ = torch.full((B * P, H), float("nan"), device=d)
    dU = torch.full((B, H), float("nan"), device=d)
    gw2 = torch.full((B, H), float("nan"), device=d)
    ops.din_att_dz(t(Hh), t(mask) if masked else None, float(keep), t(dz), t(w2), B, P, dZ, dU, gw2)
    # dZ: the kernel's fp32 sequence, each step one IEEE-rounded numpy float32 op
    ref = dz[:, None] * w2[None, :]
    if masked:
        ref = (ref * mask) / keep
    ref = np.where(Hh > 0, ref, np.float32(0)).astype(np.float32)
    _bits_equal(dZ, torch.from_numpy(ref), f"dZ H={H} P={P} mask={masked}")
    # dU: the sum over p in order, fp32
    r3 = ref.reshape(B, P, H)
    su = np.zeros((B, H), dtype=np.float32)
    for p in range(P):
        su = su + r3[:, p, :]
    _bits_equal(dU, torch.from_numpy(su), f"dU H={H} P={P} mask={masked}")
    # gw2_part = sum_p Hh*dz with fmaf: P roundings of U, each of a partial sum <= sum_p |Hh*dz|
    terms = Hh.astype(np.float64).reshape(B, P, H) * dz.astype(np.float64).reshape(B, P, 1)
    _within(gw2, terms.sum(1), P * U * np.abs(terms).sum(1), f"gw2_part H={H} P={P}")


# ---------------------------------------------------------------------------------------------------------------------
# colsum_rows: 8 row groups per column, each summed in row order, then a fixed 8-way sequence
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,ncols", [(1, 31), (7, 1), (8, 33), (9, 256), (12_800, 300), (409_601, 45)])
def test_colsum_rows(rows, ncols):
    from tf_repos_b200 import ops
    d = _dev()
    rng = np.random.default_rng(rows + ncols)
    x = (rng.standard_normal((rows, ncols)) * np.exp(rng.standard_normal((rows, 1)))).astype(np.float32)
    out = torch.full((ncols,), float("nan"), device=d)
    xd = torch.from_numpy(x).to(d)
    ops.colsum_rows(xd, out)
    # fp64: the longest chain is ceil(rows/8) adds in a group plus 8 in the final sequence, each <= U of <= sum|x|
    x64 = x.astype(np.float64)
    _within(out, x64.sum(0), (-(-rows // 8) + 8) * U * np.abs(x64).sum(0), f"colsum_rows {rows}x{ncols}")
    # exact: the kernel's order restated in fp32 (group q adds rows q, q+8, ...; then groups 0..7 in order)
    nblk = -(-rows // 8)
    pad = np.zeros((nblk * 8, ncols), dtype=np.float32)
    pad[:rows] = x
    blk = pad.reshape(nblk, 8, ncols)
    valid = (np.arange(nblk * 8) < rows).reshape(nblk, 8, 1)
    acc = np.zeros((8, ncols), dtype=np.float32)
    for i in range(nblk):
        acc = np.where(valid[i], acc + blk[i], acc)
    t = np.zeros(ncols, dtype=np.float32)
    for q in range(8):
        t = t + acc[q]
    _bits_equal(out, torch.from_numpy(t), f"colsum_rows order {rows}x{ncols}")
    out2 = torch.empty_like(out)
    ops.colsum_rows(xd, out2)
    _bits_equal(out2, out, "colsum_rows run to run")


# ---------------------------------------------------------------------------------------------------------------------
# din_pool_fwd / bwd: att = sigmoid(z); u = sum_p (id > 0) att E (DIN.py:169-172) and its gradient
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [1, 7, 31, 33, 100])
@pytest.mark.parametrize("K", DIN_K)
def test_din_pool_fwd_bwd(K, P):
    from tf_repos_b200 import ops
    d = _dev()
    B = 21
    g = torch.Generator().manual_seed(K * 131 + P)
    E = torch.randn(B * P, K, generator=g)
    z = torch.randn(B * P, generator=g) * 3
    ids = torch.randint(1, 1000, (B, P), generator=g, dtype=torch.int32)
    lens = torch.randint(1, P + 1, (B,), generator=g)
    ids[torch.arange(P)[None, :] >= lens[:, None]] = 0
    ids[3] = 0; ids[B - 1] = 0                         # samples with every position padding: u = 0, dz = 0
    zv = z.view(B, P)
    zv[5, 0] = 90.0; zv[6, 0] = -90.0                   # expf(-z) underflows / overflows: att exactly 1 / exactly 0
    ids[5, 0] = 7; ids[6, 0] = 9
    ids = ids.reshape(-1).contiguous()
    ld = 2 * K + 4                                      # u and du live in a strided slice of a wider row
    X = torch.full((B, ld), 7.0, device=d)
    att = torch.full((B * P,), float("nan"), device=d)
    ops.din_pool_fwd(E.to(d), z.to(d), ids.to(d), B, P, K, att, X[:, 4:], ld)
    Xc = X.cpu()
    assert torch.all(Xc[:, :4] == 7.0) and torch.all(Xc[:, 4 + K:] == 7.0), "din_pool_fwd wrote outside u"
    u = Xc[:, 4:4 + K]
    att_c = att.cpu()
    assert att_c[5 * P].item() == 1.0 and att_c[6 * P].item() == 0.0
    assert torch.all(u[3] == 0) and torch.all(u[B - 1] == 0)

    m = (ids > 0).double().view(B, P, 1)
    z64 = z.double().requires_grad_()
    E64 = E.double().requires_grad_()
    a64 = torch.sigmoid(z64)
    u64 = (E64.view(B, P, K) * a64.view(B, P, 1) * m).sum(1)
    DU = torch.randn(B, ld, generator=g)
    du = DU[:, 4:4 + K]
    u64.backward(du.double())
    a = a64.detach()
    # att = 1/(1 + expf(-z)): expf is within 2 ulp (2*2^-23), 1 + e and the division round once each: 3*2^-23 of att;
    # below 2^-126 the fp32 sigmoid may flush to 0 through expf's overflow (z = -90 above).
    ea = 3 * TRUNC * a + 2.0 ** -126
    _within(att, a, ea, f"att K={K} P={P}")
    # u: per term the att error; the warp adds ceil(P/RPW) fmas per slot, then log2(RPW) shuffle adds (RPW = 32/LPR)
    lpr = min(K // 4, 32)
    rpw = 32 // lpr
    n_add = -(-P // rpw) + int(math.log2(rpw))
    absE = E.double().abs().view(B, P, K)
    _within(u, u64.detach(), ((ea.view(B, P, 1) * absE * m).sum(1) + n_add * U * (a.view(B, P, 1) * absE * m).sum(1)) * 1.01,
            f"u K={K} P={P}")

    DUd = DU.to(d)
    dE = torch.full((B * P, K), float("nan"), device=d)
    dz = torch.full((B * P,), float("nan"), device=d)
    ops.din_pool_bwd(E.to(d), att, ids.to(d), DUd[:, 4:], ld, B, P, K, dE, dz)
    # dE = (m*att)*du: the att error plus one rounding
    _within(dE, E64.grad, ((ea + U * a).view(B, P, 1) * du.double().abs().view(B, 1, K) * m).reshape(B * P, K),
            f"dE K={K} P={P}")
    # dz = ((m*att)*(1-att))*dot: dot = e.du over K (<= K roundings of U of sum|e du|); s = att(1-att) moves by
    # <= |1-2att|*ea + ea^2 <= 1.01 ea from att's error, and 1-att, s and s*dot round once each (3U)
    dot = (E.double().view(B, P, K) * du.double().view(B, 1, K)).sum(2).reshape(-1)
    sdot = (E.double().view(B, P, K) * du.double().view(B, 1, K)).abs().sum(2).reshape(-1)
    s = a * (1 - a)
    mz = m.reshape(-1)
    _within(dz, z64.grad, ((1.01 * ea + 3 * U * s) * dot.abs() + s * (K + 1) * U * sdot) * mz * 1.01, f"dz K={K} P={P}")
    dzc = dz.cpu().view(B, P)
    assert torch.all(dzc[3] == 0) and torch.all(dzc[B - 1] == 0) and torch.all(dzc.reshape(-1)[ids == 0] == 0)
    assert torch.all(dE.cpu()[ids == 0] == 0)


# ---------------------------------------------------------------------------------------------------------------------
# gather_scale_rows, bag_sum_fwd/bwd, scale_rows at every supported K
# ---------------------------------------------------------------------------------------------------------------------
def _bags(B, N, g, max_len=9):
    lens = torch.randint(0, max_len + 1, (B,), generator=g)
    lens[0] = 0; lens[B // 2] = 0; lens[B - 1] = 0                     # empty bags, first / middle / last
    off = torch.zeros(B + 1, dtype=torch.int32)
    off[1:] = torch.cumsum(lens, 0).to(torch.int32)
    ids = torch.randint(0, N, (int(off[-1]),), generator=g, dtype=torch.int32)
    return ids, off, lens


def _seq_bag_sum(V, ids, off):
    """unweighted bag sums in occurrence order, one rounded fp32 add per occurrence"""
    B = off.numel() - 1
    lens = (off[1:] - off[:-1]).long()
    acc = torch.zeros(B, V.shape[1])
    for j in range(int(lens.max()) if B else 0):
        have = lens > j
        idx = (off[:-1].long() + j).clamp_max(max(ids.numel() - 1, 0))
        acc = torch.where(have[:, None], acc + V[ids.long()[idx]], acc)
    return acc


@pytest.mark.parametrize("K", DIN_K)
def test_gather_bag_scale_rows(K):
    from tf_repos_b200 import ops
    d = _dev()
    g = torch.Generator().manual_seed(K)
    N, B, G = 777, 45, 5
    V = torch.randn(N, K, generator=g)
    Vd = V.to(d)
    # gather, G > 1 with ld_group: rows land inside a wider [B, ld] buffer (the MLP input layout); then weighted, G = 1
    ld = G * K + 8
    ids = torch.randint(0, N, (B * G,), generator=g, dtype=torch.int32)
    x = torch.full((B, ld), 3.0, device=d)
    oob = torch.zeros(2, dtype=torch.int32, device=d)
    ops.gather_scale_rows(ids.to(d), None, Vd, x, G, ld, oob)
    assert torch.equal(x.cpu()[:, :G * K], V[ids.long()].reshape(B, G * K)) and torch.all(x.cpu()[:, G * K:] == 3.0)
    w = torch.rand(B * G, generator=g) * 3
    E = torch.empty(B * G, K, device=d)
    ops.gather_scale_rows(ids.to(d), w.to(d), Vd, E, 1, K, oob)
    assert torch.equal(E.cpu(), V[ids.long()] * w[:, None]), "gather: one rounded multiply per element"
    assert oob.tolist() == [0, 0]

    # bag_sum_fwd unweighted (fma with w = 1 is a rounded add): bit-exact against the in-order fp32 sum
    bids, off, lens = _bags(B, N, g)
    out = torch.full((B, K + 4), 5.0, device=d)
    ops.bag_sum_fwd(bids.to(d), None, off.to(d), Vd, out[:, 4:], K + 4, oob)
    oc = out.cpu()
    assert torch.equal(oc[:, 4:], _seq_bag_sum(V, bids, off)) and torch.all(oc[:, :4] == 5.0)
    empty = (lens == 0)
    assert torch.all(oc[:, 4:][empty].view(torch.int32) == 0), "an empty bag is a +0 row"
    # weighted: n fmas per bag, each rounding once a partial sum <= sum|V w|
    bw = torch.rand(bids.numel(), generator=g) * 3
    outw = torch.full((B, K), float("nan"), device=d)
    ops.bag_sum_fwd(bids.to(d), bw.to(d), off.to(d), Vd, outw, K, oob)
    seg = torch.repeat_interleave(torch.arange(B), lens)
    terms = V.double()[bids.long()] * bw.double()[:, None]
    ref = torch.zeros(B, K, dtype=torch.float64).index_add(0, seg, terms)
    mag = torch.zeros(B, K, dtype=torch.float64).index_add(0, seg, terms.abs())
    _within(outw, ref, lens.double()[:, None] * U * mag, f"weighted bag_sum_fwd K={K}")
    assert torch.all(outw.cpu()[empty].view(torch.int32) == 0)
    assert oob.tolist() == [0, 0]

    # bag_sum_bwd: one rounded multiply per element, unweighted and weighted, d_out read from a strided slice
    D = torch.randn(B, K + 4, generator=g)
    gr = torch.full((bids.numel(), K), float("nan"), device=d)
    Dd = D.to(d)
    ops.bag_sum_bwd(Dd[:, 4:], K + 4, None, off.to(d), K, gr)
    assert torch.equal(gr.cpu(), D[:, 4:][seg])
    ops.bag_sum_bwd(Dd[:, 4:], K + 4, bw.to(d), off.to(d), K, gr)
    assert torch.equal(gr.cpu(), D[:, 4:][seg] * bw[:, None])

    # scale_rows: (x + add) * w, two rounded ops, G > 1 reading a strided x; and each of add / w alone
    Xs = torch.randn(B, ld, generator=g)
    add = torch.randn(B * G, K, generator=g)
    ws = torch.rand(B * G, generator=g) * 3
    xin = Xs[:, :G * K].reshape(B * G, K)
    o = torch.full((B * G, K), float("nan"), device=d)
    Xd = Xs.to(d)
    ops.scale_rows(Xd, add.to(d), ws.to(d), B * G, K, G, ld, o)
    assert torch.equal(o.cpu(), (xin + add) * ws[:, None])
    ops.scale_rows(Xd, None, ws.to(d), B * G, K, G, ld, o)
    assert torch.equal(o.cpu(), xin * ws[:, None])
    ops.scale_rows(Xd, add.to(d), None, B * G, K, G, ld, o)
    assert torch.equal(o.cpu(), xin + add)
    ops.scale_rows(Xd[:, 8:], None, None, B, K, 1, ld, o[:B])
    assert torch.equal(o.cpu()[:B], Xs[:, 8:8 + K])


def test_unsupported_k_is_rejected_before_any_launch():
    from tf_repos_b200 import _lib, ops
    from tf_repos_b200._lib import CtrError
    d = _dev()
    K, B, P = 12, 4, 3
    V = torch.zeros(10, K, device=d)
    ids = torch.ones(B * P, dtype=torch.int32, device=d)
    off = torch.arange(B + 1, dtype=torch.int32, device=d) * P
    rows = torch.zeros(B * P, K, device=d)
    out = torch.zeros(B, K, device=d)
    z = torch.zeros(B * P, device=d)
    calls = [
        lambda: ops.gather_scale_rows(ids, None, V, rows, 1, K),
        lambda: ops.bag_sum_fwd(ids, None, off, V, out, K),
        lambda: ops.bag_sum_bwd(out, K, None, off, K, rows),
        lambda: ops.scale_rows(rows, None, None, B * P, K, 1, K, rows.clone()),
        lambda: ops.din_pool_fwd(rows, z, ids, B, P, K, z.clone(), out, K),
        lambda: ops.din_pool_bwd(rows, z, ids, out, K, B, P, K, rows.clone(), z.clone()),
    ]
    torch.cuda.synchronize()
    for i, call in enumerate(calls):
        n0 = _lib.launch_count()
        with pytest.raises(CtrError, match="K=12 unsupported"):
            call()
        assert _lib.launch_count() == n0, f"call {i} launched a kernel for K=12"


# ---------------------------------------------------------------------------------------------------------------------
# out-of-range bag ids: counted (TensorFlow's embedding_lookup_sparse raises), and they add nothing
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [4, 32, 256])
def test_bag_sum_fwd_counts_out_of_range_ids(K):
    from tf_repos_b200 import ops
    d = _dev()
    g = torch.Generator().manual_seed(K + 5)
    N, B = 300, 33
    bids, off, lens = _bags(B, N, g)
    bad = bids.clone()
    pos = torch.nonzero(lens > 2).reshape(-1)[:4]
    bad_at = torch.cat([off[pos].long(), off[pos].long() + 2])        # 8 bad occurrences in 4 bags
    bad[bad_at[:4]] = N
    bad[bad_at[4:]] = -1
    V = torch.randn(N, K, generator=g)
    oob = torch.zeros(2, dtype=torch.int32, device=d)
    out = torch.full((B, K), float("nan"), device=d)
    ops.bag_sum_fwd(bad.to(d), None, off.to(d), V.to(d), out, K, oob)
    cnt, first = oob.tolist()
    assert cnt == 8 and first in (N, -1), oob.tolist()
    # the good occurrences alone, in order (a bad one adds +0 * V[0], which leaves the partial sum as it is)
    good = torch.ones(bids.numel(), dtype=torch.bool)
    good[bad_at] = False
    keep_lens = torch.zeros(B, dtype=torch.int64).index_add(0, torch.repeat_interleave(torch.arange(B), lens), good.long())
    off_g = torch.zeros(B + 1, dtype=torch.int32)
    off_g[1:] = torch.cumsum(keep_lens, 0).to(torch.int32)
    assert torch.equal(out.cpu(), _seq_bag_sum(V, bids[good], off_g))
    # weighted: same count again, and the bad occurrences' weights do not reach the sum
    w = torch.rand(bids.numel(), generator=g) + 0.5
    oob.zero_()
    ops.bag_sum_fwd(bad.to(d), w.to(d), off.to(d), V.to(d), out, K, oob)
    assert oob[0].item() == 8
    wz = w.clone(); wz[bad_at] = 0
    seg = torch.repeat_interleave(torch.arange(B), lens)
    terms = V.double()[bids.long()] * wz.double()[:, None]
    ref = torch.zeros(B, K, dtype=torch.float64).index_add(0, seg, terms)
    mag = torch.zeros(B, K, dtype=torch.float64).index_add(0, seg, terms.abs())
    _within(out, ref, lens.double()[:, None] * U * mag, "weighted bag sum without the bad occurrences")
    # without a counter (the original entry point) the sums are the same and nothing is written
    out2 = torch.empty_like(out)
    ops.bag_sum_fwd(bad.to(d), w.to(d), off.to(d), V.to(d), out2, K)
    assert torch.equal(out2, out)


def _small_din(attn, B=32, P=9, N=500):
    from tf_repos_b200.din import DIN
    return DIN(11, N, 8, B, P, max_a_int=8, deep_layers="16,8", dropout="1.0,1.0", attention_pooling=attn,
               device="cuda:0")


def _cuda(batch):
    return {k: v.cuda() for k, v in batch.items()}


@pytest.mark.parametrize("bad_id", ["N", -1])
def test_din_check_ids_raises_for_a_bad_a_int_id(bad_id):
    from tf_repos_b200 import synth
    B, P, N = 32, 9, 500
    m = _small_din(True, B, P, N)
    bad = N if bad_id == "N" else -1
    batch, labels = synth.din_batch(B, N, 11, P, 8, seed=3)
    m.predict(_cuda(batch)); m.check_ids()                  # a clean batch passes
    batch["a_int_ids"][5] = bad
    m.predict(_cuda(batch))
    with pytest.raises(IndexError, match=f"first: {bad}"):
        m.check_ids()
    m.check_ids()                                           # the counter was reset
    m.train_step(_cuda(batch), labels.cuda())
    with pytest.raises(IndexError, match=r"^1 feature ids"):
        m.check_ids()


def test_din_check_ids_raises_for_a_bad_behaviour_id_without_attention():
    from tf_repos_b200 import synth
    B, P, N = 32, 9, 500
    m = _small_din(False, B, P, N)
    batch, labels = synth.din_batch(B, N, 11, P, 8, seed=4, fixed_len=True)
    batch["u_ids"][2, 7, 3] = N
    batch["u_ids"][0, 1, 0] = -1
    m.predict(_cuda(batch))
    with pytest.raises(IndexError, match=r"^2 feature ids"):
        m.check_ids()
    m.train_step(_cuda(batch), labels.cuda())
    with pytest.raises(IndexError, match=r"^2 feature ids"):
        m.check_ids()


# ---------------------------------------------------------------------------------------------------------------------
# DIN at the reference's default configuration (DIN.py:35-46) against the oracle
# ---------------------------------------------------------------------------------------------------------------------
DEF = dict(deep_layers="256,128,64", dropout="0.5,0.5,0.5", attention_layers="256", attention_pooling=True, l2_reg=1e-4,
           learning_rate=5e-4, optimizer="Adam")
DB, DN, DK, DFP, DP = 128, 20_000, 32, 11, 100
ATT = "Field-wise-Pooling-layer"


def _oracle(dtype):
    from oracle import models as om
    ref = om.DIN(DFP, DN, DK, seed=4, dtype=dtype, **DEF)
    g = torch.Generator().manual_seed(1)
    ref.params["embeddings"].copy_(torch.randn(DN, DK, generator=g) * 0.1)
    for p in ref.params.values():
        p.copy_(p.float().to(dtype))                        # both sides start from the same fp32 values
    return ref


def _gpu_din(mode="exact", epoch_steps=8):
    from tf_repos_b200.din import DIN
    return DIN(DFP, DN, DK, DB, DP, max_a_int=8, update_mode=mode, epoch_steps=epoch_steps, device="cuda:0", **DEF)


def _masks(step):
    g = torch.Generator().manual_seed(900 + step)
    att = [(torch.rand(DB * DP, 256, generator=g) < 0.5).float() for _ in range(4)]
    mlp = [(torch.rand(DB, w, generator=g) < 0.5).float() for w in (256, 128, 64)]
    cpu = {"att": att, "mlp": mlp}
    return cpu, {"att": [m.cuda() for m in att], "mlp": [m.cuda() for m in mlp]}


def _batch(step):
    from tf_repos_b200 import synth
    batch, labels = synth.din_batch(DB, DN, DFP, DP, 8, seed=300 + step)
    long = {k: (v.long() if v.dtype == torch.int32 else v) for k, v in batch.items()}
    return batch, long, labels


# One step's gradients pass through at most these rounded stages, each within its bound of the magnitude of the terms
# it sums (gemm_rel for GEMMs, n*U for fixed-order sums, the pooling's derivation above); to first order the
# gradient error is their sum.  Forward: grouped attention layer (R = 3K folded to K, 2 adds), att_out (R = 256 fmas),
# sigmoid (3*2^-23), pooling (P + 5 adds), MLP layers (R = 19K = 608, 256, 128) and the output (R = 64); backward: the
# same GEMMs' dIn (R = 64, 128, 256, 608), din_pool_bwd's dot (R = K), the attention dW over B*P rows split in
# chunks of <= 256 (+ <= 64 partial adds) and the four units' axpby sums (3 adds).  Evaluated: ~3.7e-4, against the
# largest magnitude of each gradient, which bounds the magnitude of its summed terms up to the cancellation that
# dW2 = dWc - dWd shows (scaled separately below).
TOL_GRAD = (gemm_rel(DK, 2) + 256 * U + 3 * TRUNC + (DP + 5) * U + gemm_rel(608) + gemm_rel(256) + gemm_rel(128)
            + gemm_rel(64) + gemm_rel(64) + gemm_rel(128) + gemm_rel(256) + gemm_rel(608) + (DK + 1) * U
            + gemm_rel(256, adds=64) + 3 * U)


def test_din_default_config_one_step_gradients_match_fp64():
    ref = _oracle(torch.float64)
    gpu = _gpu_din()
    gpu.load_variables(ref.params)
    batch, long, labels = _batch(0)
    mc, mg = _masks(0)
    _, out, _, dgrads = ref.gradients(long, labels, mc)
    gpu.train_step(_cuda(batch), labels.cuda(), masks=mg)
    gpu.check_ids()
    torch.cuda.synchronize()
    assert set(dgrads) == set(gpu.dense.grads), (sorted(dgrads), sorted(gpu.dense.grads))
    for name, gref in dgrads.items():
        got = gpu.dense.grads[name].cpu()
        if name == f"{ATT}/att_fc0/weights":
            K = DK
            for blk, sl in (("dW1 = dWc", slice(0, K)), ("dW3 = dWd", slice(2 * K, 3 * K))):
                _within(got[sl], gref[sl], TOL_GRAD * gref[sl].abs().max(), f"{name} {blk}")
            # dW2 = dWc - dWd cancels: the errors of both operands stay, so the bound scales with |dWc| + |dWd|
            scale = gref[:K].abs().max() + gref[2 * K:].abs().max()
            _within(got[K:2 * K], gref[K:2 * K], TOL_GRAD * scale, f"{name} dW2 = dWc - dWd")
        else:
            _within(got, gref.reshape(got.shape), TOL_GRAD * gref.abs().max(), name)
    per = out["per_occurrence"]
    g = gpu.g_all.cpu()
    s = gpu.seg
    segs = [("common", "common", DB * DFP), ("a0", "a_cat", DB), ("a1", "a_shop", DB), ("a2", "a_brand", DB),
            ("a_int", "a_int", long["a_int_ids"].numel())]
    segs += [(f"u{f}", f"u_{nm}", DB * DP) for f, nm in enumerate(("cat", "shop", "brand", "int"))]
    for seg, site, n in segs:
        o = s[seg][0]
        r = per[site].reshape(n, DK)
        _within(g[o:o + n], r, TOL_GRAD * r.abs().max(), f"per-occurrence rows {site}")
    o, n = s["a_int"]
    nnz = long["a_int_ids"].numel()
    assert torch.all(g[o + nnz:o + n] == 0)


def _state(m):
    m.flush()
    out = [m.V.var] + list(m.V.slots) + [m.dense.flat] + list(m.dense.slots)
    return [t.clone() for t in out]


@pytest.mark.parametrize("mode", ["exact", "exact_deferred"])
def test_din_default_config_three_steps_match_the_fp32_oracle(mode):
    ref = _oracle(torch.float32)
    gpu = _gpu_din(mode, epoch_steps=2)
    gpu.load_variables(ref.params)
    for step in range(3):
        batch, long, labels = _batch(step)
        mc, mg = _masks(step)
        ref.train_step(long, labels, mc)
        gpu.train_step(_cuda(batch), labels.cuda(), masks=mg)
        gpu.check_ids()
        vs = gpu.variables()
        for name, want in ref.params.items():
            # the tolerance test_gpu_din.py holds DIN's parameters to
            got, want = vs[name].cpu().double().numpy(), want.double().numpy()
            np.testing.assert_allclose(got.reshape(want.shape), want, rtol=2e-5, atol=2e-5 * max(np.abs(want).max(), 1e-30),
                                       err_msg=f"{name} after step {step} ({mode})")


def test_din_default_config_deferred_equals_exact_bit_for_bit():
    a = _gpu_din("exact")
    b = _gpu_din("exact_deferred", epoch_steps=4)
    ref = _oracle(torch.float32)
    a.load_variables(ref.params); b.load_variables(ref.params)
    for step in range(8):                                   # two epochs
        batch, _, labels = _batch(10 + step)
        _, mg = _masks(10 + step)
        la = a.train_step(_cuda(batch), labels.cuda(), masks=mg)
        lb = b.train_step(_cuda(batch), labels.cuda(), masks=mg)
        assert torch.equal(la[0], lb[0]), f"CE differs at step {step}"
        if step in (1, 5):                                  # mid-epoch flushes
            for x, y in zip(_state(a), _state(b)):
                _bits_equal(y, x, f"exact_deferred vs exact after step {step}")
    for x, y in zip(_state(a), _state(b)):
        _bits_equal(y, x, "exact_deferred vs exact after two epochs")


def test_din_default_config_is_bit_reproducible():
    ref = _oracle(torch.float32)
    states = []
    for _ in range(2):
        m = _gpu_din("exact")
        m.load_variables(ref.params)
        for step in range(3):
            batch, _, labels = _batch(20 + step)
            _, mg = _masks(20 + step)
            m.train_step(_cuda(batch), labels.cuda(), masks=mg)
        states.append(_state(m) + [m.g_all.clone(), m.dense.grad.clone()])
    for x, y in zip(*states):
        _bits_equal(y, x, "two fresh models")
