"""The wgmma 3xTF32 GEMM (tc_gemm.cu) behind every dense layer, through the entry points the models use: ops.fc_fwd,
ops.fc_fwd_grouped and ops.fc_bwd.

A. Exact known answers.  The operands are built on a grid (tests/tf32_oracle.py) on which the exact product is an fp32
   number and any 24-bit accumulator reaches it whatever its rounding: every output, including the fused epilogues
   (bias, group bias, relu, dropout, accumulate), the dZ pass, the bias gradient and the split-R reduce, is compared bit
   for bit.  A kernel that drops a cross term, reads the wrong lo slice or loses an element on a fallback path fails.
   The layers cover every BN class x interior/edge tile x aligned/misaligned x one/two-stage combination.
B. Bit identities on normal data: moving rows or columns across tiles, misaligned copies and a second call leave the
   bits unchanged.
C. fp64 accuracy at the reference's layer shapes: max |C - C64| / (|A| |B|) under 1/16 of the best of plain TF32 and
   the two 2xTF32 emulations on the same data, so a kernel that drops a cross term cannot pass.
D. Contracts: M = 0 is a no-op, bad arguments raise CtrError.
"""
import numpy as np
import pytest
import torch

from tests import tf32_oracle as o
from tests.test_gpu_din_attention import _bits_equal, _sm_count

pytestmark = pytest.mark.gpu

NAN = float("nan")


def _dev():
    return torch.device("cuda:0")


class Buf:
    """A contiguous tensor placed `off` floats into a larger buffer whose guard cells hold a sentinel: a view that is not
    16 B-aligned when off % 4 != 0, and a check that nothing outside it was written."""

    def __init__(self, shape, off, fill=NAN, data=None):
        n = int(np.prod(shape))
        self.off, self.n = off, n
        self.raw = torch.full((off + n + 4,), -7.25, dtype=torch.float32, device=_dev())
        self.t = self.raw[off:off + n].view(*shape)
        if data is not None:
            self.t.copy_(torch.from_numpy(np.ascontiguousarray(data, dtype=np.float32)).view(*shape))
        else:
            self.t.fill_(fill)

    def guards_intact(self, what):
        g = torch.cat([self.raw[:self.off], self.raw[self.off + self.n:]]).cpu()
        assert torch.all(g == -7.25), f"{what}: a write landed outside the output"

    def np(self):
        return self.t.cpu().numpy()


def _exact_equal(got, want, what):
    got = got.detach().cpu() if torch.is_tensor(got) else torch.from_numpy(np.ascontiguousarray(got))
    want = torch.from_numpy(np.ascontiguousarray(want, dtype=np.float32))
    if not torch.equal(got.contiguous().view(torch.int32), want.view(torch.int32)):
        d = (got.view(torch.int32) != want.view(torch.int32))
        i = tuple(int(v) for v in torch.nonzero(d)[0])
        raise AssertionError(f"{what}: {int(d.sum())} of {d.numel()} elements differ in their bits; first at {i}: "
                             f"got {float(got[i])!r} want {float(want[i])!r}")


def _f32(x):
    return np.asarray(x, dtype=np.float32)


def _mm(A, B):
    """The exact product in fp64; + 0.0 turns a -0 sum of -0 products into the +0 the kernel's accumulator holds."""
    return np.asarray(A, np.float64) @ np.asarray(B, np.float64) + 0.0


def _colsum(Z):
    return np.asarray(Z, np.float64).sum(0) + 0.0


def _epilogue_ref(C, bias, gbias, gP, act, mask, keep):
    """tc_epilogue_rows EPI 1 in fp32: ((C + b) + gb[i/gP]), relu, then v / keep * mask (IEEE division)."""
    v = _f32(C)
    if bias is not None:
        v = _f32(v + bias[None, :])
    if gbias is not None:
        v = _f32(v + gbias[np.arange(v.shape[0]) // gP])
    if act == 1:
        v = np.maximum(v, np.float32(0))
    if mask is not None:
        v = _f32(_f32(v / np.float32(keep)) * mask)
    return v


def _ws(M, Kd, Nd):
    return torch.empty(max(ops().fc_bwd_workspace_bytes(M, Kd, Nd), 16), dtype=torch.uint8, device=_dev())


def ops():
    from tf_repos_b200 import ops as _ops
    return _ops


# ---------------------------------------------------------------------------------------------------------------------
# A. exact known answers over the covering design
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", o.covering_cases(), ids=o.case_id)
def test_exact_layer(case):
    c = case
    M, Kd, Nd, act, keep, gP = c["M"], c["Kd"], c["Nd"], c["act"], c["keep"], c["group_P"]
    rng = np.random.default_rng(1000 + c["i"])
    x, W, dOut = o.exact_layer(rng, M, Kd, Nd, c["lo"])
    o.assert_exact(x, W, "fwd")
    bias = o.grid_lo(rng, Nd) if c["bias"] else None
    gbias = o.grid_lo(rng, (-(-M // gP), Nd)) if gP else None
    mask = (rng.random((M, Nd)) < keep).astype(np.float32) if keep else None
    off = o.offsets(c)

    # forward: act(in @ W + b + gb[i / P]) (/ keep * mask)
    bx, bW, bout = Buf((M, Kd), off[0], data=x), Buf((Kd, Nd), off[1], data=W), Buf((M, Nd), off[2])
    bmask = Buf((M, Nd), off[3], data=mask) if keep else None
    tb = torch.from_numpy(bias).to(_dev()) if c["bias"] else None
    if gP:
        ops().fc_fwd_grouped(bx.t, bW.t, tb, torch.from_numpy(gbias).to(_dev()), gP, bmask and bmask.t, keep or 1.0,
                             act, bout.t)
    else:
        ops().fc_fwd(bx.t, bW.t, tb, bmask and bmask.t, keep or 1.0, act, bout.t)
    C = _mm(x, W)
    out = _epilogue_ref(C, bias, gbias, gP, act, mask, keep)
    _exact_equal(bout.t, out, f"fwd {o.case_id(c)}")
    bout.guards_intact("fwd out")

    # backward: dZ = dOut (* mask / 0.5) * (out > 0) in place, db = colsum dZ, dW = in^T dZ, dIn (+)= dZ W^T
    bmask_b = bmask if keep == 0.5 else None
    dZ = dOut.copy()
    if bmask_b is not None:
        dZ = _f32(_f32(dZ * mask) / np.float32(0.5))
    if act == 1:
        dZ = np.where(out > 0, dZ, np.float32(0)).astype(np.float32)
    o.assert_exact(dZ, W.T, "dIn")
    o.assert_exact(x.T, dZ, "dW")
    old = o.grid_lo(rng, (M, Kd)) if c["accumulate_din"] else None
    bdO = Buf((M, Nd), off[4], data=dOut)
    bdIn = Buf((M, Kd), off[2], data=old) if c["accumulate_din"] else Buf((M, Kd), off[2])
    bdW, bdb = Buf((Kd, Nd), off[5]), Buf((Nd,), off[5])
    ops().fc_bwd(bx.t, bW.t, bout.t, bmask_b and bmask_b.t, 0.5 if bmask_b else 1.0, bdO.t, act, bdIn.t, bdW.t,
                 bdb.t, _ws(M, Kd, Nd), accumulate_din=c["accumulate_din"])
    _exact_equal(bdO.t, dZ, "dZ in place")
    _exact_equal(bdb.t, _colsum(dZ), "db")
    _exact_equal(bdW.t, _mm(x.T, dZ), f"dW (S={o.dw_split(M, Kd, Nd, _sm_count())[0]})")
    dIn = _mm(dZ, W.T)
    _exact_equal(bdIn.t, _f32(dIn) + old if c["accumulate_din"] else dIn, "dIn")
    for b, what in ((bdO, "dOut"), (bdIn, "dIn"), (bdW, "dW"), (bdb, "db")):
        b.guards_intact(what)


def test_exact_relu_boundary():
    """Pre-activations exactly 0 (and exactly +-2^-11): relu gives +0 and the dZ pass zeroes the gradient where
    out == 0; act 2 takes dOut as dZ and leaves it (and db) untouched."""
    rng = np.random.default_rng(7)
    M, Kd, Nd = 300, 40, 96
    x = o.grid_int(rng, (M, Kd), 0.1, vmax=1)
    W = o.grid_lo(rng, (Kd, Nd), 0.2)
    bias = np.zeros(Nd, np.float32)
    bias[::3] = o.GRID
    d = _dev()
    out = torch.full((M, Nd), NAN, device=d)
    ops().fc_fwd(torch.from_numpy(x).to(d), torch.from_numpy(W).to(d), torch.from_numpy(bias).to(d), None, 1.0, 1, out)
    pre = _f32(_mm(x, W)) + bias
    assert (pre == 0).mean() > 0.2 and (pre > 0).any() and (pre < 0).any()
    _exact_equal(out, np.maximum(pre, np.float32(0)), "relu at 0")
    dOut = o.grid_int(rng, (M, Nd), 0.05)
    dOut[dOut == 0] = 1.0          # a gradient everywhere, so that a wrong gate at out == 0 shows
    dO = torch.from_numpy(dOut).to(d)
    dW, db = torch.full((Kd, Nd), NAN, device=d), torch.full((Nd,), NAN, device=d)
    ops().fc_bwd(torch.from_numpy(x).to(d), torch.from_numpy(W).to(d), out, None, 1.0, dO, 1, None, dW, db,
                 _ws(M, Kd, Nd))
    dZ = np.where(pre > 0, dOut, np.float32(0)).astype(np.float32)
    _exact_equal(dO, dZ, "dZ gated at out == 0")
    _exact_equal(db, _colsum(dZ), "db")
    # act 2: dOut already holds dZ, no dZ pass, db untouched
    dO2, db2 = torch.from_numpy(dOut).to(d), torch.full((Nd,), NAN, device=d)
    dIn2 = torch.full((M, Kd), NAN, device=d)
    ops().fc_bwd(torch.from_numpy(x).to(d), torch.from_numpy(W).to(d), None, None, 1.0, dO2, 2, dIn2, dW, db2,
                 _ws(M, Kd, Nd))
    _exact_equal(dO2, dOut, "act 2 leaves dOut")
    assert torch.isnan(db2).all(), "act 2 wrote db"
    _exact_equal(dW, _mm(x.T, dOut), "dW from act 2")
    _exact_equal(dIn2, _mm(dOut, W.T), "dIn from act 2")


@pytest.mark.parametrize("lo", ["in", "dOut"])
@pytest.mark.parametrize("split", o.DW_SPLITS)
@pytest.mark.parametrize("shape", o.DW_EDGES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_exact_dw_edges(shape, split, lo):
    """dW plain and transposed at the edges of the transposed rule, with one chunk, a middle split whose chunk is not
    a multiple of 4, and the 64-chunk cap with a short last chunk."""
    Kd, Nd = shape
    sm = _sm_count()
    M = o.dw_edge_m(Kd, Nd, split, sm)
    S, chunk = o.dw_split(M, Kd, Nd, sm)
    assert (S == 1) == (split == "one")
    rng = np.random.default_rng(Kd * 1000 + Nd + len(split) + len(lo))
    x, W, dOut = o.exact_layer(rng, M, Kd, Nd, lo)
    o.assert_exact(x.T, dOut, "dW")
    d = _dev()
    dO = torch.from_numpy(dOut).to(d)
    dW, db, dIn = torch.full((Kd, Nd), NAN, device=d), torch.full((Nd,), NAN, device=d), torch.full((M, Kd), NAN, device=d)
    out = torch.ones((M, Nd), device=d)
    ops().fc_bwd(torch.from_numpy(x).to(d), torch.from_numpy(W).to(d), out, None, 1.0, dO, 0, dIn, dW, db, _ws(M, Kd, Nd))
    what = f"M={M} S={S} chunk={chunk} {'transposed' if o.dw_transposed(Kd, Nd) else 'plain'}"
    _exact_equal(dW, _mm(x.T, dOut), f"dW {what}")
    _exact_equal(db, _colsum(dOut), f"db {what}")
    _exact_equal(dIn, _mm(dOut, W.T), f"dIn {what}")


@pytest.mark.parametrize("lo", ["in", "dOut"])
@pytest.mark.parametrize("case", o.LONG_DW, ids=lambda c: c[0].replace(" ", "_"))
def test_exact_long_dw(case, lo):
    """The longest dW reductions of the reference's models (split into 64 chunks of 6400 / 1482 rows) on sparse dZ."""
    import scipy.sparse as sp
    name, M, Kd, Nd, per_col = case
    S, chunk = o.dw_split(M, Kd, Nd, _sm_count())
    rng = np.random.default_rng(M + len(lo))
    x = o.grid_lo(rng, (M, Kd)) if lo == "in" else o.grid_int(rng, (M, Kd))
    rows, cols, vals = o.sparse_dz(rng, M, Nd, per_col, lo)
    d = _dev()
    dO = torch.zeros((M, Nd), device=d)
    dO[torch.from_numpy(rows).to(d), torch.from_numpy(cols).to(d)] = torch.from_numpy(vals).to(d)
    dW = torch.full((Kd, Nd), NAN, device=d)
    ops().fc_bwd(torch.from_numpy(x).to(d), torch.empty((Kd, Nd), device=d), None, None, 1.0, dO, 2, None, dW, None,
                 _ws(M, Kd, Nd))
    Z = sp.csc_matrix((vals.astype(np.float64), (rows, cols)), shape=(M, Nd))
    want = np.asarray((Z.T @ x.astype(np.float64)).T) + 0.0
    assert np.abs(np.asarray((abs(Z).T @ np.abs(x.astype(np.float64))))).max() <= o.EXACT_LIMIT
    _exact_equal(dW, want, f"{name} dW S={S} chunk={chunk}")


# ---------------------------------------------------------------------------------------------------------------------
# B. bit identities on normal data
# ---------------------------------------------------------------------------------------------------------------------
def _layer(rng, M, Kd, Nd, keep=0.5):
    x = rng.standard_normal((M, Kd)).astype(np.float32)
    W = (rng.standard_normal((Kd, Nd)) / np.sqrt(Kd)).astype(np.float32)
    b = (rng.standard_normal(Nd) * 0.1).astype(np.float32)
    mask = (rng.random((M, Nd)) < keep).astype(np.float32)
    dOut = rng.standard_normal((M, Nd)).astype(np.float32)
    return x, W, b, mask, dOut


def _run(x, W, b, mask, dOut, keep=0.5, act=1, offs=(0,) * 8, accumulate_din=None):
    """fwd + bwd on device copies placed at the given float offsets; returns numpy out, dZ, dIn, dW, db."""
    M, Kd = x.shape
    Nd = W.shape[1]
    bx, bW, bb = Buf((M, Kd), offs[0], data=x), Buf((Kd, Nd), offs[1], data=W), Buf((Nd,), offs[2], data=b)
    bm, bo = Buf((M, Nd), offs[3], data=mask), Buf((M, Nd), offs[4])
    ops().fc_fwd(bx.t, bW.t, bb.t, bm.t, keep, act, bo.t)
    bd = Buf((M, Nd), offs[5], data=dOut)
    bdIn = Buf((M, Kd), offs[6], data=accumulate_din) if accumulate_din is not None else Buf((M, Kd), offs[6])
    bdW, bdb = Buf((Kd, Nd), offs[7]), Buf((Nd,), offs[7])
    ops().fc_bwd(bx.t, bW.t, bo.t, bm.t, keep, bd.t, act, bdIn.t, bdW.t, bdb.t, _ws(M, Kd, Nd),
                 accumulate_din=accumulate_din is not None)
    return bo.np(), bd.np(), bdIn.np(), bdW.np(), bdb.np()


def _bits(a, b, what):
    _bits_equal(torch.from_numpy(np.ascontiguousarray(a)), torch.from_numpy(np.ascontiguousarray(b)), what)


@pytest.mark.parametrize("z", [1, 64, 127])
def test_rows_shift(z):
    """Prepending z rows to in / mask / dOut moves every row across warpgroup halves, tile edges and fast/slow loads:
    out[z:] and dIn[z:] (and dZ) keep their bits."""
    rng = np.random.default_rng(z)
    M, Kd, Nd = 300, 256, 200
    x, W, b, mask, dOut = _layer(rng, M + z, Kd, Nd)
    base = _run(x[z:], W, b, mask[z:], dOut[z:])
    shifted = _run(x, W, b, mask, dOut)
    for k, what in ((0, "out"), (1, "dZ"), (2, "dIn")):
        _bits(shifted[k][z:], base[k], f"{what} with {z} rows prepended")


@pytest.mark.parametrize("z", [1, 3])
def test_cols_shift(z):
    """Columns prepended to Wt (N 200 -> 200 + z, one BN class, the same dW split) shift out, dZ, dW and db; rows
    prepended to Wt and columns to in (Kd 200 -> 200 + z) shift dIn's columns and dW's rows."""
    rng = np.random.default_rng(10 + z)
    M, Kd, Nd = 777, 200, 200
    sm = _sm_count()
    x, W, b, mask, dOut = _layer(rng, M, Kd + z, Nd + z)
    assert o.dw_split(M, Kd, Nd, sm) == o.dw_split(M, Kd, Nd + z, sm) == o.dw_split(M, Kd + z, Nd, sm)
    base = _run(x[:, z:], W[z:, z:], b[z:], mask[:, z:], dOut[:, z:])
    wide = _run(x[:, z:], W[z:], b, mask, dOut)
    for k, what in ((0, "out"), (1, "dZ"), (3, "dW"), (4, "db")):
        _bits(wide[k][..., z:], base[k], f"{what} with {z} output columns prepended")
    # act 0: dZ does not depend on the forward, whose reduction the extra input columns change
    base0 = _run(x[:, z:], W[z:, z:], b[z:], mask[:, z:], dOut[:, z:], act=0)
    deep = _run(x, W[:, z:], b[z:], mask[:, z:], dOut[:, z:], act=0)
    _bits(deep[2][:, z:], base0[2], f"dIn with {z} input columns prepended")
    _bits(deep[3][z:], base0[3], f"dW with {z} input columns prepended")


@pytest.mark.parametrize("shape", [(1000, 256, 128), (300, 64, 256), (8192, 624, 256)])
def test_misaligned_and_repeat(shape):
    """Misaligned copies of every operand take the load_tile fallback and the scalar epilogue: same bits as the
    aligned call.  A second aligned call repeats them too (split-R dW and db included)."""
    M, Kd, Nd = shape
    rng = np.random.default_rng(M)
    x, W, b, mask, dOut = _layer(rng, M, Kd, Nd)
    old = rng.standard_normal((M, Kd)).astype(np.float32)
    ref = _run(x, W, b, mask, dOut, accumulate_din=old)
    again = _run(x, W, b, mask, dOut, accumulate_din=old)
    mis = _run(x, W, b, mask, dOut, offs=(1, 2, 3, 1, 2, 3, 1, 2), accumulate_din=old)
    for k, what in enumerate(("out", "dZ", "dIn", "dW", "db")):
        _bits(again[k], ref[k], f"{what} on a second call")
        _bits(mis[k], ref[k], f"{what} from misaligned operands")


# ---------------------------------------------------------------------------------------------------------------------
# C. fp64 accuracy at the reference's layer shapes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layer", o.accuracy_layers(), ids=lambda l: f"{l[0].replace(' ', '_')}-L{l[1]}")
def test_accuracy(layer):
    name, i, M, Kd, Nd = layer
    x, W, dZ = o.accuracy_operands(M, Kd, Nd, i, seed=i)
    d = _dev()
    tx, tW, tdZ = (torch.from_numpy(a).to(d) for a in (x, W, dZ))
    out = torch.full((M, Nd), NAN, device=d)
    ops().fc_fwd(tx, tW, None, None, 1.0, 0, out)
    dIn, dW = torch.full((M, Kd), NAN, device=d), torch.full((Kd, Nd), NAN, device=d)
    ops().fc_bwd(tx, tW, None, None, 1.0, tdZ, 2, dIn, dW, None, _ws(M, Kd, Nd))
    got = {"fwd": out, "dIn": dIn, "dW": dW, "dW^T": dW.T}
    for p, A, B, chunk in o.products(x, W, dZ, _sm_count()):
        broken, C64, mag = o.broken_metrics(A, B)
        tol = min(broken.values()) / 16
        err = o.rel_metric(got[p].cpu().numpy(), A, B, C64, mag)
        print(f"RATIO {name} layer {i} {p} ({A.shape[0]}x{A.shape[1]}x{B.shape[1]}, chunk {chunk}): kernel {err:.3e} "
              f"tol {tol:.3e} best broken {min(broken.values()):.3e} -> {err / tol:.3g}")
        assert err <= tol, f"{name} layer {i} {p}: {err:.3e} > {tol:.3e} ({broken})"


# ---------------------------------------------------------------------------------------------------------------------
# D. contracts
# ---------------------------------------------------------------------------------------------------------------------
def test_empty_and_bad_arguments():
    from tf_repos_b200._lib import CtrError
    d = _dev()
    Kd, Nd = 16, 32
    W, x0 = torch.randn(Kd, Nd, device=d), torch.empty(0, Kd, device=d)
    out, dW, db = torch.full((4, Nd), NAN, device=d), torch.full((Kd, Nd), NAN, device=d), torch.full((Nd,), NAN, device=d)
    ops().fc_fwd(x0, W, None, None, 1.0, 1, out)
    ops().fc_fwd_grouped(x0, W, None, out, 3, None, 1.0, 1, out)
    ops().fc_bwd(x0, W, out, None, 1.0, out, 1, out, dW, db, torch.empty(16, dtype=torch.uint8, device=d))
    torch.cuda.synchronize()
    assert torch.isnan(out).all() and torch.isnan(dW).all() and torch.isnan(db).all(), "M = 0 wrote an output"
    x = torch.randn(4, Kd, device=d)
    mask = torch.ones(4, Nd, device=d)
    ws = _ws(4, Kd, Nd)
    with pytest.raises(CtrError):
        ops().fc_fwd(x, W, None, None, 1.0, 2, out)                                  # act 2 is backward-only
    with pytest.raises(CtrError):
        ops().fc_fwd(x, W, None, None, 1.0, -1, out)
    with pytest.raises(CtrError):
        ops().fc_fwd(torch.empty(4, 0, device=d), torch.empty(0, Nd, device=d), None, None, 1.0, 0, out)   # Kd = 0
    with pytest.raises(CtrError):
        ops().fc_fwd_grouped(x, W, None, out, 0, None, 1.0, 0, out)                  # group_P = 0
    for keep in (0.0, -0.5):
        with pytest.raises(CtrError):
            ops().fc_fwd(x, W, None, mask, keep, 0, out)
        with pytest.raises(CtrError):
            ops().fc_bwd(x, W, out, mask, keep, out.clone(), 1, None, dW, db, ws)
    with pytest.raises(CtrError):
        ops().fc_bwd(x, W, out, None, 1.0, out.clone(), 3, None, dW, db, ws)
    with pytest.raises(CtrError):
        ops().fc_bwd(torch.empty(4, 0, device=d), torch.empty(0, Nd, device=d), out, None, 1.0, out.clone(), 0, None,
                     torch.empty(0, Nd, device=d), db, ws)
    with pytest.raises(CtrError):
        ops().fc_bwd(x, W, out, None, 1.0, out.clone(), 1, None, dW, db, ws[:ws.numel() - 4])
    torch.cuda.synchronize()
