"""wide_n_deep's kernels one by one, against exact restatements or fp64, at the reference's default configuration
(wide_n_deep.py:31-34: embedding_size=32, batch_size=128, deep_layers=256,128,64) and at the edges of their dispatch:

  ctr_wd_input_fwd / ctr_wd_input_bwd (csrc/wide_deep.cu): the stacked flat ids f*NB + id, out-of-range ids -> bucket 0
      of their own column, the name-sorted numeric order, the linear sum, the per-occurrence gradients and the fixed
      tree of the dense linear gradients;
  ctr_segment_sum_rows (csrc/segment_sum.cu) on the paths only wide_n_deep reaches: K = 1 and other generic K, the
      non-split long-run kernel, the split kernel when its scratch runs out (base = -1) and the CTR_LONG_SEG boundary;
  the first DNN layer's D = 26*32 + 13 = 845 inputs (lda % 4 != 0, ldc = 845) and the 256 -> 128 -> 64 layers;
  the three models at the reference's default configuration against oracle/wide_deep.py run in fp64.

Error bounds (each comparison states which one and why):
  U = 2^-24 is the unit roundoff of one round-to-nearest fp32 operation.  A value computed with n rounded operations
  chained along any one path of a fixed summation tree is within gamma(n) = n*U/(1 - n*U) of the exact result,
  relative to the sum of the absolute values of its terms (Higham, Accuracy and Stability, 4.2).  A fused
  multiply-add rounds once.  gemm_rel is the 3xTF32 product bound derived in test_gpu_din_attention.py.
"""
import math

import numpy as np
import pytest
import torch

from tests.test_gpu_din_attention import U, _bits_equal, _np, _pick_split, _within, gemm_rel

pytestmark = pytest.mark.gpu

I32_MAX, I32_MIN = 2 ** 31 - 1, -2 ** 31
LONG_SEG = 128          # CTR_LONG_SEG: a run longer than this leaves the short kernel
SEG_CHUNK = 1024        # segment_sum.cu: occurrences per partial row of the split long-run path
# input_layer / linear_model order columns by name: I1, I10, I11, I12, I13, I2, ..., I9 (as indices into I1..I13)
NUM_NAME_SORTED = [0, 9, 10, 11, 12, 1, 2, 3, 4, 5, 6, 7, 8]


def _dev():
    return torch.device("cuda:0")


def gamma(n):
    return n * U / (1 - n * U)


def _check(got, ref, bound, what):
    """_within, and the largest err/bound ratio printed (pytest -s shows the margin of every bounded comparison)."""
    _within(got, ref, bound, what)
    err, b = np.abs(_np(got) - _np(ref)), np.broadcast_to(_np(bound), np.shape(_np(ref)))
    r = float(np.max(np.where(b > 0, err / np.maximum(b, 1e-300), 0.0))) if err.size else 0.0
    print(f"RATIO {what}: {r:.3g}")


# ---------------------------------------------------------------------------------------------------------------------
# ctr_wd_input_fwd: flat ids, the DNN input row and the linear part's per-sample sum
# ---------------------------------------------------------------------------------------------------------------------
def _ids(B, Fc, NB, g):
    """Random in-range ids, with every special value present: 0, NB-1, NB, -1, INT32_MAX, INT32_MIN first, then
    again at random places."""
    ids = torch.randint(0, NB, (B * Fc,), generator=g, dtype=torch.int64)
    special = torch.tensor([0, NB - 1, NB, -1, I32_MAX, I32_MIN], dtype=torch.int64)
    ids[: min(6, ids.numel())] = special[: min(6, ids.numel())]
    at = torch.randint(0, ids.numel(), (max(ids.numel() // 20, 1),), generator=g)
    ids[at] = special[torch.randint(0, 6, (at.numel(),), generator=g)]
    return ids.to(torch.int32).reshape(B, Fc)


def _fwd_case(B, Fc, Fd, K, NB, seed):
    g = torch.Generator().manual_seed(seed)
    d = _dev()
    perm = list(range(Fd))
    if Fd == 13:
        perm = NUM_NAME_SORTED
    elif Fd:
        perm = torch.randperm(Fd, generator=g).tolist()
    case = dict(
        ids=_ids(B, Fc, NB, g), dense=torch.randn(B, Fd, generator=g),
        emb=torch.randn(Fc * NB, K, generator=torch.Generator(device=d).manual_seed(seed), device=d),
        wide_cat=torch.randn(Fc * NB, generator=g), wide_num=torch.randn(Fd, generator=g),
        wide_bias=torch.randn(1, generator=g), num_perm=torch.tensor(perm, dtype=torch.int32))
    return {k: v.to(d) for k, v in case.items()}


def _fwd_ref(c, NB, with_bias=True):
    ids = c["ids"].cpu().long()
    B, Fc = ids.shape
    clamped = torch.where((ids < 0) | (ids >= NB), torch.zeros_like(ids), ids)
    flat = (torch.arange(Fc) * NB + clamped).to(torch.int32)
    x = torch.cat([c["emb"][flat.reshape(-1).long().to(c["emb"].device)].reshape(B, -1).cpu(),
                   c["dense"].cpu()[:, c["num_perm"].cpu().long()]], 1)
    cat64 = c["wide_cat"].cpu().double()[flat.long()]
    num64 = c["dense"].cpu().double() * c["wide_num"].cpu().double()
    bias64 = c["wide_bias"].cpu().double() if with_bias else torch.zeros(1, dtype=torch.float64)
    lin = cat64.sum(1) + num64.sum(1) + bias64
    mag = cat64.abs().sum(1) + num64.abs().sum(1) + bias64.abs()
    # each lane adds its ceil(Fc/32) table weights, then fmas its ceil(Fd/32) numeric terms; 5 butterfly levels; + bias
    n_ops = -(-Fc // 32) + -(-c["dense"].shape[1] // 32) + 5 + 1
    return flat, x, lin, gamma(n_ops) * mag


def _run_fwd(c, NB, K, emb=True, wide=True, bias=True):
    from tf_repos_b200 import ops
    B, Fc = c["ids"].shape
    Fd = c["dense"].shape[1]
    d = _dev()
    flat = torch.full((B, Fc), -7, dtype=torch.int32, device=d)
    x = torch.full((B, Fc * K + Fd), float("nan"), device=d) if emb else None
    lin = torch.full((B,), float("nan"), device=d) if wide else None
    ops.wd_input_fwd(c["ids"], c["dense"], c["emb"] if emb else None, c["wide_cat"] if wide else None,
                     c["wide_num"] if wide else None, c["wide_bias"] if (wide and bias) else None, c["num_perm"], NB, K,
                     flat, x, lin)
    return flat, x, lin


def test_numeric_columns_are_name_sorted():
    """The model and the oracle both derive the numeric order with sorted(); pin it to the literal name order."""
    from oracle import wide_deep as owd
    from tf_repos_b200 import wide_deep
    assert wide_deep.NUM_SORTED == NUM_NAME_SORTED
    assert owd.NUM_SORTED == NUM_NAME_SORTED


# every value of each axis is covered, plus the reference point (Fc, Fd, K, NB) = (26, 13, 32, 10000) at B = 128
@pytest.mark.parametrize("B,Fc,Fd,K,NB", [
    (128, 26, 13, 32, 10000),     # the reference default
    (1, 1, 0, 1, 1),              # one id, no numerics, a one-bucket column: every id but 0 is out of range
    (7, 33, 40, 33, 10000),       # Fc and Fd above a warp: lanes take two columns; K not a multiple of 4
    (8193, 26, 13, 8, 10000),     # B one past a multiple of the 8 warps of a CTA
    (128, 70, 40, 256, 1),        # three column rounds per lane, x rows of 17960
    (8193, 1, 40, 256, 10000),
    (1, 70, 13, 1, 10000),
    (7, 32, 0, 32, 1),
])
def test_wd_input_fwd(B, Fc, Fd, K, NB):
    c = _fwd_case(B, Fc, Fd, K, NB, seed=B * 7 + Fc * 5 + Fd * 3 + K + NB)
    flat_ref, x_ref, lin_ref, bound = _fwd_ref(c, NB)
    flat, x, lin = _run_fwd(c, NB, K)
    _bits_equal(flat, flat_ref, f"flat_ids B={B} Fc={Fc} NB={NB}")
    _bits_equal(x, x_ref, f"x B={B} Fc={Fc} Fd={Fd} K={K}")
    _check(lin, lin_ref, bound, f"lin B={B} Fc={Fc} Fd={Fd}")
    flat2, x2, lin2 = _run_fwd(c, NB, K)
    _bits_equal(lin2, lin, "lin on a second call")


def test_wd_input_fwd_pointer_combinations_and_empty_batch():
    """emb only (DNNClassifier), wide only (LinearClassifier), both, and no bias; B = 0 writes nothing."""
    from tf_repos_b200 import ops
    B, Fc, Fd, K, NB = 128, 26, 13, 32, 10000
    c = _fwd_case(B, Fc, Fd, K, NB, seed=11)
    flat_ref, x_ref, lin_ref, bound = _fwd_ref(c, NB)
    _, _, lin_nb_ref, bound_nb = _fwd_ref(c, NB, with_bias=False)
    for emb, wide, bias in ((True, False, False), (False, True, True), (True, True, True), (True, True, False)):
        what = f"emb={emb} wide={wide} bias={bias}"
        flat, x, lin = _run_fwd(c, NB, K, emb=emb, wide=wide, bias=bias)
        _bits_equal(flat, flat_ref, f"flat_ids {what}")
        if emb:
            _bits_equal(x, x_ref, f"x {what}")
        if wide:
            _check(lin, lin_ref if bias else lin_nb_ref, bound if bias else bound_nb, f"lin {what}")
    d = _dev()
    flat = torch.full((B, Fc), -7, dtype=torch.int32, device=d)
    x = torch.full((B, Fc * K + Fd), float("nan"), device=d)
    lin = torch.full((B,), float("nan"), device=d)
    ops.wd_input_fwd(c["ids"][:0], c["dense"][:0], c["emb"], c["wide_cat"], c["wide_num"], c["wide_bias"],
                     c["num_perm"], NB, K, flat, x, lin)
    assert bool((flat == -7).all()) and bool(x.isnan().all()) and bool(lin.isnan().all()), "B = 0 wrote output"


def _raw_fwd(**over):
    from tf_repos_b200 import _lib, ops
    d = _dev()
    B, Fc, Fd, NB, K = 4, 2, 3, 10, 4
    t = dict(ids=torch.zeros(B, Fc, dtype=torch.int32, device=d), dense=torch.zeros(B, Fd, device=d),
             emb=torch.zeros(Fc * NB, K, device=d), wide_cat=torch.zeros(Fc * NB, device=d),
             wide_num=torch.zeros(Fd, device=d), wide_bias=torch.zeros(1, device=d),
             num_perm=torch.arange(Fd, dtype=torch.int32, device=d), flat_ids=torch.zeros(B, Fc, dtype=torch.int32, device=d),
             x=torch.zeros(B, Fc * K + Fd, device=d), lin=torch.zeros(B, device=d))
    a = {k: v.data_ptr() for k, v in t.items()}
    a.update(B=B, Fc=Fc, Fd=Fd, NB=NB, K=K)
    a.update(over)
    _lib.check(_lib.raw().ctr_wd_input_fwd(a["ids"], a["dense"], a["emb"], a["wide_cat"], a["wide_num"], a["wide_bias"],
                                           a["num_perm"], a["B"], a["Fc"], a["Fd"], a["NB"], a["K"], a["flat_ids"], a["x"],
                                           a["lin"], ops._stream()), "ctr_wd_input_fwd")


def _raw_bwd(**over):
    from tf_repos_b200 import _lib, ops
    d = _dev()
    B, Fc, Fd, K = 4, 2, 3, 4
    t = dict(dX=torch.zeros(B, Fc * K + Fd, device=d), dy=torch.zeros(B, device=d), dense=torch.zeros(B, Fd, device=d),
             g_rows=torch.zeros(B * Fc, K, device=d), g_cat=torch.zeros(B * Fc, device=d), g_num=torch.zeros(Fd, device=d),
             g_bias=torch.zeros(1, device=d))
    a = {k: v.data_ptr() for k, v in t.items()}
    a.update(B=B, Fc=Fc, Fd=Fd, K=K)
    a.update(over)
    _lib.check(_lib.raw().ctr_wd_input_bwd(a["dX"], a["dy"], a["dense"], a["B"], a["Fc"], a["Fd"], a["K"], a["g_rows"],
                                           a["g_cat"], a["g_num"], a["g_bias"], ops._stream()), "ctr_wd_input_bwd")


@pytest.mark.parametrize("call,over,msg", [
    ("fwd", dict(B=-1), "ctr_wd_input_fwd: bad sizes"),
    ("fwd", dict(Fc=0), "ctr_wd_input_fwd: bad sizes"),
    ("fwd", dict(Fd=-1), "ctr_wd_input_fwd: bad sizes"),
    ("fwd", dict(NB=0), "ctr_wd_input_fwd: bad sizes"),
    ("fwd", dict(K=0), "ctr_wd_input_fwd: bad sizes"),
    ("fwd", dict(ids=None), "ctr_wd_input_fwd: null ids/dense"),
    ("fwd", dict(flat_ids=None), "ctr_wd_input_fwd: null ids/dense"),
    ("fwd", dict(dense=None), "ctr_wd_input_fwd: null ids/dense"),
    ("fwd", dict(x=None), "ctr_wd_input_fwd: emb needs x and num_perm"),
    ("fwd", dict(num_perm=None), "ctr_wd_input_fwd: emb needs x and num_perm"),
    ("fwd", dict(lin=None), "ctr_wd_input_fwd: wide part needs lin"),
    ("fwd", dict(lin=None, wide_cat=None), "ctr_wd_input_fwd: wide part needs lin"),
    ("bwd", dict(B=-1), "ctr_wd_input_bwd: bad sizes"),
    ("bwd", dict(Fc=0), "ctr_wd_input_bwd: bad sizes"),
    ("bwd", dict(Fd=-1), "ctr_wd_input_bwd: bad sizes"),
    ("bwd", dict(K=0), "ctr_wd_input_bwd: bad sizes"),
    ("bwd", dict(dX=None), "ctr_wd_input_bwd: g_rows needs dX"),
    ("bwd", dict(dy=None), "ctr_wd_input_bwd: wide gradients need dy"),
    ("bwd", dict(dy=None, g_cat=None, g_num=None), "ctr_wd_input_bwd: wide gradients need dy"),
    ("bwd", dict(dense=None), "ctr_wd_input_bwd: g_num needs dense and g_bias"),
    ("bwd", dict(g_bias=None), "ctr_wd_input_bwd: g_num needs dense and g_bias"),
])
def test_wd_input_requires_raise(call, over, msg):
    from tf_repos_b200._lib import CtrError
    with pytest.raises(CtrError, match=msg):
        (_raw_fwd if call == "fwd" else _raw_bwd)(**over)
    torch.cuda.synchronize()


def test_wd_input_optional_pointers_pass_their_checks():
    """The combinations the three model types pass must not trip a check: no wide part at all, Fd = 0 without dense
    or num_perm, and g_bias without g_num (or dense)."""
    _raw_fwd(wide_cat=None, wide_num=None, wide_bias=None, lin=None)
    _raw_fwd(emb=None, x=None, num_perm=None)
    _raw_fwd(Fd=0, dense=None, num_perm=None)
    _raw_fwd(B=0, ids=None, dense=None, flat_ids=None)
    _raw_bwd(g_num=None, dense=None)
    _raw_bwd(g_rows=None, dX=None)
    _raw_bwd(g_cat=None, g_num=None, g_bias=None, dy=None)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# ctr_wd_input_bwd: per-occurrence gradients and the linear part's dense gradients
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,Fc,Fd,K", [
    (128, 26, 13, 32),     # the reference default
    (8192, 26, 13, 32),    # B*Fc*K = 6.8 M > 16 CTAs per SM * 256: the grid-stride loop goes round many times
    (7, 33, 40, 33),
    (1, 1, 0, 1),
    (8193, 70, 40, 1),     # B one past a multiple of the 256 threads that stride the dense gradients
    (300, 1, 256, 256),    # Fd = 256 numeric columns: 257 CTAs of the dense-gradient kernel
])
def test_wd_input_bwd(B, Fc, Fd, K):
    from tf_repos_b200 import ops
    d = _dev()
    g = torch.Generator().manual_seed(B + Fc + Fd + K)
    dX = torch.randn(B, Fc * K + Fd, generator=g)
    dX[:, Fc * K:] = 1e30                                   # numeric columns of dX: must not reach g_rows
    dy = torch.randn(B, generator=g)
    dense = torch.randn(B, Fd, generator=g)

    def run(with_num=True):
        g_rows = torch.full((B * Fc, K), float("nan"), device=d)
        g_cat = torch.full((B * Fc,), float("nan"), device=d)
        g_num = torch.full((Fd,), float("nan"), device=d) if with_num else None
        g_bias = torch.full((1,), float("nan"), device=d)
        ops.wd_input_bwd(dX.to(d), dy.to(d), dense.to(d) if with_num else None, B, Fc, Fd, K, g_rows, g_cat, g_num,
                         g_bias)
        return g_rows, g_cat, g_num, g_bias

    g_rows, g_cat, g_num, g_bias = run()
    _bits_equal(g_rows, dX[:, :Fc * K].reshape(B * Fc, K), f"g_rows B={B} Fc={Fc} K={K}")
    _bits_equal(g_cat, dy.repeat_interleave(Fc), f"g_cat B={B} Fc={Fc}")
    # each thread adds (fmas) its ceil(B/256) samples in order, then 8 levels of the shared-memory tree; +1 for the
    # product the bias column does not have (a conservative round for the fma's single rounding)
    bnd = gamma(-(-B // 256) + 8 + 1)
    p64 = dy.double()[:, None] * dense.double()
    _check(g_num, p64.sum(0), bnd * p64.abs().sum(0), f"g_num B={B} Fd={Fd}")
    _check(g_bias, dy.double().sum().reshape(1), bnd * dy.double().abs().sum().reshape(1), f"g_bias B={B}")
    g_rows2, g_cat2, g_num2, g_bias2 = run()
    for a, b_, w in ((g_rows2, g_rows, "g_rows"), (g_cat2, g_cat, "g_cat"), (g_num2, g_num, "g_num"),
                     (g_bias2, g_bias, "g_bias")):
        _bits_equal(a, b_, f"{w} on a second call")
    _, _, _, g_bias3 = run(with_num=False)
    _bits_equal(g_bias3, g_bias, "g_bias without g_num")


# ---------------------------------------------------------------------------------------------------------------------
# ctr_segment_sum_rows on the paths wide_n_deep reaches and the K3 tests do not
# ---------------------------------------------------------------------------------------------------------------------
def _runs_ids(lengths, n_short_ids, n_short, rng):
    """ids with one run of each given length and n_short occurrences spread over n_short_ids other ids, shuffled.  Short
    ids are even, the long runs' ids odd and spread evenly between them, so the long runs' positions u in the sorted
    unique ids are spread over the whole range (and over many CTAs of the kernel that lists them)."""
    ids = [np.full(L, 100_001 + 2 * (i * n_short_ids // len(lengths)), dtype=np.int64) for i, L in enumerate(lengths)]
    ids.append(100_000 + 2 * rng.integers(0, n_short_ids, size=n_short))
    ids = np.concatenate(ids)
    rng.shuffle(ids)
    return ids.astype(np.int32)


def _segsum(ids, K, rng, with_w, ws_bytes=None):
    """unique_segment + segment_sum_rows; with ws_bytes the sum gets a workspace of that size instead of the sort's.
    run(resegment=True) repeats unique_segment first (its long_list comes out in no fixed order)."""
    from tf_repos_b200 import ops
    d = _dev()
    n = ids.size
    uw = ops.UniqueWorkspace(n, 1 << 20, d)
    sort_ws = uw.ws
    sum_ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=d) if ws_bytes is not None else sort_ws
    g = rng.standard_normal((n, K)).astype(np.float32)
    gw = rng.standard_normal(n).astype(np.float32) if with_w else None

    def segment():
        uw.ws = sort_ws
        ops.unique_segment(torch.from_numpy(ids).to(d), uw)
        uw.ws = sum_ws

    def run(resegment=False):
        if resegment:
            segment()
        g_uniq = torch.full((n, K), float("nan"), device=d)
        gw_uniq = torch.full((n,), float("nan"), device=d) if with_w else None
        ops.segment_sum_rows(torch.from_numpy(g).to(d), torch.from_numpy(gw).to(d) if with_w else None, uw, K,
                             g_uniq, gw_uniq)
        return g_uniq, gw_uniq

    segment()
    out = run()
    U_ = int(uw.n_uniq.item())
    _, inv, lens = np.unique(ids, return_inverse=True, return_counts=True)
    assert lens.size == U_
    return uw, g, gw, inv, lens, out, run


def _seq32(v, inv, U_):
    """np.add.at on fp32 adds each occurrence in index order, one fp32 rounding each: sequential occurrence order."""
    s = np.zeros((U_,) + v.shape[1:], dtype=np.float32)
    np.add.at(s, inv, v)
    return s


def _sum64(v, inv, U_):
    s = np.zeros((U_,) + v.shape[1:]); np.add.at(s, inv, v.astype(np.float64))
    m = np.zeros((U_,) + v.shape[1:]); np.add.at(m, inv, np.abs(v).astype(np.float64))
    return s, m


@pytest.mark.parametrize("K", [1, 2, 3, 12, 33])
@pytest.mark.parametrize("with_w", [False, True])
def test_segment_sum_generic_k_is_sequential_for_every_run(K, with_w):
    """segsum_generic_kernel (every K without a vector kernel; K = 1 is the wide model's scalar table) adds each run in
    perm order, i.e. in occurrence order, however long the run: bit-exact against sequential fp32."""
    rng = np.random.default_rng(K * 2 + with_w)
    ids = _runs_ids([1, 2, 127, 128, 129, 300, 1000, 4000], 3000, 9000, rng)
    uw, g, gw, inv, lens, (g_uniq, gw_uniq), run = _segsum(ids, K, rng, with_w)
    U_ = lens.size
    assert lens.max() == 4000
    _bits_equal(g_uniq[:U_], torch.from_numpy(_seq32(g, inv, U_)), f"generic K={K} g_uniq")
    if with_w:
        _bits_equal(gw_uniq[:U_], torch.from_numpy(_seq32(gw, inv, U_)), f"generic K={K} gw_uniq")


def _long_bound(lens, G, split):
    """A long run: each of the G lane groups adds its ceil(len/G) occurrences in order, log2(G) tree levels, and on the
    split path the final kernel adds the run's ceil(len/SEG_CHUNK) chunk partials in order."""
    n = -(-lens // G) + int(math.log2(G)) + (-(-lens // SEG_CHUNK) if split else 0)
    return np.array([gamma(int(k)) for k in n])


def _lanes_per_row(K):
    return {4: 1, 8: 2, 16: 4, 32: 8, 64: 16, 128: 32, 256: 32}[K]


def _check_runs(uw, g, gw, inv, lens, g_uniq, gw_uniq, K, split, what):
    U_ = lens.size
    short = lens <= LONG_SEG
    _bits_equal(g_uniq[:U_][torch.from_numpy(short).to(g_uniq.device)], torch.from_numpy(_seq32(g, inv, U_)[short]),
                f"{what}: short runs")
    G = 256 // _lanes_per_row(K)
    bnd = _long_bound(lens[~short], G, split)
    s, m = _sum64(g, inv, U_)
    _check(g_uniq[:U_].cpu().numpy()[~short], s[~short], bnd[:, None] * m[~short], f"{what}: long runs")
    if gw is not None:
        sw, mw = _sum64(gw, inv, U_)
        _bits_equal(gw_uniq[:U_][torch.from_numpy(short).to(g_uniq.device)], torch.from_numpy(_seq32(gw, inv, U_)[short]),
                    f"{what}: gw short runs")
        _check(gw_uniq[:U_].cpu().numpy()[~short], sw[~short], bnd * mw[~short], f"{what}: gw long runs")


def _want_rows(n):
    """ctr_segment_sum_rows: the partial rows the split path asks for; below 16 it uses the non-split kernel."""
    max_long = n // (LONG_SEG + 1) + 1
    return n // SEG_CHUNK + max_long, max_long


@pytest.mark.parametrize("K", [4, 32, 256])
@pytest.mark.parametrize("lengths,n_short", [([300], 0), ([129, 130, 500], 700), ([1800], 0), ([129, 1024], 600)])
def test_segment_sum_non_split_long_kernel(K, lengths, n_short):
    """n small enough that the split path would get fewer than 16 partial rows: segsum_long_kernel sums each long run
    with one CTA.  Runs from 129 up to the whole of n."""
    rng = np.random.default_rng(K + sum(lengths))
    ids = _runs_ids(lengths, max(n_short // 3, 1), n_short, rng)
    assert _want_rows(ids.size)[0] < 16
    uw, g, gw, inv, lens, (g_uniq, gw_uniq), run = _segsum(ids, K, rng, True)
    _check_runs(uw, g, gw, inv, lens, g_uniq, gw_uniq, K, False, f"non-split K={K} runs={lengths}")
    g2, gw2 = run()
    _bits_equal(g2[:lens.size], g_uniq[:lens.size], "non-split g_uniq on a second call")
    _bits_equal(gw2[:lens.size], gw_uniq[:lens.size], "non-split gw_uniq on a second call")


def _expected_plan(lens, cap):
    """segsum_long_plan_kernel's rule: long runs take partial rows in ascending u; a run's base is the chunk count of
    the long runs before it, and it gets no rows (base -1, summed whole by one CTA) if base + chunks > cap."""
    plan, base = {}, 0
    for u in np.nonzero(lens > LONG_SEG)[0]:
        chunks = -(-int(lens[u]) // SEG_CHUNK)
        plan[int(u)] = (base, chunks) if base + chunks <= cap else (-1, 1)
        base += chunks
    return plan


def _plan_of(uw, plan_bytes):
    n_long = int(uw.long_list[0].item())
    us = uw.long_list[1:1 + n_long].cpu().numpy()
    plan = uw.ws[:plan_bytes].view(torch.int32).cpu().numpy()
    return {int(u): (int(plan[1 + 2 * li]), int(plan[2 + 2 * li])) for li, u in enumerate(us)}


def test_segment_sum_split_path_when_scratch_runs_out():
    """With 16 <= cap_rows < want_rows the split path's partial rows run out: the long runs past the limit get
    base = -1 and are summed whole by one CTA straight into g_uniq.  K = 256; 36 long runs of 1 to 5 chunks in mixed
    order, their u spread past the first CTAs of the kernel that lists them.  Which runs get rows must not depend on
    the order long_list comes out in, so a second unique_segment + sum must give the same plan and the same bits."""
    K = 256
    rng = np.random.default_rng(256)
    lengths = rng.permutation([2100] * 12 + [3100] * 6 + [1025] * 14 + [129, 200, 1024, 4100]).tolist()
    ids = _runs_ids(lengths, 4000, 8000, rng)
    n = ids.size
    want, max_long = _want_rows(n)
    # workspace layout (segment_sum.cu): int32 plan[1 + 2*max_long] padded to 16 bytes | float partial[cap][K + 4]
    plan_bytes = ((1 + 2 * max_long) * 4 + 15) & ~15
    cap = 40
    assert 16 <= cap < want and sum(-(-L // SEG_CHUNK) for L in lengths) > cap
    uw, g, gw, inv, lens, (g_uniq, gw_uniq), run = _segsum(ids, K, rng, True, ws_bytes=plan_bytes + cap * (K + 4) * 4)
    long_u = np.nonzero(lens > LONG_SEG)[0]
    assert long_u.size == 36 and long_u.max() > 256
    want_plan = _expected_plan(lens, cap)
    assert _plan_of(uw, plan_bytes) == want_plan
    bases = np.array([b for b, _ in want_plan.values()])
    assert (bases < 0).any() and (bases >= 0).any(), f"want runs on both sides of the scratch limit, plan {want_plan}"
    # a run that got a base may have several chunks; one without sums everything in one CTA: the bound covers both
    _check_runs(uw, g, gw, inv, lens, g_uniq, gw_uniq, K, True, "scratch exhausted")
    g2, gw2 = run(resegment=True)
    assert _plan_of(uw, plan_bytes) == want_plan
    _bits_equal(g2[:lens.size], g_uniq[:lens.size], "scratch exhausted g_uniq after a second unique_segment")
    _bits_equal(gw2[:lens.size], gw_uniq[:lens.size], "scratch exhausted gw_uniq after a second unique_segment")


@pytest.mark.parametrize("K", [4, 32, 256])
def test_segment_sum_long_seg_boundary(K):
    """A run of exactly CTR_LONG_SEG = 128 stays on the short kernel (sequential, bit-exact); 129 leaves it."""
    rng = np.random.default_rng(K + 7)
    ids = _runs_ids([128, 129, 128, 129], 2000, 6000, rng)
    assert _want_rows(ids.size)[0] >= 16
    uw, g, gw, inv, lens, (g_uniq, gw_uniq), run = _segsum(ids, K, rng, True)
    assert sorted(lens[lens >= LONG_SEG].tolist()) == [128, 128, 129, 129]
    assert int(uw.long_list[0].item()) == 2
    _check_runs(uw, g, gw, inv, lens, g_uniq, gw_uniq, K, True, f"boundary K={K}")


# ---------------------------------------------------------------------------------------------------------------------
# the DNN layers at the reference default: D = 26*32 + 13 = 845 inputs, then 256 -> 128 -> 64
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,Kd,Nd", [(128, 845, 256), (8192, 845, 256), (128, 256, 128), (128, 128, 64)])
@pytest.mark.parametrize("act", [0, 1])
def test_fc_wide_deep_layers(M, Kd, Nd, act):
    from tf_repos_b200 import ops
    d = _dev()
    g = torch.Generator().manual_seed(M + Kd + Nd + act)
    x = torch.randn(M, Kd, generator=g)
    W = torch.randn(Kd, Nd, generator=g) / Kd ** 0.5
    b = torch.randn(Nd, generator=g) * 0.1
    dOut = torch.randn(M, Nd, generator=g)
    x64, W64, b64 = x.double(), W.double(), b.double()
    out = torch.full((M, Nd), float("nan"), device=d)
    ops.fc_fwd(x.to(d), W.to(d), b.to(d), None, 1.0, act, out)
    pre = x64 @ W64 + b64
    # one product over Kd, then the bias add; relu is 1-Lipschitz, so it cannot widen the error
    _check(out, pre.clamp_min(0.0) if act else pre, gemm_rel(Kd, adds=1) * (x64.abs() @ W64.abs() + b64.abs()),
           f"fc_fwd act={act} M={M} Kd={Kd} Nd={Nd}")
    ws = torch.empty(ops.fc_bwd_workspace_bytes(M, Kd, Nd), dtype=torch.uint8, device=d)

    def run():
        dO = dOut.to(d).clone()
        dIn = torch.full((M, Kd), float("nan"), device=d)
        dW = torch.full((Kd, Nd), float("nan"), device=d)
        db = torch.full((Nd,), float("nan"), device=d)
        ops.fc_bwd(x.to(d), W.to(d), out, None, 1.0, dO, act, dIn, dW, db, ws)
        return dO, dIn, dW, db

    dZ, dIn, dW, db = run()
    # the relu gate is the GPU's own out > 0 (a pre-activation within rounding of 0 may land on either side)
    gate = (out.cpu() > 0).float() if act else torch.ones(M, Nd)
    dZ32 = torch.where(gate > 0, dOut, torch.zeros(()))      # the kernel stores +0 where the gate is closed
    _bits_equal(dZ, dZ32, f"dZ in place act={act} M={M}")
    dZ64 = dZ32.double()
    _check(dIn, dZ64 @ W64.T, gemm_rel(Nd) * (dZ64.abs() @ W64.abs().T), f"dIn act={act} M={M} Kd={Kd} Nd={Nd}")
    S = _pick_split(Kd, Nd, M)                               # Kd > 64: the plain (not transposed) dW product
    _check(dW, x64.T @ dZ64, gemm_rel(-(-M // S), adds=S) * (x64.abs().T @ dZ64.abs()),
           f"dW act={act} M={M} Kd={Kd} Nd={Nd} S={S}")
    # db: 8 row lanes add <= 16 rows of a 128-row chunk, 8 lanes combined in order, then ceil(chunks/8) chunk partials
    # per group and the 8 groups in order
    chunks = -(-M // 128)
    _check(db, dZ64.sum(0), gamma(16 + 8 + -(-chunks // 8) + 8) * dZ64.abs().sum(0), f"db act={act} M={M} Nd={Nd}")
    _, dIn2, dW2, db2 = run()
    _bits_equal(dIn2, dIn, "dIn on a second call")
    _bits_equal(dW2, dW, "dW on a second call")
    _bits_equal(db2, db, "db on a second call")


# ---------------------------------------------------------------------------------------------------------------------
# the three models at the reference default against the oracle in fp64
# ---------------------------------------------------------------------------------------------------------------------
def _model_batch(B, seed, shared_column=None):
    g = torch.Generator().manual_seed(seed)
    dense = torch.rand(B, 13, generator=g)
    cat = torch.randint(1, 10000, (B, 26), generator=g, dtype=torch.int64).to(torch.int32)   # bucket 0 left free
    cat[0, 0] = 12345                     # out of range: lands in bucket 0 of column C14
    cat[min(1, B - 1), 5] = -3            # and of column C19
    cat[min(2, B - 1), 5] = I32_MIN
    if shared_column is not None:
        cat[:, shared_column] = 7         # one id in every sample: a run of B
    labels = (torch.rand(B, generator=g) < 0.3).float()
    return dense, cat, labels


def _oracles(model_type, K, layers):
    from oracle import wide_deep as owd
    o32 = owd.WideDeep(embedding_size=K, deep_layers=layers, model_type=model_type, seed=3)
    if model_type == "wide":         # an all-zero start is a degenerate parity case: give the linear part some weights
        g = torch.Generator().manual_seed(1)
        for n in o32.params:
            o32.params[n] = (torch.randn(o32.params[n].shape, generator=g) * 0.05).float()
    o64 = owd.WideDeep(embedding_size=K, deep_layers=layers, model_type=model_type, seed=3, dtype=torch.float64)
    o64.params = {n: p.double() for n, p in o32.params.items()}
    o64.slots = {n: [s.double() for s in v] for n, v in o32.slots.items()}
    return o32, o64


def _close_to_fp64(got, want32, want64, what, scale):
    """max|got - fp64| <= scale * max(4 * max|fp32 oracle - fp64|, 1e-6 * max|fp64|).  The fp32 oracle's distance from
    fp64 calibrates the tolerance: the GPU may be off the exact result by four times what a plain fp32 evaluation of
    the same steps is, times `scale`, the expected error of the GPU's reductions relative to the oracle's.

    scale = 1 for the wide model: every sum on its path is a rounded fp32 add, like the oracle's.
    scale = sqrt(3 R) where the DNN's GEMMs feed the result, R = D = 845 its longest reduction (~50).  The oracle's fp32
    dot products round to nearest: each add errs by a zero-mean amount of standard deviation ulp/sqrt(12), so R adds
    drift by ~sqrt(R/12) ulp.  The tensor core truncates its accumulator (test_gpu_din_attention.py, TRUNC): each add
    errs by ulp/2 on average, all the same way while the partial sum keeps its sign, so R adds drift by ~R/2 ulp.
    The ratio is sqrt(3 R).  This is an estimate of typical error, not a bound: the worst-case bounds (gemm_rel against
    gamma(R)) differ by only ~2.3, which is why the GEMMs themselves are pinned by bounds in test_fc_wide_deep_layers.
    On one H100 80GB HBM3 at 700 W the DNN models sat up to ~54x the fp32 oracle's distance (a hidden-layer bias after
    four deep steps, at 7.3e-6 of max|value|), under 0.3 of this tolerance."""
    got, want32, want64 = _np(got), _np(want32), _np(want64)
    ref = float(np.max(np.abs(want32 - want64))) if want64.size else 0.0
    tol = scale * max(4 * ref, 1e-6 * float(np.max(np.abs(want64))) if want64.size else 0.0)
    err = float(np.max(np.abs(got - want64))) if want64.size else 0.0
    assert err <= tol, f"{what}: max err {err:.3e} > tol {tol:.3e} (fp32 oracle is {ref:.3e} off fp64)"
    print(f"RATIO model {what}: {err / tol if tol else 0.0:.3g}")


def _run_model(model_type, B, steps, shared_column=None):
    from tf_repos_b200.wide_deep import NUM_BUCKETS, WideDeep
    K, layers = 32, "256,128,64"
    o32, o64 = _oracles(model_type, K, layers)
    m = WideDeep(embedding_size=K, batch_size=B, deep_layers=layers, model_type=model_type, seed=3)
    m.load_variables(o32.params)
    d = m.device
    scale = math.sqrt(3 * m.D) if m.has_dnn else 1.0
    tables = ([m.emb.var] if m.has_dnn else []) + ([m.wide_cat.var] if m.has_linear else [])
    for step, Bs in enumerate(steps):
        dense, cat, labels = _model_batch(Bs, seed=40 + step, shared_column=shared_column)
        what = f"{model_type} B={B} step={step} Bs={Bs}"
        m.predict(dense.to(d), cat.to(d))
        _close_to_fp64(m.y[:Bs], o32.predict(dense, cat)["y"], o64.predict(dense, cat)["y"], f"{what} logits",
                       scale)
        before = [t.clone() for t in tables]
        loss = float(m.train_step(dense.to(d), cat.to(d), labels.to(d)))
        l32, l64 = o32.train_step(dense, cat, labels), o64.train_step(dense, cat, labels)
        _close_to_fp64(np.array([loss]), np.array([l32]), np.array([l64]), f"{what} loss", scale)
        for name, v in m.variables().items():
            _close_to_fp64(v.reshape(o64.params[name].shape), o32.params[name], o64.params[name], f"{what} {name}",
                           scale)
        # no L2: only the rows a clamped id of this step gathers may move, and an out-of-range id's row is bucket 0
        ids = cat.long()
        clamped = torch.where((ids < 0) | (ids >= NUM_BUCKETS), torch.zeros_like(ids), ids)
        touched = torch.zeros(26 * NUM_BUCKETS, dtype=torch.bool)
        touched[(torch.arange(26) * NUM_BUCKETS + clamped).reshape(-1)] = True
        t_dev = touched.to(d)
        for t_old, t_new in zip(before, tables):
            _bits_equal(t_new[~t_dev], t_old[~t_dev], f"{what}: rows no id touched")
            for f in (0, 5):                          # bucket 0 of C14 and C19 is reached only through the bad ids
                assert not torch.equal(t_new[f * NUM_BUCKETS], t_old[f * NUM_BUCKETS]), \
                    f"{what}: the out-of-range id's gradient did not reach bucket 0 of column {f}"


@pytest.mark.parametrize("model_type", ["wide", "deep", "wide_n_deep"])
def test_model_default_config_matches_fp64_oracle(model_type):
    """K = 32, deep_layers = 256,128,64, batch 128, five steps, the third a partial batch of 50."""
    _run_model(model_type, 128, [128, 128, 50, 128, 128])


def test_wide_n_deep_shared_id_batch_512_matches_fp64_oracle():
    """Batch 512 with C16's id shared by all samples: a run of 512 takes the split long path, which carries the wide
    part's scalar gradient (gw) next to the embedding rows."""
    from tf_repos_b200 import ops
    B, K = 512, 32
    n = B * 26
    want, max_long = _want_rows(n)
    ws = max(ops.unique_segment_workspace_bytes(n, 26 * 10000), 16)
    assert min(want, (ws - (((1 + 2 * max_long) * 4 + 15) & ~15)) // ((K + 4) * 4)) >= 16, "not the split path"
    _run_model("wide_n_deep", B, [512, 512, 50, 512, 512], shared_column=2)
