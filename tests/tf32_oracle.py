"""Plain fp64 references for tc_gemm.cu's 3xTF32 GEMM (numpy only, no GPU).

- split(a): the kernel's operand split, hi = cvt.rna.tf32(a) and lo = a - hi (exact in fp32).  The tensor core reads
  the top 19 bits of an operand register, so lo enters the product truncated to TF32 (tf32_trunc); hi is already TF32.
- gemm_emulated(A, B, terms): exact fp64 products of the split operands.  terms picks any subset of hi*hi, lo*hi and
  hi*lo, so plain TF32 ({"hh"}) and a kernel that dropped one cross term ({"hh", "lh"} / {"hh", "hl"}) are one call each.
- gemm_model(A, B, chunk): a MODEL of the kernel's arithmetic, not a measurement of the H100's accumulator: every
  k8 block sum is exact, and each wgmma adds it to an fp32 accumulator truncated toward zero -- hi*hi in one, the two
  cross terms in a second, the two added once (round to nearest) at the end.  With a split-R chunk it also models
  fc.cu's fixed-order fp32 reduce of the chunk partials.
- pick_split / dw_transposed / bn_class: mirrors of fc.cu's split and transposed-dW rules and tc_gemm.cu's tile width.
- Exact-data constructors: one operand takes p + q*2^-11 (p in [-3, 3], q in {-1, 0, 1}: 12-13 significant bits, so
  lo is 0 or +-2^-11, a TF32 number), the others small integers (lo = 0).  With sum_r |a_r b_r| <= 2^11 for every output
  element, every addend and every partial sum is a multiple of 2^-11 below 2^12: an accumulator that keeps 24
  significant bits adds them exactly, whatever its rounding, and the fp64 product rounded to fp32 is the exact answer.
  A kernel that drops a cross term, or reads a lo tile at the wrong k offset, misses the 2^-11 parts.
"""
from __future__ import annotations

import numpy as np

GRID = 2.0 ** -11                 # the lo part of every exact-data value is a multiple of this
EXACT_LIMIT = 2.0 ** 11           # sum_r |a_r b_r| bound that keeps every partial sum exact in 24 bits
TC_BM = 128                       # tc_gemm.cu's output tile rows (and fc.cu's pick_split tile)
TERMS_3X = ("hh", "lh", "hl")
BROKEN = {"1xTF32": ("hh",), "2xTF32 without hi*lo": ("hh", "lh"), "2xTF32 without lo*hi": ("hh", "hl")}


# ---------------------------------------------------------------------------------------------------------------------
# the split
# ---------------------------------------------------------------------------------------------------------------------
def rna_tf32(a):
    """cvt.rna.tf32.f32: round to 10 explicit mantissa bits, ties away from zero (bit-level: (bits + 0x1000) & ~0x1FFF)."""
    b = np.asarray(a, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return ((b + 0x1000) & 0xFFFFE000).astype(np.uint32).view(np.float32)


def tf32_trunc(a):
    """What the tensor core reads of an fp32 register: the low 13 mantissa bits dropped."""
    return (np.asarray(a, dtype=np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def is_tf32(a):
    return not np.any(np.asarray(a, dtype=np.float32).view(np.uint32) & np.uint32(0x1FFF))


def split(a):
    """(hi, lo) as tf32_hi / store_tile_fast compute them: hi = rna_tf32(a), lo = a - hi in fp32 (exact)."""
    a = np.asarray(a, dtype=np.float32)
    hi = rna_tf32(a)
    with np.errstate(over="ignore", invalid="ignore"):
        lo = (a - hi).astype(np.float32)
    return hi, lo


def _parts(A):
    hi, lo = split(A)
    return hi.astype(np.float64), tf32_trunc(lo).astype(np.float64)


# ---------------------------------------------------------------------------------------------------------------------
# products
# ---------------------------------------------------------------------------------------------------------------------
def gemm_emulated(A, B, terms=TERMS_3X):
    """sum of the chosen split products, each exact in fp64 (no accumulation error): A[M,R] @ B[R,N]."""
    Ah, Al = _parts(A)
    Bh, Bl = _parts(B)
    C = np.zeros((Ah.shape[0], Bh.shape[1]))
    if "hh" in terms:
        C += Ah @ Bh
    if "lh" in terms:
        C += Al @ Bh
    if "hl" in terms:
        C += Ah @ Bl
    return C


def trunc_fp32(x):
    """fp64 -> fp32 rounded toward zero."""
    x = np.asarray(x, dtype=np.float64)
    f = x.astype(np.float32)
    over = np.abs(f.astype(np.float64)) > np.abs(x)
    f[over] = np.nextafter(f[over], np.float32(0))
    return f


def _model_chunk(Ah, Al, Bh, Bl):
    M, R = Ah.shape
    acc = np.zeros((M, Bh.shape[1]), np.float32)
    acc2 = np.zeros_like(acc)
    for k in range(0, R, 8):
        s = slice(k, k + 8)
        acc2 = trunc_fp32(acc2 + Al[:, s] @ Bh[s])          # the kernel's wgmma order within a k-step
        acc2 = trunc_fp32(acc2 + Ah[:, s] @ Bl[s])
        acc = trunc_fp32(acc + Ah[:, s] @ Bh[s])
    return (acc + acc2).astype(np.float32)


def gemm_model(A, B, chunk=None):
    """Model of the kernel's fp32 result of A[M,R] @ B[R,N] (see the module docstring).  chunk: split-R chunk length;
    the partials are then added in chunk order in fp32, as splitk_reduce_kernel does."""
    Ah, Al = _parts(A)
    Bh, Bl = _parts(B)
    R = Ah.shape[1]
    chunk = R if not chunk else chunk
    out = np.zeros((Ah.shape[0], Bh.shape[1]), np.float32)
    for r0 in range(0, max(R, 1), chunk):
        s = slice(r0, min(R, r0 + chunk))
        out = (out + _model_chunk(Ah[:, s], Al[:, s], Bh[s], Bl[s])).astype(np.float32)
    return out


def rel_metric(C, A, B, C64=None, mag=None):
    """max_ij |C - A@B| / (|A| @ |B|)_ij in fp64 (elements with a zero magnitude must be exactly 0)."""
    A64, B64 = np.asarray(A, np.float64), np.asarray(B, np.float64)
    C64 = A64 @ B64 if C64 is None else C64
    mag = np.abs(A64) @ np.abs(B64) if mag is None else mag
    err = np.abs(np.asarray(C, np.float64) - C64)
    assert np.all(err[mag == 0] == 0)
    return float(np.max(np.where(mag > 0, err / np.where(mag > 0, mag, 1.0), 0.0))) if err.size else 0.0


def broken_metrics(A, B):
    """{variant: metric} of each broken emulation on this data, and the fp64 product and magnitude (reusable)."""
    A64, B64 = np.asarray(A, np.float64), np.asarray(B, np.float64)
    C64, mag = A64 @ B64, np.abs(A64) @ np.abs(B64)
    return {k: rel_metric(gemm_emulated(A, B, t), A, B, C64, mag) for k, t in BROKEN.items()}, C64, mag


def tolerance(A, B, headroom=16.0):
    """The accuracy tolerance of a product: 1/16 of the best of the three broken emulations on the same data."""
    m, _, _ = broken_metrics(A, B)
    return min(m.values()) / headroom, m


# ---------------------------------------------------------------------------------------------------------------------
# dispatch mirrors
# ---------------------------------------------------------------------------------------------------------------------
def pick_split(M, N, R, sm_count):
    """fc.cu pick_split: split-R chunks of a dW product of M x N outputs over R."""
    tiles = -(-M // TC_BM) * -(-N // TC_BM)
    s = max(-(-2 * sm_count // tiles), 1)
    return max(min(s, (R + 255) // 256, 64), 1)


def dw_transposed(Kd, Nd):
    """fc.cu: dW runs as dW^T = dZ^T @ in when the layer input is narrow and the output wide."""
    return Kd <= 64 and Nd >= 128


def dw_split(M, Kd, Nd, sm_count):
    """(S, chunk) of fc_bwd's dW product for a layer Kd -> Nd over M rows."""
    S = pick_split(Nd, Kd, M, sm_count) if dw_transposed(Kd, Nd) else pick_split(Kd, Nd, M, sm_count)
    return S, -(-M // S)


def bn_class(N):
    """tc_gemm.cu launch_tc: the output tile width of a product N wide."""
    return 32 if N <= 32 else 64 if N <= 64 else 128


# ---------------------------------------------------------------------------------------------------------------------
# exact data
# ---------------------------------------------------------------------------------------------------------------------
def grid_lo(rng, shape, density=1.0):
    """p + q*2^-11, p in [-3, 3], q in {-1, 0, 1}; zero with probability 1 - density."""
    v = rng.integers(-3, 4, shape) + rng.integers(-1, 2, shape) * GRID
    if density < 1.0:
        v = np.where(rng.random(shape) < density, v, 0.0)
    return v.astype(np.float32)


def grid_int(rng, shape, density=1.0, vmax=3):
    v = rng.integers(-vmax, vmax + 1, shape).astype(np.float64)
    if density < 1.0:
        v = np.where(rng.random(shape) < density, v, 0.0)
    return v.astype(np.float32)


def assert_exact(A, B, what="product"):
    """The exact-data precondition of A[M,R] @ B[R,N]: every value on the 2^-11 grid, with lo a TF32 number, and
    sum_r |a_r b_r| <= 2^11 for every output element."""
    for X in (A, B):
        X = np.asarray(X, np.float32)
        assert np.all(np.asarray(X, np.float64) / GRID == np.round(np.asarray(X, np.float64) / GRID)), what
        assert is_tf32(split(X)[1]), what
    A64, B64 = np.asarray(A, np.float64), np.asarray(B, np.float64)
    mag = np.abs(A64) @ np.abs(B64)
    assert mag.size == 0 or mag.max() <= EXACT_LIMIT, f"{what}: sum |ab| reaches {mag.max()} > 2^11"


def exact_layer(rng, M, Kd, Nd, lo, budget=192.0):
    """in [M,Kd], W [Kd,Nd], dOut [M,Nd] on the exact grid; `lo` in {"in", "W", "dOut"} names the operand that carries
    lo parts (the others are small integers).  Densities keep the mean of sum |ab| near 3*budget in all three products
    (fwd over Kd, dIn over Nd, dW over M), so that dZ = dOut*mask/0.5 stays within the precondition too."""
    dw = min(1.0, budget / Kd)
    dz = min(1.0, budget / M, budget / (Nd * dw))
    x = grid_lo(rng, (M, Kd)) if lo == "in" else grid_int(rng, (M, Kd))
    W = grid_lo(rng, (Kd, Nd), dw) if lo == "W" else grid_int(rng, (Kd, Nd), dw)
    dOut = grid_lo(rng, (M, Nd), dz) if lo == "dOut" else grid_int(rng, (M, Nd), dz)
    return x, W, dOut


# ---------------------------------------------------------------------------------------------------------------------
# the accuracy cases: the reference's layer shapes on realistic data
# ---------------------------------------------------------------------------------------------------------------------
# (name, rows M of the layer input, layer widths, input dropout-like sparsity of the hidden layers)
ACCURACY_CASES = [
    ("bench DeepFM", 8192, (624, 256, 128, 64)),
    ("DeepFM defaults", 64, (39 * 32, 256, 128, 64)),
    ("wide_n_deep", 128, (845, 256, 128, 64)),
    ("NFM", 128, (64, 128, 64)),
    ("DIN attention", 64 * 100, (32, 256)),
    ("AFM attention", 128 * 741, (256, 256)),
]


def accuracy_layers():
    """[(case name, layer index, M, Kd, Nd)] of every layer of ACCURACY_CASES."""
    out = []
    for name, M, widths in ACCURACY_CASES:
        for i in range(len(widths) - 1):
            out.append((name, i, M, widths[i], widths[i + 1]))
    return out


def accuracy_operands(M, Kd, Nd, layer, seed):
    """Realistic operands of one layer: in ~ N(0,1) for the first layer and relu(N(0,1)) after it, W ~ N(0, 1/Kd),
    dZ ~ N(0,1) with half of it zeroed (relu gate / dropout)."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((M, Kd)).astype(np.float32)
    if layer > 0:
        x = np.maximum(x, 0.0).astype(np.float32)
    W = (rng.standard_normal((Kd, Nd)) / np.sqrt(Kd)).astype(np.float32)
    dZ = (rng.standard_normal((M, Nd)) * (rng.random((M, Nd)) < 0.5)).astype(np.float32)
    return x, W, dZ


def products(x, W, dZ, sm_count):
    """The three products fc.cu launches for one layer, as (name, A, B, chunk) in the orientation the kernel computes."""
    M, Kd = x.shape
    Nd = W.shape[1]
    S, chunk = dw_split(M, Kd, Nd, sm_count)
    dw = ("dW^T", dZ.T, x, chunk) if dw_transposed(Kd, Nd) else ("dW", x.T, dZ, chunk)
    return [("fwd", x, W, None), ("dIn", dZ, W.T, None), dw]


# ---------------------------------------------------------------------------------------------------------------------
# the exact-answer designs of the GPU tests (shared with the CPU test that pins their constructions)
# ---------------------------------------------------------------------------------------------------------------------
N_BY_BN = {32: (1, 31, 32), 64: (33, 64), 128: (65, 128, 129, 256, 400)}
M_BY_TILE = {"interior": (128, 8192), "edge": (1, 63, 64, 127, 129, 300)}
R_BY_STAGES = {1: (1, 3, 4, 8, 31, 32), 2: (33, 100, 624, 845, 1248)}
MASKS = (None, 0.5, 0.8)
GROUP_P = (None, 1, 3, 128, 129)
LO = ("in", "W", "dOut")


def covering_cases():
    """One layer per (BN class x interior/edge rows x aligned/misaligned x 1 or 2 stages) of the forward product, the
    values of every axis (N, M, R = Kd) taken in turn within their class, and the epilogue options cycled so that each
    appears: bias, act, dropout keep, group_P, the lo-carrying operand, accumulate_din.  Misaligned layers place each
    operand 1, 2 or 3 floats into its buffer."""
    cases, seen = [], {}
    for bn in (32, 64, 128):
        for tile in ("interior", "edge"):
            for misaligned in (False, True):
                for stages in (1, 2):
                    i = len(cases)
                    k = {a: seen.get(a, 0) for a in (bn, tile, stages)}
                    for a in k:
                        seen[a] = k[a] + 1
                    cases.append(dict(
                        i=i, Nd=N_BY_BN[bn][k[bn] % len(N_BY_BN[bn])], M=M_BY_TILE[tile][k[tile] % len(M_BY_TILE[tile])],
                        Kd=R_BY_STAGES[stages][k[stages] % len(R_BY_STAGES[stages])], misaligned=misaligned,
                        bias=i % 2 == 0, act=(i // 2) % 2, keep=MASKS[i % 3], group_P=GROUP_P[i % 5], lo=LO[(i // 3) % 3],
                        accumulate_din=(i // 4) % 2 == 1))
    return cases


def case_id(c):
    return (f"M{c['M']}-K{c['Kd']}-N{c['Nd']}-{'mis' if c['misaligned'] else 'al'}-b{int(c['bias'])}-a{c['act']}"
            f"-k{c['keep']}-g{c['group_P']}-{c['lo']}-acc{int(c['accumulate_din'])}")


def offsets(c, n=6):
    """Pointer offsets (floats) of in, Wt, out/dIn, mask, dOut, dW/db for a case: 0, or 1-3 when misaligned."""
    return [((c["i"] + j) % 3 + 1) if c["misaligned"] else 0 for j in range(n)]


DW_EDGES = ((64, 128), (65, 128), (64, 127), (8, 300))
DW_SPLITS = ("one", "middle", "cap")


def dw_edge_m(Kd, Nd, which, sm_count):
    """Rows M of a dW product of a Kd -> Nd layer with the named split: S = 1; 1 < S < 64 with a chunk that is not a
    multiple of 4; S = 64 with a short last chunk."""
    if which == "one":
        return 200
    M = 300 if which == "middle" else 63 * 256 + 1
    while True:
        S, chunk = dw_split(M, Kd, Nd, sm_count)
        if which == "middle" and 1 < S < 64 and chunk % 4:
            return M
        if which == "cap" and S == 64 and M % chunk and chunk % 4:
            return M
        M += 1


# long sparse dW reductions at the reference's shapes: (name, M, Kd, Nd, nonzeros per dZ column)
LONG_DW = (("DIN config 4", 4096 * 100, 32, 256, 200), ("AFM attention", 128 * 741, 256, 256, 200))


def sparse_dz(rng, M, Nd, per_col, lo):
    """dZ[M, Nd] with per_col distinct nonzero rows per column, as (rows, cols, values): relu / dropout zeros make the
    long dW reductions sparse, which keeps sum |in * dZ| <= per_col * 3 * (3 + 2^-11) below 2^11."""
    rows, cols = [], []
    for n in range(Nd):
        r = np.unique(rng.integers(0, M, 2 * per_col))[:per_col]
        rows.append(r)
        cols.append(np.full(r.size, n))
    rows, cols = np.concatenate(rows), np.concatenate(cols)
    vals = grid_lo(rng, rows.size) if lo == "dOut" else grid_int(rng, rows.size)
    vals[vals == 0] = 1.0
    return rows, cols, vals
