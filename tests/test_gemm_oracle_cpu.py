"""Pins tests/tf32_oracle.py, the reference of test_gpu_dense_gemm.py (CPU only).

- The split is exact: hi + lo == a, hi a TF32 number, |lo| at most half an ulp of hi.
- The exact constructions of the GPU tests are exact under the kernel's model and the 3-term emulation, and a kernel
  that drops either cross term, or runs plain TF32, gets most of their elements wrong.
- The accuracy tolerances (1/16 of the best broken emulation) sit above the model's error at every case of the GPU
  file, so that the kernel, if it behaves like the model, passes, and every broken emulation fails.
"""
import numpy as np
import pytest

from tests import tf32_oracle as o

SM = 132   # H100 SXM; the GPU tests read the device's own count


def _bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def _split_values():
    rng = np.random.default_rng(0)
    ones = np.array([0x3FFFFFFF, 0x3F7FFFFF, 0x7F7FFFFF, 0x3F800FFF, 0x3F801000, 0x3F801FFF, 0x3F803000, 0x00001000,
                     0x00000001, 0x007FFFFF, 0x00800000, 0x3F800000, 0x00000000, 0x80000000], np.uint32)
    return np.concatenate([rng.standard_normal(100000).astype(np.float32),
                           (rng.standard_normal(1000) * 1e-39).astype(np.float32),          # subnormals
                           rng.integers(0, 2 ** 31, 100000, dtype=np.uint64).astype(np.uint32).view(np.float32),
                           ones.view(np.float32), (ones | 0x80000000).view(np.float32)])


def test_split_is_exact():
    a = _split_values()
    a = a[np.isfinite(a)]
    hi, lo = o.split(a)
    ok = np.isfinite(hi)
    assert o.is_tf32(hi)
    assert np.array_equal(hi[ok] + lo[ok], a[ok])                         # exact: fp32 add of the two halves
    assert np.array_equal(hi[ok].astype(np.float64) + lo[ok].astype(np.float64), a[ok].astype(np.float64))
    ulp = np.spacing(np.abs(hi[ok]).astype(np.float32)).astype(np.float64) * 2.0 ** 13
    assert np.all(np.abs(lo[ok].astype(np.float64)) <= ulp / 2)
    # lo itself needs up to 13 bits: the tensor core reads it truncated, which the emulation models
    assert not o.is_tf32(lo)


def test_split_known_answers():
    f = lambda b: np.array([b], np.uint32).view(np.float32)
    # a mantissa of all ones rounds up into the next binade
    hi, lo = o.split(f(0x3FFFFFFF))
    assert _bits(hi)[0] == 0x40000000 and lo[0] == f(0x3FFFFFFF)[0] - np.float32(2.0)
    # ties: exactly half an ulp of TF32 rounds away from zero, both signs
    for b, want in ((0x3F801000, 0x3F802000), (0xBF801000, 0xBF802000), (0x3F800FFF, 0x3F800000)):
        assert _bits(o.split(f(b))[0])[0] == want, hex(b)
    # +-0 and the largest subnormal
    for b in (0x00000000, 0x80000000):
        hi, lo = o.split(f(b))
        assert _bits(hi)[0] == b and lo[0] == 0
    hi, lo = o.split(f(0x007FFFFF))
    assert _bits(hi)[0] == 0x00800000 and hi[0] + lo[0] == f(0x007FFFFF)[0]
    # overflow of the rounding: the largest finite fp32 rounds to inf in TF32 (the kernel's inputs never get there)
    assert np.isinf(o.split(f(0x7F7FFFFF))[0][0])


def test_exact_grid():
    rng = np.random.default_rng(1)
    a = o.grid_lo(rng, 100000)
    hi, lo = o.split(a)
    assert set(np.unique(lo).tolist()) <= {-o.GRID, 0.0, o.GRID} and o.is_tf32(lo)
    assert np.unique(lo).size == 3


def test_model_and_emulation_known():
    """Plain TF32 loses the 2^-11 parts; the 3-term emulation and the model keep all but lo*lo; the accumulator of the
    model truncates toward zero."""
    A = np.array([[1 + o.GRID, 3.0]], np.float32)      # 1 + 2^-11 is a tie: hi = 1 + 2^-10, lo = -2^-11
    B = np.array([[1 + o.GRID], [1.0]], np.float32)
    three = (1 + o.GRID) ** 2 - o.GRID ** 2 + 3.0        # everything but lo*lo
    assert o.gemm_emulated(A, B)[0, 0] == three
    assert o.gemm_emulated(A, B, ("hh",))[0, 0] == (1 + 2 * o.GRID) ** 2 + 3.0
    assert o.gemm_model(A, B)[0, 0] == np.float32(three)
    # truncation toward zero of the accumulator: 1 + 2^-24 is cut back to 1
    A = np.ones((1, 16), np.float32)
    B = np.zeros((16, 1), np.float32)
    B[0], B[8] = 1.0, 2.0 ** -24
    assert o.gemm_model(A, B)[0, 0] == 1.0 and o.gemm_model(-A, B)[0, 0] == -1.0
    assert o.trunc_fp32(np.array([1 + 2.0 ** -30]))[0] == 1.0


def test_dispatch_mirrors():
    assert o.pick_split(624, 256, 8192, SM) == 27          # ceil(264 / 10) tiles, under the ceil(8192 / 256) cap
    assert o.pick_split(256, 32, 409600, SM) == 64         # DIN config 4, transposed: the 64 cap
    assert o.pick_split(128, 64, 200, SM) == 1
    assert o.dw_transposed(64, 128) and not o.dw_transposed(65, 128) and not o.dw_transposed(64, 127)
    assert o.dw_split(409600, 32, 256, SM) == (64, 6400) and o.dw_split(128 * 741, 256, 256, SM) == (64, 1482)
    assert [o.bn_class(n) for n in (1, 32, 33, 64, 65, 400)] == [32, 32, 64, 64, 128, 128]


def test_covering_design():
    """Every value of every axis, and every BN x tile x alignment x stages combination of the forward product."""
    cs = o.covering_cases()
    combos = {(o.bn_class(c["Nd"]), c["M"] % o.TC_BM == 0, c["misaligned"], c["Kd"] > 32) for c in cs}
    assert len(combos) == 24
    for key, values in (("Nd", sum(o.N_BY_BN.values(), ())), ("M", sum(o.M_BY_TILE.values(), ())),
                        ("Kd", sum(o.R_BY_STAGES.values(), ())), ("keep", o.MASKS), ("group_P", o.GROUP_P),
                        ("lo", o.LO), ("act", (0, 1)), ("bias", (False, True)), ("accumulate_din", (False, True))):
        assert {c[key] for c in cs} == set(values), key
    # EPI 2 on both epilogue paths: whole float4 column groups and a partial one
    acc = [c for c in cs if c["accumulate_din"]]
    assert any(c["Kd"] % 4 == 0 and not c["misaligned"] for c in acc) and any(c["Kd"] % 4 for c in acc)
    for c in cs:
        off = o.offsets(c)
        assert all(0 < v < 4 for v in off) if c["misaligned"] else not any(off)
    for (Kd, Nd) in o.DW_EDGES:
        got = {s: o.dw_split(o.dw_edge_m(Kd, Nd, s, SM), Kd, Nd, SM) for s in o.DW_SPLITS}
        assert got["one"][0] == 1 and 1 < got["middle"][0] < 64 and got["middle"][1] % 4
        M = o.dw_edge_m(Kd, Nd, "cap", SM)
        assert got["cap"][0] == 64 and M - 63 * got["cap"][1] < got["cap"][1]


def _exact_products(x, W, dZ):
    """The three products of a layer on exact data, as (name, A, B, which operand carries lo: "A" / "B" / None)."""
    has = lambda X: bool(np.any(o.split(X)[1]))
    out = []
    for name, A, B in (("fwd", x, W), ("dIn", dZ, W.T), ("dW", x.T, dZ), ("dW^T", dZ.T, x)):
        out.append((name, A, B, "A" if has(A) else "B" if has(B) else None))
    return out


def _busiest(A, B, n):
    """The n rows of A and columns of B with the most nonzeros: an output corner that sparse operands still reach."""
    r = np.sort(np.argsort(-np.count_nonzero(A, axis=1), kind="stable")[:n])
    c = np.sort(np.argsort(-np.count_nonzero(B, axis=0), kind="stable")[:n])
    return np.ascontiguousarray(A[r]), np.ascontiguousarray(B[:, c])


def _check_discriminates(A, B, lo, chunk, what, counts, n=40):
    A, B = _busiest(A, B, n)
    o.assert_exact(A, B, what)
    exact = A.astype(np.float64) @ B.astype(np.float64)
    assert np.array_equal(o.gemm_model(A, B, chunk), exact.astype(np.float32)), f"{what}: model is not exact"
    assert np.array_equal(o.gemm_emulated(A, B), exact), f"{what}: 3-term emulation is not exact"
    if lo is None:
        return
    dropped = "2xTF32 without lo*hi" if lo == "A" else "2xTF32 without hi*lo"
    for k in ("1xTF32", dropped):
        wrong = int(np.sum(o.gemm_emulated(A, B, o.BROKEN[k]) != exact))
        assert wrong > 0, f"{what}: {k} is not caught"
        counts[k] = (counts[k][0] + wrong, counts[k][1] + exact.size)


def test_exact_constructions_discriminate():
    """The covering layers and the dW edge layers of the GPU file (output subsets of the big ones, full reductions)."""
    counts = {"1xTF32": (0, 0), "2xTF32 without lo*hi": (0, 0), "2xTF32 without hi*lo": (0, 0)}
    for c in o.covering_cases():
        rng = np.random.default_rng(1000 + c["i"])
        x, W, dOut = o.exact_layer(rng, c["M"], c["Kd"], c["Nd"], c["lo"])
        for name, A, B, lo in _exact_products(x, W, dOut * np.float32(2)):
            chunk = o.dw_split(c["M"], c["Kd"], c["Nd"], SM)[1] if name.startswith("dW") else None
            _check_discriminates(A, B, lo, chunk, f"{o.case_id(c)} {name}", counts)
    for (Kd, Nd) in o.DW_EDGES:
        for s in o.DW_SPLITS:
            M = o.dw_edge_m(Kd, Nd, s, SM)
            for lo in ("in", "dOut"):
                x, W, dOut = o.exact_layer(np.random.default_rng(M + len(lo)), M, Kd, Nd, lo)
                A, B = (dOut.T, x) if o.dw_transposed(Kd, Nd) else (x.T, dOut)
                _check_discriminates(A, B, "A" if np.any(o.split(A)[1]) else "B", o.dw_split(M, Kd, Nd, SM)[1],
                                     f"dW {Kd}x{Nd} {s} lo={lo}", counts, n=24)
    for k, (wrong, n) in counts.items():
        assert wrong > 0.85 * n, f"{k} differs in only {wrong} of {n} exact outputs"


@pytest.mark.parametrize("lo", ["in", "dOut"])
@pytest.mark.parametrize("case", o.LONG_DW, ids=lambda c: c[0].replace(" ", "_"))
def test_long_sparse_construction(case, lo):
    """The long dW reductions: the precondition holds at the full M, and the model over its 64 chunks is exact."""
    name, M, Kd, Nd, per_col = case
    rng = np.random.default_rng(M + len(lo))
    x = o.grid_lo(rng, (M, Kd)) if lo == "in" else o.grid_int(rng, (M, Kd))
    rows, cols, vals = o.sparse_dz(rng, M, Nd, per_col, lo)
    assert per_col * 3 * (3 + o.GRID) <= o.EXACT_LIMIT
    keep = cols < 6
    Z = np.zeros((M, 6), np.float32)
    Z[rows[keep], cols[keep]] = vals[keep]
    assert np.count_nonzero(Z) == per_col * 6
    counts = {"1xTF32": (0, 0), "2xTF32 without lo*hi": (0, 0), "2xTF32 without hi*lo": (0, 0)}
    A, B = (Z.T, x[:, :6]) if o.dw_transposed(Kd, Nd) else (x[:, :6].T, Z)
    _check_discriminates(A, B, "A" if np.any(o.split(A)[1]) else "B", o.dw_split(M, Kd, Nd, SM)[1], name, counts, n=6)


def test_accuracy_tolerances_discriminate():
    """For every accuracy case of the GPU file (a 32 x 32 output corner, the full reduction): every broken emulation
    fails the tolerance, and the model of the kernel passes it, its error at least 16x below the best broken one."""
    for name, i, M, Kd, Nd in o.accuracy_layers():
        x, W, dZ = o.accuracy_operands(M, Kd, Nd, i, seed=i)
        for p, A, B, chunk in o.products(x, W, dZ, SM):
            A, B = np.ascontiguousarray(A[:32]), np.ascontiguousarray(B[:, :32])
            tol, broken = o.tolerance(A, B)
            assert all(v > tol for v in broken.values())
            model = o.rel_metric(o.gemm_model(A, B, chunk), A, B)
            assert model * 16 <= min(broken.values()), f"{name} layer {i} {p}: model {model:.3e} tol {tol:.3e}"
