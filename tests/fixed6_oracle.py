"""A restatement, in exact integers, of how ctr_format_preds prints a float32 the way Python's "%f" % float(x) does,
and of the ctr_auc_counts histogram; tests/test_scoring_cpu.py holds both against Python and auc_200.

x = M * 2^E with M < 2^24.  E < 0: q = (M * 10^6) >> -E rounded half to even on the exact remainder (M * 10^6 < 2^44;
a shift of 64 or more gives 0); the text is q // 10^6 "." q % 10^6.  E >= 0: x is the integer M << E, fraction .000000.
NaN of either sign prints "nan"; the sign of everything else is kept ("-0.000000", "-inf")."""
import numpy as np

N_THR = 200


def fixed6_bits(b: int) -> str:
    """"%f" of the float32 with bit pattern b"""
    s, e8, m = b >> 31, (b >> 23) & 0xFF, b & 0x7FFFFF
    if e8 == 0xFF:
        return "nan" if m else ("-inf" if s else "inf")
    M, E = (m | 0x800000, e8 - 150) if e8 else (m, -149)
    if E < 0:
        sh, q = -E, 0
        if sh < 64:
            P = M * 1000000
            q, r, half = P >> sh, P & ((1 << sh) - 1), 1 << (sh - 1)
            if r > half or (r == half and q & 1):
                q += 1
        ip, fr = divmod(q, 1000000)
    else:
        ip, fr = M << E, 0
    return ("-" if s else "") + "%d.%06d" % (ip, fr)


def fixed6(x) -> str:
    return fixed6_bits(int(np.float32(x).view(np.uint32)))


def auc_histogram(pred: np.ndarray, label: np.ndarray, thresholds: np.ndarray) -> np.ndarray:
    """int64 [2, 201]: per class (label == 0, label != 0 or NaN) the count of predictions with k thresholds below them;
    a NaN prediction has k = 200"""
    pred = np.asarray(pred, np.float32)
    k = np.searchsorted(thresholds, pred, side="left")            # #{t : t < p}
    k = np.where(np.isnan(pred), N_THR, k)
    cls = np.asarray(label, np.float32).astype(bool).astype(np.int64)
    return np.bincount(cls * (N_THR + 1) + k, minlength=2 * (N_THR + 1)).reshape(2, N_THR + 1).astype(np.int64)


# ---- the value sets both the CPU and the GPU tests run -------------------------------------------------------------
def ties_and_neighbours(ulps: int = 8) -> np.ndarray:
    """float32: the 64 exact ties j/128 (j odd) of [0, 1] and `ulps` ulps either side of each"""
    t = (np.arange(1, 128, 2, dtype=np.float64) / 128).astype(np.float32).view(np.int32)
    return (t[:, None] + np.arange(-ulps, ulps + 1, dtype=np.int32)[None, :]).reshape(-1).view(np.float32)


def rounding_boundaries() -> np.ndarray:
    """float32: the values nearest below and above every k * 1e-6 + 5e-7 in [0, 1] (2 M values)"""
    b = np.arange(1_000_000, dtype=np.float64) * 1e-6 + 5e-7
    f = b.astype(np.float32)
    lo = np.where(f.astype(np.float64) <= b, f, np.nextafter(f, np.float32(-1)))
    hi = np.nextafter(lo, np.float32(2))
    return np.concatenate([lo, hi])


def specials() -> np.ndarray:
    bits = [0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00000, 0x7F800001, 0xFF800001,
            0x7FBFFFFF, 0xFFFFFFFF, 0x7FD23456, 0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x00800000,
            0x7F7FFFFF, 0xFF7FFFFF, 0x3F800000, 0xBF800000, 0x4B7FFFFF, 0x4B800000, 0x4B800001, 0x3F7FFFFF,
            0x358637BD, 0x3500_0000, 0x34FF_FFFF]
    return np.array(bits, dtype=np.uint32).view(np.float32)


def random_patterns(n: int, seed: int) -> np.ndarray:
    return np.random.default_rng(seed).integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32)
