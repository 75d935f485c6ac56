"""The scoring path's host side without a GPU: the integer restatement of ctr_format_preds' "%f" against Python's own
"%f" on every rounding case that matters, and tf.metrics.auc from ctr_auc_counts' histogram (scoring.auc_of_histogram)
against estimator.auc_200 bit for bit."""
import numpy as np
import pytest

from tests import fixed6_oracle as fo
from tf_repos_b200.estimator import auc_200, auc_thresholds
from tf_repos_b200.scoring import auc_of_histogram


def _same_as_python(x: np.ndarray):
    bits = x.view(np.uint32).tolist()
    with np.errstate(invalid="ignore"):
        vals = x.astype(np.float64).tolist()
    bad = [(hex(b), fo.fixed6_bits(b), "%f" % v) for b, v in zip(bits, vals) if fo.fixed6_bits(b) != "%f" % v]
    assert not bad, bad[:10]


def test_ties_and_their_neighbours():
    x = fo.ties_and_neighbours()
    assert len(x) == 64 * 17
    _same_as_python(x)
    assert fo.fixed6(1 / 128) == "0.007812" and fo.fixed6(3 / 128) == "0.023438"


def test_both_sides_of_every_rounding_boundary_in_0_1():
    x = fo.rounding_boundaries()
    assert len(x) == 2_000_000
    _same_as_python(x)


def test_random_bit_patterns_over_the_whole_range():
    _same_as_python(fo.random_patterns(1_000_000, seed=7))


def test_specials():
    x = fo.specials()
    _same_as_python(x)
    got = [fo.fixed6_bits(b) for b in x.view(np.uint32).tolist()]
    assert got[:8] == ["0.000000", "-0.000000", "inf", "-inf", "nan", "nan", "nan", "nan"]
    flt_max = fo.fixed6_bits(0xFF7FFFFF)
    assert flt_max == "-340282346638528859811704183484516925440.000000" and len(flt_max) == 47


def _auc_cases():
    rng = np.random.default_rng(3)
    thr = auc_thresholds()
    on = np.concatenate([thr, np.nextafter(thr, np.float32(-2)), np.nextafter(thr, np.float32(2))])
    skew = rng.beta(0.6, 6.0, 50_000).astype(np.float32)
    yield "random", rng.random(20_000).astype(np.float32), (rng.random(20_000) < 0.3).astype(np.float32)
    yield "skewed", skew, (rng.random(50_000) < skew).astype(np.float32)
    yield "on_thresholds", np.tile(on, 3), (rng.random(3 * len(on)) < 0.5).astype(np.float32)
    p = rng.random(5000).astype(np.float32)
    p[::7] = np.nan
    lab = (rng.random(5000) < 0.4).astype(np.float32)
    lab[::11] = np.nan
    lab[1::13] = 0.5
    lab[2::17] = -0.0
    yield "nan_and_half_labels", p, lab
    yield "only_positives", rng.random(1000).astype(np.float32), np.ones(1000, np.float32)
    yield "only_negatives", rng.random(1000).astype(np.float32), np.zeros(1000, np.float32)
    yield "n1", np.array([0.3], np.float32), np.array([1.0], np.float32)
    yield "outside_0_1", np.array([-np.inf, -1, 0, -0.0, 1, 2, np.inf], np.float32), np.array([1, 0, 1, 0, 1, 0, 1], np.float32)


@pytest.mark.parametrize("case", [c[0] for c in _auc_cases()])
def test_auc_of_histogram_is_auc_200_bit_for_bit(case):
    _, p, lab = next(c for c in _auc_cases() if c[0] == case)
    h = fo.auc_histogram(p, lab, auc_thresholds())
    assert h.sum() == len(p)
    got, want = auc_of_histogram(h), auc_200(lab, p)
    assert np.float64(got).tobytes() == np.float64(want).tobytes() or (np.isnan(got) and np.isnan(want)), (got, want)


def test_histogram_counts_are_auc_200s_tp_and_fp():
    rng = np.random.default_rng(5)
    p = np.concatenate([auc_thresholds(), rng.random(3000).astype(np.float32), [np.nan]]).astype(np.float32)
    lab = (rng.random(len(p)) < 0.5).astype(np.float32)
    thr = auc_thresholds()
    h = fo.auc_histogram(p, lab, thr)
    pos = np.sort(p[lab.astype(bool)])
    tp = len(pos) - np.searchsorted(pos, thr, side="right")
    assert np.array_equal(np.cumsum(h[1][::-1])[::-1][1:], tp)
