"""wide_n_deep's serving input on the CPU: known answers for the restatement in tests/wd_serving_oracle.py (parse spec,
map-entry rules, identity buckets, combiners, errors and the reference client's request, quirk Q13)."""
import numpy as np
import pytest
import torch

from oracle import wide_deep as owd
from tests import wd_serving_oracle as so

F64 = torch.float64


def _model(model_type="wide_n_deep", K=4):
    m = owd.WideDeep(K, "8,4", model_type, seed=1, dtype=F64)
    g = torch.Generator().manual_seed(2)
    for name, p in m.params.items():        # the linear weights start at zero: give every variable a value
        p.copy_(torch.randn(p.shape, generator=g, dtype=F64))
    return m


def _rows(n, seed):
    g = np.random.default_rng(seed)
    dense = g.standard_normal((n, 13)).astype(np.float32)
    cat = g.integers(0, 10000, (n, 26))
    return dense, cat


@pytest.mark.parametrize("model_type", ["wide", "deep", "wide_n_deep"])
def test_single_value_bags_equal_predict_on_the_csv_row(model_type):
    m = _model(model_type)
    dense, cat = _rows(5, 0)
    reqs = [so.request_row(dense[i], [[int(v)] for v in cat[i]], packed=i % 2 == 0) for i in range(5)]
    got = so.classify(m, reqs)
    want = m.predict(torch.from_numpy(dense), torch.from_numpy(cat))["prob"].numpy()
    assert np.array_equal(got["scores"][:, 1], want)
    assert np.array_equal(got["scores"][:, 0], 1 - want)
    assert got["classes"].tolist() == [[b"0", b"1"]] * 5


def test_empty_and_missing_bags_give_zero_rows():
    m = _model()
    dense = [0.25] * 13
    entries = [(owd.NUM_NAMES[j], so.float_feature([dense[j]])) for j in range(13)]
    entries += [("C14", so.int64_feature([])), ("C15", None), ("C16", so.int64_feature([7]))]   # C17..C39 missing
    rows, lin_rows, _ = so.columns(m, [so.example(entries)])
    for c in owd.CAT_NAMES:
        if c == "C16":
            assert torch.equal(rows[c][0], m.params[m.emb_name(c)][7])
            continue
        assert torch.equal(rows[c], torch.zeros(1, m.K, dtype=F64)), c
        assert float(lin_rows[c]) == 0.0, c


def test_mean_of_two_rows_and_duplicate_ids():
    m = _model()
    t = m.params[m.emb_name("C20")]
    w = m.params["linear/linear_model/C20/weights"].reshape(-1)
    bags = [[1]] * 26
    bags[6] = [11, 12]
    rows, lin_rows, _ = so.columns(m, [so.request_row([0.0] * 13, bags)])
    assert torch.allclose(rows["C20"][0], (t[11] + t[12]) / 2, rtol=0, atol=1e-15)
    assert float(lin_rows["C20"]) == pytest.approx(float(w[11] + w[12]), abs=1e-15)
    bags[6] = [11, 11, 12]                      # a duplicate counts each time it appears
    rows, lin_rows, _ = so.columns(m, [so.request_row([0.0] * 13, bags, packed=False)])
    assert torch.allclose(rows["C20"][0], (2 * t[11] + t[12]) / 3, rtol=0, atol=1e-15)
    assert float(lin_rows["C20"]) == pytest.approx(float(2 * w[11] + w[12]), abs=1e-15)


@pytest.mark.parametrize("v", [2 ** 32 + 5, -1, 10000, 2 ** 63 - 1, -2 ** 63])
def test_out_of_range_ids_use_all_64_bits(v):
    m = _model()
    bags = [[3]] * 26
    bags[0] = [v]
    dense, b = so.parse(so.request_row([1.0] * 13, bags))
    assert b[0] == [v & (2 ** 64 - 1)] and so.bucket(b[0][0]) == 0
    rows, _, _ = so.columns(m, [so.request_row([1.0] * 13, bags)])
    assert torch.equal(rows["C14"][0], m.params[m.emb_name("C14")][0])
    assert so.bucket(9999) == 9999 and so.bucket(5) == 5


def test_last_entry_wins_and_unknown_keys_are_ignored():
    base = [(owd.NUM_NAMES[j], so.float_feature([j + 0.5])) for j in range(13)]
    ex = so.example([("C14", so.int64_feature([1])), ("I3", so.float_feature([9.0])), ("C1", so.int64_feature([5])),
                     ("C40", so.int64_feature([5])), ("I14", so.float_feature([1.0, 2.0])), ("C014", so.float_feature([1])),
                     ("I0", so.bytes_feature([b"x"])), ("foo", so.float_feature([1.0])), ("c15", so.int64_feature([8])),
                     (None, so.float_feature([1.0]))] + base + [("C14", so.int64_feature([2, 3])),
                                                                ("C15", so.float_feature([1.0])), ("C15", None)])
    dense, bags = so.parse(ex)
    assert dense == [j + 0.5 for j in range(13)]    # I3 = 9.0 came first and lost
    assert bags[0] == [2, 3] and bags[1] == [] and all(b == [] for b in bags[2:])


def test_shuffled_entries_and_unpacked_lists_parse_alike():
    dense, cat = _rows(1, 3)
    bags = [[int(v), int(v) + 1] for v in cat[0]]
    a = so.request_row(dense[0], bags)
    entries = [(owd.NUM_NAMES[j], so.float_feature([dense[0][j]], packed=False)) for j in range(13)]
    entries += [(c, so.int64_feature(bags[f], packed=False)) for f, c in enumerate(owd.CAT_NAMES)]
    np.random.default_rng(4).shuffle(entries)
    assert so.parse(a) == so.parse(so.example(entries))


def _good_entries():
    return [(owd.NUM_NAMES[j], so.float_feature([1.0])) for j in range(13)] + \
           [(c, so.int64_feature([1])) for c in owd.CAT_NAMES]


def _with(key, feat):
    return so.example([(k, f) for k, f in _good_entries() if k != key] + ([(key, feat)] if feat is not False else []))


ERROR_CASES = [
    ("truncated", so.request_row([1.0] * 13, [[1]] * 26)[:-3], so.MALFORMED, 0),
    ("wire type 3", b"\x0b" + so.request_row([1.0] * 13, [[1]] * 26), so.MALFORMED, 0),
    ("packed floats not a multiple of 4", _with("I2", b"\x12\x05\x0a\x03abc"), so.MALFORMED, 0),
    ("bad varint in a bag", _with("C30", b"\x1a\x03\x0a\x01\x80"), so.MALFORMED, 0),
    ("key not UTF-8", so.example(_good_entries() + [(b"\xff", so.float_feature([1.0]))]), so.MALFORMED, 0),
    ("I missing", _with("I5", False), so.MISSING, 4),
    ("I empty Feature", _with("I13", None), so.COUNT, 12),
    ("I empty FloatList", _with("I1", so.float_feature([])), so.COUNT, 0),
    ("I two values", _with("I7", so.float_feature([1.0, 2.0])), so.COUNT, 6),
    ("Int64List under I", _with("I3", so.int64_feature([1])), so.KIND, 2),
    ("BytesList under I", _with("I3", so.bytes_feature([b"1"])), so.KIND, 2),
    ("FloatList under C", _with("C20", so.float_feature([1.0])), so.KIND, 19),
    ("BytesList under C", _with("C39", so.bytes_feature([b"1"])), so.KIND, 38),
    ("several kinds", _with("C14", so.int64_feature([1]) + so.float_feature([1.0])), so.KIND, 13),
    ("first failing key wins", so.example([(k, f) for k, f in _good_entries() if k not in ("I9", "C15")] +
                                          [("C15", so.float_feature([1.0]))]), so.MISSING, 8),
]


@pytest.mark.parametrize("what,ex,check,key", ERROR_CASES, ids=[c[0] for c in ERROR_CASES])
def test_errors_name_the_example_and_the_key(what, ex, check, key):
    m = _model()
    good = so.request_row([1.0] * 13, [[1]] * 26)
    with pytest.raises(so.Rejected) as e:
        so.classify(m, [good, good, good, ex, ex])
    assert (e.value.index, e.value.check, e.value.key) == (3, check, key)
    assert str(e.value).startswith("example 3: ")
    if check != so.MALFORMED:
        assert repr(so.KEYS[key]) in str(e.value)


def test_q13_the_reference_clients_request():
    dense, bags = so.parse(so.client_request())
    assert dense == [0.5] * 13
    assert bags[:13] == [[123]] * 13 and bags[13:] == [[]] * 13
    m = _model()
    p = so.classify(m, [so.client_request()])["scores"][0, 1]
    rows = {c: (m.params[m.emb_name(c)][123] if f < 13 else torch.zeros(m.K, dtype=F64)).reshape(1, -1)
            for f, c in enumerate(owd.CAT_NAMES)}
    lin = {c: (m.params[f"linear/linear_model/{c}/weights"][123] if f < 13 else torch.zeros(1, dtype=F64)).reshape(1, 1)
           for f, c in enumerate(owd.CAT_NAMES)}
    want = float(torch.sigmoid(m._forward(m.params, rows, lin, torch.full((1, 13), 0.5, dtype=F64))))
    assert p == pytest.approx(want, rel=1e-15)
