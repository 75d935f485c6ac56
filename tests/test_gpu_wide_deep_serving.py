"""wide_n_deep's serving input on the H100: ctr_wd_serve_input (csrc/wd_serving.cu) and serving.WideDeepServable against
ctr_wd_input_fwd / WideDeep.predict bit for bit on one-value requests, against the fp64 restatement in
tests/wd_serving_oracle.py on everything else, and end to end from the drop-in's export."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import wide_deep as owd
from tests import wd_serving_oracle as so

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
I32_MAX, I32_MIN = 2 ** 31 - 1, -2 ** 31


def _model(model_type, K=32, B=128, layers="256,128,64", seed=0):
    """a WideDeep on cuda:0 with every variable random (the linear part starts at zero otherwise)"""
    from tf_repos_b200.wide_deep import WideDeep
    m = WideDeep(K, B, layers, model_type, device="cuda:0", seed=seed)
    g = torch.Generator().manual_seed(seed + 100)
    m.load_variables({n: torch.randn(v.shape, generator=g) * 0.3 for n, v in m.variables().items()})
    return m


def _servable(m):
    from tf_repos_b200.serving import WideDeepServable
    return WideDeepServable(m)


def _oracle(m):
    o = owd.WideDeep(m.K, ",".join(map(str, m.layers)), m.model_type, dtype=torch.float64)
    for n, v in m.variables().items():
        o.params[n].copy_(v.detach().cpu().double().reshape(o.params[n].shape))
    return o


def _stage(examples, dev="cuda:0"):
    lens = [len(e) for e in examples]
    off = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int64, device=dev)
    data = torch.tensor(np.frombuffer(b"".join(examples) or b"\0", dtype=np.uint8), device=dev)
    return data, off


def _run_kernel(m, examples, example_base=0):
    from tf_repos_b200 import ops
    from tf_repos_b200.wide_deep import NUM_BUCKETS
    n = len(examples)
    data, off = _stage(examples)
    x = torch.full((n, m.D), float("nan"), device="cuda:0") if m.has_dnn else None
    lin = torch.full((n,), float("nan"), device="cuda:0") if m.has_linear else None
    err = torch.full((1,), -1, dtype=torch.int64, device="cuda:0")
    ops.wd_serve_input(data, off, example_base, m.emb.var if m.has_dnn else None,
                       m.wide_cat.var if m.has_linear else None,
                       m.dense_lin["linear/numeric"] if m.has_linear else None,
                       m.dense_lin["linear/linear_model/bias_weights"] if m.has_linear else None,
                       m.num_perm, NUM_BUCKETS, m.K, x, lin, err)
    return x, lin, int(err.item())


def _one_value_rows(n, seed):
    g = np.random.default_rng(seed)
    dense = g.standard_normal((n, 13)).astype(np.float32)
    cat = g.integers(0, 10000, (n, 26))
    special = [0, 9999, 10000, -1, I32_MAX, I32_MIN]       # ids ctr_wd_input_fwd sees the same as int32
    cat.reshape(-1)[: len(special)] = special
    cat.reshape(-1)[g.integers(0, cat.size, n)] = g.choice(special, n)
    return dense, cat


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model_type", ["wide", "deep", "wide_n_deep"])
def test_one_value_requests_are_bit_identical_to_wd_input_fwd_and_predict(model_type):
    from tf_repos_b200 import ops
    from tf_repos_b200.wide_deep import NUM_BUCKETS
    m = _model(model_type, B=128)
    n = 300                                                   # three slices of the 128-row servable
    dense, cat = _one_value_rows(n, 1)
    reqs = [so.request_row(dense[i], [[int(v)] for v in cat[i]], packed=i % 3 != 0) for i in range(n)]
    x, lin, err = _run_kernel(m, reqs)
    assert err == -1
    d_dense, d_cat = torch.from_numpy(dense).cuda(), torch.from_numpy(cat.astype(np.int32)).cuda()
    x_ref = torch.full_like(x, float("nan")) if x is not None else None
    lin_ref = torch.full_like(lin, float("nan")) if lin is not None else None
    flat = torch.empty(n, 26, dtype=torch.int32, device="cuda:0")
    ops.wd_input_fwd(d_cat, d_dense, m.emb.var if m.has_dnn else None, m.wide_cat.var if m.has_linear else None,
                     m.dense_lin["linear/numeric"] if m.has_linear else None,
                     m.dense_lin["linear/linear_model/bias_weights"] if m.has_linear else None,
                     m.num_perm, NUM_BUCKETS, m.K, flat, x_ref, lin_ref)
    for got, want in ((x, x_ref), (lin, lin_ref)):
        if want is not None:
            assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    out = _servable(m).classify(reqs)
    want = np.concatenate([m.predict(d_dense[lo:lo + 128], d_cat[lo:lo + 128]).cpu().numpy() for lo in range(0, n, 128)])
    assert np.array_equal(out["scores"][:, 1].view(np.int32), want.view(np.int32))
    assert np.array_equal(out["scores"][:, 0], np.float32(1) - want)
    assert out["scores"].dtype == np.float32 and out["classes"].tolist() == [[b"0", b"1"]] * n


def _random_request(i, g):
    """multi-valued, empty and missing bags, packed and unpacked lists, shuffled entries, duplicate keys (the last
    wins), unknown keys and ids outside [0, 10000) in all 64 bits"""
    packed = bool(g.integers(2))
    entries = [(owd.NUM_NAMES[j], so.float_feature([g.standard_normal()], packed)) for j in range(13)]
    for c in owd.CAT_NAMES:
        r = g.integers(10)
        if r == 0:
            continue                                         # missing
        bag = [] if r == 1 else list(g.integers(0, 10000, g.integers(1, 6)))
        if bag and g.integers(4) == 0:
            bag[0] = int(g.choice([-1, 10000, 2 ** 32 + 5, 2 ** 63 - 1, -2 ** 63, I32_MIN]))
        if len(bag) > 1 and g.integers(3) == 0:
            bag.append(bag[0])                              # a duplicate id
        entries.append((c, so.int64_feature(bag, bool(g.integers(2)))))
    for _ in range(g.integers(3)):                           # a superseded entry of a model key
        k = so.KEYS[g.integers(39)]
        entries.insert(0, (k, so.int64_feature([1, 2]) if k[0] == "C" else so.float_feature([7.0])))
    entries += [("C%d" % (j + 1), so.int64_feature([123])) for j in range(g.integers(0, 14))]   # unknown keys
    entries += [("I14", so.float_feature([1.0, 2.0])), ("label", so.bytes_feature([b"1"]))]
    head, tail = entries[: len(entries) // 2], entries[len(entries) // 2:]
    g.shuffle(tail)                                          # shuffled, but a superseded entry stays ahead
    return so.example(head + tail)


@pytest.mark.parametrize("K", [8, 32])
@pytest.mark.parametrize("model_type", ["wide", "deep", "wide_n_deep"])
def test_kernel_matches_the_fp64_oracle_on_random_requests(model_type, K):
    m = _model(model_type, K=K, B=256, layers="64,32", seed=K)
    g = np.random.default_rng(K)
    reqs = [_random_request(i, g) for i in range(200)] + [so.client_request()]
    x, lin, err = _run_kernel(m, reqs)
    assert err == -1
    o = _oracle(m)
    o_abs = _oracle(m)
    for v in o_abs.params.values():
        v.abs_()

    def inputs(model):
        """the x row and the linear logit of every request in fp64, from the oracle's columns"""
        rows, lin_rows, dense = so.columns(model, reqs)
        if model is o_abs:
            dense = dense.abs()
        xs = torch.cat([rows[c] for c in owd.CAT_NAMES] + [dense[:, j:j + 1] for j in owd.NUM_SORTED], 1) \
            if m.has_dnn else None
        if not m.has_linear:
            return xs, None
        w = model.params
        lin = sum(lin_rows[c].reshape(-1) for c in owd.CAT_NAMES) + w["linear/linear_model/bias_weights"]
        lin = lin + sum(dense[:, j] * w[f"linear/linear_model/{owd.NUM_NAMES[j]}/weights"].reshape(()) for j in range(13))
        return xs, lin

    # U = 2^-24 per rounded fp32 operation: a bag of <= 7 rows summed and divided (x), <= 7 weights + one fma + five
    # butterfly levels + the bias per lane (lin) stay within 1e-6 of the sum of the absolute values of their terms
    (x_want, lin_want), (x_mag, lin_mag) = inputs(o), inputs(o_abs)
    if m.has_dnn:
        err_x = (x.cpu().double() - x_want).abs()
        assert torch.all(err_x <= 1e-6 * x_mag), (err_x / x_mag.clamp_min(1e-300)).max()
    if m.has_linear:
        err_l = (lin.cpu().double() - lin_want).abs()
        assert torch.all(err_l <= 1e-6 * lin_mag), (err_l / lin_mag).max()
    p = _servable(m).classify(reqs)["scores"][:, 1].astype(np.float64)
    p_ref = so.classify(o, reqs)["scores"][:, 1]
    np.testing.assert_allclose(p, p_ref, rtol=1e-5, atol=1e-6)


def _good():
    return so.request_row([1.0] * 13, [[1]] * 26)


ERRORS = [
    ("truncated", _good()[:-3]),
    ("packed floats not a multiple of 4", so.example([("I2", b"\x12\x05\x0a\x03abc")] + [
        (k, so.float_feature([1.0])) for k in owd.NUM_NAMES[2:]])),
    ("key not UTF-8", so.example([(b"\xc3\x28", so.float_feature([1.0]))])),
    ("I missing", so.example([(k, so.float_feature([1.0])) for k in owd.NUM_NAMES[1:]])),
    ("I empty Feature", so.example([(k, so.float_feature([1.0]) if k != "I13" else None) for k in owd.NUM_NAMES])),
    ("I two values", so.example([(k, so.float_feature([1.0, 2.0] if k == "I7" else [1.0], packed=False))
                                 for k in owd.NUM_NAMES])),
    ("Int64List under I", so.example([(k, so.float_feature([1.0]) if k != "I3" else so.int64_feature([1]))
                                      for k in owd.NUM_NAMES])),
    ("FloatList under C", so.example([(k, so.float_feature([1.0])) for k in owd.NUM_NAMES] +
                                     [("C20", so.float_feature([1.0]))])),
    ("BytesList under C", so.example([(k, so.float_feature([1.0])) for k in owd.NUM_NAMES] +
                                     [("C39", so.bytes_feature([b"1"]))])),
    ("several kinds", so.example([(k, so.float_feature([1.0])) for k in owd.NUM_NAMES] +
                                 [("C14", so.int64_feature([1]) + so.float_feature([1.0]))])),
]


@pytest.mark.parametrize("what,bad", ERRORS, ids=[e[0] for e in ERRORS])
def test_errors_name_the_first_bad_example_and_the_servable_recovers(what, bad):
    m = _model("wide_n_deep", K=8, B=64, layers="16")
    s = _servable(m)
    reqs = [_good()] * 150
    reqs[97] = bad                                           # in the second 64-row slice
    reqs[140] = bad
    with pytest.raises(ValueError) as e:
        so.classify(_oracle(m), reqs)
    msg = str(e.value)
    assert msg.startswith("example 97: ")
    with pytest.raises(ValueError) as e:
        s.classify(reqs)
    assert str(e.value) == msg
    good = [_good(), so.client_request()]
    np.testing.assert_allclose(s.classify(good)["scores"], so.classify(_oracle(m), good)["scores"], rtol=1e-5, atol=1e-6)


def test_request_sizes():
    m = _model("wide_n_deep", K=8, B=64, layers="16")
    s = _servable(m)
    from tf_repos_b200 import _lib
    n0 = _lib.launch_count()
    out = s.classify([])
    assert out["scores"].shape == (0, 2) and out["scores"].dtype == np.float32 and out["classes"].shape == (0, 2)
    assert _lib.launch_count() == n0                         # n = 0: no launch
    g = np.random.default_rng(5)
    reqs = [_random_request(i, g) for i in range(64 * 3 + 5)]
    o = _oracle(m)
    for n in (1, 64, 65, len(reqs)):
        got, want = s.classify(reqs[:n]), so.classify(o, reqs[:n])
        assert got["scores"].shape == (n, 2) and got["classes"].shape == (n, 2)
        np.testing.assert_allclose(got["scores"], want["scores"], rtol=1e-5, atol=1e-6)


# ---------------------------------------------------------------------------------------------------------------------
def _csv(path, n, seed):
    g = np.random.default_rng(seed)
    with open(path, "w") as fh:
        for _ in range(n):
            dense = ["%.4f" % v for v in g.random(13)]
            cat = [str(v) for v in g.integers(0, 12000, 26)]      # a few ids out of range
            fh.write(",".join([str(int(g.integers(2)))] + dense + cat) + "\n")


@pytest.mark.parametrize("model_type", ["wide", "deep", "wide_n_deep"])
def test_export_model_answers_the_serving_request_with_pred_txt(tmp_path, model_type):
    from tf_repos_b200.serving import Servable
    from tf_repos_b200.wide_deep_main import decode_csv_file
    tmp = str(tmp_path)
    os.makedirs(tmp + "/data")
    _csv(tmp + "/data/tr0.csv", 300, 1)
    _csv(tmp + "/data/te0.csv", 77, 2)
    common = [sys.executable, os.path.join(ROOT, "Model_pipeline", "wide_n_deep.py"), "--model_type=" + model_type,
              "--embedding_size=8", "--batch_size=32", "--deep_layers=32,16", "--num_epochs=2", "--log_steps=5",
              "--data_dir=" + tmp + "/data", "--model_dir=" + tmp + "/ckpt/m_", "--dt_dir=20261016",
              "--servable_model_dir=" + tmp + "/export"]
    for task in ("train", "predict", "export_model"):
        r = subprocess.run(common + ["--task_type=" + task], capture_output=True, text=True, timeout=280)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    want = np.array([float(l) for l in open(tmp + "/data/pred.txt").read().split()], dtype=np.float64)
    _, dense, cat = decode_csv_file(tmp + "/data/te0.csv")
    reqs = [so.request_row(dense[i], [[int(v)] for v in cat[i]]) for i in range(len(dense))]
    s = Servable.load(tmp + "/export", max_batch=32)
    out = s.classify(reqs)
    assert len(want) == 77 and out["scores"].shape == (77, 2)
    np.testing.assert_allclose(out["scores"][:, 1], want, atol=1e-6)
    assert out["classes"].tolist() == [[b"0", b"1"]] * 77
