"""ESMM serving on the GPU (csrc/tfrecord_device.cu ctr_esmm_serve_scan + ctr_tfrecord_emit_esmm,
serving.ESMMServable; DESIGN.md §2.14) against the training path (esmm_main.make_batch + ESMM.predict), the fp64 oracle
tests/esmm_oracle.py and DeepCvrMTL.py's pred.txt.  ESMM's Examples have DIN's schema plus the label z, and serving
reads neither label, so tests/din_serving_oracle.py is the CPU restatement of the request's parse and checks."""
import os
import struct
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import din_serving_oracle as so

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F, N, K, LAYERS = 5, 3000, 8, "32,16"
OUTPUTS = ("pctr", "pcvr", "pctcvr")


def _randomize(m, seed):
    g = torch.Generator().manual_seed(100 + seed)
    vals = {}
    for k, v in m.variables().items():
        if "moving_variance" in k:
            vals[k] = torch.rand(v.shape, generator=g, dtype=torch.float64).float() + 0.5
        else:
            vals[k] = (torch.rand(v.shape, generator=g, dtype=torch.float64) * 0.6 - 0.3).float()
    m.load_variables(vals)
    return m


def _model(B=16, cap=4096, batch_norm=False, seed=0):
    from tf_repos_b200.esmm import ESMM
    return _randomize(ESMM(F, N, K, B, cap, deep_layers=LAYERS, dropout="0.9,0.9", batch_norm=batch_norm,
                           update_mode="lazy", seed=seed), seed)


def _servable(m):
    from tf_repos_b200.serving import ESMMServable
    return ESMMServable(m)


def _encoded(rng, maxlen, labels=True):
    """one Example with the training schema, written by tfrecord.encode_example"""
    from tf_repos_b200.tfrecord import encode_example
    ex = {"feat_ids": rng.randint(0, N, F).astype(np.int64), "a_catids": np.int64(rng.randint(0, N)),
          "a_shopids": np.int64(rng.randint(0, N)), "a_brandids": np.int64(rng.randint(0, N)),
          "a_intids": rng.randint(0, N, rng.randint(0, 4)).astype(np.int64)}
    if labels:
        ex["y"], ex["z"] = np.float32(rng.rand() < 0.4), np.float32(rng.rand() < 0.2)
    for u in so.U:
        ln = rng.randint(0, maxlen + 1)
        ex["u_%sids" % u] = rng.randint(0, N, ln).astype(np.int64)
        ex["u_%svals" % u] = (rng.randn(ln) * 2).astype(np.float32)
    return encode_example(ex)


def _request(n, seed, maxlen=6):
    rng = np.random.RandomState(seed)
    return [_encoded(rng, maxlen, labels=bool(rng.rand() < 0.5)) for _ in range(n)]


def _decode(examples, N_=None):
    """the request as esmm_main.decode's dict (z = 0.0 beside so.decode's y = 0.0, so that make_batch takes it)"""
    d = so.decode(examples, F, N_)
    d["z"] = [0.0] * len(examples)
    return d


def _training_path(m, examples):
    """ESMM.predict(make_batch(decode(...))) over slices of m.B, as esmm_main scores a data set"""
    from tf_repos_b200 import esmm_main as em
    d = _decode(examples, m.N)
    out = {k: [] for k in OUTPUTS}
    for lo in range(0, len(examples), m.B):
        idx = list(range(lo, min(lo + m.B, len(examples))))
        batch, _, n = em.make_batch(d, idx, m.B, m.device)
        for k, p in zip(OUTPUTS, m.predict(batch)):
            out[k].append(p[:n].cpu().numpy().copy())
    return {k: np.concatenate(v) for k, v in out.items()}


def _bits(a):
    return np.asarray(a, dtype=np.float32).view(np.uint32)


def _same(got, want):
    assert set(got) == set(OUTPUTS)
    for k in OUTPUTS:
        assert got[k].dtype == np.float32 and got[k].shape == want[k].shape, k
        np.testing.assert_array_equal(_bits(got[k]), _bits(want[k]), err_msg=k)


# ---- 1. the emitted batch is make_batch's -------------------------------------------------------------------------
def _emit(examples, B, cap):
    from tf_repos_b200 import ops
    dev = torch.device("cuda")
    lens = [len(e) for e in examples]
    off = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int64, device=dev)
    data = torch.tensor(np.frombuffer(b"".join(examples), np.uint8), device=dev)
    i32 = dict(dtype=torch.int32, device=dev)
    slot_off, slot_len = torch.empty(B, dtype=torch.int64, device=dev), torch.empty(B, **i32)
    total, err = torch.full((1,), -5, dtype=torch.int64, device=dev), torch.full((1,), -1, dtype=torch.int64, device=dev)
    batch = {"feat_ids": torch.full((B, F), -7, **i32), "a_ids": torch.full((3, B), -7, **i32),
             "bag_ids": torch.full((cap + 40,), -7, **i32), "bag_wgt": torch.full((cap + 40,), 7.0, device=dev),
             "bag_off": torch.full((5 * B + 1,), -7, **i32)}
    ops.esmm_serve_scan(data, off, 0, F, B, cap, slot_off, slot_len, batch["bag_off"], total, err)
    ops.tfrecord_emit_esmm(data, slot_off, slot_len, B, F, batch["bag_off"], batch["feat_ids"], batch["a_ids"],
                           batch["bag_ids"], batch["bag_wgt"], torch.empty(B, device=dev), torch.empty(B, device=dev))
    return {k: v.cpu() for k, v in batch.items()}, int(total.item()), int(err.item())


def _edge_request(n, seed):
    """random Examples, one with every bag empty or missing and one with bags of 1 to 300 values, NaN weights and ids
    at the top of [0, 2^31)"""
    req = _request(n, seed)
    nan_bits = [0x7FC00001, 0xFFC12345, 0x7F800001, 0x00000001, 0x80000000, 0x7F800000]
    nans = [struct.unpack("<f", struct.pack("<I", b))[0] for b in nan_bits]
    if n > 2:
        req[n // 2] = so.din_example([1, 2, 3, 4, 5], [1, 1, 1])
    long_ex = so.din_example([(1 << 31) - 1, (1 << 30) + 3, 0, 1, 2], [(1 << 31) - 1, 0, 5], [(1 << 31) - 2] * 4,
                             (list(range(300)), [], [7] * 6, [(1 << 31) - 1]),
                             ([0.25] * 300, [], nans, [-0.0]), packed=False)
    req[n - 1 if n > 1 else 0] = long_ex
    return req


@pytest.mark.parametrize("n", [1, 15, 16])
def test_emitted_batch_equals_make_batch_bit_for_bit(n):
    from tf_repos_b200 import esmm_main as em
    B = 16
    req = _edge_request(n, 7 + n)
    d = _decode(req)
    want, _, _ = em.make_batch(d, list(range(n)), B, "cpu")
    nnz = want["bag_ids"].numel()
    batch, total, err = _emit(req, B, nnz + 3)
    assert err == -1 and total == nnz
    for k in ("feat_ids", "a_ids", "bag_off"):
        assert torch.equal(batch[k], want[k]), k
    assert torch.equal(batch["bag_ids"][:nnz], want["bag_ids"])
    assert torch.equal(batch["bag_wgt"][:nnz].view(torch.int32), want["bag_wgt"].view(torch.int32))
    assert torch.all(batch["bag_ids"][nnz:] == -7) and torch.all(batch["bag_wgt"][nnz:] == 7.0)


def test_a_slice_past_the_capacity_gets_empty_bags_and_reports_its_total():
    from tf_repos_b200 import esmm_main as em
    B = 16
    req = _edge_request(16, 9)
    want, _, _ = em.make_batch(_decode(req), list(range(16)), B, "cpu")
    nnz = want["bag_ids"].numel()
    batch, total, err = _emit(req, B, nnz - 1)
    assert err == -1 and total == nnz
    assert torch.all(batch["bag_off"] == 0)
    assert torch.all(batch["bag_ids"] == -7) and torch.all(batch["bag_wgt"] == 7.0)
    assert torch.equal(batch["feat_ids"], want["feat_ids"]) and torch.equal(batch["a_ids"], want["a_ids"])


# ---- 2. predict is ESMM.predict on the host-built batch -------------------------------------------------------------
@pytest.mark.parametrize("batch_norm", [False, True])
def test_predict_is_bit_identical_to_the_training_path(batch_norm):
    m = _model(B=16, batch_norm=batch_norm)
    s = _servable(m)
    for seed, n in ((1, 1), (2, 17), (3, 3 * 16 + 5)):
        req = _request(n, seed)
        _same(s.predict(req), _training_path(m, req))
    assert m.cap == 4096


def test_request_sizes():
    m = _model(B=16)
    s = _servable(m)
    empty = s.predict([])
    assert set(empty) == set(OUTPUTS) and all(v.shape == (0,) and v.dtype == np.float32 for v in empty.values())
    for n in (1, 15, 16, 32, 33):
        req = _request(n, 40 + n, maxlen=40)
        _same(s.predict(req), _training_path(m, req))


# ---- 3. fp64 ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bn", [False, True])
def test_predict_agrees_with_the_fp64_oracle(bn):
    from tests.test_gpu_esmm_deepmvm_fp64 import (ESMM_CFGS, FP, HALF_SUB, N_ESMM, U, _esmm_oracle, _long,
                                                  _tol_esmm, _within, gam)
    from tf_repos_b200 import esmm_main as em
    from tf_repos_b200.esmm import ESMM
    from tf_repos_b200.tfrecord import encode_example
    cfg = "flags"
    K_, B, layers, dropout = ESMM_CFGS[cfg][:4]
    ref = _esmm_oracle(cfg, bn, torch.float64)
    if bn:
        g = torch.Generator().manual_seed(5)
        for k, v in ref.bn_state.items():
            v.copy_(torch.rand(v.shape, generator=g, dtype=torch.float64) + 0.5 if "variance" in k
                    else torch.randn(v.shape, generator=g, dtype=torch.float64) * 0.2)
            v.copy_(v.float().double())
    m = ESMM(FP, N_ESMM, K_, B, 1 << 14, deep_layers=layers, dropout=dropout, batch_norm=bn, update_mode="lazy")
    m.load_variables({**ref.params, **ref.bn_state})
    rng = np.random.RandomState(3)
    req = []
    for _ in range(B + 37):
        ex = {"feat_ids": rng.randint(0, N_ESMM, FP).astype(np.int64), "a_intids": rng.randint(0, N_ESMM, 5)}
        for k in ("a_catids", "a_shopids", "a_brandids"):
            ex[k] = np.int64(rng.randint(0, N_ESMM))
        for u in so.U:
            ln = rng.randint(0, 50)
            ex["u_%sids" % u] = rng.randint(0, N_ESMM, ln).astype(np.int64)
            ex["u_%svals" % u] = rng.rand(ln).astype(np.float32) * 2
        req.append(encode_example(ex))
    got = _servable(m).predict(req)
    d = so.decode(req, FP, N_ESMM)
    d["z"] = [0.0] * len(req)
    tol = _tol_esmm(cfg, bn)
    for lo in range(0, len(req), B):
        idx = list(range(lo, min(lo + B, len(req))))
        batch, _, n = em.make_batch(d, idx, B, "cpu")
        out = ref.predict(_long(batch))
        pt, pv, P = (out[k][:n].numpy() for k in OUTPUTS)
        E = {t: tol * float(out[f"y_{t}"].abs().max()) for t in ("ctr", "cvr")}
        dpt, dpv = E["ctr"] / 4 + gam(6) * pt + HALF_SUB, E["cvr"] / 4 + gam(6) * pv + HALF_SUB
        dP = dpt * pv + pt * dpv + dpt * dpv + U * P
        tag = f"batch_norm={bn} examples {lo}..{lo + n - 1}"
        _within(torch.from_numpy(got["pctr"][lo:lo + n]), pt, dpt, f"{tag}: pctr")
        _within(torch.from_numpy(got["pcvr"][lo:lo + n]), pv, dpv, f"{tag}: pcvr")
        _within(torch.from_numpy(got["pctcvr"][lo:lo + n]), P, dP, f"{tag}: pctcvr")


# ---- 4. DeepCvrMTL.py train -> serve ------------------------------------------------------------------------------
def test_a_trained_model_dir_answers_with_pred_txt(tmp_path):
    from tests.test_gpu_esmm_cli import _write
    from tf_repos_b200 import tf_checkpoint
    from tf_repos_b200.serving import ESMMServable
    from tf_repos_b200.tfrecord import read_records
    tmp = str(tmp_path)
    os.makedirs(tmp + "/data/tr"); os.makedirs(tmp + "/data/te"); os.makedirs(tmp + "/ckpt")
    _write(tmp + "/data/tr/part0.tfrecord", 150, 1)
    _write(tmp + "/data/te/part0.tfrecord", 70, 3)
    common = [sys.executable, os.path.join(ROOT, "Model_pipeline", "DeepCvrMTL.py"), "--field_size=11",
              "--feature_size=5000", "--embedding_size=8", "--batch_size=64", "--deep_layers=16,8", "--dropout=0.9,0.9",
              "--ctr_task_wgt=0.3", "--log_steps=100", "--num_epochs=1", "--data_dir=" + tmp + "/data",
              "--model_dir=" + tmp + "/ckpt/m_", "--dt_dir=20261019"]
    for task in ("train", "infer"):
        r = subprocess.run(common + ["--task_type=" + task], capture_output=True, text=True, timeout=280)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    mdir = tmp + "/ckpt/m_20261019"
    te = list(read_records(tmp + "/data/te/part0.tfrecord"))
    s = ESMMServable.load(mdir, 11, 5000, 8, deep_layers="16,8", max_batch=32)
    got = s.predict(te)
    lines = open(tmp + "/data/pred.txt").read().split("\n")[:-1]
    assert ["%f\t%f" % (a, b) for a, b in zip(got["pctr"], got["pcvr"])] == lines
    assert np.array_equal(_bits(got["pctcvr"]), _bits(got["pctr"] * got["pcvr"]))
    # the same variables as a TensorFlow bundle
    tf_checkpoint.save(s.model, tmp + "/tf")
    t = ESMMServable.load(tmp + "/tf", 11, 5000, 8, deep_layers="16,8", max_batch=32, checkpoint_format="tf",
                          occ_capacity=s.model.cap)
    _same(t.predict(te), got)


# ---- 5. rejections ---------------------------------------------------------------------------------------------------
def _good(i):
    return so.din_example([1 + i, 2, 3, 4, 5], [6, 7, 8], [9], ([10], [], [], []), ([0.5], [], [], []),
                          extra=[("y", so.float_feature([1.0])), ("z", so.float_feature([0.0]))])


BAD = {
    "malformed": so.example([]) + b"\x0a\x81",
    "non-utf8 key": so.example([("feat_ids", so.int64_feature([1, 2, 3, 4, 5])), (b"\xc3\x28", b"")]),
    "malformed z": so.din_example([1, 2, 3, 4, 5], [1, 2, 3], extra=[("z", b"\x12\x05\x0a")]),
    "required": so.example([("feat_ids", so.int64_feature([1, 2, 3, 4, 5]))]),
    "required a_brandids": so.din_example([1, 2, 3, 4, 5], [1, 2, 3], extra=[("a_brandids", so.int64_feature([]))]),
    "count": so.din_example([1, 2], [1, 2, 3]),
    "mismatch": so.din_example([1, 2, 3, 4, 5], [1, 2, 3], [], ([], [7], [], []), ([], [1.0, 2.0], [], [])),
    "kind": so.din_example([1, 2, 3, 4, 5], [1, 2, 3], [], ([], [4], [], []), ([], [1.0], [], []),
                           extra=[("u_shopvals", so.int64_feature([1]))]),
    "several kinds": so.din_example([1, 2, 3, 4, 5], [1, 2, 3],
                                    extra=[("a_intids", so.int64_feature([1]) + so.float_feature([1.0]))]),
    "range": so.din_example([1, 2, 3, 4, 5], [1, 2, 3], [1 << 35]),
    "range feat_ids": so.din_example([1, 2, 3, (1 << 64) - 1, 5], [1, 2, 3]),
    "feature_size": so.din_example([1, 2, 3, 4, 5], [1, 2, 3], [], ([], [], [N], []), ([], [], [1.0], [])),
    "feature_size a_catids": so.din_example([1, 2, 3, 4, 5], [N, 2, 3]),
    "feature_size feat_ids": so.din_example([1, 2, 3, N + 7, 5], [1, 2, 3]),
}


@pytest.mark.parametrize("what", sorted(BAD))
@pytest.mark.parametrize("at", [5, 37])
def test_errors_name_the_bad_example_and_the_servable_recovers(what, at):
    m = _model(B=16)
    s = _servable(m)
    req = [_good(i) for i in range(45)]
    req[at] = BAD[what]
    req[at + 3] = BAD["malformed"]
    with pytest.raises(so.Rejected) as want:
        so.decode(req, F, N)
    assert want.value.index == at
    with pytest.raises(ValueError) as got:
        s.predict(req)
    assert str(got.value) == str(want.value)
    assert m.oob.tolist()[0] == 0
    good = [_good(i) for i in range(20)]
    _same(s.predict(good), _training_path(m, good))


# ---- 6. growth -------------------------------------------------------------------------------------------------------
CAP = 128      # above every slice of _request(20, 21, maxlen=2) and the first of _long_request, below its second


def _long_request():
    req = _request(35, 22, maxlen=2)
    req[30] = so.din_example([1, 2, 3, 4, 5], [1, 2, 3], list(range(1, 60)),
                             ([7] * 130, [], [8] * 50, []), ([0.5] * 130, [], [1.5] * 50, []))
    return req


def _slice_totals(req, B):
    occ = [sum(len(v) for k, v in so.parse(r, 0, F).items() if k.startswith(("u_", "a_int")) and k.endswith("ids"))
           for r in req]
    return [sum(occ[lo:lo + B]) + (B - len(occ[lo:lo + B])) * occ[lo] for lo in range(0, len(req), B)]


def test_a_slice_past_the_capacity_is_answered_by_growing():
    m = _model(B=16, cap=CAP)
    s = _servable(m)
    small = _request(20, 21, maxlen=2)
    before = s.predict(small)
    assert m.cap == CAP
    long = _long_request()
    got = s.predict(long)
    assert m.cap == max(_slice_totals(long, 16)) > CAP
    big = _model(B=16, cap=1 << 14)
    _same(got, _servable(big).predict(long))
    _same(got, _training_path(m, long))
    cap = m.cap
    _same(s.predict(small), before)
    assert m.cap == cap and s._batch["bag_ids"].numel() == cap


class _FailingTorch:
    """torch, except that torch.empty raises CUDA out-of-memory after `after` calls"""

    def __init__(self, after):
        self.calls, self.after = 0, after

    def __getattr__(self, name):
        return getattr(torch, name)

    def empty(self, *args, **kw):
        self.calls += 1
        if self.calls > self.after:
            raise torch.cuda.OutOfMemoryError("injected allocation failure")
        return torch.empty(*args, **kw)


@pytest.mark.parametrize("after", [0, 5, 6])   # the first, bag_ids' and bag_wgt's allocation
def test_a_failed_growth_leaves_the_servable_as_it_was(monkeypatch, after):
    from tf_repos_b200 import serving
    m = _model(B=16, cap=CAP)
    s = _servable(m)
    small = _request(20, 21, maxlen=2)
    before = s.predict(small)
    monkeypatch.setattr(serving, "torch", _FailingTorch(after))
    with pytest.raises(torch.cuda.OutOfMemoryError):
        s.predict(_long_request())
    monkeypatch.undo()
    assert m.cap == CAP and m.ids_all is not None and s._batch["bag_ids"].numel() == CAP
    _same(s.predict(small), before)
    long = _long_request()
    _same(s.predict(long), _training_path(m, long))
    assert m.cap > CAP


def test_a_grown_model_no_longer_trains():
    m = _model(B=8, cap=32)
    m.grow(16)
    assert m.cap == 32 and m.ids_all is not None
    m.grow(100)
    assert m.cap == 100 and m.ids_all is None
    with pytest.raises(RuntimeError, match="grew its occurrence capacity for inference"):
        m.train_step(None, None)


def test_an_id_past_feature_size_in_a_slice_that_grows_is_rejected():
    # the id is only read, and counted, when the slice is run again at the grown capacity
    m = _model(B=16, cap=64)
    s = _servable(m)
    req = [_good(i) for i in range(24)]
    req[17] = so.din_example([1, 2, 3, 4, 5], [1, 2, 3], [], (list(range(1, 90)) + [N], [], [], []),
                             ([1.0] * 90, [], [], []))
    with pytest.raises(so.Rejected) as want:
        so.decode(req, F, N)
    with pytest.raises(ValueError) as got:
        s.predict(req)
    assert str(got.value) == str(want.value) and m.cap > 64
    assert m.oob.tolist()[0] == 0
    good = [_good(i) for i in range(20)]
    _same(s.predict(good), _training_path(m, good))
