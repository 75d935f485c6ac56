"""DIN serving on the GPU (csrc/tfrecord_device.cu ctr_din_serve_scan + ctr_tfrecord_emit_din, serving.DINServable;
DESIGN.md §2.10) against the training path (din_main.make_batch + DIN.predict), the CPU restatement
tests/din_serving_oracle.py and the fp64 oracle DIN."""
import json
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


def _model(B=16, P=8, A=4, attention_pooling=True, batch_norm=False, seed=0):
    from tf_repos_b200.din import DIN
    m = DIN(F, N, K, B, P, max_a_int=A, deep_layers=LAYERS, dropout="0.9,0.9", attention_pooling=attention_pooling,
            batch_norm=batch_norm, update_mode="lazy", seed=seed)
    g = torch.Generator().manual_seed(100 + seed)
    vals = {}
    for k, v in m.variables().items():
        if "moving_variance" in k:
            vals[k] = torch.rand(v.shape, generator=g, dtype=torch.float64).float() + 0.5
        else:
            vals[k] = (torch.rand(v.shape, generator=g, dtype=torch.float64) * 0.6 - 0.3).float()
    m.load_variables(vals)
    return m


def _servable(m):
    from tf_repos_b200.serving import DINServable
    return DINServable(m)


def _random_request(n, seed, maxlen=6, max_a=3):
    rng = np.random.RandomState(seed)
    out = []
    for i in range(n):
        lens = rng.randint(0, maxlen + 1, 4)
        u_ids = [rng.randint(0, N, l).tolist() for l in lens]
        u_vals = [(rng.randn(l) * 2).astype(np.float32).tolist() for l in lens]
        extra = []
        if rng.rand() < 0.3:
            extra.append(("y", so.float_feature([1.0])))
        if rng.rand() < 0.2:
            extra.append(("z", so.int64_feature([3])))
        if rng.rand() < 0.2:
            extra.append(("u_catids", so.int64_feature(u_ids[0], packed=False)))
        out.append(so.din_example(rng.randint(0, N, F).tolist(), rng.randint(0, N, 3).tolist(),
                                  rng.randint(0, N, rng.randint(0, max_a + 1)).tolist(), u_ids, u_vals,
                                  packed=bool(rng.rand() < 0.7), extra=extra))
    return out


def _training_path(m, examples, P=None):
    """DIN.predict(make_batch(decode(...))) over slices of m.B, as din_main scores a data set"""
    from tf_repos_b200 import din_main as dm
    d = so.decode(examples, F, N)
    out = []
    for lo in range(0, len(examples), m.B):
        idx = list(range(lo, min(lo + m.B, len(examples))))
        batch, _, n = dm.make_batch(d, idx, m.B, P or m.P, m.device)
        out.append(m.predict(batch)[:n].cpu().numpy().copy())
    return np.concatenate(out) if out else np.zeros(0, np.float32)


def _bits(a):
    return np.asarray(a, dtype=np.float32).view(np.uint32)


@pytest.mark.parametrize("attention_pooling,batch_norm", [(True, False), (False, False), (False, True)])
def test_predict_is_bit_identical_to_the_training_path(attention_pooling, batch_norm):
    m = _model(attention_pooling=attention_pooling, batch_norm=batch_norm)
    s = _servable(m)
    for seed, n in ((1, 7), (2, 16), (3, 41)):
        req = _random_request(n, seed)
        got = s.predict(req)
        assert got.dtype == np.float32 and got.shape == (n,)
        np.testing.assert_array_equal(_bits(got), _bits(_training_path(m, req)))


def _emit(m, examples):
    from tf_repos_b200 import ops
    dev, B, P, A = m.device, m.B, m.P, m.max_a_int
    lens = [len(e) for e in examples]
    off = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int64, device=dev)
    data = torch.tensor(np.frombuffer(b"".join(examples), np.uint8), device=dev)
    i32 = dict(dtype=torch.int32, device=dev)
    slot_off, slot_len = torch.empty(B, dtype=torch.int64, device=dev), torch.empty(B, **i32)
    maxima, err = torch.zeros(2, **i32), torch.full((1,), -1, dtype=torch.int64, device=dev)
    batch = {"feat_ids": torch.empty(B, F, **i32), "a_ids": torch.empty(3, B, **i32),
             "a_int_ids": torch.full((B * A,), -7, **i32), "a_int_off": torch.empty(B + 1, **i32),
             "u_ids": torch.full((4, B, P), -7, **i32), "u_wgt": torch.full((4, B, P), 7.0, device=dev)}
    ops.din_serve_scan(data, off, 0, F, B, A, slot_off, slot_len, batch["a_int_off"], maxima, err)
    ops.tfrecord_emit_din(data, slot_off, slot_len, B, F, P, batch["a_int_off"], batch["feat_ids"], batch["a_ids"],
                          batch["a_int_ids"], batch["u_ids"], batch["u_wgt"], torch.empty(B, device=dev))
    return batch, maxima.tolist(), int(err.item())


def test_emitted_batch_equals_make_batch_bit_for_bit():
    from tf_repos_b200 import din_main as dm
    m = _model(B=16, P=6, A=4)
    nan_bits = [0x7FC00001, 0xFFC12345, 0x7F800001, 0x00000001, 0x80000000, 0x7F800000]
    nans = [struct.unpack("<f", struct.pack("<I", b))[0] for b in nan_bits]
    req = _random_request(9, 7, maxlen=6, max_a=4)
    req[2] = so.din_example([(1 << 31) - 1, (1 << 30) + 3, 0, 1, 2], [(1 << 31) - 1, 0, 5], [(1 << 31) - 2] * 4,
                            ([1] * 6, [], [], [(1 << 31) - 1]), (nans, [], [], [-0.0]), packed=False)
    req[5] = so.din_example([1, 2, 3, 4, 5], [1, 1, 1])               # every list empty or missing
    batch, maxima, err = _emit(m, req)
    assert err == -1 and maxima == [6, 4]
    d = so.decode(req, F)
    want, _, _ = dm.make_batch(d, list(range(len(req))), m.B, m.P, "cpu")
    for k, v in want.items():
        got = batch[k].cpu()
        if k == "a_int_ids":
            got = got[:v.numel()]
        assert got.dtype == v.dtype and got.shape == v.shape, k
        assert torch.equal(got.view(torch.int32), v.view(torch.int32)), k
    assert batch["u_wgt"][0, 2].cpu().view(torch.int32).tolist() == \
        [0x7FC00001, 0xFFC12345 - (1 << 32), 0x7FC00001, 0x00000001, 0x80000000 - (1 << 32), 0x7F800000]


def test_predict_agrees_with_the_fp64_oracle():
    from oracle import models as om
    from tf_repos_b200 import din_main as dm
    m = _model(B=16, P=8)
    ref = om.DIN(F, N, K, deep_layers=LAYERS, dropout="0.9,0.9", attention_layers="256", seed=0,
                 dtype=torch.float64)
    for k, v in m.variables().items():
        ref.params[k] = v.detach().cpu().double().reshape(ref.params[k].shape).clone()
    req = _random_request(30, 11)
    got = _servable(m).predict(req)
    d = so.decode(req, F, N)
    want = []
    for lo in range(0, 30, 16):
        idx = list(range(lo, min(lo + 16, 30)))
        batch, _, n = dm.make_batch(d, idx, 16, 8, "cpu")
        lb = {k: (v.long() if v.dtype == torch.int32 else v.double()) for k, v in batch.items()}
        want.append(ref.predict(lb)["prob"][:n].numpy())
    np.testing.assert_allclose(got, np.concatenate(want), rtol=2e-5, atol=2e-6)


def test_longer_lists_than_the_buffers_are_answered_by_growing():
    m = _model(B=16, P=4, A=2)
    s = _servable(m)
    small = _random_request(20, 21, maxlen=4, max_a=2)
    before = s.predict(small)
    long = _random_request(35, 22, maxlen=4, max_a=2)
    long[30] = so.din_example([1, 2, 3, 4, 5], [1, 2, 3], list(range(1, 10)),
                              ([7] * 13, [], [8] * 5, []), ([0.5] * 13, [], [1.5] * 5, []))
    long[3] = so.din_example([1, 2, 3, 4, 5], [1, 2, 3], [], ([], [], [], [9] * 6), ([], [], [], [2.0] * 6))
    got = s.predict(long)
    assert (m.P, m.max_a_int) == (13, 9)
    np.testing.assert_array_equal(_bits(got), _bits(_training_path(m, long)))
    # din.cu's pooling adds position p into lane slot p % (32 / LPR) in position order and bag_sum_fwd adds in position
    # order: the zero-weight padding a larger P adds contributes exact zeros, so results do not depend on P
    np.testing.assert_array_equal(_bits(s.predict(small)), _bits(before))


def test_growth_without_attention_pooling_keeps_the_bits():
    m = _model(B=8, P=3, A=1, attention_pooling=False)
    s = _servable(m)
    req = _random_request(12, 31, maxlen=3, max_a=1)
    before = s.predict(req)
    s.predict([so.din_example([1, 2, 3, 4, 5], [1, 2, 3], [4] * 7, ([5] * 40, [], [], []), ([1.0] * 40, [], [], []))])
    assert (m.P, m.max_a_int) == (40, 7)
    np.testing.assert_array_equal(_bits(s.predict(req)), _bits(before))


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


def _long_request():
    req = _random_request(35, 22, maxlen=4, max_a=2)
    req[30] = so.din_example([1, 2, 3, 4, 5], [1, 2, 3], list(range(1, 10)),
                             ([7] * 13, [], [8] * 5, []), ([0.5] * 13, [], [1.5] * 5, []))
    return req


@pytest.mark.parametrize("where,after", [("din", 0), ("din", 5), ("serving", 0), ("serving", 4)])
def test_a_failed_growth_leaves_the_servable_as_it_was(monkeypatch, where, after):
    from tf_repos_b200 import din, serving
    m = _model(B=16, P=4, A=2)
    s = _servable(m)
    small = _random_request(20, 21, maxlen=4, max_a=2)
    before = s.predict(small)
    monkeypatch.setattr(din if where == "din" else serving, "torch", _FailingTorch(after))
    with pytest.raises(torch.cuda.OutOfMemoryError):
        s.predict(_long_request())
    monkeypatch.undo()
    assert (m.P, m.max_a_int) == (4, 2) and m.ids_all is not None
    assert s._batch["u_ids"].shape[2] == 4 and s._batch["a_int_ids"].numel() == 16 * 2
    np.testing.assert_array_equal(_bits(s.predict(small)), _bits(before))
    long = _long_request()
    got = s.predict(long)
    assert (m.P, m.max_a_int) == (13, 9)
    np.testing.assert_array_equal(_bits(got), _bits(_training_path(m, long)))


def test_a_grown_model_no_longer_trains():
    m = _model(B=8, P=4, A=2)
    m.grow(9, 3)
    assert (m.P, m.max_a_int) == (9, 3)
    with pytest.raises(RuntimeError, match="grew its buffers for inference"):
        m.train_step(None, None)


@pytest.mark.parametrize("later_malformed", [False, True])
@pytest.mark.parametrize("key", ["u_catids", "a_intids"])
def test_an_id_past_the_starting_buffers_that_reaches_feature_size_is_rejected(key, later_malformed):
    # without a later error the id is only read, and counted, when the slice is run again at the grown sizes
    m = _model(B=16, P=4, A=2)
    s = _servable(m)
    req = [_good(i) for i in range(24)]
    ids = list(range(1, 13)) + [N]
    if key == "u_catids":
        req[17] = so.din_example([1, 2, 3, 4, 5], [1, 2, 3], [], (ids, [], [], []), ([1.0] * 13, [], [], []))
    else:
        req[17] = so.din_example([1, 2, 3, 4, 5], [1, 2, 3], ids[-5:])
    if later_malformed:
        req[20] = BAD["malformed"]
    with pytest.raises(so.Rejected) as want:
        so.decode(req, F, N)
    assert (want.value.index, want.value.check) == (17, so.VOCAB)
    with pytest.raises(ValueError) as got:
        s.predict(req)
    assert str(got.value) == str(want.value)
    assert m.oob.tolist()[0] == 0
    good = [_good(i) for i in range(20)]
    np.testing.assert_array_equal(_bits(s.predict(good)), _bits(_training_path(m, good)))


def _good(i):
    return so.din_example([1 + i, 2, 3, 4, 5], [6, 7, 8], [9], ([10], [], [], []), ([0.5], [], [], []))


BAD = {
    "malformed": so.example([]) + b"\x0a\x81",
    "non-utf8 key": so.example([("feat_ids", so.int64_feature([1, 2, 3, 4, 5])), (b"\xc3\x28", b"")]),
    "required": so.example([("feat_ids", so.int64_feature([1, 2, 3, 4, 5]))]),
    "count": so.din_example([1, 2], [1, 2, 3]),
    "mismatch": so.din_example([1, 2, 3, 4, 5], [1, 2, 3], [], ([], [], [], [1, 2]), ([], [], [], [1.0])),
    "kind": so.din_example([1, 2, 3, 4, 5], [1, 2, 3], extra=[("u_shopvals", so.int64_feature([1]))]),
    "several kinds": so.din_example([1, 2, 3, 4, 5], [1, 2, 3],
                                    extra=[("a_intids", so.int64_feature([1]) + so.float_feature([1.0]))]),
    "range": so.din_example([1, 2, 3, 4, 5], [1, 2, 3], [1 << 35]),
    "feature_size": so.din_example([1, 2, 3, 4, 5], [1, 2, 3], [], ([], [], [N], []), ([], [], [1.0], [])),
    "feature_size a_catids": so.din_example([1, 2, 3, 4, 5], [N, 2, 3]),
}


@pytest.mark.parametrize("what", sorted(BAD))
@pytest.mark.parametrize("at", [0, 5, 37])
def test_errors_name_the_first_bad_example_and_the_servable_recovers(what, at):
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
    good = [_good(i) for i in range(20)]
    np.testing.assert_array_equal(_bits(s.predict(good)), _bits(_training_path(m, good)))
    assert m.oob.tolist()[0] == 0


def test_request_sizes():
    m = _model(B=16)
    s = _servable(m)
    assert s.predict([]).shape == (0,)
    for n in (1, 16, 17, 3 * 16 + 5):
        req = _random_request(n, 40 + n)
        np.testing.assert_array_equal(_bits(s.predict(req)), _bits(_training_path(m, req)))


def _write_din(path, n, seed, maxlen=6):
    from tf_repos_b200 import tfrecord as tfr
    rng = np.random.RandomState(seed)
    recs = []
    for _ in range(n):
        ex = {"y": np.float32(rng.rand() < 0.3), "z": np.float32(0.0), "feat_ids": rng.randint(1, 5000, 11).astype(np.int64),
              "a_catids": np.int64(rng.randint(1, 5000)), "a_shopids": np.int64(rng.randint(1, 5000)),
              "a_brandids": np.int64(rng.randint(1, 5000)),
              "a_intids": rng.randint(1, 5000, rng.randint(0, 4)).astype(np.int64)}
        for f in so.U:
            ln = rng.randint(0, maxlen + 1)
            ex["u_%sids" % f] = rng.randint(1, 5000, ln).astype(np.int64)
            ex["u_%svals" % f] = (rng.rand(ln) * 3).astype(np.float32)
        recs.append(tfr.encode_example(ex))
    tfr.write_records(path, recs)
    return recs


def test_export_answers_the_serving_request_with_pred_txt(tmp_path):
    from tf_repos_b200 import din_main as dm
    from tf_repos_b200.din import DIN
    from tf_repos_b200.estimator import restore_checkpoint
    from tf_repos_b200.serving import DINServable, Servable
    tmp = str(tmp_path)
    os.makedirs(tmp + "/data/tr"); os.makedirs(tmp + "/data/te"); os.makedirs(tmp + "/ckpt")
    _write_din(tmp + "/data/tr/part0.tfrecord", 150, 1)
    te = _write_din(tmp + "/data/te/part0.tfrecord", 70, 3)
    common = [sys.executable, os.path.join(ROOT, "Model_pipeline", "DIN.py"), "--field_size=11", "--feature_size=5000",
              "--embedding_size=8", "--batch_size=64", "--deep_layers=16,8", "--dropout=0.9,0.9", "--log_steps=100",
              "--num_epochs=1", "--data_dir=" + tmp + "/data", "--model_dir=" + tmp + "/ckpt/m_", "--dt_dir=20260922"]
    for task in ("train", "infer", "export"):
        r = subprocess.run(common + ["--task_type=" + task, "--servable_model_dir=" + tmp + "/export"],
                           capture_output=True, text=True, timeout=280)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    sub = os.listdir(tmp + "/export")
    s = Servable.load(os.path.join(tmp, "export", sub[0]), max_batch=64)
    assert isinstance(s, DINServable)
    got = s.predict(te)
    want = np.array([float(x) for x in open(tmp + "/data/pred.txt").read().split()], dtype=np.float32)
    assert np.array_equal(np.array(["%f" % p for p in got]), np.array(["%f" % p for p in want]))
    # and DIN.predict at the training P, bit for bit
    meta = json.load(open(tmp + "/ckpt/m_20260922/din_shapes.json"))
    m = DIN(11, 5000, 8, 64, meta["P"], max_a_int=meta["max_a_int"], deep_layers="16,8", dropout="0.9,0.9",
            update_mode="lazy")
    restore_checkpoint(m, tmp + "/ckpt/m_20260922")
    d = dm.decode_tfrecord_files([tmp + "/data/te/part0.tfrecord"], 11)
    ref = []
    for idx in dm.index_stream(70, 1, 64):
        batch, _, n = dm.make_batch(d, idx, 64, meta["P"], m.device)
        ref.append(m.predict(batch)[:n].cpu().numpy().copy())
    np.testing.assert_array_equal(_bits(got), _bits(np.concatenate(ref)))
