"""DeepMVM (DeepMVM.py:100-230) on the GPU: the multi-view product kernels bit for bit against fp32 CPU restatements,
N-step training parity against the oracle, exact-deferred / CUDA-graph bit identity, and the drop-in script end to
end (train -> eval -> resume -> infer -> export -> serving) with TF-named state."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.deepmvm_oracle import DeepMVM as OracleDeepMVM

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _close(got, ref, rtol, what=""):
    got = got.detach().cpu().double().numpy(); ref = ref.detach().cpu().double().numpy()
    s = max(float(np.abs(ref).max()), 1e-30)
    np.testing.assert_allclose(got, ref, rtol=rtol, atol=rtol * s, err_msg=what)


def _same(a, b):
    """bitwise-equal values, NaN where the other has NaN (CPU and GPU NaNs differ in sign/payload bits only)"""
    a, b = a.cpu(), b.cpu()
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a.masked_fill(na, 0), b.masked_fill(nb, 0))


def _inputs(B, F, K, regime, seed):
    g = torch.Generator().manual_seed(seed)
    sign = torch.where(torch.rand(F, K, generator=g) < 0.5, -1.0, 1.0)
    if regime == "o1":            # factors ~ +-[0.9, 1.1], plus exact zeros (e = -b)
        mb = sign * (0.9 + 0.2 * torch.rand(F, K, generator=g))
        x = torch.randn(B, F, K, generator=g) * 0.01
        z = torch.rand(B, F, K, generator=g) < 0.003
        z[0, 0, 0] = z[1, F - 1, K - 1] = z[2, F // 2, K // 2] = True
        x[z] = -mb.expand(B, F, K)[z]
    elif regime == "glorot":      # the reference's initialisation: most products are denormal or zero
        mb = (torch.randn(F, K, generator=g).clamp(-2, 2) * (2.0 / (F + K)) ** 0.5)
        x = torch.randn(B, F, K, generator=g) * 1e-4
    else:                         # |b| = 10^U(-6,6): partial products overflow and underflow
        mb = sign * 10.0 ** (12 * torch.rand(F, K, generator=g) - 6)
        x = torch.randn(B, F, K, generator=g) * 1e-3
    return x.reshape(B, F * K).contiguous(), mb.contiguous(), torch.randn(B, K, generator=g), torch.randn(B, F * K, generator=g)


@pytest.mark.parametrize("regime", ["o1", "glorot", "extreme"])
@pytest.mark.parametrize("K", [4, 8, 16, 32, 64, 256])
@pytest.mark.parametrize("F", [1, 2, 39, 64])
def test_mvm_kernels_bit_exact(F, K, regime):
    from tf_repos_b200 import ops
    d = torch.device("cuda:0")
    B = 257
    x, mb, gx, dX = _inputs(B, F, K, regime, seed=F * 1000 + K + len(regime))
    # fp32 CPU restatement of DeepMVM.py:145-148 and torch autograd of it
    xl = x.clone().requires_grad_()
    a = xl.view(B, F, K) + mb
    p = a[:, 0]
    for i in range(1, F):
        p = p * a[:, i]
    (da,) = torch.autograd.grad(p, xl, gx)
    x_mvm = torch.empty(B, K, device=d)
    ops.mvm_fwd(x.to(d), mb.to(d), x_mvm)
    assert _same(x_mvm, p.detach()), "x_mvm"
    if regime == "o1":
        assert p.abs().median() > 1e-3 and torch.all(torch.isfinite(p))      # the product is not trivially small
        assert torch.any(p == 0)                                              # ... and has exact zero factors
    d_e = torch.empty(B, F * K, device=d)
    d_b = torch.empty(F, K, device=d)
    ws = torch.empty(ops.mvm_bwd_workspace_bytes(B, F, K), dtype=torch.uint8, device=d)
    ops.mvm_bwd(x.to(d), mb.to(d), gx.to(d), dX.to(d), d_e, d_b, ws)
    assert _same(d_e, da + dX), "d_e"
    # d mvm_b: an fp32 batch reduction in a fixed order, against the fp64 sum of the same da
    da3 = da.view(B, F, K).double()
    ref, scale = da3.sum(0), da3.abs().sum(0)
    got = d_b.cpu().double()
    fin = torch.isfinite(ref) & (scale < 3e38)
    assert torch.all(torch.isfinite(got[fin]))
    assert torch.all((got - ref).abs()[fin] <= 1e-5 * scale[fin]), "d mvm_b"
    inf = ~torch.isfinite(ref)
    assert not torch.any(torch.isfinite(got[inf])), "d mvm_b non-finite entries"
    # inf / nan propagate like the fp64 sum unless the finite terms themselves can overflow an fp32 partial sum
    scale_fin = torch.where(torch.isfinite(da3), da3, 0.0).abs().sum(0)
    strict = inf & (scale_fin < 3e38)
    assert _same(got[strict], ref[strict]), "d mvm_b non-finite entries"
    d_e2 = torch.empty_like(d_e); d_b2 = torch.empty_like(d_b)
    ops.mvm_bwd(x.to(d), mb.to(d), gx.to(d), None, d_e2, d_b2, ws)
    assert _same(d_b2, d_b), "deterministic d mvm_b"
    assert _same(d_e2, da), "d_e without dX"


def test_mvm_empty_batch_zeroes_the_bias_gradient():
    from tf_repos_b200 import ops
    d = torch.device("cuda:0")
    d_b = torch.full((39, 16), 7.0, device=d)
    ws = torch.empty(16, dtype=torch.uint8, device=d)
    e = torch.empty(0, 39 * 16, device=d)
    ops.mvm_bwd(e, torch.ones(39, 16, device=d), torch.empty(0, 16, device=d), None, e, d_b, ws)
    assert torch.all(d_b == 0)


def _o1_init(ref, N, K, F, seed):
    g = torch.Generator().manual_seed(seed)
    sign = torch.where(torch.rand(F, K, generator=g) < 0.5, -1.0, 1.0)
    ref.params["mvm_b"].copy_(sign * (0.9 + 0.2 * torch.rand(F, K, generator=g)))
    ref.params["mvm_w"].copy_(torch.randn(N, K, generator=g) * 0.02)


@pytest.mark.parametrize("opt,mode", [("Adam", "exact"), ("Adam", "exact_deferred"), ("Adam", "lazy"), ("Adagrad", "exact")])
def test_deepmvm_train_steps_match_oracle(opt, mode):
    from oracle import tf_semantics as tfs
    from tf_repos_b200 import synth
    from tf_repos_b200.deepmvm import DeepMVM
    B, N, K, F = 256, 10_000, 8, 39
    lr = 5e-4 if opt == "Adam" else 0.01
    kw = dict(deep_layers="64,32", dropout="1.0,1.0", l2_reg=1e-4, learning_rate=lr, optimizer=opt)
    ref = OracleDeepMVM(F, N, K, update_mode=("lazy" if mode == "lazy" else "exact"), seed=5, **kw)
    _o1_init(ref, N, K, F, 9)
    gpu = DeepMVM(F, N, K, B, update_mode=mode, epoch_steps=3, device="cuda:0", **kw)
    gpu.load_variables(ref.params)
    for step in range(4):
        ids, vals, labels = synth.criteo_batch(B, N, F, seed=200 + step)
        batch = {"feat_ids": ids.long(), "feat_vals": vals}
        gpu.predict(ids.cuda(), vals.cuda())
        out = ref.predict(batch)
        assert out["x_mvm"].abs().median() > 1e-3                         # the product term is not negligible
        _close(gpu.y[:B], out["y"], 1e-5, f"logits step {step}")
        reg_w = 1e-4 * float(tfs.l2_loss(ref.params["mvm_w"].double()))
        reg_b = 1e-4 * float(tfs.l2_loss(ref.params["mvm_b"].double()))
        loss_ref = ref.train_step(batch, labels)
        parts = gpu.train_step(ids.cuda(), vals.cuda(), labels.cuda())
        gpu.check_ids()
        if mode == "exact":
            assert abs(gpu.loss_value(parts) - loss_ref) <= 1e-5 * abs(loss_ref)
            ce, t_w, t_b = parts.tolist()                                 # CE, l2*l2_loss(mvm_w), l2*l2_loss(mvm_b)
            assert abs(t_w - reg_w) <= 1e-5 * reg_w and abs(t_b - reg_b) <= 1e-5 * reg_b
        vs = gpu.variables()
        for name in ("mvm_w", "mvm_b", "Deep-part/mlp0/weights", "DeepMVM-out/deep_out/weights"):
            _close(vs[name], ref.params[name], 2e-5, f"{name} after step {step} ({opt},{mode})")


def test_deepmvm_batch_norm_matches_oracle():
    """batch_norm after each relu (DeepMVM.py:174-175).  The batch moments are fp32 reductions in another order than the
    oracle's, and Adam's m/sqrt(v) turns the last-bit differences of a near-zero table gradient into a visible step, so
    the table is held to 1e-4 here; every dense variable, the moving statistics and the logits keep 2e-5 / 1e-5."""
    from tf_repos_b200 import synth
    from tf_repos_b200.deepmvm import DeepMVM
    B, N, K, F = 256, 10_000, 8, 39
    kw = dict(deep_layers="64,32", dropout="1.0,1.0", l2_reg=1e-4, learning_rate=5e-4, optimizer="Adam", batch_norm=True)
    ref = OracleDeepMVM(F, N, K, update_mode="exact", seed=5, **kw)
    _o1_init(ref, N, K, F, 9)
    gpu = DeepMVM(F, N, K, B, update_mode="exact", device="cuda:0", **kw)
    gpu.load_variables(ref.params)
    for step in range(4):
        ids, vals, labels = synth.criteo_batch(B, N, F, seed=300 + step)
        gpu.predict(ids.cuda(), vals.cuda())
        _close(gpu.y[:B], ref.predict({"feat_ids": ids.long(), "feat_vals": vals})["y"], 1e-5, f"logits step {step}")
        loss_ref = ref.train_step({"feat_ids": ids.long(), "feat_vals": vals}, labels)
        parts = gpu.train_step(ids.cuda(), vals.cuda(), labels.cuda())
        assert abs(gpu.loss_value(parts) - loss_ref) <= 1e-5 * abs(loss_ref)
    vs = gpu.variables()
    _close(vs["mvm_w"], ref.params["mvm_w"], 1e-4, "mvm_w")
    for name in ("mvm_b", "Deep-part/mlp0/weights", "Deep-part/bn_0/gamma", "DeepMVM-out/deep_out/weights"):
        _close(vs[name], ref.params[name], 2e-5, name)
    for name, v in ref.bn_state.items():
        _close(vs[name], v, 2e-5, name)


def test_deferred_and_graphed_steps_are_bit_identical():
    from tf_repos_b200 import synth
    from tf_repos_b200.deepmvm import DeepMVM
    B, N, K, F = 512, 20_000, 16, 39
    mk = lambda mode: DeepMVM(F, N, K, B, deep_layers="64,32", update_mode=mode, epoch_steps=3, device="cuda:0", seed=3)
    a, b, c = mk("exact"), mk("exact_deferred"), mk("exact_deferred")
    for m in (b, c):
        m.V.var.copy_(a.V.var); m.dense.flat.copy_(a.dense.flat)
    batches = [synth.criteo_batch(B, N, F, seed=30 + i, device="cuda:0") for i in range(11)]
    for bt in batches:
        a.train_step(*bt); b.train_step(*bt); c.train_step_graphed(*bt)
    assert c.replayed_launches > 0
    b.flush(); c.flush()
    assert torch.equal(a.V.var, b.V.var) and all(torch.equal(x, y) for x, y in zip(a.V.slots, b.V.slots))
    assert torch.equal(a.dense["mvm_b"], b.dense["mvm_b"])
    assert all(torch.equal(x, y) for x, y in zip(a.dense.slots, b.dense.slots))
    vb, vc = b.variables(), c.variables()
    for name in vb:
        assert torch.equal(vb[name], vc[name]), name


def test_model_fn_builds_deepmvm():
    from tf_repos_b200 import synth
    from tf_repos_b200.model_fn import ModeKeys, model_fn
    params = {"model": "DeepMVM", "field_size": 39, "feature_size": 5000, "embedding_size": 8, "deep_layers": "16,8",
              "batch_size": 64, "update_mode": "exact"}
    ids, vals, labels = synth.criteo_batch(64, 5000, 39, seed=1)
    parts = model_fn({"feat_ids": ids, "feat_vals": vals}, labels, ModeKeys.TRAIN, params).train_op()
    assert parts.shape == (3,) and params["_model"].global_step == 1
    prob = model_fn({"feat_ids": ids, "feat_vals": vals}, None, ModeKeys.PREDICT, params).predictions["prob"]
    assert prob.shape == (64,) and torch.all((prob > 0) & (prob < 1))


def _write(tmp, name, rows, seed, N=10_000):
    from tf_repos_b200 import synth
    ids, vals, labels = synth.criteo_batch(rows, N, 39, seed=seed)
    synth.write_libsvm(os.path.join(tmp, name), ids, vals, labels)


def test_cli_train_eval_infer_export(tmp_path):
    tmp = str(tmp_path)
    os.makedirs(tmp + "/data"); os.makedirs(tmp + "/ckpt")
    for name, rows, seed in (("tr0.libsvm", 600, 1), ("tr1.libsvm", 400, 2), ("va.libsvm", 200, 3), ("te.libsvm", 150, 4)):
        _write(tmp + "/data", name, rows, seed)
    common = [sys.executable, os.path.join(ROOT, "Model_pipeline", "DeepMVM.py"), "--field_size=39", "--feature_size=10000",
              "--embedding_size=8", "--batch_size=128", "--deep_layers=32,16", "--dropout=0.8,0.8", "--log_steps=5",
              "--num_epochs=1", "--data_dir=" + tmp + "/data", "--model_dir=" + tmp + "/ckpt/m_", "--dt_dir=20260922"]

    def run(*args):
        r = subprocess.run(common + list(args), capture_output=True, text=True, timeout=280)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        return r.stdout
    out = run("--task_type=train")
    assert "global_step/sec" in out and "Loss for final step" in out
    assert os.path.exists(tmp + "/ckpt/m_20260922/ctr_b200.ckpt")
    ev = json.loads(run("--task_type=eval").strip().splitlines()[-1])
    assert 0.0 <= ev["auc"] <= 1.0 and ev["global_step"] == 8
    out2 = run("--task_type=train")
    assert "restored checkpoint" in out2
    assert json.loads(run("--task_type=eval").strip().splitlines()[-1])["global_step"] == 16
    run("--task_type=infer")
    lines = open(tmp + "/data/pred.txt").read().split("\n")
    assert len(lines) == 151 and lines[-1] == "" and all(len(l.split(".")[1]) == 6 and 0 <= float(l) <= 1 for l in lines[:-1])
    run("--task_type=export", "--servable_model_dir=" + tmp + "/export")
    sub = os.listdir(tmp + "/export")
    sig = json.load(open(os.path.join(tmp, "export", sub[0], "signature.json")))
    assert sig["model"] == "DeepMVM" and sig["inputs"]["feat_ids"] == {"dtype": "int64", "shape": [None, 39]}
    from tf_repos_b200.input_fn import decode_libsvm_file
    from tf_repos_b200.serving import Servable
    ids, vals, _ = decode_libsvm_file(tmp + "/data/te.libsvm", 39)
    s = Servable.load(os.path.join(tmp, "export", sub[0]), max_batch=64)
    prob = s.predict(ids.astype(np.int64), vals)
    want = np.array([float(l) for l in lines[:-1]], dtype=np.float32)
    np.testing.assert_allclose(prob.numpy(), want, atol=1e-6)


def test_tf_named_training_state_roundtrip(tmp_path):
    from tf_repos_b200 import synth, tf_names
    from tf_repos_b200.deepmvm import DeepMVM
    F, N, K, B = 39, 5000, 8, 64
    mk = lambda: DeepMVM(F, N, K, B, deep_layers="16,8", dropout="1.0,1.0", update_mode="exact_deferred", epoch_steps=4,
                         device="cuda:0", seed=5)
    a = mk()
    batches = [synth.criteo_batch(B, N, F, seed=40 + i, device="cuda:0") for i in range(6)]
    for bt in batches[:3]:
        a.train_step(*bt)
    sd = tf_names.state_dict_tf(a)
    assert sd["mvm_w"].shape == (N, K) and sd["mvm_w/Adam"].shape == (N, K) and sd["mvm_w/Adam_1"].shape == (N, K)
    assert sd["mvm_b"].shape == (F, K) and sd["mvm_b/Adam"].shape == (F, K) and sd["mvm_b/Adam_1"].shape == (F, K)
    assert sd["Deep-part/mlp0/weights/Adam"].shape == (F * K, 16)
    assert sd["DeepMVM-out/deep_out/weights"].shape == (K + 8, 1) and "DeepMVM-out/deep_out/biases/Adam_1" in sd
    assert int(sd["global_step"]) == 3 and "beta1_power" in sd
    path = os.path.join(str(tmp_path), "state.npz")
    tf_names.export_npz(a, path)
    b2 = mk()
    tf_names.import_npz(b2, path)
    for bt in batches[3:]:
        a.train_step(*bt); b2.train_step(*bt)
    va, vb = a.variables(), b2.variables()
    for name in va:
        assert torch.equal(va[name], vb[name]), name
