"""DeepMVM on the CPU: the oracle restatement (tests/deepmvm_oracle.py) against per-sample, per-element Python loops read
from DeepMVM.py:139-199, closed forms of the multi-view product, the hand-derived prefix-product backward that
csrc/mvm.cu implements against fp64 autograd, argument validation of the ctr_mvm_* entries (no GPU touched) and the
flag surface of Model_pipeline/DeepMVM.py."""
import importlib.util
import math
import os

import pytest
import torch

from tests.deepmvm_oracle import DeepMVM

F64 = torch.float64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _fc(x, W, b):
    out = []
    for j in range(len(b)):
        s = b[j]
        for i in range(len(x)):
            s += x[i] * W[i][j]
        out.append(s)
    return out


def _ce(y, z):            # tf.nn.sigmoid_cross_entropy_with_logits
    return max(y, 0.0) - y * z + math.log1p(math.exp(-abs(y)))


def _l2(t):               # tf.nn.l2_loss = sum(t^2)/2
    flat = torch.tensor(t, dtype=F64).reshape(-1).tolist()
    return sum(v * v for v in flat) / 2


def _batch(B, F, N, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, N, (B, F), generator=g)
    vals = torch.rand(B, F, generator=g, dtype=F64) + 0.2
    labels = (torch.rand(B, generator=g) < 0.4).to(F64)
    return ids, vals, labels


def test_forward_and_loss_match_per_element_loops():
    B, F, N, K = 3, 5, 17, 4
    m = DeepMVM(F, N, K, deep_layers="6,3", dropout="1.0,1.0", l2_reg=0.01, dtype=F64, seed=1)
    g = torch.Generator().manual_seed(11)
    for n, p in m.params.items():            # random values everywhere (the initialisers leave the biases at 0)
        p.copy_(torch.randn(p.shape, generator=g, dtype=F64) * 0.7)
    p = {n: t.tolist() for n, t in m.params.items()}
    ids, vals, labels = _batch(B, F, N, 3)
    ys = []
    for b in range(B):
        e = [[p["mvm_w"][ids[b, f]][k] * float(vals[b, f]) for k in range(K)] for f in range(F)]   # :140-142
        x_mvm = []
        for k in range(K):                                                                        # :145-148
            prod = e[0][k] + p["mvm_b"][0][k]
            for f in range(1, F):
                prod = prod * (e[f][k] + p["mvm_b"][f][k])
            x_mvm.append(prod)
        h = [v for row in e for v in row]                                                        # :166, without mvm_b
        for i in range(2):
            h = [max(s, 0.0) for s in _fc(h, p[f"Deep-part/mlp{i}/weights"], p[f"Deep-part/mlp{i}/biases"])]
        ys.append(_fc(x_mvm + h, p["DeepMVM-out/deep_out/weights"], p["DeepMVM-out/deep_out/biases"])[0])  # x_mvm first
    batch = {"feat_ids": ids, "feat_vals": vals}
    y = m.predict(batch)["y"].tolist()
    for a, r in zip(y, ys):
        assert abs(a - r) <= 1e-12 * max(1.0, abs(r)), (a, r)
    loss = sum(_ce(v, z) for v, z in zip(ys, labels.tolist())) / B + 0.01 * _l2(p["mvm_w"]) + 0.01 * _l2(p["mvm_b"])
    got = m.evaluate(batch, labels)["loss"]
    assert abs(got - loss) <= 1e-12 * max(1.0, abs(loss)), (got, loss)
    assert m.l2_vars == ("mvm_w", "mvm_b")           # the table term comes first (DeepMVM.py:197-199)


def test_single_field_is_the_biased_embedding():
    m = DeepMVM(1, 13, 4, deep_layers="3", dropout="1.0", dtype=F64, seed=2)
    ids, vals, _ = _batch(6, 1, 13, 4)
    out = m.predict({"feat_ids": ids, "feat_vals": vals})
    want = m.params["mvm_w"][ids[:, 0]] * vals[:, :1] + m.params["mvm_b"][0]
    assert torch.equal(out["x_mvm"], want)


def test_zero_values_give_the_product_of_the_biases():
    F, K = 7, 5
    m = DeepMVM(F, 50, K, deep_layers="4", dropout="1.0", seed=3)
    ids, vals, _ = _batch(4, F, 50, 5)
    out = m.predict({"feat_ids": ids, "feat_vals": torch.zeros_like(vals)})
    prod = m.params["mvm_b"][0].clone()
    for f in range(1, F):
        prod = prod * m.params["mvm_b"][f]
    assert torch.equal(out["x_mvm"], prod.expand(4, K))


def test_unit_biases_and_zero_table_give_one():
    F, K = 39, 8
    m = DeepMVM(F, 100, K, deep_layers="4", dropout="1.0", seed=4)
    m.params["mvm_b"].fill_(1.0)
    m.params["mvm_w"].zero_()
    ids, vals, _ = _batch(5, F, 100, 6)
    assert torch.equal(m.predict({"feat_ids": ids, "feat_vals": vals.float()})["x_mvm"], torch.ones(5, K))


def test_one_zero_factor_zeroes_the_product_and_all_other_field_gradients():
    F, K, B, f0 = 6, 4, 8, 2
    m = DeepMVM(F, F, K, deep_layers="5", dropout="1.0", l2_reg=0.0, dtype=F64, seed=5)
    g = torch.Generator().manual_seed(7)
    m.params["mvm_b"].copy_(torch.rand(F, K, generator=g, dtype=F64) + 0.5)
    m.params["mvm_w"].copy_(torch.randn(F, K, generator=g, dtype=F64) * 0.1)
    m.params["mvm_w"][f0] = -m.params["mvm_b"][f0]          # e = -b on field f0 (val 1): a[:, f0, :] == 0 exactly
    ids = torch.arange(F).repeat(B, 1)
    vals = torch.ones(B, F, dtype=F64)
    vals[:, [0, 1, 3, 4, 5]] = torch.rand(B, 5, generator=g, dtype=F64) + 0.5
    batch = {"feat_ids": ids, "feat_vals": vals}
    labels = (torch.arange(B) % 2).to(F64)
    assert torch.all(m.predict(batch)["x_mvm"] == 0)
    _, _, _, dense = m.gradients(batch, labels)
    d_b = dense["mvm_b"]                                     # = sum_b da[b]: mvm_b reaches the loss only through x_mvm
    assert torch.all(d_b[f0] != 0)
    assert torch.all(torch.cat([d_b[:f0], d_b[f0 + 1:]]) == 0)


def _prefix_bwd(a, g):
    """The backward csrc/mvm.cu runs: prefix products P_i as the forward rounds them, then
    da_i = g*P_{i-1}; g = g*a_i for i = F-1..1; da_0 = g.  a: [B,F,K], g: [B,K]."""
    F = a.shape[1]
    P = [a[:, 0]]
    for i in range(1, F - 1):
        P.append(P[-1] * a[:, i])
    da = torch.empty_like(a)
    for i in range(F - 1, 0, -1):
        da[:, i] = g * P[i - 1]
        g = g * a[:, i]
    da[:, 0] = g
    return da


@pytest.mark.parametrize("F", [1, 2, 5, 39])
def test_prefix_backward_matches_autograd_with_zero_factors(F):
    B, K = 9, 6
    gen = torch.Generator().manual_seed(F)
    a = (torch.rand(B, F, K, generator=gen, dtype=F64) + 0.5) * torch.where(torch.rand(B, F, K, generator=gen) < 0.5, -1.0, 1.0)
    a[torch.rand(B, F, K, generator=gen) < 0.08] = 0.0     # exact zeros, one or several per column
    a[0, :, 0] = 0.0
    a.requires_grad_()
    g = torch.randn(B, K, generator=gen, dtype=F64)
    p = a[:, 0]
    for i in range(1, F):
        p = p * a[:, i]
    p.backward(g)
    assert torch.equal(_prefix_bwd(a.detach(), g), a.grad)


def test_argument_validation_needs_no_gpu():
    from tf_repos_b200 import _lib
    L = _lib.raw()
    n0 = L.ctr_launch_count()
    fake = 256                                               # never dereferenced: every call below fails validation
    assert L.ctr_mvm_fwd(None, None, 4, 39, 16, None, None) == -1 and "null" in _lib.last_error()
    assert L.ctr_mvm_fwd(fake, fake, 4, 0, 16, fake, None) == -1
    assert L.ctr_mvm_fwd(fake, fake, -1, 39, 16, fake, None) == -1
    assert L.ctr_mvm_fwd(fake, fake, 4, 65, 16, fake, None) == -2 and "F <= 64" in _lib.last_error()
    assert L.ctr_mvm_fwd(fake, fake, 4, 39, 257, fake, None) == -2 and "K <= 256" in _lib.last_error()
    assert L.ctr_mvm_bwd(fake, fake, fake, None, 4, 39, 16, None, fake, fake, 1 << 30, None) == -1
    assert L.ctr_mvm_bwd(fake, fake, fake, None, 4, 39, 16, fake, None, fake, 1 << 30, None) == -1
    assert L.ctr_mvm_bwd(fake, fake, fake, None, 4, 100, 16, fake, fake, fake, 1 << 30, None) == -2
    assert L.ctr_mvm_bwd(fake, fake, fake, None, 4, 39, 16, fake, fake, fake, 0, None) == -4
    assert "workspace" in _lib.last_error()
    assert L.ctr_mvm_bwd_workspace_bytes(8192, 39, 16) >= 39 * 16 * 4
    assert L.ctr_launch_count() == n0


def test_script_takes_the_reference_flags():
    from tf_repos_b200 import flags
    importlib.reload(flags)
    spec = importlib.util.spec_from_file_location("deepmvm_script", os.path.join(ROOT, "Model_pipeline", "DeepMVM.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)                             # defines the flags; main() is not run
    F = mod.FLAGS
    # defaults of DeepMVM.py:35-60
    assert (F.dist_mode, F.num_threads, F.feature_size, F.field_size, F.embedding_size, F.num_epochs, F.batch_size,
            F.log_steps, F.learning_rate, F.l2_reg, F.loss_type, F.optimizer, F.deep_layers, F.dropout, F.batch_norm,
            F.batch_norm_decay, F.task_type, F.clear_existing_model) == \
           (0, 16, 0, 0, 32, 10, 64, 1000, 0.0005, 0.0001, "log_loss", "Adam", "256,128,64", "0.5,0.5,0.5", False, 0.9,
            "train", False)
    rest = F._parse("--task_type=train --learning_rate=0.0005 --optimizer=Adam --num_epochs=1 --batch_size=256 "
                    "--field_size=39 --feature_size=117581 --embedding_size=16 --deep_layers=400,400,400 "
                    "--dropout=0.5,0.5,0.5 --loss_type=log_loss --batch_norm=True --batch_norm_decay=0.99 "
                    "--log_steps=1000 --num_threads=8 --model_dir=./model_ckpt/criteo/DeepMVM/ "
                    "--data_dir=./data/criteo/".split())
    assert rest == [] and F.feature_size == 117581 and F.embedding_size == 16 and F.batch_norm and F.batch_norm_decay == 0.99
    with pytest.raises(SystemExit):
        F._parse(["--cross_layers=3"])                       # DeepMVM has no model-specific flag
    importlib.reload(flags)
