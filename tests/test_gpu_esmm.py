"""ESMM (DeepCvrMTL.py:107-259) on the GPU: the embedding kernels bit for bit against the oracle's sequential fp32
restatement, the multi-task head against its fp32 restatement, CUDA-graph replay, and N-step training parity."""
import numpy as np
import pytest
import torch

from tests import esmm_oracle as eo

pytestmark = pytest.mark.gpu
KS = [4, 8, 16, 32, 64, 128, 256]


def _close(got, ref, rtol, what=""):
    got = got.detach().cpu().double().numpy(); ref = ref.detach().cpu().double().numpy()
    s = max(float(np.abs(ref).max()), 1e-30)
    np.testing.assert_allclose(got, ref, rtol=rtol, atol=rtol * s, err_msg=what)


def _cuda(batch):
    return {k: v.cuda() for k, v in batch.items()}


def _long(batch):
    return {k: (v.long() if k.endswith("ids") else v) for k, v in batch.items()}


def _edge_batch(B, Fp, N, seed):
    """bags of length 0 (first, middle and last sample), 1 and >= 500, duplicates, zero / negative weights, id 0"""
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(0, 7, (5, B), generator=g)
    lens[:, 0] = 0; lens[1, B // 2] = 0; lens[:, B - 1] = 0
    lens[0, 1] = 1; lens[1, 2] = 517; lens[4, 3] = 1
    off = torch.zeros(5 * B + 1, dtype=torch.int32)
    off[1:] = torch.cumsum(lens.reshape(-1), 0).to(torch.int32)
    nnz = int(off[-1])
    ids = torch.randint(0, N, (nnz,), generator=g, dtype=torch.int32)
    ids[::7] = 0
    ids[1::11] = 5                                        # duplicates inside bags
    wgt = torch.rand(nnz, generator=g) * 4 - 1            # negative weights
    wgt[::5] = 0.0
    feat = torch.randint(0, N, (B, Fp), generator=g, dtype=torch.int32)
    feat[0, 0] = 0
    a_ids = torch.randint(0, N, (3, B), generator=g, dtype=torch.int32)
    return {"feat_ids": feat, "a_ids": a_ids, "bag_ids": ids, "bag_wgt": wgt, "bag_off": off}


def _ref_embed(V, batch, dx, cap):
    """x and the per-occurrence gradient rows (model order, zero rows up to the capacity) from the oracle restatement"""
    B, Fp = batch["feat_ids"].shape
    K = V.shape[1]
    rows = {"common": V[batch["feat_ids"].long()], "a": V[batch["a_ids"].long()], "occ": V[batch["bag_ids"].long()]}
    rows = {k: v.detach().requires_grad_() for k, v in rows.items()}
    bags = eo.bag_sums(rows["occ"], batch["bag_wgt"], batch["bag_off"], 4 * B).reshape(5, B, K)
    a = rows["a"]
    x = torch.cat([rows["common"].reshape(B, Fp * K), bags[0], bags[1], bags[2], bags[3], a[0], a[1], a[2], bags[4]], 1)
    x.backward(dx)
    nnz = batch["bag_ids"].numel()
    g = torch.cat([rows["common"].grad.reshape(-1, K), rows["a"].grad.reshape(-1, K), rows["occ"].grad.reshape(-1, K),
                   torch.zeros(cap - nnz, K)])
    return x.detach(), g


@pytest.mark.parametrize("K", KS)
def test_embed_kernels_bit_exact(K):
    from tf_repos_b200 import ops
    B, Fp, N = 41, 3, 2000
    batch = _edge_batch(B, Fp, N, seed=K)
    g = torch.Generator().manual_seed(K + 1)
    V = torch.randn(N, K, generator=g)
    dx = torch.randn(B, (Fp + 8) * K, generator=g)
    cap = batch["bag_ids"].numel() + 13
    x_ref, g_ref = _ref_embed(V, batch, dx, cap)
    d = torch.device("cuda:0")
    x = torch.full((B, (Fp + 8) * K), float("nan"), device=d)
    oob = torch.zeros(2, dtype=torch.int32, device=d)
    bd = _cuda(batch)
    ops.esmm_embed_fwd(bd["feat_ids"], bd["a_ids"], bd["bag_ids"], bd["bag_wgt"], bd["bag_off"], V.to(d), x, oob)
    assert oob.tolist() == [0, 0]
    assert torch.equal(x.cpu(), x_ref)
    g_rows = torch.full((B * (Fp + 3) + cap, K), float("nan"), device=d)
    ops.esmm_embed_bwd(dx.to(d), bd["bag_wgt"], bd["bag_off"], B, Fp, K, g_rows)
    assert torch.equal(g_rows.cpu(), g_ref)


def test_embed_rejects_other_k_and_counts_out_of_range_ids():
    from tf_repos_b200 import ops
    from tf_repos_b200._lib import CtrError
    d = torch.device("cuda:0")
    B, Fp, N, K = 9, 2, 100, 8
    batch = _cuda(_edge_batch(B, Fp, N, seed=3))
    x = torch.zeros(B, (Fp + 8) * 12, device=d)
    with pytest.raises(CtrError, match="K=12 unsupported"):
        ops.esmm_embed_fwd(batch["feat_ids"], batch["a_ids"], batch["bag_ids"], batch["bag_wgt"], batch["bag_off"],
                           torch.zeros(N, 12, device=d), x)
    batch["bag_ids"][4] = N + 7
    batch["feat_ids"][2, 1] = -3
    x = torch.zeros(B, (Fp + 8) * K, device=d)
    oob = torch.zeros(2, dtype=torch.int32, device=d)
    ops.esmm_embed_fwd(batch["feat_ids"], batch["a_ids"], batch["bag_ids"], batch["bag_wgt"], batch["bag_off"],
                       torch.randn(N, K, device=d), x, oob)
    cnt, first = oob.tolist()
    assert cnt == 2 and first in (N + 7, -3)
    assert torch.all(x[2, K:2 * K] == 0)


def _head_inputs(B, seed):
    g = torch.Generator().manual_seed(seed)
    y_ctr = torch.randn(B, generator=g) * 4
    y_cvr = torch.randn(B, generator=g) * 4
    y_ctr[:6] = torch.tensor([30.0, -30.0, 30.0, -60.0, 0.0, -110.0])
    y_cvr[:6] = torch.tensor([30.0, -30.0, -30.0, -60.0, 0.0, 5.0])     # pctcvr = 1 (row 0) and 0 (rows 3, 5)
    y = (torch.rand(B, generator=g) < 0.4).float()
    z = y * (torch.rand(B, generator=g) < 0.5).float()
    y[:6] = torch.tensor([0.0, 1.0, 1.0, 1.0, 0.0, 1.0]); z[:6] = torch.tensor([0.0, 1.0, 0.0, 1.0, 0.0, 1.0])
    return y_ctr, y_cvr, y, z


@pytest.mark.parametrize("w", [0.0, 0.3, 0.5, 1.0])
def test_head_matches_restatement_deterministic_and_zero_past_n(w):
    from tf_repos_b200 import ops
    d = torch.device("cuda:0")
    B, n = 3000, 2777
    y_ctr, y_cvr, y, z = _head_inputs(B, seed=int(w * 10))
    ref = eo.head_reference(y_ctr[:n], y_cvr[:n], y[:n], z[:n], w, 1.0 - w)
    outs = []
    for _ in range(2):
        o = [torch.full((B,), float("nan"), device=d) for _ in range(5)] + [torch.zeros(2, device=d)]
        pt, pv, p, dc, dv, losses = o
        ops.esmm_head(y_ctr.to(d), y_cvr.to(d), y.to(d), z.to(d), n, w, 1.0 - w, pt, pv, p, losses, dc, dv)
        outs.append([t.cpu() for t in o])
    assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(*outs))     # run to run, bitwise
    pt, pv, p, dc, dv, losses = outs[0]
    assert p[0] == 1.0 and p[3] == 0.0 and p[5] == 0.0
    # rtol 1e-5 with an absolute floor of 1e-5 of the largest element: p - y and the log terms cancel for rows the
    # model already classifies well, whose gradients are then tiny in absolute terms
    for got, want, what in ((pt[:n], ref[0], "pctr"), (pv[:n], ref[1], "pcvr"), (p[:n], ref[2], "pctcvr"),
                            (losses[0], ref[3], "ctr_loss"), (losses[1], ref[4], "cvr_loss"),
                            (dc[:n], ref[5], "d y_ctr"), (dv[:n], ref[6], "d y_cvr")):
        _close(got, want, 1e-5, what)
    assert torch.all(dc[n:].view(torch.int32) == 0) and torch.all(dv[n:].view(torch.int32) == 0)
    if w == 1.0:
        assert torch.all(dv == 0)
    # inference: probabilities only
    q = [torch.zeros(B, device=d) for _ in range(3)]
    ops.esmm_head(y_ctr.to(d), y_cvr.to(d), None, None, 0, w, 1.0 - w, *q)
    assert torch.equal(q[2].cpu(), p)


def test_kernels_replay_in_a_cuda_graph():
    from tf_repos_b200 import ops
    d = torch.device("cuda:0")
    B, Fp, N, K = 64, 4, 3000, 16
    batch = _cuda(_edge_batch(B, Fp, N, seed=9))
    V = torch.randn(N, K, device=d)
    dx = torch.randn(B, (Fp + 8) * K, device=d)
    y_ctr, y_cvr, y, z = (t.to(d) for t in _head_inputs(B, seed=2))
    cap = batch["bag_ids"].numel() + 5
    x = torch.zeros(B, (Fp + 8) * K, device=d)
    g = torch.zeros(B * (Fp + 3) + cap, K, device=d)
    oob = torch.zeros(2, dtype=torch.int32, device=d)
    h = [torch.zeros(B, device=d) for _ in range(5)] + [torch.zeros(2, device=d)]

    def run():
        ops.esmm_embed_fwd(batch["feat_ids"], batch["a_ids"], batch["bag_ids"], batch["bag_wgt"], batch["bag_off"], V, x, oob)
        ops.esmm_head(y_ctr, y_cvr, y, z, B - 3, 0.3, 0.7, h[0], h[1], h[2], h[5], h[3], h[4])
        ops.esmm_embed_bwd(dx, batch["bag_wgt"], batch["bag_off"], B, Fp, K, g)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run()
    torch.cuda.current_stream().wait_stream(s)
    want = [t.clone() for t in [x, g] + h]
    for t in [x, g] + h:
        t.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        run()
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip([x, g] + h, want))


KW = dict(deep_layers="16,8", dropout="1.0,1.0", ctr_task_wgt=0.3, l2_reg=1e-4)
LENS = (6, 40, 6, 6, 4)


def _models(opt, mode, bn, cap, B=64, N=3000, K=8, Fp=5, epoch_steps=3):
    from tf_repos_b200.esmm import ESMM
    lr = 5e-4 if opt == "Adam" else 0.01
    ref = eo.ESMM(Fp, N, K, update_mode=("lazy" if mode == "lazy" else "exact"), seed=4, batch_norm=bn,
                  learning_rate=lr, optimizer=opt, **KW)
    g = torch.Generator().manual_seed(1)
    ref.params["embeddings"].copy_(torch.randn(N, K, generator=g) * 0.1)
    gpu = ESMM(Fp, N, K, B, cap, update_mode=mode, epoch_steps=epoch_steps, device="cuda:0", batch_norm=bn,
               learning_rate=lr, optimizer=opt, **KW)
    gpu.load_variables({**ref.params, **ref.bn_state})
    return ref, gpu


@pytest.mark.parametrize("opt,mode,bn", [("Adam", "exact", False), ("Adam", "exact_deferred", False),
                                         ("Adam", "lazy", False), ("Adagrad", "exact", False), ("Adam", "exact", True)])
def test_esmm_train_steps_match_oracle(opt, mode, bn):
    from tf_repos_b200 import synth
    B, N, K, Fp = 64, 3000, 8, 5
    batches = [synth.esmm_batch(B, N, Fp, max_lens=LENS, min_len=0, seed=60 + s) for s in range(4)]
    cap = max(b["bag_ids"].numel() for b, _ in batches) + 10
    ref, gpu = _models(opt, mode, bn, cap)
    for step, (batch, labels) in enumerate(batches):
        pt, pv, _ = gpu.predict(_cuda(batch))
        out = ref.predict(_long(batch))
        _close(pt, out["pctr"], 1e-5, f"pctr step {step}"); _close(pv, out["pcvr"], 1e-5, f"pcvr step {step}")
        loss_ref = ref.train_step(_long(batch), labels)
        parts = gpu.train_step(_cuda(batch), tuple(l.cuda() for l in labels))
        gpu.check_ids()
        if mode == "exact":
            assert abs(gpu.loss_value(parts) - loss_ref) <= 1e-5 * abs(loss_ref)
        vs = gpu.variables()
        names = ["embeddings", "cvr_mlp0/weights", "ctr_mlp0/weights", "cvr_mlp1/biases", "cvr_out/weights",
                 "ctr_out/weights", "ctr_out/biases"]
        if bn:
            names += ["cvr_bn_0/gamma", "ctr_bn_1/beta", "ctr_bn_0/moving_mean", "cvr_bn_1/moving_variance"]
        for name in names:
            want = ref.params[name] if name in ref.params else ref.bn_state[name]
            _close(vs[name], want, 2e-5, f"{name} after step {step} ({opt},{mode},bn={bn})")


def test_exact_deferred_state_equals_exact():
    from tf_repos_b200 import synth
    B, N, K, Fp = 64, 3000, 8, 5
    batches = [synth.esmm_batch(B, N, Fp, max_lens=LENS, min_len=0, seed=80 + s, device="cuda") for s in range(5)]
    cap = max(b["bag_ids"].numel() for b, _ in batches)
    _, a = _models("Adam", "exact", False, cap)
    _, b = _models("Adam", "exact_deferred", False, cap)
    for batch, labels in batches:
        a.train_step(batch, labels); b.train_step(batch, labels)
    b.flush()
    assert torch.equal(a.V.var, b.V.var) and all(torch.equal(x, y) for x, y in zip(a.V.slots, b.V.slots))
    assert torch.equal(a.dense.flat, b.dense.flat)


def _pad(batch, labels, B):
    """pad a CSR batch of n samples to B with copies of sample 0 (what esmm_main.make_batch does)"""
    n = batch["feat_ids"].shape[0]
    off = batch["bag_off"].tolist()
    ids, wgt, new_off = [], [], [0]
    for j in range(5):
        for b in list(range(n)) + [0] * (B - n):
            lo, hi = off[j * n + b], off[j * n + b + 1]
            ids.append(batch["bag_ids"][lo:hi]); wgt.append(batch["bag_wgt"][lo:hi])
            new_off.append(new_off[-1] + hi - lo)
    rep = lambda t, dim: torch.cat([t, t.narrow(dim, 0, 1).repeat_interleave(B - n, dim)], dim)
    padded = {"feat_ids": rep(batch["feat_ids"], 0), "a_ids": rep(batch["a_ids"], 1), "bag_ids": torch.cat(ids),
              "bag_wgt": torch.cat(wgt), "bag_off": torch.tensor(new_off, dtype=torch.int32)}
    return padded, tuple(rep(l, 0) for l in labels)


@pytest.mark.parametrize("mode", ["exact", "exact_deferred"])
def test_partial_final_batch_equals_the_smaller_batch(mode):
    from tf_repos_b200 import synth
    B, n, N, K, Fp = 64, 23, 3000, 8, 5
    full, lab = synth.esmm_batch(B, N, Fp, max_lens=LENS, min_len=0, seed=7)
    small, lab_s = synth.esmm_batch(n, N, Fp, max_lens=LENS, min_len=0, seed=8)
    padded, lab_p = _pad(small, lab_s, B)
    cap = max(full["bag_ids"].numel(), padded["bag_ids"].numel())
    ref, gpu = _models("Adam", mode, False, cap)
    ref.train_step(_long(full), lab)
    gpu.train_step(_cuda(full), tuple(l.cuda() for l in lab))
    loss_ref = ref.train_step(_long(small), lab_s)
    parts = gpu.train_step(_cuda(padded), tuple(l.cuda() for l in lab_p), n_valid=n)
    if mode == "exact":
        assert abs(gpu.loss_value(parts) - loss_ref) <= 1e-5 * abs(loss_ref), (gpu.loss_value(parts), loss_ref)
    vs = gpu.variables()
    for name in ("embeddings", "cvr_mlp0/weights", "ctr_mlp0/weights", "cvr_out/biases", "ctr_out/weights"):
        _close(vs[name], ref.params[name], 2e-5, f"{name} after the partial batch ({mode})")


def test_out_of_range_ids_raise_and_capacity_overflow_raises():
    from tf_repos_b200 import synth
    from tf_repos_b200.esmm import ESMM
    B, N, K, Fp = 32, 500, 8, 3
    batch, labels = synth.esmm_batch(B, N, Fp, max_lens=LENS, min_len=0, seed=1, device="cuda")
    m = ESMM(Fp, N, K, B, batch["bag_ids"].numel(), device="cuda:0", **KW)
    batch["bag_ids"][0] = N
    m.train_step(batch, labels)
    with pytest.raises(IndexError, match="outside"):
        m.check_ids()
    small = ESMM(Fp, N, K, B, batch["bag_ids"].numel() - 1, device="cuda:0", **KW)
    with pytest.raises(ValueError, match="capacity"):
        small.train_step(batch, labels)
