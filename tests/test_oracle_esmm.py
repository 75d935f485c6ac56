"""ESMM (DeepCvrMTL.py:107-259) on the CPU: the oracle restatement against per-element loops and closed forms, the
hand-derived head gradient against fp64 autograd, the CSR input pipeline from TFRecords, and the flag surface."""
import importlib.util
import os
import types

import numpy as np
import pytest
import torch

from tests import esmm_oracle as eo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _csr(bags_per_kind):
    """bags_per_kind[j][b] = list of (id, weight) -> bag_ids, bag_wgt, bag_off"""
    ids, wgt, off = [], [], [0]
    for kind in bags_per_kind:
        for bag in kind:
            ids += [i for i, _ in bag]; wgt += [w for _, w in bag]
            off.append(len(ids))
    return (torch.tensor(ids, dtype=torch.int32), torch.tensor(wgt, dtype=torch.float32),
            torch.tensor(off, dtype=torch.int32))


def test_forward_matches_per_element_loops():
    """x = [common | u_cat u_shop u_brand u_int | a_cat a_shop a_brand | a_int] (DeepCvrMTL.py:164); weighted bags are
    e*w then a sequential sum, a_int is unweighted, id 0 is a real row, empty bags (first, middle, last sample) are 0."""
    B, Fp, N, K = 4, 2, 12, 4
    g = torch.Generator().manual_seed(0)
    ref = eo.ESMM(Fp, N, K, deep_layers="3", dropout="1.0", seed=1)
    ref.params["embeddings"].copy_(torch.randn(N, K, generator=g))
    feat = torch.tensor([[0, 1], [2, 3], [4, 0], [5, 6]], dtype=torch.int32)
    a_ids = torch.tensor([[1, 2, 3, 0], [4, 5, 6, 7], [0, 8, 9, 10]], dtype=torch.int32)
    bags = [
        [[], [(0, 0.5), (3, -1.25)], [(7, 0.0)], []],                          # u_cat: empty first and last
        [[(1, 1.0), (1, 2.0), (1, 3.0)], [], [(2, 0.75)], [(11, 1.5)]],        # u_shop: duplicates, empty middle
        [[(4, 2.5)], [(5, -0.5)], [], [(6, 1.0), (0, 0.25)]],
        [[(8, 1.0)], [(9, 3.0), (10, 0.1), (0, 7.0)], [(3, 1e-3)], []],
        [[(2, 9.0), (2, 9.0)], [], [(0, 9.0)], [(11, 9.0)]],                   # a_int: weights must be ignored
    ]
    bag_ids, bag_wgt, bag_off = _csr(bags)
    batch = {"feat_ids": feat, "a_ids": a_ids, "bag_ids": bag_ids, "bag_wgt": bag_wgt, "bag_off": bag_off}
    x = ref.predict({k: (v.long() if k.endswith("ids") else v) for k, v in batch.items()})["x"]
    V = ref.params["embeddings"].numpy()
    want = np.zeros((B, (Fp + 8) * K), np.float32)
    for b in range(B):
        cols = []
        for f in range(Fp):
            cols.append(V[feat[b, f]])
        sums = []
        for j in range(5):
            acc = np.zeros(K, np.float32)
            for i, w in bags[j][b]:
                term = V[i] if j == 4 else (V[i] * np.float32(w)).astype(np.float32)
                acc = (acc + term).astype(np.float32)
            sums.append(acc)
        cols += sums[:4] + [V[a_ids[0, b]], V[a_ids[1, b]], V[a_ids[2, b]]] + [sums[4]]
        want[b] = np.concatenate(cols)
    assert torch.equal(x, torch.from_numpy(want))
    assert torch.equal(x[0, Fp * K:(Fp + 1) * K], torch.zeros(K))          # empty u_cat bag of the first sample


def test_log_loss_closed_form():
    p = torch.tensor([0.0, 1e-9, 0.25, 0.5, 0.999, 1.0], dtype=torch.float64)
    z = torch.tensor([0.0, 1.0, 1.0, 0.0, 1.0, 0.0], dtype=torch.float64)
    eps = 1e-7
    want = np.mean([-(zi * np.log(pi + eps)) - (1 - zi) * np.log(1 - pi + eps) for pi, zi in zip(p.tolist(), z.tolist())])
    assert abs(float(eo.log_loss(p, z)) - want) <= 1e-12 * abs(want)
    # p = 0 with z = 1 and p = 1 with z = 0 stay finite: -log(eps)
    assert abs(float(eo.log_loss(torch.zeros(1, dtype=torch.float64), torch.ones(1, dtype=torch.float64))) + np.log(eps)) < 1e-9


@pytest.mark.parametrize("w", [0.0, 0.3, 0.5, 1.0])
def test_hand_derived_head_gradient_matches_fp64_autograd(w):
    g = torch.Generator().manual_seed(int(w * 10))
    n = 300
    y_ctr = torch.randn(n, generator=g) * 4
    y_cvr = torch.randn(n, generator=g) * 4
    y_ctr[:4] = torch.tensor([30.0, -30.0, 0.0, -60.0]); y_cvr[:4] = torch.tensor([30.0, -30.0, 0.0, -60.0])
    y = (torch.rand(n, generator=g) < 0.4).float()
    z = y * (torch.rand(n, generator=g) < 0.5).float()
    a, c = y_ctr.double().requires_grad_(), y_cvr.double().requires_grad_()
    from oracle import tf_semantics as tfs
    pctr, pcvr = torch.sigmoid(a), torch.sigmoid(c)
    ctr = tfs.sigmoid_cross_entropy_with_logits(a, y.double()).mean()
    cvr = eo.log_loss(pctr * pcvr, z.double())
    (w * ctr + (1 - w) * cvr).backward()
    # the derivation, evaluated in fp64: equal to autograd up to fp64 rounding
    pt, pv, p, lc, lv, dc, dv = eo.head_reference(y_ctr, y_cvr, y, z, w, 1.0 - w, dtype=torch.float64)
    for got, ref in ((lc, ctr), (lv, cvr), (p, pctr * pcvr), (dc, a.grad), (dv, c.grad)):
        np.testing.assert_allclose(got.detach().numpy(), ref.detach().numpy(), rtol=1e-9, atol=1e-15)
    # the fp32 evaluation (what the kernel computes) within 1e-5 of the largest gradient: near p = 1 the term
    # (1-p)+eps cancels in fp32 and the saturated rows lose their relative accuracy, but never more than that
    pt, pv, p, lc, lv, dc, dv = eo.head_reference(y_ctr, y_cvr, y, z, w, 1.0 - w)
    for got, ref in ((lc, ctr), (lv, cvr), (dc, a.grad), (dv, c.grad)):
        s = max(float(ref.detach().abs().max()), 1e-30)
        np.testing.assert_allclose(got.double().detach().numpy(), ref.detach().numpy(), rtol=1e-5, atol=1e-4 * s)
    if w == 1.0:
        assert torch.all(dv == 0)       # the CVR tower gets exactly no gradient
    assert torch.isfinite(dc).all() and torch.isfinite(dv).all()   # logits of +-30, -60: eps keeps the logs finite


def _write(path, n, seed, F=3, N=50, drop=None, mismatch=False):
    from tf_repos_b200 import tfrecord as tfr
    rng = np.random.RandomState(seed)
    recs = []
    for k in range(n):
        ex = {"y": np.float32(rng.rand() < 0.5), "z": np.float32(rng.rand() < 0.2),
              "feat_ids": rng.randint(0, N, F).astype(np.int64), "a_catids": np.int64(rng.randint(0, N)),
              "a_shopids": np.int64(rng.randint(0, N)), "a_brandids": np.int64(rng.randint(0, N)),
              "a_intids": rng.randint(0, N, rng.randint(0, 4)).astype(np.int64)}
        for f in ("cat", "shop", "brand", "int"):
            ln = rng.randint(0, 7)
            ex["u_%sids" % f] = rng.randint(0, N, ln).astype(np.int64)
            ex["u_%svals" % f] = (rng.rand(ln + (1 if mismatch and k == n - 1 else 0)) * 3).astype(np.float32)
        if drop:
            del ex[drop]
        recs.append(tfr.encode_example(ex))
    tfr.write_records(path, recs)


def test_csr_batching_from_tfrecords(tmp_path):
    from tf_repos_b200 import esmm_main as em
    p = os.path.join(tmp_path, "a.tfrecord")
    _write(p, 37, seed=1)
    d = em.decode([p], 3)
    assert len(d["y"]) == 37 and len(d["z"]) == 37
    batch, (y, z), n = em.make_batch(d, list(range(30, 37)), 8, "cpu")
    assert n == 7 and batch["bag_off"].shape == (41,) and y.shape == (8,) and z.shape == (8,)
    off = batch["bag_off"].tolist()
    for j, key in enumerate(("u_catids", "u_shopids", "u_brandids", "u_intids", "a_int")):
        for b in range(8):
            i = 30 + b if b < 7 else 30                                       # padding = copies of the first sample
            assert batch["bag_ids"][off[j * 8 + b]:off[j * 8 + b + 1]].tolist() == d[key][i].tolist()
            if j < 4:
                vals = d[key.replace("ids", "vals")][i]
                assert np.array_equal(batch["bag_wgt"][off[j * 8 + b]:off[j * 8 + b + 1]].numpy(), vals)
    # capacity: the largest batch of the stream, the padded final one included
    occ = em.sample_occurrences(d)
    want = 0
    for idx in em.index_stream(37, 3, 8):
        want = max(want, int(occ[idx].sum() + (8 - len(idx)) * occ[idx[0]]))
    assert em.max_batch_occurrences(d, 3, 8) == want
    # a batch larger than the capacity is refused, never truncated
    from tf_repos_b200.esmm import ESMM
    with pytest.raises(ValueError, match="capacity"):
        ESMM._stage_ids(types.SimpleNamespace(cap=int(off[-1]) - 1), batch)
    # z is required (FixedLenFeature without default), and ids / vals lengths must agree
    _write(p, 5, seed=2, drop="z")
    with pytest.raises(ValueError, match="Feature: z"):
        em.decode([p], 3)
    from tf_repos_b200 import din_main as dm
    assert len(dm.decode_tfrecord_files([p], 3)["y"]) == 5                   # DIN does not read z
    _write(p, 5, seed=3, mismatch=True)
    with pytest.raises(ValueError, match="lengths differ"):
        em.decode([p], 3)


def test_flag_surface_and_defaults():
    """the flags of DeepCvrMTL.py:34-60 with their defaults, plus the engine-only ones"""
    import importlib
    from tf_repos_b200 import flags
    importlib.reload(flags)
    spec = importlib.util.spec_from_file_location("esmm_script", os.path.join(ROOT, "Model_pipeline", "DeepCvrMTL.py"))
    spec.loader.exec_module(importlib.util.module_from_spec(spec))
    F = flags.FLAGS
    want = {"dist_mode": 0, "ps_hosts": "", "worker_hosts": "", "job_name": "", "task_index": 0, "num_threads": 16,
            "feature_size": 0, "field_size": 0, "embedding_size": 32, "num_epochs": 10, "batch_size": 64,
            "log_steps": 1000, "learning_rate": 0.0005, "l2_reg": 0.0001, "loss_type": "log_loss", "ctr_task_wgt": 0.5,
            "optimizer": "Adam", "deep_layers": "256,128,64", "dropout": "0.5,0.5,0.5", "batch_norm": False,
            "batch_norm_decay": 0.9, "data_dir": "", "dt_dir": "", "model_dir": "", "servable_model_dir": "",
            "task_type": "train", "clear_existing_model": False}
    items = F._items()
    assert set(items) - set(want) == {"update_mode", "input_parse"}
    assert {k: items[k] for k in want} == want
    F._parse(["--ctr_task_wgt=0.3", "--deep_layers=256,128", "--dropout=0.8,0.5", "--update_mode=lazy"])
    assert F.ctr_task_wgt == 0.3 and F.deep_layers == "256,128" and F.update_mode == "lazy"
    importlib.reload(flags)
