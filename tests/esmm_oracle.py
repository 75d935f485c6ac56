"""CPU restatement of ESMM's model_fn (DeepMTL/Model_pipeline/DeepCvrMTL.py:107-259), op for op, on the shared oracle
machinery of oracle/models.py (variables, slots, TF update semantics).  Test infrastructure, like oracle/: the GPU parity
tests compare tf_repos_b200.esmm.ESMM against it, and test_oracle_esmm.py pins it with per-element loops, closed forms
and an fp64 autograd check of the hand-derived head gradient.

The shared OracleModel.gradients is written for one logit and one label (sigmoid CE); ESMM overrides it with the
two-task loss and leaves the shared machinery untouched.  Batches use the CSR layout of tf_repos_b200.esmm."""
from __future__ import annotations

import numpy as np
import torch

from oracle import models as om
from oracle import tf_semantics as tfs

TOWERS = ("cvr", "ctr")
LOG_EPS = 1e-7          # tf.losses.log_loss default epsilon


def bag_sums(rows, wgt, off, n_weighted):
    """embedding_lookup_sparse(combiner="sum") over CSR bags, sequentially: acc = +0; acc = acc + e_i*w_i in occurrence
    order (one rounded multiply, then one rounded add); bags >= n_weighted are unweighted (acc = acc + e_i)."""
    off = off.long()
    nb = off.numel() - 1
    lens = off[1:] - off[:-1]
    acc = torch.zeros(nb, rows.shape[1], dtype=rows.dtype)
    weighted = torch.arange(nb) < n_weighted
    for p in range(int(lens.max()) if nb else 0):
        sel = torch.nonzero(lens > p).reshape(-1)
        i = off[sel] + p
        w = weighted[sel]
        term = torch.where(w.unsqueeze(1), rows[i] * wgt[i].to(rows.dtype).unsqueeze(1), rows[i])
        acc = acc.index_add(0, sel, term)
    return acc


def log_loss(p, z, eps=LOG_EPS):
    """tf.losses.log_loss(labels=z, predictions=p) [TF-sem]: -z*log(p+eps) - (1-z)*log(1-p+eps), reduced with
    SUM_BY_NONZERO_WEIGHTS (weights 1: the mean over the batch)."""
    losses = -(z * torch.log(p + eps)) - ((1 - z) * torch.log(1 - p + eps))
    return losses.sum() / losses.numel()


def head_reference(y_ctr, y_cvr, y, z, w_ctr, w_cvr, dtype=torch.float32, pt=None, pv=None):
    """The head gradient csrc/esmm.cu implements, one rounded op at a time in TF's autodiff order (include/ctr_b200.h,
    ctr_esmm_head); fp32 like the kernel, or fp64 to check the derivation.  Given pt / pv (e.g. the kernel's own
    sigmoids), the chain starts from them instead of recomputing the sigmoids, so every later op can be compared bit
    for bit.  Returns (pctr, pcvr, pctcvr, ctr_loss, cvr_loss, d_ctr, d_cvr)."""
    f = dtype
    one = torch.ones((), dtype=f)
    n = y_ctr.numel()
    a, c, t, zz = y_ctr.to(f), y_cvr.to(f), y.to(f), z.to(f)
    pt = tfs.sigmoid(a) if pt is None else pt.to(f)
    pv = tfs.sigmoid(c) if pv is None else pv.to(f)
    p = pt * pv
    g_ctr = torch.tensor(w_ctr, dtype=f) / torch.tensor(float(n), dtype=f)
    g_cvr = torch.tensor(w_cvr, dtype=f) / torch.tensor(float(n), dtype=f)
    q1, q2 = p + LOG_EPS, (one - p) + LOG_EPS
    nz = one - zz
    ctr_loss = tfs.sigmoid_cross_entropy_with_logits(a, t).sum() / n
    cvr_loss = (-(zz * torch.log(q1)) - (nz * torch.log(q2))).sum() / n
    ng = -g_cvr
    dp = (ng * zz) * (one / q1) + (-((ng * nz) * (one / q2)))
    d_cvr = ((dp * pt) * pv) * (one - pv)
    d_ctr = (pt - t) * g_ctr + ((dp * pv) * pt) * (one - pt)
    return pt, pv, p, ctr_loss, cvr_loss, d_ctr, d_cvr


class ESMM(om.OracleModel):
    """DeepCvrMTL.py:107-259.  Labels are (y, z)."""

    tables = ("embeddings",)
    l2_vars = ("embeddings",)  # DeepCvrMTL.py:223

    def __init__(self, field_size, feature_size, embedding_size, deep_layers="256,128,64", dropout="0.5,0.5,0.5",
                 ctr_task_wgt=0.5, batch_norm=False, batch_norm_decay=0.9, seed=0, **kw):
        super().__init__(**kw)
        self.Fp, self.N, self.K = field_size, feature_size, embedding_size
        self.layers, self.keep = om._ints(deep_layers), om._floats(dropout)
        self.w = float(ctr_task_wgt)
        self.batch_norm, self.bn_decay = batch_norm, batch_norm_decay
        self.bn_state = {}
        gen = torch.Generator().manual_seed(seed)
        self.add_param("embeddings", tfs.glorot_normal((self.N, self.K), gen, self.dtype))     # :122
        for t in TOWERS:                                                                        # :171-203
            d = (self.Fp + 8) * self.K
            for i, h in enumerate(self.layers):
                self.add_param(f"{t}_mlp{i}/weights", tfs.xavier_uniform((d, h), gen, self.dtype))
                self.add_param(f"{t}_mlp{i}/biases", torch.zeros(h, dtype=self.dtype))
                if batch_norm:
                    self.add_param(f"{t}_bn_{i}/gamma", torch.ones(h, dtype=self.dtype))
                    self.add_param(f"{t}_bn_{i}/beta", torch.zeros(h, dtype=self.dtype))
                    self.bn_state[f"{t}_bn_{i}/moving_mean"] = torch.zeros(h, dtype=self.dtype)
                    self.bn_state[f"{t}_bn_{i}/moving_variance"] = torch.ones(h, dtype=self.dtype)
                d = h
            self.add_param(f"{t}_out/weights", tfs.xavier_uniform((d, 1), gen, self.dtype))
            self.add_param(f"{t}_out/biases", torch.zeros(1, dtype=self.dtype))
        self.init_slots()

    def sites(self, batch):
        return {"common": ("embeddings", batch["feat_ids"]), "a": ("embeddings", batch["a_ids"]),
                "occ": ("embeddings", batch["bag_ids"])}

    def _tower(self, t, x, dense, train, masks):
        for i in range(len(self.layers)):
            x = tfs.fully_connected(x, dense[f"{t}_mlp{i}/weights"], dense[f"{t}_mlp{i}/biases"], "relu")
            if self.batch_norm:
                x = tfs.batch_norm(x, dense[f"{t}_bn_{i}/gamma"], dense[f"{t}_bn_{i}/beta"],
                                   self.bn_state[f"{t}_bn_{i}/moving_mean"],
                                   self.bn_state[f"{t}_bn_{i}/moving_variance"], train, self.bn_decay)
            if train:
                x = tfs.dropout(x, self.keep[i], None if masks is None or masks.get(t) is None else masks[t][i])
        return tfs.fully_connected(x, dense[f"{t}_out/weights"], dense[f"{t}_out/biases"], None).reshape(-1)

    def forward(self, rows, dense, batch, train, masks=None):
        B, K = batch["feat_ids"].shape[0], self.K
        common = rows["common"].reshape(B, self.Fp * K)                                         # :153
        a = rows["a"]                                                                           # :160-162
        bags = bag_sums(rows["occ"], batch["bag_wgt"], batch["bag_off"], 4 * B).reshape(5, B, K)  # :155-159
        x = torch.cat([common, bags[0], bags[1], bags[2], bags[3], a[0], a[1], a[2], bags[4]], 1)  # :164
        y = {t: self._tower(t, x, dense, train, masks) for t in TOWERS}
        pctr, pcvr = tfs.sigmoid(y["ctr"]), tfs.sigmoid(y["cvr"])                              # :205-208
        return {"y_ctr": y["ctr"], "y_cvr": y["cvr"], "pctr": pctr, "pcvr": pcvr, "pctcvr": pctr * pcvr, "x": x}

    def predict(self, batch):
        with torch.no_grad():
            dense = {n: p for n, p in self.params.items() if n not in self.tables}
            return self.forward(self._gather(batch, False), dense, batch, train=False)

    def task_losses(self, out, labels):
        y, z = (l.to(self.dtype) for l in labels)
        ctr = tfs.sigmoid_cross_entropy_with_logits(out["y_ctr"], y).mean()                     # :220
        cvr = log_loss(out["pctcvr"], z)                                                        # :222
        return ctr, cvr

    def gradients(self, batch, labels, masks=None):
        """OracleModel.gradients with loss = w*ctr_loss + (1-w)*cvr_loss + l2*l2_loss(embeddings) (:223); the weights
        are the fp32 constants TF makes of the Python floats w and 1 - w."""
        rows = self._gather(batch, True)
        dense = {n: p.detach().requires_grad_() for n, p in self.params.items() if n not in self.tables}
        out = self.forward(rows, dense, batch, train=True, masks=masks)
        ctr, cvr = self.task_losses(out, labels)
        obj = torch.tensor(self.w, dtype=self.dtype) * ctr + torch.tensor(1.0 - self.w, dtype=self.dtype) * cvr
        obj.backward()
        loss = obj.detach() + self.reg_loss()
        sites = self.sites(batch)
        table_grads = {}
        vals, idx = [], []
        for site, (tn, ids) in sites.items():
            g = rows[site].grad if rows[site].grad is not None else torch.zeros_like(rows[site])
            vals.append(g.reshape(-1, self.K).numpy())
            idx.append(ids.reshape(-1).numpy())
        summed, uniq = tfs.deduplicate_indexed_slices(np.concatenate(vals), np.concatenate(idx))
        table_grads["embeddings"] = (torch.from_numpy(summed), torch.from_numpy(uniq.astype(np.int64)))
        dense_grads = {n: (p.grad if p.grad is not None else torch.zeros_like(p)) for n, p in dense.items()}
        out = {k: v.detach() for k, v in out.items()}
        out["per_occurrence"] = {s: (rows[s].grad.detach() if rows[s].grad is not None else None) for s in rows}
        return loss, out, table_grads, dense_grads
