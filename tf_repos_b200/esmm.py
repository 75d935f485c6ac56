"""ESMM (Entire Space Multi-task Model) on the H100 engine: mirror of `model_fn` in
DeepMTL/Model_pipeline/DeepCvrMTL.py:107-259.

Inputs (the TFRecord features of DeepCvrMTL.py:66-83, the Ali-CCP layout DIN reads; no densification: the reference
calls embedding_lookup_sparse on the var-len SparseTensors, :155-159):
    feat_ids [B,F'] int32                        common fields (no feat_vals, :153-154)
    a_ids    [3,B]  int32                        a_catids, a_shopids, a_brandids
    bag_ids [nnz] int32, bag_wgt [nnz] f32,      one CSR over 5B bags: bag j*B+b is field j of sample b, j = u_cat,
    bag_off [5B+1] int32                         u_shop, u_brand, u_int (weighted by u_*vals), a_int (unweighted)
Id 0 is an ordinary row.  Labels: y (click) and z (conversion).
Variables (TF names; tf.name_scope("CVR_Task") does not prefix get_variable names): `embeddings [N,K]`;
`cvr_mlp{i}/{weights,biases}`, `cvr_out/...`, `ctr_mlp{i}/...`, `ctr_out/...`; with --batch_norm `cvr_bn_{i}/...` and
`ctr_bn_{i}/...`.  Only the table is L2-regularised (the fully_connected regularizers never reach `loss`, quirk Q4).

loss = w * mean CE(y_ctr, y) + (1-w) * log_loss(pctr*pcvr, z) + l2 * l2_loss(embeddings)   (:220-223); the head and
the embedding layer are csrc/esmm.cu, the towers the wgmma MLP.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import ops
from .base import floats, ints
from .engine import DenseVars, OptimizerState, SparseModel, SparseUpdater, Table
from .mlp import MLP

BAGS = ("u_cat", "u_shop", "u_brand", "u_int", "a_int")
TOWERS = ("cvr", "ctr")          # creation order of DeepCvrMTL.py:166-203


class ESMM(SparseModel):
    def __init__(self, field_size: int, feature_size: int, embedding_size: int, batch_size: int, occ_capacity: int,
                 deep_layers="256,128,64", dropout="0.5,0.5,0.5", ctr_task_wgt: float = 0.5, l2_reg: float = 1e-4,
                 learning_rate: float = 5e-4, optimizer: str = "Adam", update_mode: str = "exact", device="cuda",
                 seed: int = 0, epoch_steps: int = 8, batch_norm: bool = False, batch_norm_decay: float = 0.9):
        self.Fp, self.N, self.K, self.B = field_size, feature_size, embedding_size, batch_size
        self.cap = int(occ_capacity)
        self.layers, self.keep = ints(deep_layers), floats(dropout)
        self.ctr_task_wgt = float(ctr_task_wgt)
        # TF turns the Python constants w and 1 - w into fp32 constants separately (:223)
        self.w_ctr, self.w_cvr = self.ctr_task_wgt, 1.0 - self.ctr_task_wgt
        self.l2_reg = float(l2_reg)
        self.device = dev = torch.device(device)
        self.seed = seed
        B, Fp, K = self.B, self.Fp, self.K
        self.opt = OptimizerState(optimizer, learning_rate, l2_reg, dev)
        self.V = Table("embeddings", self.N, K, self.opt, dev, seed=seed * 2 + 1)          # :122
        self.tables = [self.V]
        self.Dx = (Fp + 8) * K                                                               # :164
        # two towers; distinct seeds so that their dropout masks differ (MLP draws them from seed*131 + layer)
        self.towers = {t: MLP(self.Dx, self.layers, self.keep, B, dev, scope="", out_scope=f"{t}_out",
                              seed=seed * 2 + k, layer_fmt=f"{t}_mlp{{i}}", batch_norm=batch_norm,
                              bn_decay=batch_norm_decay, bn_fmt=f"{t}_bn_{{i}}")
                       for k, t in enumerate(TOWERS)}
        self.dense = DenseVars(self.towers["cvr"].specs() + self.towers["ctr"].specs(), self.opt, dev)
        gen = torch.Generator().manual_seed(seed)
        for t in TOWERS:
            self.towers[t].init(self.dense, gen)
        f32 = dict(dtype=torch.float32, device=dev)
        self.x = torch.empty(B, self.Dx, **f32)
        self.dx = torch.empty(B, self.Dx, **f32)
        self.pctr, self.pcvr, self.pctcvr = (torch.empty(B, **f32) for _ in range(3))
        self.dy = {t: torch.empty(B, **f32) for t in TOWERS}
        self.d_last = {t: torch.empty(B, self.towers[t].out_in, **f32) for t in TOWERS}
        self.losses = self.dense.tail[0:2]                                                   # ctr_loss, cvr_loss
        self.oob = torch.zeros(2, dtype=torch.int32, device=dev)
        # per-occurrence ids / gradient rows: [common B*F' | a_cat a_shop a_brand | bag occurrences (capacity)]
        self.n_fixed = B * Fp + 3 * B
        self.n_total = self.n_fixed + self.cap
        self.ids_all = torch.zeros(self.n_total, dtype=torch.int32, device=dev)
        self.g_all = torch.zeros(self.n_total, K, **f32)
        self.updater = SparseUpdater(self.n_total, self.N, K, self.opt, dev, False, self.tables, update_mode,
                                     epoch_steps, l2_reg)
        self._a = {}
        self.global_step = 0

    def grow(self, occ_capacity: int):
        """For inference: let the model take batches of up to occ_capacity bag occurrences (sizes never shrink).  The
        forward reads the bags through bag_off and holds no occurrence-sized buffer of its own, so growing allocates
        nothing and cannot fail half way; the caller sizes its bag_ids / bag_wgt.  The training buffers, sized to the
        old capacity, are released: a grown model predicts but no longer trains.  Variables, optimizer slots and
        batch-norm statistics stay."""
        cap = max(self.cap, int(occ_capacity))
        if cap == self.cap:
            return
        self.cap, self.n_total = cap, self.n_fixed + cap
        self.ids_all = self.g_all = None

    # ---- plumbing -------------------------------------------------------------------------------------
    def variables(self) -> Dict[str, torch.Tensor]:
        self.flush()
        out = {"embeddings": self.V.var}
        out.update(self.dense.views)
        for t in TOWERS:
            out.update(self.towers[t].bn_state)
        return out

    def _stage_ids(self, batch):
        """ids of every lookup of the step in gradient-row order; unused occurrence slots repeat the batch's first
        common id (gathered anyway) with zero gradient rows, so they change neither the unique set nor its sums."""
        nnz = batch["bag_ids"].numel()
        if nnz > self.cap:
            raise ValueError(f"batch has {nnz} bag occurrences, the model's capacity is {self.cap}")
        B, Fp, o = self.B, self.Fp, self.n_fixed
        ids = self.ids_all
        ids[:B * Fp].copy_(batch["feat_ids"].reshape(-1))
        ids[B * Fp:o].copy_(batch["a_ids"].reshape(-1))
        ids[o:o + nnz].copy_(batch["bag_ids"])
        if nnz < self.cap:
            ids[o + nnz:].copy_(batch["feat_ids"].reshape(-1)[:1].expand(self.cap - nnz))

    # ---- f(x) -------------------------------------------------------------------------------------------
    def _forward(self, batch, train: bool, masks=None):
        ops.esmm_embed_fwd(batch["feat_ids"], batch["a_ids"], batch["bag_ids"], batch["bag_wgt"], batch["bag_off"],
                           self.V.var, self.x, self.oob)                                     # :153-164
        y = {}
        for t in TOWERS:                                                                     # :166-203
            m = masks.get(t) if masks else None
            self._a[t] = self.towers[t].forward_hidden(self.x, self.dense, train, m, step_dev=self.opt.state[3:4])
            y[t] = self.towers[t].forward_out(self._a[t], self.dense)
        return y

    def predict(self, batch, labels=None, n: Optional[int] = None):
        """pctr, pcvr, pctcvr [B] (:205-210).  With labels = (y, z): also ctr_loss, cvr_loss over the first n rows in
        self.losses (eval)."""
        self.flush()
        y = self._forward(batch, train=False)
        yl, zl = labels if labels is not None else (None, None)
        ops.esmm_head(y["ctr"], y["cvr"], yl, zl, self.B if n is None else n, self.w_ctr, self.w_cvr, self.pctr,
                      self.pcvr, self.pctcvr, self.losses if labels is not None else None)
        return self.pctr, self.pcvr, self.pctcvr

    def _backward(self, batch):
        dxs = []
        for t in TOWERS:
            tw = self.towers[t]
            tw.backward_out(self._a[t], self.dy[t], self.dense, self.d_last[t])
            dxs.append(tw.backward_hidden(self.x, self.d_last[t], self.dense))
        ops.axpby(dxs[0], 1.0, dxs[1], 1.0, self.dx)              # AddN of the two towers' d x_concat
        ops.esmm_embed_bwd(self.dx, batch["bag_wgt"], batch["bag_off"], self.B, self.Fp, self.K, self.g_all)

    def train_step(self, batch, labels, masks=None, n_valid: Optional[int] = None) -> torch.Tensor:
        """one optimizer.minimize(loss) (DeepCvrMTL.py:220-251); labels = (y, z).  Returns
        {ctr_loss, cvr_loss, l2*l2_loss(embeddings)}.  n_valid < batch_size: the final partial batch, padded by the
        caller; the losses are means over the n_valid real samples and the padded rows' logit gradients are exactly 0,
        so the step equals TensorFlow's step on the smaller batch (not with --batch_norm: the padded rows would enter
        the batch moments)."""
        if self.ids_all is None:
            raise RuntimeError("this ESMM grew its occurrence capacity for inference (ESMM.grow) and no longer trains")
        upd = self.updater
        self._stage_ids(batch)
        upd.begin_step()
        upd.catch_up(self.ids_all)
        y = self._forward(batch, train=True, masks=masks)
        n = self.B if n_valid is None else int(n_valid)
        assert 0 < n <= self.B
        if n < self.B and self.towers["ctr"].batch_norm:
            raise NotImplementedError("a partial final batch with --batch_norm (padded rows would enter the batch moments)")
        ops.esmm_head(y["ctr"], y["cvr"], labels[0], labels[1], n, self.w_ctr, self.w_cvr, self.pctr, self.pcvr,
                      self.pctcvr, self.losses, self.dy["ctr"], self.dy["cvr"])
        self._backward(batch)
        upd.finish_step(self.ids_all, self.g_all)
        self.dense.apply()
        self.global_step += 1
        return torch.cat([self.losses, upd.reg[0:1]])

    def loss_value(self, parts: torch.Tensor) -> float:
        """ctr_task_wgt*ctr_loss + (1 - ctr_task_wgt)*cvr_loss + l2_reg*l2_loss(embeddings)   (:223)"""
        p = parts.tolist()
        return self.w_ctr * p[0] + self.w_cvr * p[1] + p[2]
