"""Shared host-side skeleton of the libsvm models (DeepFM, DCN, PNN, NFM, AFM): one embedding table
`[N,K]` (+ an optional first-order table `[N]`) gathered with the same `feat_ids`, a dense part, the
sigmoid-CE head and `optimizer.minimize` with TensorFlow's update semantics.

Sub-classes implement
    _forward(ids, vals, train, masks) -> (bias, y_a, y_b, y_c)   logit terms, summed left to right
    _backward(ids, vals)                                          from self.dy: fill self.g_rows
                                                                  (+ self.g_w) and the dense gradients
The update modes (exact / exact_deferred / lazy) and their step schedule: engine.SparseUpdater.  In
exact_deferred mode the l2*l2_loss terms of `loss` become available at the end of each epoch (`epoch_reg_terms`).
Data parallel (world > 1): tables are replicated; every rank all-gathers the per-occurrence sparse
gradients and applies the identical de-duplicated update; dense gradients + loss ride in one
all-reduce.  Synchronous DP replaces the reference's asynchronous parameter server
(DeepFM.py:237-282) -- a documented deviation.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from . import ops
from .engine import DenseVars, OptimizerState, SparseModel, SparseUpdater, Table


def ints(s) -> List[int]:
    return [int(t) for t in s.split(",")] if isinstance(s, str) else list(s)


def floats(s) -> List[float]:
    return [float(t) for t in s.split(",")] if isinstance(s, str) else list(s)


class CTRModel(SparseModel):
    replayed_launches = 0               # kernels launched through CUDA-graph replays (train_step_graphed)
    batch_norm, bn_decay = False, 0.9   # --batch_norm / --batch_norm_decay (set by the sub-class before _build)
    table_name = "emb"          # TF variable name of the [N,K] table
    linear_name: Optional[str] = None  # TF variable name of the [N] first-order table, if any

    def __init__(self, field_size: int, feature_size: int, embedding_size: int, batch_size: int,
                 l2_reg: float, learning_rate: float, optimizer: str, update_mode: str = "exact",
                 device="cuda", seed: int = 0, world: int = 1, epoch_steps: int = 8):
        self.F, self.N, self.K, self.B = field_size, feature_size, embedding_size, batch_size
        self.l2_reg = float(l2_reg)
        self.device = torch.device(device)
        self.world, self.seed = world, seed
        dev = self.device
        self.opt = OptimizerState(optimizer, learning_rate, l2_reg, dev)
        self.V = Table(self.table_name, self.N, self.K, self.opt, dev, seed=seed * 2 + 1)
        self.W = Table(self.linear_name, self.N, 1, self.opt, dev, seed=seed * 2 + 2) if self.linear_name else None
        self.tables = [self.V] + ([self.W] if self.W is not None else [])
        B, F, K = self.B, self.F, self.K
        f32 = dict(dtype=torch.float32, device=dev)
        self.y = torch.empty(B, **f32)
        self.pred = torch.empty(B, **f32)
        self.dy = torch.empty(B, **f32)
        self.g_rows = torch.empty(B * F, K, **f32)
        self.g_w = torch.empty(B * F, **f32) if self.W is not None else None
        self.oob = torch.zeros(2, dtype=torch.int32, device=dev)
        G = world
        self.updater = SparseUpdater(G * B * F, self.N, K, self.opt, dev, self.W is not None, self.tables, update_mode,
                                     epoch_steps, l2_reg)
        if G > 1:
            self.ids_all = torch.empty(G * B * F, dtype=torch.int32, device=dev)
            self.g_rows_all = torch.empty(G * B * F, K, **f32)
            self.g_w_all = torch.empty(G * B * F, **f32) if self.W is not None else None
        self.global_step = 0
        self.dense: DenseVars = None  # set by the sub-class (_build)
        self._build()
        self.loss_ce = self.dense.tail[0:1]

    # ---- to be provided --------------------------------------------------------------------------------
    def _build(self):
        raise NotImplementedError

    def _forward(self, ids, vals, train: bool, masks=None):
        raise NotImplementedError

    def _backward(self, ids, vals):
        raise NotImplementedError

    def _dense_reg_terms(self) -> Optional[torch.Tensor]:
        """l2*l2_loss of regularised DENSE variables (DCN's cross_w/cross_b), device tensor or None."""
        return None

    def epoch_reg_terms(self) -> torch.Tensor:
        """exact_deferred: [n_tables, epoch_steps] l2*l2_loss(table) for every step of the epoch that just
        ended, in loss order (linear table first when present)."""
        ep = self.updater.ep
        order = ([self.W] if self.W is not None else []) + [self.V]
        return torch.stack([ep[t.name]["reg"][: self.epoch_steps] for t in order])

    # ---- variable access by TF name --------------------------------------------------------------------------
    def variables(self) -> Dict[str, torch.Tensor]:
        self.flush()
        out = {t.name: t.var for t in self.tables}
        out.update(self.dense.views)
        mlp = getattr(self, "mlp", None)
        if mlp is not None:
            out.update(mlp.bn_state)      # non-trainable moving_mean / moving_variance (batch_norm=True)
        return out

    # ---- modes --------------------------------------------------------------------------------------------------
    def predict(self, ids: torch.Tensor, vals: torch.Tensor) -> torch.Tensor:
        """mode == PREDICT (DeepFM.py:178-185): returns prob [B]."""
        B = ids.shape[0]
        self.flush()
        bias, y_a, y_b, y_c = self._forward(ids, vals, train=False)
        ops.logit_loss(bias, y_a, y_b, y_c, None, B, y=self.y[:B], pred=self.pred[:B])
        return self.pred[:B]

    def train_step(self, ids: torch.Tensor, vals: torch.Tensor, labels: torch.Tensor, masks=None) -> torch.Tensor:
        """mode == TRAIN: one optimizer.minimize(loss) (DeepFM.py:188-213).  Returns a device tensor
        {mean CE, l2*l2_loss terms in the order of the reference's loss expression} whose left-to-right
        sum is `loss` (table terms come from the dense sweep in exact mode; zeros otherwise)."""
        B, F, K = ids.shape[0], self.F, self.K
        assert B <= self.B, "batch larger than the configured batch_size"
        assert B == self.B or self.world == 1, "partial batches are not supported under data parallelism"
        deferred = self.update_mode == "exact_deferred"
        upd = self.updater
        upd.begin_step()
        ids_u = ids.reshape(-1)
        if deferred and self.world > 1:
            import torch.distributed as dist
            dist.all_gather_into_tensor(self.ids_all, ids_u)
            ids_u = self.ids_all
        # gathered rows (of every rank) must hold the state at the start of this step
        upd.catch_up(ids_u)
        bias, y_a, y_b, y_c = self._forward(ids, vals, train=True, masks=masks)
        ops.logit_loss(bias, y_a, y_b, y_c, labels, B, y=self.y[:B], pred=self.pred[:B], loss_ce=self.loss_ce,
                       dy=self.dy[:B], dbias=(self.dense.grads[self.bias_name] if self.bias_name else None),
                       B_total=B * self.world)
        self._backward(ids, vals)
        g_rows = self.g_rows[: B * F]
        g_w = self.g_w[: B * F] if self.g_w is not None else None
        if self.world > 1:
            import torch.distributed as dist
            if not deferred:
                dist.all_gather_into_tensor(self.ids_all, ids.reshape(-1))
            dist.all_gather_into_tensor(self.g_rows_all, g_rows)
            if g_w is not None:
                dist.all_gather_into_tensor(self.g_w_all, g_w)
            dist.all_reduce(self.dense.grad)  # dense gradients + the loss tail, summed over ranks
            g_rows, g_w = self.g_rows_all, (self.g_w_all if g_w is not None else None)
        upd.finish_step(self.ids_all if self.world > 1 else ids.reshape(-1), g_rows, g_w)
        dense_reg = self._dense_reg_terms()
        self.dense.apply()
        self.global_step += 1
        parts = [self.loss_ce]
        if dense_reg is not None and not self.table_reg_first:
            parts.append(dense_reg)
        if self.W is not None:
            parts.append(upd.reg[1:2])
        parts.append(upd.reg[0:1])
        if dense_reg is not None and self.table_reg_first:
            parts.append(dense_reg)
        return torch.cat(parts)

    bias_name: Optional[str] = None
    # loss-term order: False = dense terms before the tables (DCN.py:198-199), True = after them (DeepMVM.py:197-199)
    table_reg_first = False

    # ---- CUDA-graph replay of the step ----------------------------------------------------------------------
    def train_step_graphed(self, ids: torch.Tensor, vals: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
        """train_step with the ~45 kernel launches of a step replayed from a CUDA graph (one graph per position in
        the epoch: the position is a launch argument of the row kernels).  Same kernels, same order, same results;
        what goes away is the per-launch host latency between them.  Full batches on one GPU only; the step that
        ends an epoch (it launches the table sweep) runs eagerly.  The returned tensor is the graph's static output:
        it is overwritten by the next replay of the same position."""
        B = ids.shape[0]
        deferred = self.update_mode == "exact_deferred"
        ends_epoch = deferred and self.epoch_pos == self.epoch_steps - 1
        if B != self.B or self.world != 1 or ends_epoch:
            return self.train_step(ids, vals, labels)
        if not hasattr(self, "_graphs"):
            self._graphs, self._graph_out, self._graph_seen = {}, {}, {}
            self._gin = (torch.empty(self.B, self.F, dtype=torch.int32, device=self.device),
                         torch.empty(self.B, self.F, dtype=torch.float32, device=self.device),
                         torch.empty(self.B, dtype=torch.float32, device=self.device))
        for dst, src in zip(self._gin, (ids, vals, labels)):
            dst.copy_(src, non_blocking=True)
        key = (self.update_mode, self.epoch_pos if deferred else 0)
        g = self._graphs.get(key)
        if g is None:
            if not self._graph_seen.get(key):       # first visit: eager (lazy allocations, cudaFuncSetAttribute, ...)
                self._graph_seen[key] = True
                return self.train_step(*self._gin)
            from . import _lib
            pos, step = self.epoch_pos, self.global_step
            n0 = _lib.launch_count()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                out = self.train_step(*self._gin)
            # capture ran the host code (bookkeeping advanced) but launched nothing: rewind, then replay below
            self.updater.epoch_pos, self.global_step = pos, step
            self._graphs[key], self._graph_out[key] = g, out
            self._graph_launches = getattr(self, "_graph_launches", {})
            self._graph_launches[key] = _lib.launch_count() - n0     # kernels of libctr_b200.so inside this graph
            self.replayed_launches -= self._graph_launches[key]      # the capture itself launched nothing
        g.replay()
        self.replayed_launches += self._graph_launches[key]
        self.global_step += 1
        if deferred:
            self.updater.epoch_pos += 1
        return self._graph_out[key]

    def predict_graphed(self, ids: torch.Tensor, vals: torch.Tensor) -> torch.Tensor:
        """predict() for full batches with the forward's launches replayed from one CUDA graph (same kernels)."""
        B = ids.shape[0]
        if B != self.B or self.world != 1:
            return self.predict(ids, vals)
        self.flush()
        if not hasattr(self, "_pg"):
            self._pg, self._pg_seen = None, 0
            self._pin = (torch.empty(self.B, self.F, dtype=torch.int32, device=self.device),
                         torch.empty(self.B, self.F, dtype=torch.float32, device=self.device))
        self._pin[0].copy_(ids, non_blocking=True); self._pin[1].copy_(vals, non_blocking=True)
        if self._pg is None:
            self._pg_seen += 1
            if self._pg_seen < 2:
                return self.predict(*self._pin)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._pg_out = self.predict(*self._pin)
            self._pg = g
        self._pg.replay()
        return self._pg_out

    def loss_value(self, parts: torch.Tensor) -> float:
        total = 0.0
        for p in parts.tolist():
            total = total + p
        return total
