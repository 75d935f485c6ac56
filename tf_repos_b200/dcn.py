"""Deep & Cross Network on the H100 engine: mirror of `model_fn` in deep_ctr/Model_pipeline/DCN.py:105-230.

Variables (TF names): `emb [N,K]`, `cross_w [L,D]`, `cross_b [L,D]` (all three L2-regularised,
DCN.py:198-199), `Deep-Network/mlp{i}/...`, `DCN-out/out_layer/...`.  No first-order term, no bias
variable.  Flag: `--cross_layers` (default 3, DCN.py:52).
"""
from __future__ import annotations

import torch

from . import ops
from .base import CTRModel, floats, ints
from .engine import DenseVars
from .mlp import MLP


class DCN(CTRModel):
    table_name = "emb"       # DCN.py:122
    linear_name = None
    bias_name = None

    def __init__(self, field_size: int, feature_size: int, embedding_size: int, batch_size: int,
                 deep_layers="256,128,64", cross_layers: int = 3, dropout="0.5,0.5,0.5", l2_reg: float = 1e-4,
                 learning_rate: float = 5e-4, optimizer: str = "Adam", update_mode: str = "exact",
                 device="cuda", seed: int = 0, world: int = 1, epoch_steps: int = 8, batch_norm: bool = False,
                 batch_norm_decay: float = 0.9):
        self.layers, self.keep, self.L = ints(deep_layers), floats(dropout), int(cross_layers)
        self.batch_norm, self.bn_decay = bool(batch_norm), float(batch_norm_decay)
        super().__init__(field_size, feature_size, embedding_size, batch_size, l2_reg, learning_rate, optimizer,
                         update_mode, device, seed, world, epoch_steps)
        self.emb = self.V

    def _build(self):
        B, F, K, L, dev = self.B, self.F, self.K, self.L, self.device
        D = F * K
        self.D = D
        f32 = dict(dtype=torch.float32, device=dev)
        # out_layer input = [x_L (D), x_deep (last hidden)]  (DCN.py:178-181)
        self.mlp = MLP(D, self.layers, self.keep, B, dev, scope="Deep-Network", out_scope="DCN-out/out_layer",
                       out_extra_in=D, seed=self.seed, batch_norm=self.batch_norm, bn_decay=self.bn_decay)
        specs = [("cross_b", (L, D)), ("cross_w", (L, D))] + self.mlp.specs()
        self.dense = DenseVars(specs, self.opt, dev, l2_names=("cross_b", "cross_w"))
        gen = torch.Generator().manual_seed(self.seed)
        self.mlp.init(self.dense, gen)
        std = (2.0 / (L + D)) ** 0.5                     # glorot_normal on [L, D] (DCN.py:118-121)
        for nm in ("cross_b", "cross_w"):
            self.dense[nm].copy_((torch.randn(L, D, generator=gen, dtype=torch.float64).clamp_(-2, 2) * std).float())
        self.x0 = torch.empty(B, D, **f32)
        self.xL = torch.empty(B, D, **f32)
        self.s = torch.empty(B, max(L, 1), **f32)
        self.d_h = torch.empty(B, self.mlp.last_dim, **f32)
        self.dx = torch.empty(B, D, **f32)
        self.cross_ws = torch.empty(max(ops.cross_bwd_workspace_bytes(B, D, max(L, 1)), 16), dtype=torch.uint8, device=dev)
        self.reg_dense = torch.zeros(2, **f32)
        self.l2_ws = torch.empty(1024, **f32)

    def _forward(self, ids, vals, train: bool, masks=None):
        B = ids.shape[0]
        ops.fm_embed_fwd(ids, vals, self.V.var, None, ops.FM_PLAIN, x=self.x0[:B], oob=self.oob)     # DCN.py:134-138
        if self.L > 0:
            ops.cross_fwd(self.x0[:B], self.dense["cross_w"], self.dense["cross_b"], self.xL[:B], self.s[:B])  # :140-145
            xl = self.xL[:B]
        else:
            xl = self.x0[:B]
        self._a = self.mlp.forward_hidden(self.x0[:B], self.dense, train, masks, step_dev=self.opt.state[3:4])  # :147-176
        y = self.mlp.forward_out(self._a, self.dense, extra=xl)                                       # :178-184
        return None, y, None, None

    def _backward(self, ids, vals):
        B = ids.shape[0]
        if self.L <= 0:
            raise NotImplementedError("cross_layers == 0 (the reference's flag default is 3)")
        dy = self.dy[:B]
        self.mlp.backward_out(self._a, dy, self.dense, self.d_h[:B], extra=self.xL[:B])  # d x_L -> mlp.d_extra, d x_deep -> d_h
        dX = self.mlp.backward_hidden(self.x0[:B], self.d_h[:B], self.dense)             # d x0 through the deep network
        ops.cross_bwd(self.x0[:B], self.dense["cross_w"], self.dense["cross_b"], self.s[:B], self.mlp.d_extra[:B], dX,
                      self.dx[:B], self.dense.grads["cross_w"], self.dense.grads["cross_b"], self.cross_ws)
        ops.fm_embed_bwd(vals, None, None, self.dx[:B], None, None, self.K, ops.FM_PLAIN, self.g_rows[: B * self.F], None)

    def _dense_reg_terms(self):
        # loss = CE + l2*l2_loss(cross_b) + l2*l2_loss(cross_w) + l2*l2_loss(emb)   (DCN.py:198-199)
        if self.l2_reg == 0.0:
            return self.reg_dense
        ops.l2_loss(self.dense["cross_b"], self.reg_dense[0:1], self.l2_ws, scale=self.l2_reg)
        ops.l2_loss(self.dense["cross_w"], self.reg_dense[1:2], self.l2_ws, scale=self.l2_reg)
        return self.reg_dense
