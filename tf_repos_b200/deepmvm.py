"""Deep & Multi-view Machines on the H100 engine: mirror of `model_fn` in deep_ctr/Model_pipeline/DeepMVM.py:100-230.

Variables (TF names): `mvm_w [N,K]` (the table), `mvm_b [F,K]` (a dense per-field bias; both L2-regularised,
DeepMVM.py:197-199), `Deep-part/mlp{i}/...`, `DeepMVM-out/deep_out/...`.  No first-order table, no bias variable.
x_mvm = prod_f (e_f + mvm_b_f) over the fields (csrc/mvm.cu); the deep part reads the scaled embeddings without
mvm_b; the head is FC([x_mvm, x_deep]) -> 1.  No model-specific flag.
"""
from __future__ import annotations

import torch

from . import ops
from .base import CTRModel, floats, ints
from .engine import DenseVars
from .mlp import MLP


class DeepMVM(CTRModel):
    table_name = "mvm_w"      # DeepMVM.py:117
    linear_name = None
    bias_name = None
    table_reg_first = True    # loss = CE + l2*l2_loss(mvm_w) + l2*l2_loss(mvm_b)   (DeepMVM.py:197-199)

    def __init__(self, field_size: int, feature_size: int, embedding_size: int, batch_size: int,
                 deep_layers="256,128,64", dropout="0.5,0.5,0.5", l2_reg: float = 1e-4, learning_rate: float = 5e-4,
                 optimizer: str = "Adam", update_mode: str = "exact", device="cuda", seed: int = 0, world: int = 1,
                 epoch_steps: int = 8, batch_norm: bool = False, batch_norm_decay: float = 0.9):
        self.layers, self.keep = ints(deep_layers), floats(dropout)
        self.batch_norm, self.bn_decay = bool(batch_norm), float(batch_norm_decay)
        super().__init__(field_size, feature_size, embedding_size, batch_size, l2_reg, learning_rate, optimizer,
                         update_mode, device, seed, world, epoch_steps)
        self.mvm_w = self.V

    def _build(self):
        B, F, K, dev = self.B, self.F, self.K, self.device
        D = F * K
        f32 = dict(dtype=torch.float32, device=dev)
        # deep_out input = [x_mvm (K), x_deep (last hidden)]  (DeepMVM.py:181-183)
        self.mlp = MLP(D, self.layers, self.keep, B, dev, scope="Deep-part", out_scope="DeepMVM-out/deep_out",
                       out_extra_in=K, seed=self.seed, batch_norm=self.batch_norm, bn_decay=self.bn_decay)
        self.dense = DenseVars([("mvm_b", (F, K))] + self.mlp.specs(), self.opt, dev, l2_names=("mvm_b",))
        gen = torch.Generator().manual_seed(self.seed)
        self.mlp.init(self.dense, gen)
        std = (2.0 / (F + K)) ** 0.5                     # glorot_normal on [F, K] (DeepMVM.py:118)
        self.dense["mvm_b"].copy_((torch.randn(F, K, generator=gen, dtype=torch.float64).clamp_(-2, 2) * std).float())
        self.x = torch.empty(B, D, **f32)
        self.x_mvm = torch.empty(B, K, **f32)
        self.d_h = torch.empty(B, self.mlp.last_dim, **f32)
        self.dx = torch.empty(B, D, **f32)
        self.mvm_ws = torch.empty(max(ops.mvm_bwd_workspace_bytes(B, F, K), 16), dtype=torch.uint8, device=dev)
        self.reg_dense = torch.zeros(1, **f32)
        self.l2_ws = torch.empty(1024, **f32)

    def _forward(self, ids, vals, train: bool, masks=None):
        B = ids.shape[0]
        ops.fm_embed_fwd(ids, vals, self.V.var, None, ops.FM_PLAIN, x=self.x[:B], oob=self.oob)      # DeepMVM.py:139-142
        ops.mvm_fwd(self.x[:B], self.dense["mvm_b"], self.x_mvm[:B])                                 # :144-150
        self._a = self.mlp.forward_hidden(self.x[:B], self.dense, train, masks, step_dev=self.opt.state[3:4])  # :152-178
        y = self.mlp.forward_out(self._a, self.dense, extra=self.x_mvm[:B])                          # :180-184
        return None, y, None, None

    def _backward(self, ids, vals):
        B = ids.shape[0]
        dy = self.dy[:B]
        self.mlp.backward_out(self._a, dy, self.dense, self.d_h[:B], extra=self.x_mvm[:B])  # d x_mvm -> mlp.d_extra
        dX = self.mlp.backward_hidden(self.x[:B], self.d_h[:B], self.dense)                # d e through the deep part
        ops.mvm_bwd(self.x[:B], self.dense["mvm_b"], self.mlp.d_extra[:B], dX, self.dx[:B],
                    self.dense.grads["mvm_b"], self.mvm_ws)
        ops.fm_embed_bwd(vals, None, None, self.dx[:B], None, None, self.K, ops.FM_PLAIN, self.g_rows[: B * self.F], None)

    def _dense_reg_terms(self):
        if self.l2_reg == 0.0:
            return self.reg_dense
        ops.l2_loss(self.dense["mvm_b"], self.reg_dense[0:1], self.l2_ws, scale=self.l2_reg)
        return self.reg_dense
