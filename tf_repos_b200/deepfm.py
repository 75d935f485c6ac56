"""DeepFM on the H100 engine: host-side mirror of `model_fn` in deep_ctr/Model_pipeline/DeepFM.py:100-221.

Same parameters (`field_size, feature_size, embedding_size, l2_reg, learning_rate, deep_layers,
dropout`, DeepFM.py:329-338), same variable names (`fm_bias, fm_w, fm_v, Deep-part/mlp{i}/...`),
same modes (TRAIN / EVAL / PREDICT).  Everything numerical runs in hand-written sm_90a kernels
through the C ABI; see tf_repos_b200/engine.py (SparseUpdater) for the update modes and
tf_repos_b200/base.py for data parallelism.
"""
from __future__ import annotations

import torch

from . import ops
from .base import CTRModel, floats, ints
from .engine import DenseVars
from .mlp import MLP


class DeepFM(CTRModel):
    table_name = "fm_v"      # DeepFM.py:116
    linear_name = "fm_w"     # DeepFM.py:115
    bias_name = "fm_bias"    # DeepFM.py:114

    def __init__(self, field_size: int, feature_size: int, embedding_size: int, batch_size: int,
                 deep_layers="256,128,64", dropout="0.5,0.5,0.5", l2_reg: float = 1e-4,
                 learning_rate: float = 5e-4, optimizer: str = "Adam", update_mode: str = "exact",
                 device="cuda", seed: int = 0, world: int = 1, epoch_steps: int = 8, batch_norm: bool = False,
                 batch_norm_decay: float = 0.9):
        self.layers, self.keep = ints(deep_layers), floats(dropout)
        self.batch_norm, self.bn_decay = bool(batch_norm), float(batch_norm_decay)
        super().__init__(field_size, feature_size, embedding_size, batch_size, l2_reg, learning_rate, optimizer,
                         update_mode, device, seed, world, epoch_steps)
        self.fm_v, self.fm_w = self.V, self.W

    def _build(self):
        B, F, K, dev = self.B, self.F, self.K, self.device
        f32 = dict(dtype=torch.float32, device=dev)
        self.mlp = MLP(F * K, self.layers, self.keep, B, dev, seed=self.seed, batch_norm=self.batch_norm,
                       bn_decay=self.bn_decay)
        self.dense = DenseVars([("fm_bias", (1,))] + self.mlp.specs(), self.opt, dev)
        self.mlp.init(self.dense, torch.Generator().manual_seed(self.seed))
        self.x = torch.empty(B, F * K, **f32)      # scaled embeddings = deep_inputs (DeepFM.py:151)
        self.S = torch.empty(B, K, **f32)          # sum_f e, saved for the backward
        self.y_w = torch.empty(B, **f32)
        self.y_v = torch.empty(B, **f32)
        self.d_last = torch.empty(B, self.mlp.out_in, **f32)

    def _forward(self, ids, vals, train: bool, masks=None):
        B = ids.shape[0]
        ops.fm_embed_fwd(ids, vals, self.V.var, self.W.var, ops.FM_DEEPFM, x=self.x[:B], y_w=self.y_w[:B],
                         y2=self.y_v[:B], S=self.S[:B], oob=self.oob)                       # :125-135,151
        self._a = self.mlp.forward_hidden(self.x[:B], self.dense, train, masks, step_dev=self.opt.state[3:4])
        y_d = self.mlp.forward_out(self._a, self.dense)                                     # :152-167
        return self.dense["fm_bias"], self.y_w[:B], self.y_v[:B], y_d                       # :172-175

    def _backward(self, ids, vals):
        B = ids.shape[0]
        dy = self.dy[:B]
        self.mlp.backward_out(self._a, dy, self.dense, self.d_last[:B])
        dX = self.mlp.backward_hidden(self.x[:B], self.d_last[:B], self.dense)
        ops.fm_embed_bwd(vals, self.x[:B], self.S[:B], dX, dy, dy, self.K, ops.FM_DEEPFM,
                         self.g_rows[: B * self.F], self.g_w[: B * self.F])
