"""FNN / Inner-PNN / Outer-PNN: mirror of `model_fn` in deep_ctr/Model_pipeline/PNN.py:102-238.
`--model_type {FNN, Inner, Outer}` (PNN.py:61).  Variables: `bias`, `linear`, `emb` (PNN.py:116-118),
`Deep-part/mlp{i}`, `Deep-part/deep_out`.  y = bias + y_linear + MLP(z), z = x | [x, inner] | [x, outer]."""
from __future__ import annotations

import torch

from . import ops
from .base import CTRModel, floats, ints
from .engine import DenseVars
from .mlp import MLP


class PNN(CTRModel):
    table_name, linear_name, bias_name = "emb", "linear", "bias"

    def __init__(self, field_size, feature_size, embedding_size, batch_size, model_type="Inner",
                 deep_layers="256,128,64", dropout="0.5,0.5,0.5", l2_reg=1e-4, learning_rate=5e-4, optimizer="Adam",
                 update_mode="exact", device="cuda", seed=0, world=1, epoch_steps=8, batch_norm=False, batch_norm_decay=0.9):
        if model_type not in ("FNN", "Inner", "Outer"):
            raise NameError(f"model_type {model_type!r}: deep_inputs is undefined (PNN.py:139-167)")
        self.model_type = model_type
        if model_type != "FNN":
            try:
                ops.pnn_product_check(field_size, embedding_size, model_type == "Outer")
            except ops.CtrError as e:
                raise ValueError(f"--embedding_size={embedding_size} with --field_size={field_size} is not supported "
                                 f"by the {model_type} product kernels: {e}") from None
        self.layers, self.keep = ints(deep_layers), floats(dropout)
        self.batch_norm, self.bn_decay = bool(batch_norm), float(batch_norm_decay)
        super().__init__(field_size, feature_size, embedding_size, batch_size, l2_reg, learning_rate, optimizer,
                         update_mode, device, seed, world, epoch_steps)

    def _build(self):
        B, F, K, dev = self.B, self.F, self.K, self.device
        f32 = dict(dtype=torch.float32, device=dev)
        P = F * (F - 1) // 2                       # py2 integer division (quirk Q8, PNN.py:113)
        self.Dz = F * K + {"FNN": 0, "Inner": P, "Outer": P * K * K}[self.model_type]
        self.mlp = MLP(self.Dz, self.layers, self.keep, B, dev, seed=self.seed, batch_norm=self.batch_norm,
                       bn_decay=self.bn_decay)
        self.dense = DenseVars([("bias", (1,))] + self.mlp.specs(), self.opt, dev)
        self.mlp.init(self.dense, torch.Generator().manual_seed(self.seed))
        self.x = torch.empty(B, F * K, **f32)
        self.y_w = torch.empty(B, **f32)
        self.z = torch.empty(B, self.Dz, **f32) if self.model_type != "FNN" else None
        self.dX = torch.empty(B, F * K, **f32)
        self.d_last = torch.empty(B, self.mlp.out_in, **f32)

    def _forward(self, ids, vals, train, masks=None):
        B = ids.shape[0]
        ops.fm_embed_fwd(ids, vals, self.V.var, self.W.var, ops.FM_PLAIN, x=self.x[:B], y_w=self.y_w[:B], oob=self.oob)
        z = self.x[:B]
        if self.model_type != "FNN":                                                         # PNN.py:141-167
            z = self.z[:B]
            ops.pnn_product_fwd(self.x[:B], B, self.F, self.K, self.model_type == "Outer", z)
        self._z = z
        mm = masks.get("mlp") if masks else None
        self._a = self.mlp.forward_hidden(z, self.dense, train, mm, step_dev=self.opt.state[3:4])
        y_d = self.mlp.forward_out(self._a, self.dense)
        return self.dense["bias"], self.y_w[:B], y_d, None                                   # PNN.py:190-193

    def _backward(self, ids, vals):
        B = ids.shape[0]
        dy = self.dy[:B]
        self.mlp.backward_out(self._a, dy, self.dense, self.d_last[:B])
        dz = self.mlp.backward_hidden(self._z, self.d_last[:B], self.dense)
        dX = dz
        if self.model_type != "FNN":
            ops.pnn_product_bwd(self.x[:B], dz, B, self.F, self.K, self.model_type == "Outer", self.dX[:B])
            dX = self.dX[:B]
        ops.fm_embed_bwd(vals, None, None, dX, None, dy, self.K, ops.FM_PLAIN, self.g_rows[: B * self.F],
                         self.g_w[: B * self.F])
