"""Attentional Factorization Machine: mirror of `model_fn` in deep_ctr/Model_pipeline/AFM.py:99-212.
Variables: `bias`, `linear`, `emb` (AFM.py:111-113); `Attention-part/mlp0/{weights [K,A],biases}`,
`Attention-part/attention_out/{weights [A,1],biases}`; `Attention-based-Pooling/deep_out/{weights [K,1],biases}`.
y = bias + y_linear + FC(dropout(sum_{i<j} dropout(softmax(att_ij)) * (e_i*e_j)))   (AFM.py:127-167);
dropout[0] acts on the softmax weights, dropout[1] on the pooled vector."""
from __future__ import annotations

import torch

from . import ops
from .base import CTRModel, floats, ints
from .engine import DenseVars

ATT, POOL = "Attention-part", "Attention-based-Pooling"


class AFM(CTRModel):
    table_name, linear_name, bias_name = "emb", "linear", "bias"

    def __init__(self, field_size, feature_size, embedding_size, batch_size, attention_layers="256", dropout="1.0,0.5",
                 l2_reg=1.0, learning_rate=0.1, optimizer="Adam", update_mode="exact", device="cuda", seed=0,
                 world=1, epoch_steps=8):
        self.att_layers, self.keep = ints(attention_layers), floats(dropout)
        if len(self.att_layers) != 1:
            raise NotImplementedError("one attention layer (the reference default '256')")
        try:
            ops.afm_pool_check(field_size * (field_size - 1) // 2, embedding_size)
        except ops.CtrError as e:
            raise ValueError(f"--field_size={field_size} gives more field pairs than the attention pooling kernels "
                             f"take: {e}") from None
        super().__init__(field_size, feature_size, embedding_size, batch_size, l2_reg, learning_rate, optimizer,
                         update_mode, device, seed, world, epoch_steps)

    def _build(self):
        B, F, K, dev = self.B, self.F, self.K, self.device
        A = self.att_layers[0]
        P = F * (F - 1) // 2
        self.P, self.A = P, A
        f32 = dict(dtype=torch.float32, device=dev)
        specs = [("bias", (1,)), (f"{ATT}/mlp0/weights", (K, A)), (f"{ATT}/mlp0/biases", (A,)),
                 (f"{ATT}/attention_out/weights", (A, 1)), (f"{ATT}/attention_out/biases", (1,)),
                 (f"{POOL}/deep_out/weights", (K, 1)), (f"{POOL}/deep_out/biases", (1,))]
        self.dense = DenseVars(specs, self.opt, dev)
        gen = torch.Generator().manual_seed(self.seed)
        for nm, shape in specs:
            if nm.endswith("weights"):
                lim = (6.0 / (shape[0] + shape[1])) ** 0.5
                self.dense[nm].copy_(((torch.rand(shape, generator=gen, dtype=torch.float64) * 2 - 1) * lim).float())
        self.x = torch.empty(B, F * K, **f32)
        self.y_w = torch.empty(B, **f32)
        self.pw = torch.empty(B * P, K, **f32)
        self.Hh = torch.empty(B * P, A, **f32)
        self.logit = torch.empty(B * P, **f32)
        self.att = torch.empty(B * P, **f32)
        self.y_emb = torch.empty(B, K, **f32)
        self.y_emb_d = torch.empty(B, K, **f32)
        self.y_deep = torch.empty(B, **f32)
        self.mask0 = torch.empty(B * P, **f32)
        self.mask1 = torch.empty(B, K, **f32)
        self.d_emb = torch.empty(B, K, **f32)
        self.d_emb2 = torch.empty(B, K, **f32)
        self.dpw = torch.empty(B * P, K, **f32)
        self.dlogit = torch.empty(B * P, **f32)
        self.dHh = torch.empty(B * P, A, **f32)
        self.dX = torch.empty(B, F * K, **f32)
        self.ws = torch.empty(max(ops.fc_bwd_workspace_bytes(B * P, K, A), ops.fc1_bwd_workspace_bytes(B * P, A, 0),
                                  ops.fc1_bwd_workspace_bytes(B, K, 0), 16), dtype=torch.uint8, device=dev)

    def _forward(self, ids, vals, train, masks=None):
        B, F, K, P = ids.shape[0], self.F, self.K, self.P
        d = self.dense
        ops.fm_embed_fwd(ids, vals, self.V.var, self.W.var, ops.FM_PLAIN, x=self.x[:B], y_w=self.y_w[:B], oob=self.oob)
        ops.afm_pairs_fwd(self.x[:B], B, F, K, self.pw[: B * P])                              # AFM.py:132-138
        ops.fc_fwd(self.pw[: B * P], d[f"{ATT}/mlp0/weights"], d[f"{ATT}/mlp0/biases"], None, 1.0, 1, self.Hh[: B * P])
        ops.fc1_fwd(self.Hh[: B * P], None, d[f"{ATT}/attention_out/weights"].view(-1), d[f"{ATT}/attention_out/biases"],
                    self.logit[: B * P])                                                      # :142-148
        self._m0 = self._m1 = None
        if train:
            if masks is not None and masks.get("att") is not None:
                self._m0 = masks["att"]
            elif self.keep[0] < 1.0:
                self._m0 = self.mask0[: B * P]
                ops.dropout_mask(self._m0, self.keep[0], self.seed * 131 + 5, self.opt.state[3:4])
            if masks is not None and masks.get("pool") is not None:
                self._m1 = masks["pool"]
            elif self.keep[1] < 1.0:
                self._m1 = self.mask1[:B]
                ops.dropout_mask(self._m1, self.keep[1], self.seed * 131 + 6, self.opt.state[3:4])
        ops.afm_pool_fwd(self.pw[: B * P], self.logit[: B * P], self._m0, self.keep[0], B, P, K, self.att[: B * P],
                         self.y_emb[:B])                                                      # :151-156
        e = self.y_emb[:B]
        if self._m1 is not None:                                                              # :157-158
            ops.dropout_apply(e, self._m1, self.keep[1], self.y_emb_d[:B])
            e = self.y_emb_d[:B]
        self._e = e
        ops.fc1_fwd(e, None, d[f"{POOL}/deep_out/weights"].view(-1), d[f"{POOL}/deep_out/biases"], self.y_deep[:B])
        return d["bias"], self.y_w[:B], self.y_deep[:B], None                                 # :164-167

    def _backward(self, ids, vals):
        B, F, K, P = ids.shape[0], self.F, self.K, self.P
        d, g = self.dense, self.dense.grads
        dy = self.dy[:B]
        ops.fc1_bwd(self._e, None, d[f"{POOL}/deep_out/weights"].view(-1), dy, self.d_emb[:B], None,
                    g[f"{POOL}/deep_out/weights"].view(-1), g[f"{POOL}/deep_out/biases"], self.ws)
        de = self.d_emb[:B]
        if self._m1 is not None:
            ops.dropout_apply(de, self._m1, self.keep[1], self.d_emb2[:B])
            de = self.d_emb2[:B]
        ops.afm_pool_bwd(self.pw[: B * P], self.att[: B * P], self._m0, self.keep[0], de, B, P, K, self.dpw[: B * P],
                         self.dlogit[: B * P])
        ops.fc1_bwd(self.Hh[: B * P], None, d[f"{ATT}/attention_out/weights"].view(-1), self.dlogit[: B * P],
                    self.dHh[: B * P], None, g[f"{ATT}/attention_out/weights"].view(-1), g[f"{ATT}/attention_out/biases"],
                    self.ws)
        ops.fc_bwd(self.pw[: B * P], d[f"{ATT}/mlp0/weights"], self.Hh[: B * P], None, 1.0, self.dHh[: B * P], 1,
                   self.dpw[: B * P], g[f"{ATT}/mlp0/weights"], g[f"{ATT}/mlp0/biases"], self.ws, accumulate_din=True)
        ops.afm_pairs_bwd(self.x[:B], self.dpw[: B * P], B, F, K, self.dX[:B])
        ops.fm_embed_bwd(vals, None, None, self.dX[:B], None, dy, K, ops.FM_PLAIN, self.g_rows[: B * F], self.g_w[: B * F])
