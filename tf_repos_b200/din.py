"""Deep Interest Network on the H100 engine: mirror of `model_fn` in deep_ctr/Model_pipeline/DIN.py:101-257.

Inputs (the TFRecord features of DIN.py:60-77, already densified the way the reference does with
sparse_tensor_to_dense, DIN.py:153-154):
    feat_ids [B,F'] int32                       common fields (no values: DIN.py:143)
    a_ids    [3,B]  int32                       a_catids, a_shopids, a_brandids
    a_int_ids [nnz] int32 + a_int_off [B+1]     a_intids bags (CSR)
    u_ids [4,B,P] int32, u_wgt [4,B,P] f32      u_cat/u_shop/u_brand/u_int ids & vals, 0-padded
                                                (id 0 is the padding sentinel: mask = id > 0, DIN.py:157)
Variables (TF names): `embeddings [N,K]`; `Field-wise-Pooling-layer/att_fc0/{weights [3K,H],biases}`,
`Field-wise-Pooling-layer/att_out/{weights [H,1],biases}` shared by the 4 attention units
(reuse=tf.AUTO_REUSE, DIN.py:150); `MLP-layer/mlp{i}/...`; `DIN-out/din_out/...`.  Quirk Q5 is
reproduced: the attention hidden width is deep_layers[0], not attention_layers[0] (DIN.py:163-164).
Only the table is L2-regularised (DIN.py:226).

The attention layer uses  [e, e-a, a] @ [W1;W2;W3] = e @ (W1+W2) + a @ (W3-W2)  (see csrc/din.cu).
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import ops
from .base import floats, ints
from .engine import DenseVars, OptimizerState, SparseUpdater, Table
from .mlp import MLP

FIELDS = ("cat", "shop", "brand", "int")
ATT = "Field-wise-Pooling-layer"


class DIN:
    def __init__(self, field_size: int, feature_size: int, embedding_size: int, batch_size: int, max_len: int,
                 max_a_int: int = 8, deep_layers="256,128,64", dropout="0.5,0.5,0.5", attention_layers="256",
                 attention_pooling: bool = True, l2_reg: float = 1e-4, learning_rate: float = 5e-4,
                 optimizer: str = "Adam", update_mode: str = "exact", device="cuda", seed: int = 0,
                 epoch_steps: int = 8, batch_norm: bool = False, batch_norm_decay: float = 0.9):
        assert update_mode in ("exact", "exact_deferred", "lazy")
        if batch_norm and attention_pooling:
            # DIN.py:166 calls batch_norm_layer(train_phase=train_phase) inside attention_unit, where train_phase is
            # not defined (it is assigned later, DIN.py:189-193): the reference raises NameError (quirk Q5)
            raise NameError("name 'train_phase' is not defined (DIN.py:166: --batch_norm with --attention_pooling)")
        if len(ints(attention_layers)) != 1:
            raise NotImplementedError("one attention hidden layer (the reference default '256')")
        self.Fp, self.N, self.K, self.B, self.P = field_size, feature_size, embedding_size, batch_size, max_len
        self.layers, self.keep = ints(deep_layers), floats(dropout)
        self.H = self.layers[0]                     # quirk Q5: width = deep_layers[0]
        self.attention_pooling = attention_pooling
        self.l2_reg, self.update_mode = float(l2_reg), update_mode
        self.device = dev = torch.device(device)
        self.seed = seed
        B, Fp, K, P, H = self.B, self.Fp, self.K, self.P, self.H
        self.opt = OptimizerState(optimizer, learning_rate, l2_reg, dev)
        self.V = Table("embeddings", self.N, K, self.opt, dev, seed=seed * 2 + 1)        # DIN.py:115
        self.tables = [self.V]
        self.Dx = Fp * K + 8 * K                                                          # DIN.py:199
        self.off_u = Fp * K
        self.off_a = Fp * K + 4 * K
        self.mlp = MLP(self.Dx, self.layers, self.keep, B, dev, scope="MLP-layer", out_scope="DIN-out/din_out",
                       seed=seed, batch_norm=batch_norm, bn_decay=batch_norm_decay)
        specs = self.mlp.specs()
        if attention_pooling:
            specs = [(f"{ATT}/att_fc0/weights", (3 * K, H)), (f"{ATT}/att_fc0/biases", (H,)),
                     (f"{ATT}/att_out/weights", (H, 1)), (f"{ATT}/att_out/biases", (1,))] + specs
        self.dense = DenseVars(specs, self.opt, dev)
        gen = torch.Generator().manual_seed(seed)
        self.mlp.init(self.dense, gen)
        if attention_pooling:
            for nm, shape in ((f"{ATT}/att_fc0/weights", (3 * K, H)), (f"{ATT}/att_out/weights", (H, 1))):
                lim = (6.0 / (shape[0] + shape[1])) ** 0.5
                self.dense[nm].copy_(((torch.rand(shape, generator=gen, dtype=torch.float64) * 2 - 1) * lim).float())
        f32 = dict(dtype=torch.float32, device=dev)
        self.x = torch.empty(B, self.Dx, **f32)
        self.y = torch.empty(B, **f32)
        self.pred = torch.empty(B, **f32)
        self.dy = torch.empty(B, **f32)
        self.d_last = torch.empty(B, self.mlp.out_in, **f32)
        self.loss_ce = self.dense.tail[0:1]
        self.oob = torch.zeros(2, dtype=torch.int32, device=dev)
        self.max_a_int = max_a_int
        # per-occurrence gradient rows: [common | a_cat a_shop a_brand | a_int (padded) | u_0..u_3]
        self.seg = {"common": (0, B * Fp)}
        o = B * Fp
        for j in range(3):
            self.seg[f"a{j}"] = (o, B); o += B
        self.seg["a_int"] = (o, B * max_a_int); o += B * max_a_int
        for f in range(4):
            self.seg[f"u{f}"] = (o, B * P); o += B * P
        self.n_total = o
        self.ids_all = torch.zeros(o, dtype=torch.int32, device=dev)
        self.g_all = torch.zeros(o, K, **f32)
        self.updater = SparseUpdater(o, self.N, K, self.opt, dev, with_scalar_table=False)
        if attention_pooling:
            self.E = [torch.empty(B * P, K, **f32) for _ in range(4)]
            self.Hh = [torch.empty(B * P, H, **f32) for _ in range(4)]
            self.att = [torch.empty(B * P, **f32) for _ in range(4)]
            self.z = torch.empty(B * P, **f32)
            self.a_c = [torch.empty(B, K, **f32) for _ in range(4)]
            self.U = torch.empty(B, H, **f32)
            self.att_mask = [torch.empty(B * P, H, **f32) if self.keep[0] < 1.0 else None for _ in range(4)]
            self._att_active = [None] * 4
            self.Wc = torch.empty(K, H, **f32)
            self.Wd = torch.empty(K, H, **f32)
            self.dE = torch.empty(B * P, K, **f32)
            self.dz = torch.empty(B * P, **f32)
            self.dHh = torch.empty(B * P, H, **f32)
            self.dU = torch.empty(B, H, **f32)
            self.gw2_part = torch.empty(B, H, **f32)
            self.dz_b = torch.empty(P, **f32)
            self.da = [torch.empty(B, K, **f32) for _ in range(4)]
            self.gWc = torch.zeros(4, K, H, **f32)
            self.gWd = torch.zeros(4, K, H, **f32)
            self.gb1 = torch.zeros(4, H, **f32)
            self.gw2 = torch.zeros(4, H, **f32)
            self.gb2 = torch.zeros(4, 1, **f32)
            self.scratch_b = torch.zeros(H, **f32)
            self.att_ws = torch.empty(max(ops.fc_bwd_workspace_bytes(B * P, K, H), ops.fc_bwd_workspace_bytes(B, K, H),
                                          ops.fc1_bwd_workspace_bytes(B * P, H, 0), 16), dtype=torch.uint8, device=dev)
        self.d_aint = torch.empty(B, K, **f32)
        self.global_step = 0
        self.epoch_steps, self.epoch_pos = epoch_steps, 0
        if update_mode == "exact_deferred":
            if self.l2_reg == 0.0 and optimizer != "Adam":
                self.update_mode = "exact"
            else:
                self.updater.enable_epochs(epoch_steps, self.tables)

    # ---- plumbing -------------------------------------------------------------------------------------
    def flush(self):
        if self.update_mode == "exact_deferred" and self.epoch_pos > self.updater.flush_pos:
            self.updater.epoch_sweep(self.tables, self.epoch_pos, reset=False, l2_reg=self.l2_reg)

    def variables(self) -> Dict[str, torch.Tensor]:
        self.flush()
        out = {"embeddings": self.V.var}
        out.update(self.dense.views)
        out.update(self.mlp.bn_state)
        return out

    def load_variables(self, values: Dict[str, torch.Tensor]):
        vs = self.variables()
        for name, v in values.items():
            vs[name].copy_(v.to(self.device, torch.float32).reshape(vs[name].shape))

    def check_ids(self):
        cnt, first = self.oob.tolist()
        if cnt:
            self.oob.zero_()
            raise IndexError(f"{cnt} feature ids outside [0, {self.N}) (first: {first})")

    def _stage_ids(self, batch):
        """ids of every embedding_lookup of the step, in gradient-segment order."""
        B, P = self.B, self.P
        s = self.seg
        self.ids_all[s["common"][0]: s["common"][0] + s["common"][1]].copy_(batch["feat_ids"].reshape(-1))
        for j in range(3):
            self.ids_all[s[f"a{j}"][0]: s[f"a{j}"][0] + B].copy_(batch["a_ids"][j])
        o, n = s["a_int"]
        nnz = batch["a_int_ids"].numel()
        assert nnz <= n, "a_int bag longer than max_a_int"
        self.ids_all[o: o + n].zero_()
        self.ids_all[o: o + nnz].copy_(batch["a_int_ids"])
        for f in range(4):
            self.ids_all[s[f"u{f}"][0]: s[f"u{f}"][0] + B * P].copy_(batch["u_ids"][f].reshape(-1))

    # ---- f(x) -------------------------------------------------------------------------------------------
    def _forward(self, batch, train: bool, masks=None):
        B, Fp, K, P, H, Dx = self.B, self.Fp, self.K, self.P, self.H, self.Dx
        V, x = self.V.var, self.x
        ops.gather_scale_rows(batch["feat_ids"].reshape(-1), None, V, x, Fp, Dx, self.oob)                 # :143
        for j in range(3):                                                                                   # :145-147
            ops.gather_scale_rows(batch["a_ids"][j], None, V, x[:, self.off_a + j * K:], 1, Dx, self.oob)
        ops.bag_sum_fwd(batch["a_int_ids"], None, batch["a_int_off"], V, x[:, self.off_a + 3 * K:], Dx)     # :148
        if self.attention_pooling:
            W = self.dense[f"{ATT}/att_fc0/weights"]
            b1 = self.dense[f"{ATT}/att_fc0/biases"]
            w2 = self.dense[f"{ATT}/att_out/weights"].view(-1)
            b2 = self.dense[f"{ATT}/att_out/biases"]
            ops.axpby(W[:K], 1.0, W[K:2 * K], 1.0, self.Wc)          # Wc = W1 + W2
            ops.axpby(W[2 * K:], 1.0, W[K:2 * K], -1.0, self.Wd)     # Wd = W3 - W2
            for f in range(4):
                ids_f = batch["u_ids"][f].reshape(-1)
                ops.gather_scale_rows(ids_f, batch["u_wgt"][f].reshape(-1), V, self.E[f], 1, K, self.oob)   # :155-156
                ops.scale_rows(x[:, self.off_a + f * K:], None, None, B, K, 1, Dx, self.a_c[f])             # a_xx_emb
                ops.fc_fwd(self.a_c[f], self.Wd, b1, None, 1.0, 0, self.U)                                   # a@(W3-W2)+b
                m = None
                if train and masks is not None and masks.get("att") is not None:
                    m = masks["att"][f]
                elif train and self.keep[0] < 1.0:
                    m = self.att_mask[f]
                    ops.dropout_mask(m, self.keep[0], self.seed * 977 + 11 + f, self.opt.state[3:4])
                self._att_active[f] = m
                ops.fc_fwd_grouped(self.E[f], self.Wc, None, self.U, P, m, self.keep[0], 1, self.Hh[f])     # :164-168
                ops.fc1_fwd(self.Hh[f], None, w2, b2, self.z)                                                # :169 (pre-sigmoid)
                ops.din_pool_fwd(self.E[f], self.z, ids_f, B, P, K, self.att[f], x[:, self.off_u + f * K:], Dx)  # :169-172
        else:
            for f in range(4):   # embedding_lookup_sparse(sp_weights, combiner="sum")  (DIN.py:180-183)
                ops.bag_sum_fwd(batch["u_ids"][f].reshape(-1), batch["u_wgt"][f].reshape(-1), self._pad_offsets(),
                                V, x[:, self.off_u + f * K:], Dx)
        mm = masks.get("mlp") if masks else None
        self._a = self.mlp.forward_hidden(x, self.dense, train, mm, step_dev=self.opt.state[3:4])            # :199-208
        return self.mlp.forward_out(self._a, self.dense)                                                    # :211-214

    def _pad_offsets(self):
        if not hasattr(self, "_poff"):
            self._poff = (torch.arange(self.B + 1, device=self.device, dtype=torch.int32) * self.P).contiguous()
        return self._poff

    def predict(self, batch) -> torch.Tensor:
        self.flush()
        y_d = self._forward(batch, train=False)
        ops.logit_loss(None, y_d, None, None, None, self.B, y=self.y, pred=self.pred)
        return self.pred

    def _backward(self, batch):
        B, Fp, K, P, H, Dx = self.B, self.Fp, self.K, self.P, self.H, self.Dx
        s = self.seg
        self.mlp.backward_out(self._a, self.dy, self.dense, self.d_last)
        dx = self.mlp.backward_hidden(self.x, self.d_last, self.dense)          # [B, Dx]
        g = self.g_all
        # common fields
        ops.scale_rows(dx, None, None, B * Fp, K, Fp, Dx, g[s["common"][0]:])
        if self.attention_pooling:
            w2 = self.dense[f"{ATT}/att_out/weights"].view(-1)
            for f in range(4):
                ids_f = batch["u_ids"][f].reshape(-1)
                ops.din_pool_bwd(self.E[f], self.att[f], ids_f, dx[:, self.off_u + f * K:], Dx, B, P, K, self.dE, self.dz)
                # output layer + relu/dropout backward + per-sample sums in ONE pass over Hh (csrc/din.cu din_att_dz_kernel)
                ops.din_att_dz(self.Hh[f], self._att_active[f], self.keep[0], self.dz, w2, B, P, self.dHh, self.dU,
                               self.gw2_part)
                ops.colsum_rows(self.gw2_part, self.gw2[f])                   # d att_out/weights
                ops.colsum_rows(self.dz.view(B, P), self.dz_b)                # d att_out/biases = sum(dz): per-position sums ...
                ops.colsum_rows(self.dz_b.view(P, 1), self.gb2[f])            # ... then over positions (fixed order)
                ops.colsum_rows(self.dU, self.gb1[f])                         # d att_fc0/biases = colsum(dZ) = colsum(dU)
                ops.fc_bwd(self.E[f], self.Wc, None, None, 1.0, self.dHh, 2, self.dE, self.gWc[f], None, self.att_ws,
                           accumulate_din=True)                               # dHh holds dZ: dWc, dE += dZ @ Wc^T
                ops.fc_bwd(self.a_c[f], self.Wd, self.U, None, 1.0, self.dU, 0, self.da[f], self.gWd[f], self.scratch_b,
                           self.att_ws)
                ops.scale_rows(self.dE, None, batch["u_wgt"][f].reshape(-1), B * P, K, 1, K, g[s[f"u{f}"][0]:])
            # shared attention weights: sum the four units' gradients
            gW = self.dense.grads[f"{ATT}/att_fc0/weights"]
            for name, src in ((f"{ATT}/att_fc0/biases", self.gb1), (f"{ATT}/att_out/weights", self.gw2),
                              (f"{ATT}/att_out/biases", self.gb2)):
                dst = self.dense.grads[name].view(-1)
                ops.axpby(src[0].reshape(-1), 1.0, src[1].reshape(-1), 1.0, dst)
                ops.axpby(dst, 1.0, src[2].reshape(-1), 1.0, dst)
                ops.axpby(dst, 1.0, src[3].reshape(-1), 1.0, dst)
            for src in (self.gWc, self.gWd):
                ops.axpby(src[0], 1.0, src[1], 1.0, src[0]); ops.axpby(src[0], 1.0, src[2], 1.0, src[0])
                ops.axpby(src[0], 1.0, src[3], 1.0, src[0])
            ops.axpby(self.gWc[0], 1.0, self.gWd[0], 0.0, gW[:K])               # dW1 = dWc
            ops.axpby(self.gWc[0], 1.0, self.gWd[0], -1.0, gW[K:2 * K])         # dW2 = dWc - dWd
            ops.axpby(self.gWd[0], 1.0, self.gWc[0], 0.0, gW[2 * K:])           # dW3 = dWd
            da = self.da
        else:
            for f in range(4):
                ops.bag_sum_bwd(dx[:, self.off_u + f * K:], Dx, batch["u_wgt"][f].reshape(-1), self._pad_offsets(), K,
                                g[s[f"u{f}"][0]:])
            da = [None] * 4
        # ad-side lookups: gradient from the MLP input slice (+ from the attention unit that used them)
        for j in range(3):
            ops.scale_rows(dx[:, self.off_a + j * K:], da[j], None, B, K, 1, Dx, g[s[f"a{j}"][0]:])
        ops.scale_rows(dx[:, self.off_a + 3 * K:], da[3], None, B, K, 1, Dx, self.d_aint)
        o, n = s["a_int"]
        g[o: o + n].zero_()
        ops.bag_sum_bwd(self.d_aint, K, None, batch["a_int_off"], K, g[o:])

    def train_step(self, batch, labels, masks=None, n_valid: Optional[int] = None) -> torch.Tensor:
        """one optimizer.minimize(loss) (DIN.py:226-247).  Returns {mean CE, l2*l2_loss(embeddings)}.
        n_valid < batch_size: the final partial batch `repeat`-before-`batch` leaves (DIN.py:93-94), padded to the
        configured batch size by the caller.  The loss is the mean over the n_valid real samples and the padded rows'
        dy is exactly 0, so their gradient rows, dZ rows and bias terms are exact zeros: the step equals TensorFlow's
        step on the n_valid-sample batch (a padded id that enters the de-duplicated update with a zero summed gradient
        takes g = 0 + l2*var, which is the untouched-row update it would have taken anyway).  Not with --batch_norm
        (the padded rows would enter the batch moments)."""
        upd = self.updater
        deferred = self.update_mode == "exact_deferred"
        self._stage_ids(batch)
        if deferred:
            j = self.epoch_pos
            if j == 0:
                upd.epoch_begin()
            self.opt.tick_epoch(j)
            upd.unique(self.ids_all)
            upd.epoch_rows([(self.V, None)], j, apply=False)
        else:
            self.opt.tick()
        y_d = self._forward(batch, train=True, masks=masks)
        n = self.B if n_valid is None else int(n_valid)
        assert 0 < n <= self.B
        if n < self.B:
            if self.mlp.batch_norm:
                raise NotImplementedError("a partial final batch with --batch_norm (padded rows would enter the batch moments)")
            self.dy[n:].zero_()
        ops.logit_loss(None, y_d[:n], None, None, labels[:n], n, y=self.y[:n], pred=self.pred[:n], loss_ce=self.loss_ce,
                       dy=self.dy[:n])
        self._backward(batch)
        if deferred:
            upd.segment_sum(self.g_all, None)
            upd.epoch_rows([(self.V, upd.g_uniq)], self.epoch_pos, apply=True)
            self.epoch_pos += 1
            if self.epoch_pos == self.epoch_steps:
                upd.epoch_sweep(self.tables, self.epoch_steps, reset=True, l2_reg=self.l2_reg)
                self.epoch_pos = 0
        else:
            upd.dedup(self.ids_all, self.g_all, None)
            upd.apply(self.V, None, exact=(self.update_mode == "exact"), l2_reg=self.l2_reg)
        self.dense.apply()
        self.global_step += 1
        return torch.cat([self.loss_ce, upd.reg[0:1]])

    def loss_value(self, parts: torch.Tensor) -> float:
        p = parts.tolist()
        return p[0] + p[1]
