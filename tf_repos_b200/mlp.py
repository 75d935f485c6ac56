"""The dense 'Deep-part' (DeepFM.py:137-167): fully_connected(relu) -> dropout stacks + the N=1 output
layer, forward and backward, through libctr_b200.so (csrc/fc.cu).  No torch compute.

fp32 throughout (the logit parity target is 1e-5 relative, which rules out TF32/BF16 tensor-core
inputs without split-precision emulation).  All buffers are allocated once (CUDA-graph capturable).
batch_norm=True inserts batch_norm_layer (DeepFM.py:159-160,231-235) between a layer's relu and its dropout
(csrc/batch_norm.cu): trainable `bn_{i}/gamma|beta` live with the other dense variables, the non-trainable
`bn_{i}/moving_mean|moving_variance` in `bn_state` (saved with checkpoints / exports).
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch

from . import ops
from .engine import DenseVars


class MLP:
    """layers: hidden widths; the output layer `{scope}/{out_scope}` maps [last hidden | extra] -> 1."""

    def __init__(self, in_dim: int, layers: Sequence[int], keep_prob: Sequence[float], B: int, device,
                 scope: str = "Deep-part", out_scope: Optional[str] = "deep_out", out_extra_in: int = 0,
                 seed: int = 0, layer_fmt: str = "mlp{i}", w_name: str = "weights", b_name: str = "biases",
                 batch_norm: bool = False, bn_decay: float = 0.9, *, bn_fmt: str = "bn_{i}"):
        # layer_fmt / w_name / b_name / bn_fmt: TF variable naming (contrib fully_connected: mlp{i}/weights|biases;
        # the canned estimators' Dense layers: hiddenlayer_{i}/kernel|bias; ESMM's towers: cvr_mlp{i}, cvr_bn_{i}).
        # An empty scope leaves the names unprefixed (DeepCvrMTL.py's tf.name_scope does not prefix get_variable).
        self.layer_fmt, self.w_name, self.b_name, self.bn_fmt = layer_fmt, w_name, b_name, bn_fmt
        self.in_dim, self.layers, self.keep = in_dim, list(layers), list(keep_prob)
        self.scope, self.out_scope, self.B, self.device = scope, out_scope, B, device
        # TF name of the output layer: "<scope>/<out_scope>", or out_scope itself when it is a full path
        self.out_name = out_scope if (out_scope and "/" in out_scope) else self._scoped(out_scope)
        self.last_dim = self.layers[-1] if self.layers else in_dim
        self.out_extra_in = out_extra_in
        self.out_in = self.last_dim + out_extra_in
        self.seed = seed
        f32 = dict(dtype=torch.float32, device=device)
        self.h = [torch.empty(B, w, **f32) for w in self.layers]          # post-activation, post-dropout
        self.masks = [torch.empty(B, w, **f32) if k < 1.0 else None for w, k in zip(self.layers, self.keep)]
        self.dh = [torch.empty(B, w, **f32) for w in self.layers]
        self.y = torch.empty(B, **f32)
        self.dx = torch.empty(B, in_dim, **f32)
        self.d_extra = torch.empty(B, out_extra_in, **f32) if out_extra_in else None
        self.batch_norm, self.bn_decay = bool(batch_norm), float(bn_decay)
        self.bn_state = {}
        if self.batch_norm:
            self.r = [torch.empty(B, w, **f32) for w in self.layers]       # relu output = batch_norm input
            self.dr = [torch.empty(B, w, **f32) for w in self.layers]
            self.bn_mean = [torch.zeros(w, **f32) for w in self.layers]    # batch moments saved for the backward
            self.bn_var = [torch.ones(w, **f32) for w in self.layers]
            for i, w in enumerate(self.layers):
                self.bn_state[self._bn(i, "moving_mean")] = torch.zeros(w, **f32)
                self.bn_state[self._bn(i, "moving_variance")] = torch.ones(w, **f32)
        dims = [in_dim] + self.layers
        ws = max([ops.fc_bwd_workspace_bytes(B, dims[i], dims[i + 1]) for i in range(len(self.layers))] +
                 [ops.fc1_bwd_workspace_bytes(B, self.last_dim, out_extra_in), 16])
        self.ws = torch.empty(ws, dtype=torch.uint8, device=device)
        self._active = [None] * len(self.layers)

    def _scoped(self, name: str) -> str:
        return f"{self.scope}/{name}" if self.scope else name

    def _w(self, i: int) -> str:
        return self._scoped(f"{self.layer_fmt.format(i=i)}/{self.w_name}")

    def _b(self, i: int) -> str:
        return self._scoped(f"{self.layer_fmt.format(i=i)}/{self.b_name}")

    def _bn(self, i: int, what: str) -> str:
        return self._scoped(f"{self.bn_fmt.format(i=i)}/{what}")

    def specs(self):
        out, d = [], self.in_dim
        for i, w in enumerate(self.layers):
            out += [(self._w(i), (d, w)), (self._b(i), (w,))]
            if self.batch_norm:
                out += [(self._bn(i, "gamma"), (w,)), (self._bn(i, "beta"), (w,))]
            d = w
        if self.out_scope:
            out += [(f"{self.out_name}/{self.w_name}", (self.out_in, 1)), (f"{self.out_name}/{self.b_name}", (1,))]
        return out

    def init(self, dv: DenseVars, gen: torch.Generator):
        """xavier_uniform weights, zero biases (tf.contrib.layers.fully_connected defaults)."""
        for name, shape in self.specs():
            if name.endswith(self.w_name):
                lim = (6.0 / (shape[0] + shape[1])) ** 0.5
                w = (torch.rand(shape, generator=gen, dtype=torch.float64) * 2 - 1) * lim
                dv[name].copy_(w.to(torch.float32))
            elif name.endswith("/gamma"):       # batch_norm: gamma ones, beta zeros (the flat buffer starts at zero)
                dv[name].fill_(1.0)

    # ---- forward -------------------------------------------------------------------------------
    def forward_hidden(self, x: torch.Tensor, dv: DenseVars, train: bool, masks=None, step_dev=None) -> torch.Tensor:
        """masks: optional injected binary keep masks (parity runs); otherwise, in TRAIN mode with
        keep_prob < 1, a fresh mask is drawn on the device from (seed, global step, element)."""
        a = x
        n = a.shape[0]
        for i in range(len(self.layers)):
            W, b = dv[self._w(i)], dv[self._b(i)]
            m = None
            if train and masks is not None and masks[i] is not None:
                m = masks[i]
            elif train and self.keep[i] < 1.0:
                m = self.masks[i][:n]
                ops.dropout_mask(m, self.keep[i], self.seed * 131 + i, step_dev)
            self._active[i] = m
            h = self.h[i][:n]
            if self.batch_norm:   # relu -> batch_norm -> dropout (DeepFM.py:156-162)
                r = self.r[i][:n]
                ops.fc_fwd(a, W, b, None, 1.0, 1, r)
                ops.bn_fwd(r, dv[self._bn(i, "gamma")], dv[self._bn(i, "beta")], self.bn_state[self._bn(i, "moving_mean")],
                           self.bn_state[self._bn(i, "moving_variance")], train, self.bn_decay, m, self.keep[i], h,
                           self.bn_mean[i], self.bn_var[i])
            else:
                ops.fc_fwd(a, W, b, m, self.keep[i], 1, h)
            a = h
        return a

    def forward_out(self, a: torch.Tensor, dv: DenseVars, extra: Optional[torch.Tensor] = None) -> torch.Tensor:
        """y = [extra | a] @ W + b when `extra` is given (DCN: [x_L, x_deep]), else a @ W + b."""
        W, b = dv[f"{self.out_name}/{self.w_name}"], dv[f"{self.out_name}/{self.b_name}"]
        y = self.y[: a.shape[0]]
        if extra is not None:
            ops.fc1_fwd(extra, a, W.view(-1), b, y)
        else:
            ops.fc1_fwd(a, None, W.view(-1), b, y)
        return y

    # ---- backward ------------------------------------------------------------------------------
    def backward_out(self, a: torch.Tensor, dy: torch.Tensor, dv: DenseVars, da: torch.Tensor,
                     extra: Optional[torch.Tensor] = None):
        W = dv[f"{self.out_name}/{self.w_name}"]
        gW = dv.grads[f"{self.out_name}/{self.w_name}"].view(-1)
        gb = dv.grads[f"{self.out_name}/{self.b_name}"]
        if extra is not None:
            ops.fc1_bwd(extra, a, W.view(-1), dy, self.d_extra[: a.shape[0]], da, gW, gb, self.ws)
        else:
            ops.fc1_bwd(a, None, W.view(-1), dy, da, None, gW, gb, self.ws)

    def backward_hidden(self, x: torch.Tensor, d_last: torch.Tensor, dv: DenseVars, need_dx: bool = True):
        """d_last: gradient w.r.t. the last hidden activation (post-dropout); overwritten."""
        d = d_last
        n = d.shape[0]
        if not self.layers:
            return d_last
        for i in reversed(range(len(self.layers))):
            W = dv[self._w(i)]
            a = self.h[i - 1][:n] if i > 0 else x
            d_in = self.dh[i - 1][:n] if i > 0 else (self.dx[:n] if need_dx else None)
            if self.batch_norm:
                r, dr = self.r[i][:n], self.dr[i][:n]
                ops.bn_bwd(d, r, self.bn_mean[i], self.bn_var[i], dv[self._bn(i, "gamma")], self._active[i], self.keep[i],
                           dr, dv.grads[self._bn(i, "gamma")], dv.grads[self._bn(i, "beta")])
                ops.fc_bwd(a, W, r, None, 1.0, dr, 1, d_in, dv.grads[self._w(i)], dv.grads[self._b(i)], self.ws)
            else:
                ops.fc_bwd(a, W, self.h[i][:n], self._active[i], self.keep[i], d, 1, d_in,
                           dv.grads[self._w(i)], dv.grads[self._b(i)], self.ws)
            d = d_in
        return self.dx[:n] if need_dx else None
