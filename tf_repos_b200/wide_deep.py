"""wide_n_deep (deep_ctr/Model_pipeline/wide_n_deep.py:92-151) on libctr_b200.so: the canned estimators
LinearClassifier / DNNClassifier / DNNLinearCombinedClassifier over the Criteo CSV columns (13 numeric I1..I13,
26 categorical C14..C39 with identity buckets of 10 000 and one [10000, K] embedding table each).

[TF-sem] defaults restated in oracle/wide_deep.py (SURVEY.md A.8): name-sorted column order, out-of-range id -> 0,
loss = SUM of sigmoid cross-entropy over the batch, Adagrad(0.05 | 0.001, accumulator 0.1) on dnn/*,
Ftrl(min(0.2 | 0.005, 1/sqrt(39))) on linear/*, sparse gradients summed per id before the apply (no L2 term, so only
gathered rows move: the sparse applies ARE TensorFlow's result here).

The 26 per-column tables are stored stacked ([26*10000, K] and [26*10000]); `variables()` exposes them under the TF
checkpoint names.  All arithmetic is in csrc/wide_deep.cu, fc.cu/tc_gemm.cu, loss.cu, sort_unique.cu, segment_sum.cu,
optim.cu; torch provides memory only.
"""
from __future__ import annotations

import math
from typing import Dict

import torch

from . import ops
from .base import ints
from .engine import HYPER_TABLE, DenseVars, OptimizerState, Table
from .mlp import MLP

N_NUM, N_CAT, NUM_BUCKETS = 13, 26, 10000
NUM_NAMES = ["I%d" % i for i in range(1, 14)]
CAT_NAMES = ["C%d" % i for i in range(14, 40)]
NUM_SORTED = sorted(range(N_NUM), key=lambda j: NUM_NAMES[j])      # input_layer / linear_model sort columns by name


class WideDeep:
    def __init__(self, embedding_size=32, batch_size=128, deep_layers="256,128,64", model_type="wide_n_deep",
                 device="cuda", seed=0):
        if model_type not in ("wide", "deep", "wide_n_deep"):
            raise ValueError("model_type must be one of {'wide', 'deep', 'wide_n_deep'} (wide_n_deep.py:46)")
        self.K, self.B, self.model_type = embedding_size, batch_size, model_type
        self.layers = ints(deep_layers)
        self.device = dev = torch.device(device)
        self.has_dnn, self.has_linear = model_type != "wide", model_type != "deep"
        self.dnn_lr = 0.05 if model_type == "deep" else 0.001
        self.linear_lr = min(0.2 if model_type == "wide" else 0.005, 1.0 / math.sqrt(N_NUM + N_CAT))
        K, B = self.K, self.B
        n = B * N_CAT
        f32 = dict(dtype=torch.float32, device=dev)
        self.opt_dnn = OptimizerState("Adagrad", self.dnn_lr, 0.0, dev, adagrad_init=0.1)
        self.opt_lin = OptimizerState("ftrl", self.linear_lr, 0.0, dev)
        self.D = N_CAT * K + N_NUM
        self.num_perm = torch.tensor(NUM_SORTED, dtype=torch.int32, device=dev)
        self.flat_ids = torch.empty(n, dtype=torch.int32, device=dev)
        # both parts look up the same flat ids: one de-duplication, gradients summed per unique id
        self.uw = ops.UniqueWorkspace(n, N_CAT * NUM_BUCKETS, dev)
        self.g_uniq = torch.empty(n * K, **f32)
        self.gw_uniq = torch.empty(n, **f32)
        self.y = torch.empty(B, **f32); self.pred = torch.empty(B, **f32); self.dy = torch.empty(B, **f32)
        self.loss = torch.zeros(1, **f32)
        self.zero_bias = torch.zeros(1, **f32)
        self.lin = torch.zeros(B, **f32)
        self.g_cat = torch.empty(n, **f32)
        if self.has_dnn:
            self.emb = Table("emb", N_CAT * NUM_BUCKETS, K, self.opt_dnn, dev, init_std=1.0 / math.sqrt(K), seed=seed * 2 + 1)
            self.mlp = MLP(self.D, self.layers, [1.0] * len(self.layers), B, dev, scope="dnn", out_scope="logits", seed=seed,
                           layer_fmt="hiddenlayer_{i}", w_name="kernel", b_name="bias")
            self.dense_dnn = DenseVars(self.mlp.specs(), self.opt_dnn, dev)
            self.mlp.init(self.dense_dnn, torch.Generator().manual_seed(seed))
            self.x = torch.empty(B, self.D, **f32)
            self.d_last = torch.empty(B, self.mlp.out_in, **f32)
            self.g_rows = torch.empty(n, K, **f32)
        if self.has_linear:
            self.wide_cat = Table("wide_cat", N_CAT * NUM_BUCKETS, 1, self.opt_lin, dev, value=torch.zeros(N_CAT * NUM_BUCKETS))
            self.dense_lin = DenseVars([("linear/numeric", (N_NUM,)), ("linear/linear_model/bias_weights", (1,))],
                                       self.opt_lin, dev)
        self.global_step = 0

    # ---- variables under their TF checkpoint names ----------------------------------------------------------
    def variables(self) -> Dict[str, torch.Tensor]:
        out: Dict[str, torch.Tensor] = {}
        if self.has_dnn:
            for f, c in enumerate(CAT_NAMES):
                out[f"dnn/input_from_feature_columns/input_layer/{c}_embedding/embedding_weights"] = \
                    self.emb.var[f * NUM_BUCKETS:(f + 1) * NUM_BUCKETS]
            out.update(self.dense_dnn.views)
        if self.has_linear:
            for f, c in enumerate(CAT_NAMES):
                out[f"linear/linear_model/{c}/weights"] = self.wide_cat.var[f * NUM_BUCKETS:(f + 1) * NUM_BUCKETS].view(-1, 1)
            for j, c in enumerate(NUM_NAMES):
                out[f"linear/linear_model/{c}/weights"] = self.dense_lin["linear/numeric"][j:j + 1].view(1, 1)
            out["linear/linear_model/bias_weights"] = self.dense_lin["linear/linear_model/bias_weights"]
        return out

    def load_variables(self, values: Dict[str, torch.Tensor]):
        for name, dst in self.variables().items():
            if name in values:
                dst.copy_(values[name].to(self.device).reshape(dst.shape))

    # ---- forward ------------------------------------------------------------------------------------------------
    def _forward(self, dense: torch.Tensor, cat: torch.Tensor):
        B = dense.shape[0]
        lin = self.lin[:B] if self.has_linear else None
        ops.wd_input_fwd(cat, dense, self.emb.var if self.has_dnn else None,
                         self.wide_cat.var if self.has_linear else None,
                         self.dense_lin["linear/numeric"] if self.has_linear else None,
                         self.dense_lin["linear/linear_model/bias_weights"] if self.has_linear else None,
                         self.num_perm, NUM_BUCKETS, self.K, self.flat_ids[: B * N_CAT],
                         self.x[:B] if self.has_dnn else None, lin)
        return lin, self._dnn(B)

    def _dnn(self, B: int):
        """the DNN logits of x[:B], or None for the linear model"""
        if not self.has_dnn:
            return None
        self._a = self.mlp.forward_hidden(self.x[:B], self.dense_dnn, train=False)
        return self.mlp.forward_out(self._a, self.dense_dnn)

    def _probabilities(self, B: int, lin, y_d, pred: torch.Tensor) -> torch.Tensor:
        ops.logit_loss(self.zero_bias, lin, y_d, None, None, B, y=self.y[:B], pred=pred)
        return pred

    def predict(self, dense: torch.Tensor, cat: torch.Tensor) -> torch.Tensor:
        """probabilities[:, 1] (wide_n_deep.py:228-232)"""
        B = dense.shape[0]
        lin, y_d = self._forward(dense, cat)
        return self._probabilities(B, lin, y_d, self.pred[:B])

    def predict_examples(self, data: torch.Tensor, offsets: torch.Tensor, err: torch.Tensor, pred: torch.Tensor,
                         example_base: int = 0) -> torch.Tensor:
        """probabilities[:, 1] of the serialized tf.Examples data[offsets[b], offsets[b+1]) (uint8 / int64 [B+1]
        device tensors, B <= batch_size) -- the serving input of wide_n_deep.py:233-242, parsed on the device
        (ops.wd_serve_input).  A rejected Example min-folds (example_base + b) << 16 | check << 8 | key into err
        (int64 [1], -1 = none) and leaves its pred[b] undefined; nothing here waits for the device."""
        B = offsets.numel() - 1
        assert B <= self.B
        lin = self.lin[:B] if self.has_linear else None
        ops.wd_serve_input(data, offsets, example_base, self.emb.var if self.has_dnn else None,
                           self.wide_cat.var if self.has_linear else None,
                           self.dense_lin["linear/numeric"] if self.has_linear else None,
                           self.dense_lin["linear/linear_model/bias_weights"] if self.has_linear else None,
                           self.num_perm, NUM_BUCKETS, self.K, self.x[:B] if self.has_dnn else None, lin, err)
        return self._probabilities(B, lin, self._dnn(B), pred)

    # ---- one optimizer step of each part ----------------------------------------------------------------------
    def train_step(self, dense: torch.Tensor, cat: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
        B = dense.shape[0]
        assert B <= self.B
        n = B * N_CAT
        self.opt_dnn.tick(); self.opt_lin.tick()
        lin, y_d = self._forward(dense, cat)
        # B_total = 1: the canned head SUMS the per-example losses (dy = pred - label)
        ops.logit_loss(self.zero_bias, lin, y_d, None, labels, B, y=self.y[:B], pred=self.pred[:B], loss_ce=self.loss,
                       dy=self.dy[:B], dbias=None, B_total=1)
        dy = self.dy[:B]
        dX = None
        if self.has_dnn:
            self.mlp.backward_out(self._a, dy, self.dense_dnn, self.d_last[:B])
            dX = self.mlp.backward_hidden(self.x[:B], self.d_last[:B], self.dense_dnn)
        ops.wd_input_bwd(dX, dy, dense, B, N_CAT, N_NUM, self.K, self.g_rows[:n] if self.has_dnn else None,
                         self.g_cat[:n] if self.has_linear else None,
                         self.dense_lin.grads["linear/numeric"] if self.has_linear else None,
                         self.dense_lin.grads["linear/linear_model/bias_weights"] if self.has_linear else None)
        uw = self.uw
        uw.n_active = n
        ops.unique_segment(self.flat_ids[:n], uw)
        if self.has_dnn:
            ops.segment_sum_rows(self.g_rows[:n], self.g_cat[:n] if self.has_linear else None, uw, self.K, self.g_uniq,
                                 self.gw_uniq if self.has_linear else None)
            o = self.opt_dnn
            ops.opt_sparse_rows(o.opt, self.emb.var, self.emb.slot(0), None, uw.uniq, uw.n_uniq, self.g_uniq, uw.n, self.K,
                                o.record(HYPER_TABLE), None)
            self.dense_dnn.apply()
        if self.has_linear:
            if not self.has_dnn:   # scalar rows only: the K=1 flavour of the segment sum
                ops.segment_sum_rows(self.g_cat[:n].view(-1, 1), None, uw, 1, self.gw_uniq, None)
            o = self.opt_lin
            ops.opt_sparse_rows(o.opt, self.wide_cat.var, self.wide_cat.slot(0), self.wide_cat.slot(1), uw.uniq, uw.n_uniq,
                                self.gw_uniq, uw.n, 1, o.record(HYPER_TABLE), None)
            self.dense_lin.apply()
        self.global_step += 1
        return self.loss
