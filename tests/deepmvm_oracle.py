"""CPU restatement of DeepMVM's model_fn (deep_ctr/Model_pipeline/DeepMVM.py:100-230), op for op, on the shared oracle
machinery of oracle/models.py (variables, slots, TF update semantics).  Test infrastructure, like oracle/: the GPU
parity tests compare tf_repos_b200.deepmvm.DeepMVM against it, and test_oracle_deepmvm.py pins it with per-element
loops and closed forms."""
from __future__ import annotations

import torch

from oracle import models as om
from oracle import tf_semantics as tfs


class DeepMVM(om.OracleModel, om.MLPMixin):
    """DeepMVM.py:100-230.  No first-order table, no bias variable."""

    tables = ("mvm_w",)
    l2_vars = ("mvm_w", "mvm_b")  # DeepMVM.py:197-199, in loss order (the table term first)

    def __init__(self, field_size, feature_size, embedding_size, deep_layers="256,128,64", dropout="0.5,0.5,0.5",
                 batch_norm=False, batch_norm_decay=0.9, seed=0, **kw):
        super().__init__(**kw)
        self.F, self.N, self.K = field_size, feature_size, embedding_size
        self.layers, self.keep = om._ints(deep_layers), om._floats(dropout)
        self.batch_norm, self.bn_decay = batch_norm, batch_norm_decay
        self.bn_state = {}
        gen = torch.Generator().manual_seed(seed)
        self.add_param("mvm_w", tfs.glorot_normal((self.N, self.K), gen, self.dtype))   # DeepMVM.py:117
        self.add_param("mvm_b", tfs.glorot_normal((self.F, self.K), gen, self.dtype))   # :118
        last = self.layers[-1] if self.layers else self.F * self.K
        self.build_mlp(self.F * self.K, self.layers, gen, scope="Deep-part", out_scope="DeepMVM-out/deep_out",
                       out_dim_in=self.K + last, batch_norm=batch_norm)
        self.init_slots()

    def sites(self, batch):
        return {"emb": ("mvm_w", batch["feat_ids"].reshape(-1, self.F))}

    def forward(self, rows, dense, batch, train, masks=None):
        B = rows["emb"].shape[0]
        vals = batch["feat_vals"].reshape(-1, self.F, 1).to(self.dtype)
        e = rows["emb"] * vals                                                         # :140-142
        a = e + dense["mvm_b"]                                                         # :145
        x_mvm = a[:, 0, :]                                                             # :146
        for i in range(1, self.F):                                                     # :147-148, in field order
            x_mvm = x_mvm * a[:, i, :]
        x = e.reshape(B, self.F * self.K)                                              # :166
        h = self.run_mlp(x, dense, self.layers, self.keep, train, masks, scope="Deep-part",
                         batch_norm=self.batch_norm, bn_decay=self.bn_decay)          # :167-178
        x_stack = torch.cat([x_mvm, h], 1)                                             # :181
        y = tfs.fully_connected(x_stack, dense["DeepMVM-out/deep_out/weights"],
                                dense["DeepMVM-out/deep_out/biases"], None).reshape(-1)  # :182-184
        return {"y": y, "x": x, "x_mvm": x_mvm}
