"""Serving entry for an exported model (SURVEY.md 8f-4): answers the request the reference's TF-Serving clients send
(`Serving_pipeline/deep_fm_serving_client.cpp:42-60`: signature `serving_default`, inputs `feat_ids` int64 [n,F] and
`feat_vals` float32 [n,F], output `prob` float32 [n]; export definition DeepFM.py:354-366) from the files that
`--task_type=export` writes (`<servable_model_dir>/<timestamp>/{variables.pt, signature.json}`).

    s = Servable.load("./servable/1700000000")
    prob = s.predict(feat_ids, feat_vals)        # torch / numpy, host or device, any n

No training state is created (update_mode='lazy': no `last` bytes, no sweeps); requests larger than the configured
batch are served in slices.  The gather kernel reads int64 ids directly (ctr_fm_embed_fwd id_bits = 64).
"""
from __future__ import annotations

import json
import os
from typing import Dict

import numpy as np
import torch


def _build(model_name: str, p: Dict, batch_size: int, device):
    common = dict(dropout=p.get("dropout", "0.5,0.5,0.5"), l2_reg=p.get("l2_reg", 1e-4), learning_rate=p.get("learning_rate", 5e-4),
                  optimizer=p.get("optimizer", "Adam"), update_mode="lazy", device=device)
    F, N, K = int(p["field_size"]), int(p["feature_size"]), int(p["embedding_size"])
    if model_name == "DeepFM":
        from .deepfm import DeepFM
        return DeepFM(F, N, K, batch_size, deep_layers=p["deep_layers"], **common)
    if model_name == "DCN":
        from .dcn import DCN
        return DCN(F, N, K, batch_size, deep_layers=p["deep_layers"], cross_layers=int(p["cross_layers"]), **common)
    if model_name == "DeepMVM":
        from .deepmvm import DeepMVM
        return DeepMVM(F, N, K, batch_size, deep_layers=p["deep_layers"], batch_norm=bool(p.get("batch_norm", False)),
                       **common)
    if model_name == "NFM":
        from .nfm import NFM
        return NFM(F, N, K, batch_size, deep_layers=p["deep_layers"], **common)
    if model_name == "PNN":
        from .pnn import PNN
        return PNN(F, N, K, batch_size, model_type=p["model_type"], deep_layers=p["deep_layers"], **common)
    if model_name == "AFM":
        from .afm import AFM
        return AFM(F, N, K, batch_size, attention_layers=p["attention_layers"], **common)
    raise ValueError(f"unknown exported model {model_name!r}")


class Servable:
    def __init__(self, model, signature: Dict):
        self.model, self.signature = model, signature
        self.F = int(signature["inputs"]["feat_ids"]["shape"][1])

    @classmethod
    def load(cls, export_dir: str, max_batch: int = 4096, device="cuda") -> "Servable":
        sig = json.load(open(os.path.join(export_dir, "signature.json")))
        model = _build(sig["model"], sig["params"], max_batch, torch.device(device))
        model.load_variables(torch.load(os.path.join(export_dir, "variables.pt"), map_location="cpu"))
        return cls(model, sig)

    def predict(self, feat_ids, feat_vals) -> torch.Tensor:
        """feat_ids int64|int32 [n,F] (or [n,F,1]), feat_vals float32 [n,F]; returns prob float32 [n] on the host."""
        dev = self.model.device
        ids = torch.as_tensor(np.asarray(feat_ids) if not torch.is_tensor(feat_ids) else feat_ids)
        vals = torch.as_tensor(np.asarray(feat_vals) if not torch.is_tensor(feat_vals) else feat_vals)
        ids = ids.reshape(-1, self.F)
        vals = vals.reshape(-1, self.F).to(torch.float32)
        if ids.dtype not in (torch.int32, torch.int64):
            ids = ids.to(torch.int64)
        ids, vals = ids.to(dev).contiguous(), vals.to(dev).contiguous()
        out = torch.empty(ids.shape[0], dtype=torch.float32)
        B = self.model.B
        for lo in range(0, ids.shape[0], B):
            hi = min(lo + B, ids.shape[0])
            out[lo:hi] = self.model.predict(ids[lo:hi], vals[lo:hi]).cpu()
        self.model.check_ids()
        return out
