"""`model_fn(features, labels, mode, params)` with the contract of deep_ctr/Model_pipeline/DeepFM.py:100-221, for callers
that are written against the reference's Estimator interface rather than against the model classes.

TensorFlow's model_fn BUILDS a graph that the Estimator then runs; here the state lives in a model object (created on
the first call from `params`, DeepFM.py:329-338, and cached in `params["_model"]`, or passed in explicitly) and the
returned spec carries results and a `train_op` callable:

    spec = model_fn({"feat_ids": ids, "feat_vals": vals}, labels, ModeKeys.TRAIN, params)
    loss_parts = spec.train_op()          # ONE optimizer.minimize(loss) (DeepFM.py:213); {CE, l2 terms...}
    spec = model_fn(features, None, ModeKeys.PREDICT, params);  spec.predictions["prob"]          # DeepFM.py:178-185
    spec = model_fn(features, labels, ModeKeys.EVAL, params);   spec.loss, spec.eval_metric_ops["auc"]   # :192-199

features: "feat_ids" int32|int64 [B,F] or [B,F,1], "feat_vals" float32 same shape (the input_fn contract, :97-98).
params: field_size, feature_size, embedding_size, learning_rate, l2_reg, deep_layers, dropout (:329-338) plus, because
the reference reads them from FLAGS inside model_fn, optional optimizer (:204-211), batch_size, update_mode, model
('DeepFM' | 'DCN' | 'DeepMVM' | 'NFM' | 'PNN' | 'AFM') and that model's extra keys (cross_layers, model_type, attention_layers).
"""
from __future__ import annotations

from typing import Any, Callable, Dict, NamedTuple, Optional

import numpy as np
import torch


class ModeKeys:
    TRAIN, EVAL, PREDICT = "train", "eval", "infer"


class EstimatorSpec(NamedTuple):
    mode: str
    predictions: Optional[Dict[str, torch.Tensor]] = None
    loss: Optional[float] = None
    train_op: Optional[Callable[[], torch.Tensor]] = None
    eval_metric_ops: Optional[Dict[str, float]] = None
    export_outputs: Optional[Dict[str, Dict[str, torch.Tensor]]] = None


def build_model(params: Dict[str, Any], batch_size: int, device="cuda"):
    name = params.get("model", "DeepFM")
    F, N, K = int(params["field_size"]), int(params["feature_size"]), int(params["embedding_size"])
    kw = dict(dropout=params.get("dropout", "0.5,0.5,0.5"), l2_reg=float(params.get("l2_reg", 1e-4)),
              learning_rate=float(params.get("learning_rate", 5e-4)), optimizer=params.get("optimizer", "Adam"),
              update_mode=params.get("update_mode", "exact_deferred"), device=device)
    if name == "DeepFM":
        from .deepfm import DeepFM
        return DeepFM(F, N, K, batch_size, deep_layers=params.get("deep_layers", "256,128,64"), **kw)
    if name == "DCN":
        from .dcn import DCN
        return DCN(F, N, K, batch_size, deep_layers=params.get("deep_layers", "256,128,64"), cross_layers=int(params.get("cross_layers", 3)), **kw)
    if name == "DeepMVM":
        from .deepmvm import DeepMVM
        return DeepMVM(F, N, K, batch_size, deep_layers=params.get("deep_layers", "256,128,64"), **kw)
    if name == "NFM":
        from .nfm import NFM
        return NFM(F, N, K, batch_size, deep_layers=params.get("deep_layers", "128,64"), **kw)
    if name == "PNN":
        from .pnn import PNN
        return PNN(F, N, K, batch_size, model_type=params.get("model_type", "Inner"), deep_layers=params.get("deep_layers", "256,128,64"), **kw)
    if name == "AFM":
        from .afm import AFM
        return AFM(F, N, K, batch_size, attention_layers=params.get("attention_layers", "256"), **kw)
    raise ValueError(f"params['model'] = {name!r} is not one of DeepFM, DCN, DeepMVM, NFM, PNN, AFM")


def model_fn(features: Dict[str, torch.Tensor], labels: Optional[torch.Tensor], mode: str, params: Dict[str, Any],
             model=None) -> EstimatorSpec:
    F = int(params["field_size"])
    ids = features["feat_ids"].reshape(-1, F)          # DeepFM.py:119-122
    vals = features["feat_vals"].reshape(-1, F)
    if model is None:
        model = params.get("_model")
        if model is None:
            model = params["_model"] = build_model(params, int(params.get("batch_size", ids.shape[0])))
    dev = model.device
    ids, vals = ids.to(dev).contiguous(), vals.to(dev, torch.float32).contiguous()
    if mode == ModeKeys.PREDICT:
        prob = model.predict(ids, vals)
        pred = {"prob": prob}
        return EstimatorSpec(mode, predictions=pred, export_outputs={"serving_default": pred})
    if labels is None:
        raise ValueError("labels are required in TRAIN and EVAL mode")
    labels = labels.reshape(-1).to(dev, torch.float32).contiguous()
    if mode == ModeKeys.EVAL:
        from .estimator import auc_200
        prob = model.predict(ids, vals)
        y = model.y[: ids.shape[0]].detach().cpu().numpy().astype(np.float64)
        t = labels.cpu().numpy()
        ce = float((np.maximum(y, 0) - y * t + np.log1p(np.exp(-np.abs(y)))).mean())          # metric only, on the host
        return EstimatorSpec(mode, predictions={"prob": prob}, loss=ce,
                             eval_metric_ops={"auc": auc_200(t, prob.detach().cpu().numpy())})
    if mode == ModeKeys.TRAIN:
        return EstimatorSpec(mode, predictions=None, train_op=lambda: model.train_step(ids, vals, labels))
    raise ValueError(f"mode must be one of {ModeKeys.TRAIN!r}, {ModeKeys.EVAL!r}, {ModeKeys.PREDICT!r}")
