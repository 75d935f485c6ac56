"""input_fn / main(_) of deep_ctr/Model_pipeline/DIN.py:57-99,300-392 on the H100 engine.

Input: TFRecord files of tf.Example (`data_dir/tr/*tfrecord`, `data_dir/te/*tfrecord`; eval files = test files, quirk
Q6, DIN.py:342-345) with the features of DIN.py:60-77:
    y, z float scalars; feat_ids int64 [field_size]; a_catids, a_shopids, a_brandids int64 scalars;
    a_intids, u_{cat,shop,brand,int}ids int64 var-len; u_{cat,shop,brand,int}vals float var-len.
`dataset.batch` turns the var-len features into SparseTensors and the model densifies them with zeros
(sparse_tensor_to_dense, DIN.py:153-154): here every batch is padded to the longest list of the whole input (P),
which gives the same numbers because id 0 is masked out (DIN.py:157).

The CUDA DIN model works on full-size buffers; the single partial batch that repeat-before-batch leaves at the very end
of TRAINING is padded and trained on with `n_valid` (the padded rows' dy is exactly 0: same step as TensorFlow's smaller
batch, see DIN.train_step); eval / infer pad the last batch and drop the padded outputs, so every sample is scored.
"""
from __future__ import annotations

import glob
import json
import os
import random
import shutil
import time
from datetime import date, timedelta
from typing import Dict, Iterator, List, Sequence, Tuple

import numpy as np
import torch

from .estimator import auc_200, restore_checkpoint, save_checkpoint
from .flags import FLAGS
from .tfrecord import parse_example, read_records

U_FIELDS = ("cat", "shop", "brand", "int")


def decode_tfrecord_files(files: Sequence[str], field_size: int, labels: Sequence[str] = ("y",)) -> Dict[str, list]:
    """All examples of `files`, feature by feature (tf.parse_single_example with the spec of DIN.py:60-77).
    `labels`: the required float label features (ESMM also requires z, DeepCvrMTL.py:67-68)."""
    print("Parsing", list(files))
    d: Dict[str, list] = {k: [] for k in tuple(labels) + ("feat_ids", "a_cat", "a_shop", "a_brand", "a_int")}
    for f in U_FIELDS:
        d["u_%sids" % f], d["u_%svals" % f] = [], []
    for path in files:
        for rec in read_records(path):
            ex = parse_example(rec)
            for key in tuple(labels) + ("feat_ids", "a_catids", "a_shopids", "a_brandids"):
                if key not in ex or len(ex[key]) == 0:
                    raise ValueError(f"{path}: Feature: {key} (data type: {'float' if key in labels else 'int64'}) is required but could not be found.")
            if len(ex["feat_ids"]) != field_size:
                raise ValueError(f"{path}: feat_ids has {len(ex['feat_ids'])} values, field_size is {field_size}")
            for key in labels:
                d[key].append(float(ex[key][0]))
            d["feat_ids"].append(np.asarray(ex["feat_ids"], dtype=np.int64))
            d["a_cat"].append(int(ex["a_catids"][0])); d["a_shop"].append(int(ex["a_shopids"][0]))
            d["a_brand"].append(int(ex["a_brandids"][0]))
            d["a_int"].append(np.asarray(ex.get("a_intids", []), dtype=np.int64))
            for f in U_FIELDS:
                ids = np.asarray(ex.get("u_%sids" % f, []), dtype=np.int64)
                vals = np.asarray(ex.get("u_%svals" % f, []), dtype=np.float32)
                if len(ids) != len(vals):
                    raise ValueError(f"{path}: u_{f}ids / u_{f}vals lengths differ ({len(ids)} vs {len(vals)})")
                d["u_%sids" % f].append(ids); d["u_%svals" % f].append(vals)
    return d


def max_lengths(*datasets: Dict[str, list]) -> Tuple[int, int]:
    """(P, max_a_int): the longest behaviour list / a_int bag anywhere in the inputs (>= 1)."""
    P = A = 1
    for d in datasets:
        for f in U_FIELDS:
            P = max([P] + [len(x) for x in d["u_%sids" % f]])
        A = max([A] + [len(x) for x in d["a_int"]])
    return P, A


def make_batch(d: Dict[str, list], idx: Sequence[int], B: int, P: int, device) -> Tuple[Dict[str, torch.Tensor], torch.Tensor, int]:
    """Samples `idx` (len <= B; padded to B with copies of the first sample) -> the model's batch dict, labels, n real."""
    n = len(idx)
    idx = list(idx) + [idx[0]] * (B - n)
    feat_ids = np.stack([d["feat_ids"][i] for i in idx]).astype(np.int32)
    a_ids = np.asarray([[d[k][i] for i in idx] for k in ("a_cat", "a_shop", "a_brand")], dtype=np.int32)
    lens = [len(d["a_int"][i]) for i in idx]
    a_off = np.zeros(B + 1, dtype=np.int32)
    a_off[1:] = np.cumsum(lens)
    a_int = np.concatenate([d["a_int"][i] for i in idx]).astype(np.int32) if a_off[-1] else np.zeros(0, np.int32)
    u_ids = np.zeros((4, B, P), dtype=np.int32)
    u_wgt = np.zeros((4, B, P), dtype=np.float32)
    for fi, f in enumerate(U_FIELDS):
        for b, i in enumerate(idx):
            ids, vals = d["u_%sids" % f][i], d["u_%svals" % f][i]
            u_ids[fi, b, :len(ids)] = ids
            u_wgt[fi, b, :len(vals)] = vals
    batch = {"feat_ids": feat_ids, "a_ids": a_ids, "a_int_ids": a_int, "a_int_off": a_off, "u_ids": u_ids, "u_wgt": u_wgt}
    labels = np.asarray([d["y"][i] for i in idx], dtype=np.float32)
    return {k: torch.from_numpy(v).to(device) for k, v in batch.items()}, torch.from_numpy(labels).to(device), n


def index_stream(n: int, num_epochs: int, batch_size: int) -> Iterator[List[int]]:
    """repeat(num_epochs) then batch(batch_size): batches straddle epochs; the last one may be partial (DIN.py:93-94)"""
    cur: List[int] = []
    for _ in range(num_epochs):
        for i in range(n):
            cur.append(i)
            if len(cur) == batch_size:
                yield cur
                cur = []
    if cur:
        yield cur


def run():
    from .din import DIN
    if FLAGS.dt_dir == "":
        FLAGS.dt_dir = (date.today() + timedelta(-1)).strftime("%Y%m%d")
    FLAGS.model_dir = FLAGS.model_dir + FLAGS.dt_dir
    for k in ("task_type", "model_dir", "data_dir", "dt_dir", "num_epochs", "feature_size", "field_size", "embedding_size",
              "batch_size", "deep_layers", "dropout", "attention_pooling", "attention_layers", "loss_type", "optimizer",
              "learning_rate", "batch_norm_decay", "batch_norm", "l2_reg"):
        print(k + " ", getattr(FLAGS, k))
    if FLAGS.dist_mode != 0:
        raise SystemExit("dist_mode=%d: the TF_CONFIG parameter-server modes are not provided (DESIGN.md 7)" % FLAGS.dist_mode)
    tr_files = glob.glob("%s/tr/*tfrecord" % FLAGS.data_dir)
    random.shuffle(tr_files)
    print("tr_files:", tr_files)
    va_files = glob.glob("%s/te/*tfrecord" % FLAGS.data_dir)
    print("va_files:", va_files)
    te_files = glob.glob("%s/te/*tfrecord" % FLAGS.data_dir)
    print("te_files:", te_files)
    if FLAGS.clear_existing_model:
        try:
            shutil.rmtree(FLAGS.model_dir)
        except Exception as e:  # noqa: BLE001
            print(e, "at clear_existing_model")
        else:
            print("existing model cleaned at %s" % FLAGS.model_dir)
    F, B = FLAGS.field_size, FLAGS.batch_size
    tr = decode_tfrecord_files(tr_files, F) if FLAGS.task_type == "train" else None
    te = decode_tfrecord_files(te_files, F) if te_files else None
    P, A = max_lengths(*[x for x in (tr, te) if x is not None])
    meta_path = os.path.join(FLAGS.model_dir, "din_shapes.json")
    if os.path.exists(meta_path):     # buffers are sized at first training; later tasks must not shrink them
        m = json.load(open(meta_path))
        P, A = max(P, m["P"]), max(A, m["max_a_int"])
    model = DIN(F, FLAGS.feature_size, FLAGS.embedding_size, B, P, max_a_int=A, deep_layers=FLAGS.deep_layers,
                dropout=FLAGS.dropout, attention_layers=FLAGS.attention_layers, attention_pooling=FLAGS.attention_pooling,
                l2_reg=FLAGS.l2_reg, learning_rate=FLAGS.learning_rate, optimizer=FLAGS.optimizer,
                update_mode=FLAGS.update_mode, batch_norm=FLAGS.batch_norm, batch_norm_decay=FLAGS.batch_norm_decay)
    restore_checkpoint(model, FLAGS.model_dir)
    dev = model.device

    def score(d) -> Tuple[np.ndarray, np.ndarray]:
        preds, labs = [], []
        for idx in index_stream(len(d["y"]), 1, B):
            batch, labels, n = make_batch(d, idx, B, P, dev)
            preds.append(model.predict(batch)[:n].cpu().numpy().copy()); labs.append(labels[:n].cpu().numpy())
        model.check_ids()
        return (np.concatenate(preds), np.concatenate(labs)) if preds else (np.zeros(0, np.float32), np.zeros(0, np.float32))

    def evaluate(d):
        p, t = score(d)
        if not len(p):
            return {}
        pc = np.clip(p.astype(np.float64), 1e-12, 1 - 1e-12)
        return {"auc": auc_200(t, p), "loss_ce": float(-(t * np.log(pc) + (1 - t) * np.log(1 - pc)).mean()),
                "global_step": model.global_step}

    if FLAGS.task_type == "train":
        t0, s0, last = time.time(), model.global_step, None
        for idx in index_stream(len(tr["y"]), FLAGS.num_epochs, B):
            batch, labels, n = make_batch(tr, idx, B, P, dev)
            last = model.train_step(batch, labels, n_valid=n)      # the final batch may be partial (kept, DIN.py:93-94)
            if model.global_step % FLAGS.log_steps == 0:
                dt = time.time() - t0
                print("INFO:global_step/sec: %g" % ((model.global_step - s0) / dt))
                print("INFO:loss = %s, step = %d" % (model.loss_value(last), model.global_step))
                t0, s0 = time.time(), model.global_step
        model.check_ids()
        if last is not None:
            print("INFO:Loss for final step: %s." % model.loss_value(last))
        save_checkpoint(model, FLAGS.model_dir)
        json.dump({"P": P, "max_a_int": A}, open(meta_path, "w"))
        if te is not None:
            print("INFO:Saving dict for global step %d: %s" % (model.global_step, json.dumps(evaluate(te))))
    elif FLAGS.task_type == "eval":
        print(json.dumps(evaluate(te)))
    elif FLAGS.task_type == "infer":
        p, _ = score(te)
        with open(FLAGS.data_dir + "/pred.txt", "w") as fo:
            for prob in p:
                fo.write("%f\n" % prob)
    elif FLAGS.task_type == "export":
        out_dir = os.path.join(FLAGS.servable_model_dir, str(int(time.time())))
        os.makedirs(out_dir, exist_ok=True)
        torch.save({k: v.detach().cpu() for k, v in model.variables().items()}, os.path.join(out_dir, "variables.pt"))
        sig = {"model": "DIN", "signature": "serving_default",     # DIN.py:383-391 declares feat_ids / feat_vals (quirk Q6)
               "inputs": {"feat_ids": {"dtype": "int64", "shape": [None, F]}, "feat_vals": {"dtype": "float32", "shape": [None, F]}},
               "outputs": {"prob": {"dtype": "float32", "shape": [None]}},
               "params": {k: v for k, v in FLAGS._items().items() if isinstance(v, (int, float, str, bool))}}
        json.dump(sig, open(os.path.join(out_dir, "signature.json"), "w"), indent=1)
        print("exported to", out_dir)
    return model
