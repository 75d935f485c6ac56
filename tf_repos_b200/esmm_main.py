"""input_fn / main(_) of DeepMTL/Model_pipeline/DeepCvrMTL.py:63-105,314-398 on the H100 engine.

Input: TFRecord files of tf.Example (`data_dir/tr/*tfrecord`, `data_dir/te/*tfrecord`; eval files = test files,
DeepCvrMTL.py:339-345) with DIN's Ali-CCP features (decoded by din_main.decode_tfrecord_files) plus the required
conversion label z.  Batches are CSR (tf_repos_b200.esmm): the reference never densifies the var-len features.

repeat-before-batch keeps the last partial batch (:97-98): it is padded to the batch size with copies of its first
sample and trained on with `n_valid`; eval / infer drop the padded outputs.  The occurrence buffers have a fixed
capacity (every step has the same shapes): the largest occurrence count of any batch of the inputs, persisted in
`<model_dir>/esmm_shapes.json` so that later runs never shrink it.
"""
from __future__ import annotations

import glob
import json
import os
import random
import shutil
import time
from datetime import date, timedelta
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

from .din_main import U_FIELDS, decode_tfrecord_files, index_stream
from .estimator import auc_200, restore_checkpoint, save_checkpoint
from .flags import FLAGS

BAG_KEYS = tuple("u_%sids" % f for f in U_FIELDS) + ("a_int",)


def decode(files: Sequence[str], field_size: int) -> Dict[str, list]:
    """tf.parse_single_example with the spec of DeepCvrMTL.py:66-83: y and z are both required."""
    return decode_tfrecord_files(files, field_size, labels=("y", "z"))


def sample_occurrences(d: Dict[str, list]) -> np.ndarray:
    """bag occurrences of every sample (the five var-len id lists)"""
    return np.sum([[len(x) for x in d[k]] for k in BAG_KEYS], axis=0).astype(np.int64) if d["y"] else np.zeros(0, np.int64)


def max_batch_occurrences(d: Dict[str, list], num_epochs: int, B: int) -> int:
    """the largest occurrence count of any batch index_stream(n, num_epochs, B) yields, the padded last one included"""
    occ = sample_occurrences(d)
    n = len(occ)
    if n == 0 or num_epochs <= 0:
        return 0
    stream = np.tile(occ, num_epochs)
    starts = np.arange(0, len(stream), B)
    sums = np.add.reduceat(stream, starts)
    tail = len(stream) - starts[-1]
    sums[-1] += (B - tail) * stream[starts[-1]]
    return int(sums.max())


def make_batch(d: Dict[str, list], idx: Sequence[int], B: int, device) -> Tuple[Dict[str, torch.Tensor], Tuple[torch.Tensor, torch.Tensor], int]:
    """Samples `idx` (len <= B; padded to B with copies of the first sample) -> the model's CSR batch, (y, z), n real."""
    n = len(idx)
    idx = list(idx) + [idx[0]] * (B - n)
    feat_ids = np.stack([d["feat_ids"][i] for i in idx]).astype(np.int32)
    a_ids = np.asarray([[d[k][i] for i in idx] for k in ("a_cat", "a_shop", "a_brand")], dtype=np.int32)
    ids: List[np.ndarray] = []
    wgt: List[np.ndarray] = []
    for f in U_FIELDS:
        ids += [d["u_%sids" % f][i] for i in idx]
        wgt += [d["u_%svals" % f][i] for i in idx]
    ids += [d["a_int"][i] for i in idx]
    wgt += [np.ones(len(d["a_int"][i]), np.float32) for i in idx]        # a_int is unweighted: never read
    off = np.zeros(5 * B + 1, dtype=np.int32)
    off[1:] = np.cumsum([len(x) for x in ids])
    batch = {"feat_ids": feat_ids, "a_ids": a_ids,
             "bag_ids": np.concatenate(ids).astype(np.int32) if off[-1] else np.zeros(0, np.int32),
             "bag_wgt": np.concatenate(wgt).astype(np.float32) if off[-1] else np.zeros(0, np.float32),
             "bag_off": off}
    y = torch.from_numpy(np.asarray([d["y"][i] for i in idx], dtype=np.float32)).to(device)
    z = torch.from_numpy(np.asarray([d["z"][i] for i in idx], dtype=np.float32)).to(device)
    return {k: torch.from_numpy(v).to(device) for k, v in batch.items()}, (y, z), n


def run():
    from . import _lib, ops
    from .esmm import ESMM
    if FLAGS.dt_dir == "":
        FLAGS.dt_dir = (date.today() + timedelta(-1)).strftime("%Y%m%d")
    FLAGS.model_dir = FLAGS.model_dir + FLAGS.dt_dir
    for k in ("task_type", "model_dir", "data_dir", "dt_dir", "num_epochs", "feature_size", "field_size", "embedding_size",
              "batch_size", "deep_layers", "dropout", "loss_type", "optimizer", "learning_rate", "l2_reg", "ctr_task_wgt"):
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
    if FLAGS.task_type == "export":                  # DeepCvrMTL.py:383-384
        print("Not Implemented, Do It Yourself!")
        return None
    F, B = FLAGS.field_size, FLAGS.batch_size
    tr = decode(tr_files, F) if FLAGS.task_type == "train" else None
    te = decode(te_files, F) if te_files else None
    cap = max([1] + ([max_batch_occurrences(tr, FLAGS.num_epochs, B)] if tr else []) +
              ([max_batch_occurrences(te, 1, B)] if te else []))
    meta_path = os.path.join(FLAGS.model_dir, "esmm_shapes.json")
    if os.path.exists(meta_path):     # sized at first training; later tasks must not shrink it
        cap = max(cap, json.load(open(meta_path))["occ_capacity"])
    model = ESMM(F, FLAGS.feature_size, FLAGS.embedding_size, B, cap, deep_layers=FLAGS.deep_layers,
                 dropout=FLAGS.dropout, ctr_task_wgt=FLAGS.ctr_task_wgt, l2_reg=FLAGS.l2_reg,
                 learning_rate=FLAGS.learning_rate, optimizer=FLAGS.optimizer, update_mode=FLAGS.update_mode,
                 batch_norm=FLAGS.batch_norm, batch_norm_decay=FLAGS.batch_norm_decay)
    restore_checkpoint(model, FLAGS.model_dir)
    dev = model.device

    def score(d, with_loss: bool):
        out, losses = {"pctr": [], "pcvr": [], "pctcvr": [], "y": [], "z": []}, []
        for idx in index_stream(len(d["y"]), 1, B):
            batch, (y, z), n = make_batch(d, idx, B, dev)
            p = model.predict(batch, (y, z) if with_loss else None, n)
            for k, v in zip(("pctr", "pcvr", "pctcvr"), p):
                out[k].append(v[:n].cpu().numpy().copy())
            out["y"].append(y[:n].cpu().numpy()); out["z"].append(z[:n].cpu().numpy())
            if with_loss:
                losses.append(model.losses.tolist())
        model.check_ids()
        return {k: (np.concatenate(v) if v else np.zeros(0, np.float32)) for k, v in out.items()}, losses

    def evaluate(d):
        s, losses = score(d, True)
        if not len(s["y"]):
            return {}
        reg = torch.zeros(1, dtype=torch.float32, device=dev)
        V = model.variables()["embeddings"]
        ws = torch.empty(max(int(_lib.raw().ctr_l2_loss_workspace_bytes(V.numel())), 16), dtype=torch.uint8, device=dev)
        ops.l2_loss(V, reg, ws, scale=model.l2_reg)
        l2 = float(reg.item())
        # tf.metrics.mean of the per-batch loss (:223), and the three AUCs of :229-233
        loss = float(np.mean([model.w_ctr * c + model.w_cvr * v + l2 for c, v in losses]))
        return {"loss": loss, "CTR_AUC": auc_200(s["y"], s["pctr"]), "CVR_AUC": auc_200(s["z"], s["pcvr"]),
                "CTCVR_AUC": auc_200(s["z"], s["pctcvr"]), "global_step": model.global_step}

    if FLAGS.task_type == "train":
        t0, s0, last = time.time(), model.global_step, None
        for idx in index_stream(len(tr["y"]), FLAGS.num_epochs, B):
            batch, labels, n = make_batch(tr, idx, B, dev)
            last = model.train_step(batch, labels, n_valid=n)      # the final batch may be partial (kept, :97-98)
            if model.global_step % FLAGS.log_steps == 0:
                dt = time.time() - t0
                print("INFO:global_step/sec: %g" % ((model.global_step - s0) / dt))
                print("INFO:loss = %s, step = %d" % (model.loss_value(last), model.global_step))
                t0, s0 = time.time(), model.global_step
        model.check_ids()
        if last is not None:
            print("INFO:Loss for final step: %s." % model.loss_value(last))
        save_checkpoint(model, FLAGS.model_dir)
        json.dump({"occ_capacity": cap}, open(meta_path, "w"))
        if te is not None:
            print("INFO:Saving dict for global step %d: %s" % (model.global_step, json.dumps(evaluate(te))))
    elif FLAGS.task_type == "eval":
        print(json.dumps(evaluate(te)))
    elif FLAGS.task_type == "infer":
        # DeepCvrMTL.py:379-382 asks Estimator.predict for predict_keys="prob", a key the predictions dict does not
        # have (TF raises before the first line, quirk Q10); this writes what the loop evidently intends
        s, _ = score(te, False)
        with open(FLAGS.data_dir + "/pred.txt", "w") as fo:
            for pctr, pcvr in zip(s["pctr"], s["pcvr"]):
                fo.write("%f\t%f\n" % (pctr, pcvr))
    return model
