"""The observable contract of `main()` + tf.estimator in deep_ctr/Model_pipeline/DeepFM.py:284-366, on the
H100 engine: same task types (train / eval / infer / export), same file globbing (tr*libsvm, va*libsvm,
te*libsvm), same `model_dir + dt_dir` quirk (Q2), `pred.txt` with "%f\\n" per row, AUC with
tf.metrics.auc's 200 thresholds, `global_step/sec` logging every log_steps, resume from the checkpoint
in model_dir.  The tf.estimator runtime itself (hooks, summaries, TF_CONFIG parameter servers) is out of
scope (SURVEY.md 2.1); --dist_mode != 0 is rejected with a pointer to the multi-GPU engine classes."""
from __future__ import annotations

import glob
import json
import os
import random
import shutil
import time
from datetime import date, timedelta
from typing import Callable, Dict

import numpy as np
import torch

from .flags import FLAGS, input_parse_device
from .input_fn import input_fn


def auc_200(labels: np.ndarray, preds: np.ndarray) -> float:
    """tf.metrics.auc(labels, pred) defaults (DeepFM.py:194) [TF-sem]: 200 thresholds, trapezoidal ROC."""
    n = 200
    eps = 1e-7
    thr = np.array([0.0 - eps] + [(i + 1) / (n - 1) for i in range(n - 2)] + [1.0 + eps], dtype=np.float32)
    lab = labels.astype(bool)
    order = np.sort(preds.astype(np.float32))
    pos_sorted = np.sort(preds[lab].astype(np.float32))
    neg_sorted = np.sort(preds[~lab].astype(np.float32))
    tp = (len(pos_sorted) - np.searchsorted(pos_sorted, thr, side="right")).astype(np.float32)
    fp = (len(neg_sorted) - np.searchsorted(neg_sorted, thr, side="right")).astype(np.float32)
    fn = len(pos_sorted) - tp
    tn = len(neg_sorted) - fp
    e = np.float32(1e-6)
    rec = (tp + e) / (tp + fn + e)
    fpr = fp / (fp + tn + e)
    del order
    return float(np.sum((fpr[: n - 1] - fpr[1:]) * (rec[: n - 1] + rec[1:]) / 2.0))


def _ckpt_path(model_dir: str) -> str:
    return os.path.join(model_dir, "ctr_b200.ckpt")


def _tf_format() -> bool:
    """--checkpoint_format=tf: model_dir holds TensorFlow bundles (tf_checkpoint.py) instead of ctr_b200.ckpt."""
    fmt = getattr(FLAGS, "checkpoint_format", "b200")
    if fmt not in ("b200", "tf"):
        raise SystemExit("checkpoint_format=%r: must be one of {b200, tf}" % fmt)
    return fmt == "tf"


def save_checkpoint(model, model_dir: str):
    if _tf_format():
        from . import tf_checkpoint
        tf_checkpoint.save(model, model_dir)
        return
    os.makedirs(model_dir, exist_ok=True)
    state = {"variables": {k: v.detach().cpu() for k, v in model.variables().items()},
             "table_slots": {t.name: [s.cpu() for s in t.slots] for t in model.tables},
             "dense_slots": [s.cpu() for s in model.dense.slots],
             "opt_state": model.opt.state.cpu(), "global_step": model.global_step}
    torch.save(state, _ckpt_path(model_dir))


def restore_checkpoint(model, model_dir: str) -> bool:
    if _tf_format():
        from . import tf_checkpoint
        p = tf_checkpoint.latest_checkpoint(model_dir)
        if p is None:
            return False
        # a PREDICT / EVAL graph has no optimizer: only training needs the slots in the bundle
        tf_checkpoint.restore(model, p, variables_only=getattr(FLAGS, "task_type", "train") != "train")
        print("restored checkpoint %s at global_step %d" % (p, model.global_step))
        return True
    p = _ckpt_path(model_dir)
    if not os.path.exists(p):
        return False
    st = torch.load(p, map_location="cpu")
    model.load_variables(st["variables"])
    for t in model.tables:
        for dst, src in zip(t.slots, st["table_slots"][t.name]):
            dst.copy_(src)
    for dst, src in zip(model.dense.slots, st["dense_slots"]):
        dst.copy_(src)
    model.opt.state.copy_(st["opt_state"])
    model.global_step = int(st["global_step"])
    print("restored checkpoint %s at global_step %d" % (p, model.global_step))
    return True


def run(build_model: Callable[[], object], model_name: str):
    """main(_) of the reference scripts (DeepFM.py:284-366)."""
    # ------check Arguments------
    if FLAGS.dt_dir == "":
        FLAGS.dt_dir = (date.today() + timedelta(-1)).strftime("%Y%m%d")
    FLAGS.model_dir = FLAGS.model_dir + FLAGS.dt_dir          # quirk Q2 (DeepFM.py:286-288)
    for k in ("task_type", "model_dir", "data_dir", "dt_dir", "num_epochs", "feature_size", "field_size",
              "embedding_size", "batch_size", "deep_layers", "dropout", "loss_type", "optimizer", "learning_rate",
              "batch_norm_decay", "batch_norm", "l2_reg"):
        if k in FLAGS._items():
            print(k + " ", getattr(FLAGS, k))
    if FLAGS.dist_mode != 0:
        raise SystemExit("dist_mode=%d: the TF_CONFIG parameter-server modes (DeepFM.py:237-282) are replaced by "
                         "synchronous multi-GPU training (tf_repos_b200.sharded.ShardedDeepFM / DeepFM(world=N) under torchrun, "
                         "see bench.py and DESIGN.md 7); this script drives one GPU" % FLAGS.dist_mode)
    # ------init Envs------
    tr_files = glob.glob("%s/tr*libsvm" % FLAGS.data_dir)
    random.shuffle(tr_files)
    print("tr_files:", tr_files)
    va_files = glob.glob("%s/va*libsvm" % FLAGS.data_dir)
    print("va_files:", va_files)
    te_files = glob.glob("%s/te*libsvm" % FLAGS.data_dir)
    print("te_files:", te_files)
    if FLAGS.clear_existing_model:
        try:
            shutil.rmtree(FLAGS.model_dir)
        except Exception as e:  # noqa: BLE001  (same catch-all as the reference)
            print(e, "at clear_existing_model")
        else:
            print("existing model cleaned at %s" % FLAGS.model_dir)

    model = build_model()
    restore_checkpoint(model, FLAGS.model_dir)
    dev = model.device
    F = FLAGS.field_size
    parse_dev = input_parse_device(dev)

    def batches(files, epochs):
        for feats, labels in input_fn(files, num_epochs=epochs, batch_size=FLAGS.batch_size, field_size=F,
                                      device=parse_dev):
            yield (feats["feat_ids"].reshape(-1, F).to(dev, non_blocking=True),
                   feats["feat_vals"].reshape(-1, F).to(dev, non_blocking=True), labels.to(dev, non_blocking=True))

    def evaluate(files) -> Dict[str, float]:
        preds, labs, losses = [], [], []
        for ids, vals, labels in batches(files, 1):
            p = model.predict(ids, vals)
            y = model.y[: ids.shape[0]].cpu().numpy().astype(np.float64)
            t = labels.cpu().numpy()
            losses.append(np.maximum(y, 0) - y * t + np.log1p(np.exp(-np.abs(y))))        # metric only, on the host
            preds.append(p.cpu().numpy().copy()); labs.append(t)
        model.check_ids()
        if not preds:
            return {}
        preds, labs = np.concatenate(preds), np.concatenate(labs)
        return {"auc": auc_200(labs, preds), "loss_ce": float(np.concatenate(losses).mean()), "global_step": model.global_step}

    if FLAGS.task_type == "train":
        t0, s0 = time.time(), model.global_step
        t_ckpt = time.time()          # RunConfig default save_checkpoints_secs = 600 (the reference does not override it)
        last = None
        for ids, vals, labels in batches(tr_files, FLAGS.num_epochs):
            step_fn = getattr(model, "train_step_graphed", model.train_step)   # full batches replay a CUDA graph
            last = step_fn(ids, vals, labels)
            if model.global_step % FLAGS.log_steps == 0:
                model.check_ids()       # TF fails on the first bad batch; here: at the next log point, before more damage
                if time.time() - t_ckpt >= 600.0:
                    save_checkpoint(model, FLAGS.model_dir)
                    print("INFO:Saving checkpoints for %d into %s." % (model.global_step, FLAGS.model_dir))
                    t_ckpt = time.time()
                dt = time.time() - t0
                print("INFO:global_step/sec: %g  samples/sec: %g" % ((model.global_step - s0) / dt,
                                                                      (model.global_step - s0) * FLAGS.batch_size / dt))
                print("INFO:loss = %s, step = %d" % (model.loss_value(last), model.global_step))
                t0, s0 = time.time(), model.global_step
        model.check_ids()
        if last is not None:
            print("INFO:Loss for final step: %s." % model.loss_value(last))
        save_checkpoint(model, FLAGS.model_dir)
        if va_files:
            print("INFO:Saving dict for global step %d: %s" % (model.global_step, json.dumps(evaluate(va_files))))
    elif FLAGS.task_type == "eval":
        print(json.dumps(evaluate(va_files)))
    elif FLAGS.task_type == "infer":
        with open(FLAGS.data_dir + "/pred.txt", "w") as fo:                  # DeepFM.py:351-353
            for ids, vals, _ in batches(te_files, 1):
                for prob in model.predict(ids, vals).cpu().tolist():
                    fo.write("%f\n" % prob)
        model.check_ids()
    elif FLAGS.task_type == "export":
        out_dir = os.path.join(FLAGS.servable_model_dir, str(int(time.time())))
        os.makedirs(out_dir, exist_ok=True)
        torch.save({k: v.detach().cpu() for k, v in model.variables().items()}, os.path.join(out_dir, "variables.pt"))
        sig = {"model": model_name, "signature": "serving_default",                      # DeepFM.py:361-366
               "inputs": {"feat_ids": {"dtype": "int64", "shape": [None, F]},
                          "feat_vals": {"dtype": "float32", "shape": [None, F]}},
               "outputs": {"prob": {"dtype": "float32", "shape": [None]}},
               "params": {k: v for k, v in FLAGS._items().items() if isinstance(v, (int, float, str, bool))}}
        json.dump(sig, open(os.path.join(out_dir, "signature.json"), "w"), indent=1)
        print("exported to", out_dir)
    return model
