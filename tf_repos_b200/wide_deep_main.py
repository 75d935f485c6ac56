"""main(_) / input_fn of deep_ctr/Model_pipeline/wide_n_deep.py:55-82,181-242 on the H100 engine.

CSV input (wide_n_deep.py:55-82): tf.decode_csv with record_defaults [[0.0]] + 13*[[0.0]] + 26*[[0]] -> label
`is_click`, I1..I13 float, C14..C39 int; TextLineDataset -> map -> repeat(num_epochs) -> batch (batches straddle
files and epochs, the last partial batch is kept); no shuffle.  Task types `train`, `predict`, `export_model`
(the dispatch strings of wide_n_deep.py:217-233; the flag help says {train, predict, export}).
"""
from __future__ import annotations

import glob
import io
import json
import os
import random
import shutil
import time
from datetime import date, timedelta
from typing import Iterator, List, Sequence, Tuple

import numpy as np
import torch

from . import ops, text_chunks
from .estimator import auc_200
from .flags import FLAGS, input_parse_device

N_NUM, N_CAT = 13, 26


def _decode_csv_lines(fh, path: str, line_base: int = 0):
    """The lines of text stream fh -> (labels, dense, cat) as decode_csv_file returns them, and how many lines were
    read; line_base = lines of `path` before fh's first one (error positions are file lines)."""
    labels: List[float] = []
    dense: List[List[float]] = []
    cat: List[List[int]] = []
    n_lines = 0
    for ln, line in enumerate(fh, line_base + 1):
        n_lines += 1
        line = line.rstrip("\r\n")
        if line == "":
            continue
        cols = line.split(",")
        if len(cols) != 1 + N_NUM + N_CAT:
            raise ValueError("%s:%d: Expect %d fields but have %d in record" % (path, ln, 1 + N_NUM + N_CAT, len(cols)))
        labels.append(float(cols[0]) if cols[0].strip() else 0.0)
        dense.append([float(c) if c.strip() else 0.0 for c in cols[1:1 + N_NUM]])
        cat.append([int(c) if c.strip() else 0 for c in cols[1 + N_NUM:]])
    return (np.asarray(labels, dtype=np.float32), np.asarray(dense, dtype=np.float32).reshape(-1, N_NUM),
            np.asarray(cat, dtype=np.int64).astype(np.int32).reshape(-1, N_CAT)), n_lines


def decode_csv_file(path: str) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """-> labels f32 [n], dense f32 [n,13], cat int32 [n,26].  Empty fields take the record defaults; a line
    without exactly 40 fields is an error (tf.decode_csv raises InvalidArgument)."""
    with open(path, "r") as fh:
        return _decode_csv_lines(fh, path)[0]


def decode_csv_bytes(data: bytes, path: str, line_base: int = 0):
    """decode_csv_file of a piece of `path` (whole lines, line_base lines of the file before it):
    -> (labels, dense, cat, lines in the piece), with the file's own line numbers in the error messages."""
    with io.TextIOWrapper(io.BytesIO(data)) as fh:      # the decoding and line ends of open(path, "r")
        arrays, n_lines = _decode_csv_lines(fh, path, line_base)
    return arrays + (n_lines,)


CSV_CHUNK = 16 << 20  # bytes of text per piece of the device path


def _tokenize(path, text, n_bytes):
    max_rows = n_bytes // (1 + N_NUM + N_CAT) + 1      # an accepted line: 39 ',' and a '\n' (the last: maybe not)
    ws = text_chunks.scratch(ops.parse_csv_device_workspace_bytes(n_bytes, max_rows), text.device)
    labels, dense, cat, info = ops.parse_csv_device(text, n_bytes, 1 + N_NUM, N_CAT, max_rows, ws)
    return (dense, cat, labels), info


def _decode(path, data, line_base):
    labels, dense, cat, n_lines = decode_csv_bytes(data, path, line_base)
    return (dense, cat, labels), n_lines


def _host_parts(files: Sequence[str], num_epochs: int):
    for _ in range(num_epochs):
        for path in files:
            labels, dense, cat = decode_csv_file(path)
            yield torch.from_numpy(dense), torch.from_numpy(cat), torch.from_numpy(labels)


def input_fn(filenames: Sequence[str], num_epochs: int, batch_size: int = 1, device=None,
             chunk_bytes: int = CSV_CHUNK) -> Iterator[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]]:
    """yields (dense f32 [B,13], cat int32 [B,26], labels f32 [B]).  device=None: host decoder, host tensors.
    device="cuda[:i]": the text is streamed to the GPU in pieces of chunk_bytes and tokenised there
    (ctr_parse_csv_device, a declined piece decoded by decode_csv_bytes); batches are CUDA tensors.  Identical values
    either way."""
    print("Parsing", filenames)
    files = [filenames] if isinstance(filenames, str) else list(filenames)
    if device is not None:
        parts = text_chunks.device_parts(files, num_epochs, torch.device(device), chunk_bytes, _tokenize, _decode)
    else:
        parts = _host_parts(files, num_epochs)
    yield from text_chunks.batches(parts, batch_size)


def _ckpt(model_dir: str) -> str:
    return os.path.join(model_dir, "ctr_b200_wide_deep.ckpt")


def save_checkpoint(model, model_dir: str):
    os.makedirs(model_dir, exist_ok=True)
    st = {"variables": {k: v.detach().cpu().clone() for k, v in model.variables().items()}, "global_step": model.global_step,
          "slots": {}}
    if model.has_dnn:
        st["slots"]["emb"] = [s.cpu() for s in model.emb.slots]
        st["slots"]["dense_dnn"] = [s.cpu() for s in model.dense_dnn.slots]
    if model.has_linear:
        st["slots"]["wide_cat"] = [s.cpu() for s in model.wide_cat.slots]
        st["slots"]["dense_lin"] = [s.cpu() for s in model.dense_lin.slots]
    torch.save(st, _ckpt(model_dir))


def restore_checkpoint(model, model_dir: str) -> bool:
    p = _ckpt(model_dir)
    if not os.path.exists(p):
        return False
    st = torch.load(p, map_location="cpu")
    model.load_variables(st["variables"])
    for key, slots in st["slots"].items():
        owner = getattr(model, key)
        for dst, src in zip(owner.slots, slots):
            dst.copy_(src)
    model.global_step = int(st["global_step"])
    print("restored checkpoint %s at global_step %d" % (p, model.global_step))
    return True


def run():
    from .wide_deep import WideDeep
    if FLAGS.dt_dir == "":
        FLAGS.dt_dir = (date.today() + timedelta(-1)).strftime("%Y%m%d")
    FLAGS.model_dir = FLAGS.model_dir + FLAGS.dt_dir
    for k in ("task_type", "model_type", "model_dir", "servable_model_dir", "dt_dir", "data_dir", "num_epochs",
              "embedding_size", "deep_layers", "batch_size"):
        print(k + " ", getattr(FLAGS, k))
    if FLAGS.dist_mode:
        raise SystemExit("dist_mode: the TF_CONFIG parameter-server mode (wide_n_deep.py:153-178) is not provided; "
                         "multi-GPU training exists for DeepFM only (DESIGN.md 7)")
    tr_files = glob.glob("%s/tr*csv" % FLAGS.data_dir)
    random.shuffle(tr_files)
    print("tr_files:", tr_files)
    va_files = glob.glob("%s/va*csv" % FLAGS.data_dir)
    print("va_files:", va_files)
    te_files = glob.glob("%s/te*csv" % FLAGS.data_dir)
    print("te_files:", te_files)
    if FLAGS.clear_existing_model:
        try:
            shutil.rmtree(FLAGS.model_dir)
        except Exception as e:  # noqa: BLE001
            print(e, "at clear_existing_model")
        else:
            print("existing model cleaned at %s" % FLAGS.model_dir)
    model = WideDeep(FLAGS.embedding_size, FLAGS.batch_size, FLAGS.deep_layers, FLAGS.model_type)
    restore_checkpoint(model, FLAGS.model_dir)
    dev = model.device

    parse_dev = input_parse_device(dev)

    def batches(files, epochs):
        for batch in input_fn(files, epochs, FLAGS.batch_size, device=parse_dev):
            yield batch if parse_dev is not None else tuple(t.to(dev) for t in batch)

    def evaluate(files):
        preds, labs = [], []
        for dense, cat, labels in batches(files, 1):
            preds.append(model.predict(dense, cat).cpu().numpy().copy()); labs.append(labels.cpu().numpy())
        if not preds:
            return {}
        p, t = np.concatenate(preds), np.concatenate(labs)
        pc = np.clip(p.astype(np.float64), 1e-12, 1 - 1e-12)
        return {"auc": auc_200(t, p), "average_loss": float(-(t * np.log(pc) + (1 - t) * np.log(1 - pc)).mean()),
                "global_step": model.global_step}

    if FLAGS.task_type == "train":
        t0, s0, last = time.time(), model.global_step, None
        for dense, cat, labels in batches(tr_files, FLAGS.num_epochs):
            last = model.train_step(dense, cat, labels)
            if model.global_step % FLAGS.log_steps == 0:
                dt = time.time() - t0
                print("INFO:global_step/sec: %g" % ((model.global_step - s0) / dt))
                print("INFO:loss = %s, step = %d" % (float(last), model.global_step))
                t0, s0 = time.time(), model.global_step
        if last is not None:
            print("INFO:Loss for final step: %s." % float(last))
        save_checkpoint(model, FLAGS.model_dir)
        if va_files:
            print("INFO:Saving dict for global step %d: %s" % (model.global_step, json.dumps(evaluate(va_files))))
    elif FLAGS.task_type == "predict":
        with open(FLAGS.data_dir + "/pred.txt", "w") as fo:
            for dense, cat, _ in batches(te_files, 1):
                for prob in model.predict(dense, cat).cpu().numpy():
                    fo.write("%f\n" % prob)
    elif FLAGS.task_type == "export_model":
        os.makedirs(FLAGS.servable_model_dir, exist_ok=True)
        torch.save({"variables": {k: v.detach().cpu().clone() for k, v in model.variables().items()},
                    "signature": {"inputs": ["is_click?"] + ["I%d" % i for i in range(1, 14)] + ["C%d" % i for i in range(14, 40)],
                                  "outputs": ["probabilities"]},
                    "model_type": FLAGS.model_type},
                   os.path.join(FLAGS.servable_model_dir, "saved_model.pt"))
        print("exported to", FLAGS.servable_model_dir)
    else:
        print("task_type must be one of {train, predict, export_model}")
