"""A tiny stand-in for `tf.app.flags` so that the drop-in scripts under Model_pipeline/ take exactly the
command lines of the reference (`--task_type=train --learning_rate=0.0005 ...`, deep_ctr/run.sh:11-24).
Supports --name=value, --name value, --bool, --nobool, --bool=True/False; unknown flags are an error."""
from __future__ import annotations

import sys
from typing import Any, Dict, List, Optional


class _Flags:
    def __init__(self):
        object.__setattr__(self, "_defs", {})
        object.__setattr__(self, "_vals", {})

    def _define(self, name: str, default: Any, help: str, typ):
        self._defs[name] = (typ, default, help)
        self._vals[name] = default

    def __getattr__(self, name):
        vals = object.__getattribute__(self, "_vals")
        if name in vals:
            return vals[name]
        raise AttributeError(name)  # e.g. FLAGS.chief_hosts (quirk Q1, DeepFM.py:240)

    def __setattr__(self, name, value):
        self._vals[name] = value

    def _parse(self, argv: Optional[List[str]] = None) -> List[str]:
        argv = list(sys.argv[1:] if argv is None else argv)
        rest, i = [], 0
        while i < len(argv):
            a = argv[i]
            i += 1
            if not a.startswith("--"):
                rest.append(a)
                continue
            key, eq, val = a[2:].partition("=")
            if key not in self._defs and key.startswith("no") and key[2:] in self._defs and self._defs[key[2:]][0] is bool:
                self._vals[key[2:]] = False
                continue
            if key not in self._defs:
                raise SystemExit(f"FATAL Flags parsing error: Unknown command line flag '{key}'")
            typ = self._defs[key][0]
            if typ is bool:
                self._vals[key] = True if not eq else val.lower() in ("1", "true", "t", "yes")
                continue
            if not eq:
                if i >= len(argv):
                    raise SystemExit(f"FATAL Flags parsing error: Missing value for flag --{key}")
                val = argv[i]
                i += 1
            self._vals[key] = typ(val)
        return rest

    def _items(self) -> Dict[str, Any]:
        return dict(self._vals)


FLAGS = _Flags()


def DEFINE_integer(name, default, help=""):
    FLAGS._define(name, default, help, int)


def DEFINE_float(name, default, help=""):
    FLAGS._define(name, default, help, float)


def DEFINE_string(name, default, help=""):
    FLAGS._define(name, default, help, str)


def DEFINE_boolean(name, default, help=""):
    FLAGS._define(name, default, help, bool)


def define_common(num_threads=16, embedding_size=32, batch_size=64, learning_rate=0.0005, l2_reg=0.0001,
                  deep_layers="256,128,64", dropout="0.5,0.5,0.5", loss_type=True, batch_norm=True,
                  checkpoint_format=True):
    """The flag block every libsvm script shares (DeepFM.py:34-60; per-model defaults: SURVEY.md app. B).
    checkpoint_format=False leaves out --checkpoint_format: DeepCvrMTL.py keeps the reference's flags plus only
    --update_mode / --input_parse, and its model_dir is always ctr_b200.ckpt (tf_checkpoint.save / restore serve ESMM
    from Python)."""
    DEFINE_integer("dist_mode", 0, "distribuion mode {0-loacal, 1-single_dist, 2-multi_dist}")
    DEFINE_string("ps_hosts", "", "Comma-separated list of hostname:port pairs")
    DEFINE_string("worker_hosts", "", "Comma-separated list of hostname:port pairs")
    DEFINE_string("job_name", "", "One of 'ps', 'worker'")
    DEFINE_integer("task_index", 0, "Index of task within the job")
    DEFINE_integer("num_threads", num_threads, "Number of threads")
    DEFINE_integer("feature_size", 0, "Number of features")
    DEFINE_integer("field_size", 0, "Number of fields")
    DEFINE_integer("embedding_size", embedding_size, "Embedding size")
    DEFINE_integer("num_epochs", 10, "Number of epochs")
    DEFINE_integer("batch_size", batch_size, "Number of batch size")
    DEFINE_integer("log_steps", 1000, "save summary every steps")
    DEFINE_float("learning_rate", learning_rate, "learning rate")
    DEFINE_float("l2_reg", l2_reg, "L2 regularization")
    if loss_type:
        DEFINE_string("loss_type", "log_loss", "loss type {square_loss, log_loss}")
    DEFINE_string("optimizer", "Adam", "optimizer type {Adam, Adagrad, GD, Momentum}")
    if deep_layers is not None:
        DEFINE_string("deep_layers", deep_layers, "deep layers")
    DEFINE_string("dropout", dropout, "dropout rate")
    if batch_norm:
        DEFINE_boolean("batch_norm", False, "perform batch normaization (True or False)")
    DEFINE_float("batch_norm_decay", 0.9, "decay for the moving average(recommend trying decay=0.9)")
    DEFINE_string("data_dir", "", "data dir")
    DEFINE_string("dt_dir", "", "data dt partition")
    DEFINE_string("model_dir", "", "model check point dir")
    DEFINE_string("servable_model_dir", "", "export servable model for TensorFlow Serving")
    DEFINE_string("task_type", "train", "task type {train, infer, eval, export}")
    DEFINE_boolean("clear_existing_model", False, "clear existing model or not")
    # engine-only flag (not in the reference): how the TF-exact table update is scheduled
    DEFINE_string("update_mode", "exact_deferred", "{exact, exact_deferred, lazy}: see tf_repos_b200/engine.py (SparseUpdater)")
    DEFINE_string("input_parse", "device", "{device, host}: where the libsvm text is tokenised (same values)")
    if checkpoint_format:   # engine-only flag: which program reads model_dir (ctr_b200.ckpt, or TensorFlow's V2 bundles)
        DEFINE_string("checkpoint_format", "b200", "{b200, tf}: ctr_b200.ckpt, or TensorFlow checkpoints "
                      "(model.ckpt-<step>.index/.data-*, see tf_repos_b200/tf_checkpoint.py)")


def input_parse_device(dev):
    """--input_parse, where the input text is tokenised: dev for "device", None (the host parser) for "host".  Any
    other value stops the script."""
    if FLAGS.input_parse not in ("device", "host"):
        raise SystemExit("input_parse must be one of {device, host}")
    return dev if FLAGS.input_parse == "device" else None
