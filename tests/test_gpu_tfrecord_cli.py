"""DIN.py and DeepCvrMTL.py, which read their TFRecords on the GPU, against the same model class trained in a plain
Python process on the host decoder's make_batch batches with the same flags: the checkpoint (variables, optimizer slots,
global step) bit for bit, and pred.txt byte for byte."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = 11

# the flags exactly as the script parses them, the host decoder's batches, then train / save / restore / score as
# din_main.run and esmm_main.run do
REFERENCE = r'''
import json, os, runpy, sys
import numpy as np
ROOT, SCRIPT, TR, TE, OUT = sys.argv[1:6]
sys.argv = [SCRIPT] + sys.argv[6:]
sys.path.insert(0, ROOT)
runpy.run_path(os.path.join(ROOT, "Model_pipeline", SCRIPT), run_name="flags_only")
from tf_repos_b200.flags import FLAGS
FLAGS._parse()
from tf_repos_b200 import din_main as dm, esmm_main as em
from tf_repos_b200.estimator import restore_checkpoint, save_checkpoint
F, B = FLAGS.field_size, FLAGS.batch_size
if SCRIPT == "DIN.py":
    from tf_repos_b200.din import DIN
    tr, te = dm.decode_tfrecord_files([TR], F), dm.decode_tfrecord_files([TE], F)
    P, A = dm.max_lengths(tr, te)
    make = lambda: DIN(F, FLAGS.feature_size, FLAGS.embedding_size, B, P, max_a_int=A, deep_layers=FLAGS.deep_layers,
                       dropout=FLAGS.dropout, attention_layers=FLAGS.attention_layers,
                       attention_pooling=FLAGS.attention_pooling, l2_reg=FLAGS.l2_reg, learning_rate=FLAGS.learning_rate,
                       optimizer=FLAGS.optimizer, update_mode=FLAGS.update_mode, batch_norm=FLAGS.batch_norm,
                       batch_norm_decay=FLAGS.batch_norm_decay)
    batch_of = lambda d, idx, dev: dm.make_batch(d, idx, B, P, dev)
else:
    from tf_repos_b200.esmm import ESMM
    tr, te = em.decode([TR], F), em.decode([TE], F)
    cap = max(1, em.max_batch_occurrences(tr, FLAGS.num_epochs, B), em.max_batch_occurrences(te, 1, B))
    make = lambda: ESMM(F, FLAGS.feature_size, FLAGS.embedding_size, B, cap, deep_layers=FLAGS.deep_layers,
                        dropout=FLAGS.dropout, ctr_task_wgt=FLAGS.ctr_task_wgt, l2_reg=FLAGS.l2_reg,
                        learning_rate=FLAGS.learning_rate, optimizer=FLAGS.optimizer, update_mode=FLAGS.update_mode,
                        batch_norm=FLAGS.batch_norm, batch_norm_decay=FLAGS.batch_norm_decay)
    batch_of = lambda d, idx, dev: em.make_batch(d, idx, B, dev)
model = make()
for idx in dm.index_stream(len(tr["y"]), FLAGS.num_epochs, B):
    batch, labels, n = batch_of(tr, idx, model.device)
    model.train_step(batch, labels, n_valid=n)
model.check_ids()
save_checkpoint(model, OUT)
model = make()
restore_checkpoint(model, OUT)
with open(os.path.join(OUT, "pred.txt"), "w") as fo:
    for idx in dm.index_stream(len(te["y"]), 1, B):
        batch, labels, n = batch_of(te, idx, model.device)
        if SCRIPT == "DIN.py":
            for p in model.predict(batch)[:n].cpu().numpy():
                fo.write("%f\n" % p)
        else:
            p = model.predict(batch, None, n)
            for a, b in zip(p[0][:n].cpu().numpy(), p[1][:n].cpu().numpy()):
                fo.write("%f\t%f\n" % (a, b))
'''


def _write(path, n, seed, N=5000, maxlen=12):
    from tf_repos_b200 import tfrecord as tfr
    rng = np.random.RandomState(seed)
    recs = []
    for _ in range(n):
        y = np.float32(rng.rand() < 0.4)
        ex = {"y": y, "z": np.float32(y * (rng.rand() < 0.5)), "feat_ids": rng.randint(1, N, F).astype(np.int64),
              "a_catids": np.int64(rng.randint(1, N)), "a_shopids": np.int64(rng.randint(1, N)),
              "a_brandids": np.int64(rng.randint(1, N)), "a_intids": rng.randint(1, N, rng.randint(0, 5)).astype(np.int64)}
        for f in ("cat", "shop", "brand", "int"):
            ln = rng.randint(0, maxlen + 1)
            ex["u_%sids" % f] = rng.randint(1, N, ln).astype(np.int64)
            ex["u_%svals" % f] = (rng.rand(ln) * 3).astype(np.float32)
        recs.append(tfr.encode_example(ex))
    tfr.write_records(path, recs)


def _run(args):
    r = subprocess.run([sys.executable] + args, capture_output=True, text=True, timeout=280, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout


@pytest.mark.parametrize("script, extra", [
    ("DIN.py", ["--deep_layers=16,8", "--dropout=1,1", "--attention_layers=16"]),
    ("DeepCvrMTL.py", ["--deep_layers=16,8", "--dropout=1,1", "--ctr_task_wgt=0.3"]),
])
def test_cli_equals_in_process_training_on_host_batches(tmp_path, script, extra):
    tmp = str(tmp_path)
    os.makedirs(tmp + "/data/tr"); os.makedirs(tmp + "/data/te"); os.makedirs(tmp + "/ref")
    tr, te = tmp + "/data/tr/part0.tfrecord", tmp + "/data/te/part0.tfrecord"
    _write(tr, 150, 1); _write(te, 70, 2)
    flags = ["--field_size=%d" % F, "--feature_size=5000", "--embedding_size=8", "--batch_size=32", "--num_epochs=3",
             "--log_steps=1000", "--data_dir=" + tmp + "/data", "--model_dir=" + tmp + "/ckpt/m_",
             "--dt_dir=20261015"] + extra
    script_path = os.path.join(ROOT, "Model_pipeline", script)
    _run([script_path, "--task_type=train"] + flags)
    _run([script_path, "--task_type=infer"] + flags)
    _run(["-c", REFERENCE, ROOT, script, tr, te, tmp + "/ref"] + flags)
    got = torch.load(tmp + "/ckpt/m_20261015/ctr_b200.ckpt", map_location="cpu")
    want = torch.load(tmp + "/ref/ctr_b200.ckpt", map_location="cpu")
    assert got["global_step"] == want["global_step"] == 15           # 450 samples / 32, the partial last batch kept
    assert got["variables"].keys() == want["variables"].keys()
    for k in want["variables"]:
        assert torch.equal(got["variables"][k], want["variables"][k]), k
    for name in want["table_slots"]:
        assert all(torch.equal(a, b) for a, b in zip(got["table_slots"][name], want["table_slots"][name])), name
    assert all(torch.equal(a, b) for a, b in zip(got["dense_slots"], want["dense_slots"]))
    assert torch.equal(got["opt_state"], want["opt_state"])
    pred = open(tmp + "/data/pred.txt").read()
    assert pred.count("\n") == 70 and pred == open(tmp + "/ref/pred.txt").read()
