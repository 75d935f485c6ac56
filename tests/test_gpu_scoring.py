"""ctr_auc_counts and ctr_format_preds on the device against the numpy histogram and Python's "%f", the pred.txt writer
across buffer sizes, and every drop-in script's eval / infer against the host path it replaced, from the same
checkpoint: the eval JSON value for value and pred.txt byte for byte."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import fixed6_oracle as fo
from tests.test_scoring_cpu import _auc_cases

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _thr():
    from tf_repos_b200.estimator import auc_thresholds
    return torch.from_numpy(auc_thresholds()).cuda()


def _counts(pairs):
    from tf_repos_b200 import ops
    c = torch.zeros(2, 201, dtype=torch.int64, device="cuda")
    thr = _thr()
    for p, y in pairs:
        ops.auc_counts(p, y, thr, c)
    return c.cpu().numpy()


@pytest.mark.parametrize("case", [c[0] for c in _auc_cases()])
def test_auc_counts_equal_the_numpy_histogram(case):
    from tf_repos_b200.estimator import auc_thresholds
    _, p, y = next(c for c in _auc_cases() if c[0] == case)
    pd, yd = torch.from_numpy(p).cuda(), torch.from_numpy(y).cuda()
    want = fo.auc_histogram(p, y, auc_thresholds())
    assert np.array_equal(_counts([(pd, yd)]), want)
    if len(p) > 1:   # unaligned columns: the scalar path
        assert np.array_equal(_counts([(pd[1:], yd[1:])]), fo.auc_histogram(p[1:], y[1:], auc_thresholds()))


def test_auc_counts_accumulate_16m_skewed_predictions_over_uneven_calls():
    from tf_repos_b200.estimator import auc_thresholds
    g = torch.Generator(device="cuda").manual_seed(11)
    n = 16 << 20
    p = torch.rand(n, generator=g, device="cuda").pow(6)        # CTR-like: most mass near 0
    y = (torch.rand(n, generator=g, device="cuda") < p).float()
    cuts = [0, 0, 1, 1, 2, 1000, 1 << 20, (1 << 20) + 3, 5 << 20, 5 << 20, n - 1, n]
    got = _counts([(p[a:b], y[a:b]) for a, b in zip(cuts[:-1], cuts[1:])])
    want = fo.auc_histogram(p.cpu().numpy(), y.cpu().numpy(), auc_thresholds())
    assert got.sum() == n and np.array_equal(got, want)


def _format(a, b=None, start=0, cap=None):
    from tf_repos_b200 import ops
    a = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    b = None if b is None else torch.from_numpy(np.ascontiguousarray(b)).cuda()
    n = a.numel()
    cap = cap or start + n * 48 * (1 if b is None else 2) + 64
    out = torch.full((cap,), ord("#"), dtype=torch.uint8, device="cuda")
    off = torch.tensor([start], dtype=torch.int64, device="cuda")
    ws = torch.empty(ops.format_preds_workspace_bytes(n), dtype=torch.uint8, device="cuda")
    ops.format_preds(a, b, out, off, ws)
    end = int(off.item())
    text = out.cpu().numpy().tobytes()
    assert text[:start] == b"#" * start and set(text[end:]) <= {ord("#")}
    return text[start:end].decode()


def _python(x):
    with np.errstate(invalid="ignore"):
        return "".join("%f\n" % v for v in x.astype(np.float64).tolist())


@pytest.mark.parametrize("name", ["specials", "ties", "boundaries", "random"])
def test_format_preds_equals_python_on_the_special_sets(name):
    x = {"specials": fo.specials, "ties": fo.ties_and_neighbours, "boundaries": fo.rounding_boundaries,
         "random": lambda: fo.random_patterns(1_000_000, seed=7)}[name]()
    assert _format(x) == _python(x)


def test_format_preds_every_64th_float_in_0_1():
    x = np.arange(0, 0x3F800001, 64, dtype=np.uint32).view(np.float32)
    assert _format(x) == _python(x)


def test_format_preds_two_columns_and_a_running_offset():
    a = np.concatenate([fo.specials(), fo.random_patterns(30_000, seed=1)])
    b = np.concatenate([fo.random_patterns(len(a) - 100, seed=2), fo.ties_and_neighbours(1)[:100]])
    with np.errstate(invalid="ignore"):
        want = "".join("%f\t%f\n" % (u, v) for u, v in zip(a.astype(np.float64).tolist(), b.astype(np.float64).tolist()))
    assert _format(a, b) == want
    assert _format(a, b, start=12_345) == want          # any alignment of the start
    assert _format(a[:1], start=3) == _python(a[:1])
    assert _format(a[:0], start=7) == ""


def test_format_preds_does_not_write_past_the_buffer_and_reports_it():
    from tf_repos_b200 import ops
    x = torch.full((100,), 0.5, device="cuda")
    out = torch.zeros(250, dtype=torch.uint8, device="cuda")
    off = torch.zeros(1, dtype=torch.int64, device="cuda")
    ws = torch.empty(ops.format_preds_workspace_bytes(100), dtype=torch.uint8, device="cuda")
    ops.format_preds(x, None, out, off, ws)
    assert int(off.item()) == 900 and out.cpu().numpy().tobytes() == (b"0.500000\n" * 28)[:250]


def test_writer_with_a_4k_buffer_writes_the_default_buffers_file(tmp_path):
    from tf_repos_b200.scoring import PredWriter
    g = torch.Generator(device="cuda").manual_seed(5)
    batches = [torch.rand(n, generator=g, device="cuda") for n in (1, 300, 0, 85, 86, 1000, 7, 4096, 13)]
    batches[3][5] = float("nan")
    files = {}
    for cols in (1, 2):
        for buf in (4096, None):
            path = str(tmp_path / f"{cols}_{buf}.txt")
            kw = {} if buf is None else {"buffer_bytes": buf}
            with PredWriter(path, "cuda", columns=cols, **kw) as w:
                for x in batches:
                    w.add(x) if cols == 1 else w.add(x, 1 - x)
            files[cols, buf] = open(path, "rb").read()
        assert files[cols, 4096] == files[cols, None]
    allx = torch.cat(batches).cpu().numpy()
    assert files[1, None].decode() == _python(allx)
    empty = str(tmp_path / "empty.txt")
    PredWriter(empty, "cuda").close()
    assert open(empty, "rb").read() == b""


# ---- the drop-in scripts against the host path they replaced -------------------------------------------------------
# The flags as the script parses them, the model built and restored as its run() does, then the loops the scripts ran
# before the device path: predictions copied to the host per batch, auc_200, the numpy losses and the "%f" loops.
REFERENCE = r'''
import glob, json, os, runpy, sys
import numpy as np, torch
ROOT, SCRIPT, OUT = sys.argv[1:4]
sys.argv = [SCRIPT] + sys.argv[4:]
sys.path.insert(0, ROOT)
mod = runpy.run_path(os.path.join(ROOT, "Model_pipeline", SCRIPT), run_name="flags_only")
from tf_repos_b200.flags import FLAGS, input_parse_device
from tf_repos_b200 import estimator as est
from tf_repos_b200.estimator import auc_200
captured = {}
est.run = lambda build, name: captured.setdefault("build", build)
if "main" in mod and SCRIPT not in ("DIN.py", "DeepCvrMTL.py", "wide_n_deep.py"):
    mod["main"]()                     # parses the flags and hands its model builder to (patched) run()
else:
    FLAGS._parse()
FLAGS.model_dir = FLAGS.model_dir + FLAGS.dt_dir
F, B = getattr(FLAGS, "field_size", 0), FLAGS.batch_size     # wide_n_deep has no --field_size
res, pred_path = None, os.path.join(OUT, "pred.txt")
if SCRIPT in ("DIN.py", "DeepCvrMTL.py"):
    from tf_repos_b200.din_main import max_lengths_of
    from tf_repos_b200.tfrecord_device import TFRecordIndex
    te_files = glob.glob("%s/te/*tfrecord" % FLAGS.data_dir)
    if SCRIPT == "DIN.py":
        from tf_repos_b200.din import DIN
        te = TFRecordIndex.build(te_files, F)
        P, A = max_lengths_of(te.lens)
        m = json.load(open(os.path.join(FLAGS.model_dir, "din_shapes.json")))
        P, A = max(P, m["P"]), max(A, m["max_a_int"])
        model = DIN(F, FLAGS.feature_size, FLAGS.embedding_size, B, P, max_a_int=A, deep_layers=FLAGS.deep_layers,
                    dropout=FLAGS.dropout, attention_layers=FLAGS.attention_layers, attention_pooling=FLAGS.attention_pooling,
                    l2_reg=FLAGS.l2_reg, learning_rate=FLAGS.learning_rate, optimizer=FLAGS.optimizer,
                    update_mode=FLAGS.update_mode, batch_norm=FLAGS.batch_norm, batch_norm_decay=FLAGS.batch_norm_decay)
        est.restore_checkpoint(model, FLAGS.model_dir)
        preds, labs = [], []
        for batch, labels, n in te.batches(1, B, "din", P):
            preds.append(model.predict(batch)[:n].cpu().numpy().copy()); labs.append(labels[:n].cpu().numpy())
        model.check_ids()
        p, t = np.concatenate(preds), np.concatenate(labs)
        pc = np.clip(p.astype(np.float64), 1e-12, 1 - 1e-12)
        res = {"auc": auc_200(t, p), "loss_ce": float(-(t * np.log(pc) + (1 - t) * np.log(1 - pc)).mean()),
               "global_step": model.global_step}
        with open(pred_path, "w") as fo:
            for prob in p:
                fo.write("%f\n" % prob)
    else:
        from tf_repos_b200 import _lib, ops
        from tf_repos_b200.esmm import ESMM
        te = TFRecordIndex.build(te_files, F, ("y", "z"))
        cap = max([1, te.max_batch_occurrences(1, B)])
        cap = max(cap, json.load(open(os.path.join(FLAGS.model_dir, "esmm_shapes.json")))["occ_capacity"])
        model = ESMM(F, FLAGS.feature_size, FLAGS.embedding_size, B, cap, deep_layers=FLAGS.deep_layers,
                     dropout=FLAGS.dropout, ctr_task_wgt=FLAGS.ctr_task_wgt, l2_reg=FLAGS.l2_reg,
                     learning_rate=FLAGS.learning_rate, optimizer=FLAGS.optimizer, update_mode=FLAGS.update_mode,
                     batch_norm=FLAGS.batch_norm, batch_norm_decay=FLAGS.batch_norm_decay)
        est.restore_checkpoint(model, FLAGS.model_dir)
        dev = model.device
        def score(d, with_loss):
            out, losses = {"pctr": [], "pcvr": [], "pctcvr": [], "y": [], "z": []}, []
            for batch, (y, z), n in d.batches(1, B, "esmm"):
                p = model.predict(batch, (y, z) if with_loss else None, n)
                for k, v in zip(("pctr", "pcvr", "pctcvr"), p):
                    out[k].append(v[:n].cpu().numpy().copy())
                out["y"].append(y[:n].cpu().numpy()); out["z"].append(z[:n].cpu().numpy())
                if with_loss:
                    losses.append(model.losses.tolist())
            model.check_ids()
            return {k: np.concatenate(v) for k, v in out.items()}, losses
        s, losses = score(te, True)
        reg = torch.zeros(1, dtype=torch.float32, device=dev)
        V = model.variables()["embeddings"]
        ws = torch.empty(max(int(_lib.raw().ctr_l2_loss_workspace_bytes(V.numel())), 16), dtype=torch.uint8, device=dev)
        ops.l2_loss(V, reg, ws, scale=model.l2_reg)
        l2 = float(reg.item())
        loss = float(np.mean([model.w_ctr * c + model.w_cvr * v + l2 for c, v in losses]))
        res = {"loss": loss, "CTR_AUC": auc_200(s["y"], s["pctr"]), "CVR_AUC": auc_200(s["z"], s["pcvr"]),
               "CTCVR_AUC": auc_200(s["z"], s["pctcvr"]), "global_step": model.global_step}
        s, _ = score(te, False)
        with open(pred_path, "w") as fo:
            for pctr, pcvr in zip(s["pctr"], s["pcvr"]):
                fo.write("%f\t%f\n" % (pctr, pcvr))
elif SCRIPT == "wide_n_deep.py":
    from tf_repos_b200 import wide_deep_main as wm
    from tf_repos_b200.wide_deep import WideDeep
    model = WideDeep(FLAGS.embedding_size, FLAGS.batch_size, FLAGS.deep_layers, FLAGS.model_type)
    wm.restore_checkpoint(model, FLAGS.model_dir)
    dev, parse_dev = model.device, input_parse_device(model.device)
    def batches(files):
        for batch in wm.input_fn(files, 1, B, device=parse_dev):
            yield batch if parse_dev is not None else tuple(t.to(dev) for t in batch)
    preds, labs = [], []
    for dense, cat, labels in batches(glob.glob("%s/va*csv" % FLAGS.data_dir)):
        preds.append(model.predict(dense, cat).cpu().numpy().copy()); labs.append(labels.cpu().numpy())
    p, t = np.concatenate(preds), np.concatenate(labs)
    pc = np.clip(p.astype(np.float64), 1e-12, 1 - 1e-12)
    res = {"auc": auc_200(t, p), "average_loss": float(-(t * np.log(pc) + (1 - t) * np.log(1 - pc)).mean()),
           "global_step": model.global_step}
    with open(pred_path, "w") as fo:
        for dense, cat, _ in batches(glob.glob("%s/te*csv" % FLAGS.data_dir)):
            for prob in model.predict(dense, cat).cpu().numpy():
                fo.write("%f\n" % prob)
else:
    from tf_repos_b200.input_fn import input_fn
    model = captured["build"]()
    est.restore_checkpoint(model, FLAGS.model_dir)
    dev, parse_dev = model.device, input_parse_device(model.device)
    def batches(files):
        for feats, labels in input_fn(files, num_epochs=1, batch_size=B, field_size=F, device=parse_dev):
            yield (feats["feat_ids"].reshape(-1, F).to(dev, non_blocking=True),
                   feats["feat_vals"].reshape(-1, F).to(dev, non_blocking=True), labels.to(dev, non_blocking=True))
    preds, labs, losses = [], [], []
    for ids, vals, labels in batches(glob.glob("%s/va*libsvm" % FLAGS.data_dir)):
        p = model.predict(ids, vals)
        y = model.y[: ids.shape[0]].cpu().numpy().astype(np.float64)
        t = labels.cpu().numpy()
        losses.append(np.maximum(y, 0) - y * t + np.log1p(np.exp(-np.abs(y))))
        preds.append(p.cpu().numpy().copy()); labs.append(t)
    model.check_ids()
    preds, labs = np.concatenate(preds), np.concatenate(labs)
    res = {"auc": auc_200(labs, preds), "loss_ce": float(np.concatenate(losses).mean()), "global_step": model.global_step}
    with open(pred_path, "w") as fo:
        for ids, vals, _ in batches(glob.glob("%s/te*libsvm" % FLAGS.data_dir)):
            for prob in model.predict(ids, vals).cpu().tolist():
                fo.write("%f\n" % prob)
print(json.dumps(res))
'''


def _run(args):
    r = subprocess.run([sys.executable] + args, capture_output=True, text=True, timeout=280, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout


def _libsvm_data(d):
    from tf_repos_b200 import synth
    for name, rows, seed in (("tr0.libsvm", 700, 1), ("va.libsvm", 333, 3), ("te.libsvm", 301, 4)):
        ids, vals, labels = synth.criteo_batch(rows, 10_000, 39, seed=seed)
        synth.write_libsvm(os.path.join(d, name), ids, vals, labels)


def _tfrecord_data(d):
    from tests.test_gpu_tfrecord_cli import _write
    os.makedirs(d + "/tr"); os.makedirs(d + "/te")
    _write(d + "/tr/part0.tfrecord", 150, 1); _write(d + "/te/part0.tfrecord", 70, 2)     # 70 = 2 * 32 + 6


def _csv_data(d):
    from tests.test_gpu_wide_deep_csv import _plain_line
    g = np.random.default_rng(3)
    for name, n in (("tr0.csv", 300), ("va0.csv", 61), ("te0.csv", 77)):
        open(os.path.join(d, name), "w").write("".join(_plain_line(g) + "\n" for _ in range(n)))


CLI = [
    ("DeepFM.py", _libsvm_data, ["--field_size=39", "--feature_size=10000", "--embedding_size=8", "--batch_size=128",
                                 "--deep_layers=32,16", "--dropout=0.8,0.8"]),
    ("NFM.py", _libsvm_data, ["--field_size=39", "--feature_size=10000", "--embedding_size=8", "--batch_size=128",
                              "--deep_layers=32,16", "--dropout=0.8,0.8,0.8"]),
    ("DIN.py", _tfrecord_data, ["--field_size=11", "--feature_size=5000", "--embedding_size=8", "--batch_size=32",
                                "--deep_layers=16,8", "--dropout=1,1", "--attention_layers=16"]),
    ("DeepCvrMTL.py", _tfrecord_data, ["--field_size=11", "--feature_size=5000", "--embedding_size=8",
                                       "--batch_size=32", "--deep_layers=16,8", "--dropout=1,1", "--ctr_task_wgt=0.3"]),
    ("wide_n_deep.py", _csv_data, ["--embedding_size=8", "--batch_size=32", "--deep_layers=32,16"]),
]


@pytest.mark.parametrize("script, make_data, extra", CLI, ids=[c[0] for c in CLI])
def test_cli_eval_and_infer_equal_the_host_path(tmp_path, script, make_data, extra):
    tmp = str(tmp_path)
    os.makedirs(tmp + "/data"); os.makedirs(tmp + "/ref")
    make_data(tmp + "/data")
    flags = ["--num_epochs=2", "--log_steps=1000", "--data_dir=" + tmp + "/data", "--model_dir=" + tmp + "/ckpt/m_",
             "--dt_dir=20261018"] + extra
    path = os.path.join(ROOT, "Model_pipeline", script)
    out = _run([path, "--task_type=train"] + flags)
    at_train_end = [ln for ln in out.splitlines() if ln.startswith("INFO:Saving dict")]
    assert len(at_train_end) == 1
    ref = json.loads(_run(["-c", REFERENCE, ROOT, script, tmp + "/ref"] + flags).strip().splitlines()[-1])
    assert json.loads(at_train_end[0].split(": ", 1)[1]) == ref
    if script != "wide_n_deep.py":                      # wide_n_deep evaluates only at the end of training
        assert json.loads(_run([path, "--task_type=eval"] + flags).strip().splitlines()[-1]) == ref
    _run([path, "--task_type=predict" if script == "wide_n_deep.py" else "--task_type=infer"] + flags)
    got = open(tmp + "/data/pred.txt", "rb").read()
    assert got == open(tmp + "/ref/pred.txt", "rb").read()
    assert got.count(b"\n") == {"DIN.py": 70, "DeepCvrMTL.py": 70, "wide_n_deep.py": 77}.get(script, 301)
