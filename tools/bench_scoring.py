#!/usr/bin/env python
"""Eval / infer scoring on the GPU (DESIGN.md §6): kernel times of ctr_auc_counts and ctr_format_preds, then DeepFM.py
--task_type=infer and eval end to end, the device path against the host loops it replaced.

Kernels: CUDA events over REPS launches on N synthetic CTR-like probabilities (p = u^6, labels ~ Bernoulli(p)); GB/s
against the bytes the kernel must move: 8 B read per sample for the counts, 4 B read plus the text written per row for
the format.  End to end: LINES Criteo-layout libsvm lines (39 pairs, the bench_libsvm.py layout; a 200 000-line file
repeated) as te and va; each of `new` (estimator.run as shipped) and `old` (the per-batch host copies, auc_200, the
numpy loss and the "%f" loop, restated below) runs in its own process, alternated, ROUNDS rounds; the time is a host
clock from before the model is built to after the output exists.  Both must produce the same pred.txt bytes and the
same eval JSON.  Prints one JSON line; --out writes it to a file too."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DRIVER = r'''
import glob, json, os, runpy, sys, time
import numpy as np
ROOT, MODE = sys.argv[1:3]
sys.argv = ["DeepFM.py"] + sys.argv[3:]
sys.path.insert(0, ROOT)
import torch
mod = runpy.run_path(os.path.join(ROOT, "Model_pipeline", "DeepFM.py"), run_name="flags_only")
from tf_repos_b200 import estimator as est
from tf_repos_b200.flags import FLAGS, input_parse_device
real_run, captured = est.run, {}
est.run = lambda build, name: captured.setdefault("build", build)
mod["main"]()
torch.zeros(1, device="cuda"); torch.cuda.synchronize()        # CUDA context outside the timed window
t0 = time.perf_counter()
if MODE == "new":
    real_run(captured["build"], "DeepFM")
else:                       # estimator.run's eval / infer before the device path
    from tf_repos_b200.input_fn import input_fn
    from tf_repos_b200.estimator import auc_200
    FLAGS.model_dir = FLAGS.model_dir + FLAGS.dt_dir
    model = captured["build"]()
    est.restore_checkpoint(model, FLAGS.model_dir)
    dev, F = model.device, FLAGS.field_size
    parse_dev = input_parse_device(dev)
    def batches(files):
        for feats, labels in input_fn(files, num_epochs=1, batch_size=FLAGS.batch_size, field_size=F, device=parse_dev):
            yield (feats["feat_ids"].reshape(-1, F).to(dev, non_blocking=True),
                   feats["feat_vals"].reshape(-1, F).to(dev, non_blocking=True), labels.to(dev, non_blocking=True))
    if FLAGS.task_type == "eval":
        preds, labs, losses = [], [], []
        for ids, vals, labels in batches(glob.glob("%s/va*libsvm" % FLAGS.data_dir)):
            p = model.predict(ids, vals)
            y = model.y[: ids.shape[0]].cpu().numpy().astype(np.float64)
            t = labels.cpu().numpy()
            losses.append(np.maximum(y, 0) - y * t + np.log1p(np.exp(-np.abs(y))))
            preds.append(p.cpu().numpy().copy()); labs.append(t)
        model.check_ids()
        preds, labs = np.concatenate(preds), np.concatenate(labs)
        print(json.dumps({"auc": auc_200(labs, preds), "loss_ce": float(np.concatenate(losses).mean()),
                          "global_step": model.global_step}))
    else:
        with open(FLAGS.data_dir + "/pred.txt", "w") as fo:
            for ids, vals, _ in batches(glob.glob("%s/te*libsvm" % FLAGS.data_dir)):
                for prob in model.predict(ids, vals).cpu().tolist():
                    fo.write("%f\n" % prob)
        model.check_ids()
torch.cuda.synchronize()
print("SECONDS %.6f" % (time.perf_counter() - t0))
'''


def kernel_times(n: int, reps: int) -> dict:
    from tf_repos_b200 import ops
    from tf_repos_b200.estimator import auc_thresholds
    g = torch.Generator(device="cuda").manual_seed(1)
    p = torch.rand(n, generator=g, device="cuda").pow(6)
    y = (torch.rand(n, generator=g, device="cuda") < p).float()
    thr = torch.from_numpy(auc_thresholds()).cuda()
    counts = torch.zeros(2, 201, dtype=torch.int64, device="cuda")
    out = torch.empty(n * 10, dtype=torch.uint8, device="cuda")      # "0.dddddd\n": 9 bytes a row for p in [0, 1)
    off = torch.zeros(1, dtype=torch.int64, device="cuda")
    ws = torch.empty(ops.format_preds_workspace_bytes(n), dtype=torch.uint8, device="cuda")

    def timed(fn):
        fn(); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e-3 / reps

    t_auc = timed(lambda: ops.auc_counts(p, y, thr, counts))
    t_fmt = timed(lambda: (off.zero_(), ops.format_preds(p, None, out, off, ws)))
    text = int(off.item())
    # correctness at this size: counts against numpy, the text of a sample of rows against Python's "%f"
    from tests import fixed6_oracle as fo
    counts.zero_(); ops.auc_counts(p, y, thr, counts)
    assert np.array_equal(counts.cpu().numpy(), fo.auc_histogram(p.cpu().numpy(), y.cpu().numpy(), auc_thresholds()))
    head = out[: 9 * 100_000].cpu().numpy().tobytes().decode()
    assert head == "".join("%f\n" % v for v in p[:100_000].double().tolist())
    return {"n": n, "reps": reps,
            "auc_counts": {"ms": t_auc * 1e3, "bytes": 8 * n, "GB_per_s": 8 * n / t_auc / 1e9},
            "format_preds": {"ms": t_fmt * 1e3, "bytes_read": 4 * n, "bytes_written": text,
                             "GB_per_s": (4 * n + text) / t_fmt / 1e9, "rows_per_s": n / t_fmt}}


def end_to_end(lines: int, rounds: int, tmp: str) -> dict:
    from tf_repos_b200 import synth
    base = 200_000
    ids, vals, labels = synth.criteo_batch(base, 117_581, 39, seed=3)
    data_dir = os.path.join(tmp, "data")
    os.makedirs(data_dir)
    one = os.path.join(tmp, "one.libsvm")
    synth.write_libsvm(one, ids, vals, labels)
    chunk = open(one, "rb").read()
    for name in ("te.libsvm", "va.libsvm"):
        with open(os.path.join(data_dir, name), "wb") as fh:
            for i in range(-(-lines // base)):
                fh.write(chunk if (i + 1) * base <= lines else b"".join(chunk.splitlines(True)[: lines - i * base]))
    flags = ["--field_size=39", "--feature_size=117581", "--embedding_size=32", "--batch_size=8192",
             "--deep_layers=400,400,400", "--dropout=0.5,0.5,0.5", "--data_dir=" + data_dir,
             "--model_dir=" + os.path.join(tmp, "ckpt_"), "--dt_dir=20261018"]
    res = {"lines": lines, "rounds": rounds, "flags": flags[:6]}
    for task in ("infer", "eval"):
        secs, outs = {"new": [], "old": []}, {}
        for _ in range(rounds):
            for mode in ("new", "old"):
                r = subprocess.run([sys.executable, "-c", DRIVER, ROOT, mode, "--task_type=" + task] + flags,
                                   capture_output=True, text=True, timeout=1200)
                assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
                secs[mode].append(float(r.stdout.split("SECONDS ")[-1]))
                if task == "infer":
                    outs[mode] = open(os.path.join(data_dir, "pred.txt"), "rb").read()
                else:
                    outs[mode] = [ln for ln in r.stdout.splitlines() if ln.startswith("{")][-1]
        assert outs["new"] == outs["old"], task
        res[task] = {m: {"seconds": s, "lines_per_s": [lines / x for x in s]} for m, s in secs.items()}
        res[task]["identical_output"] = True
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=64 << 20)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--lines", type=int, default=2_600_000)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_scoring.py measures the GPU path: no CUDA device"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    res = {"card": card, "kernels": kernel_times(a.n, a.reps)}
    with tempfile.TemporaryDirectory() as tmp:
        res["end_to_end"] = end_to_end(a.lines, a.rounds, tmp)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
