#!/usr/bin/env python
"""Saving and restoring a DeepFM training state as a TensorFlow checkpoint (tf_checkpoint.save / restore) on one GPU,
against the engine's own format (estimator.save_checkpoint / restore_checkpoint, a torch.save pickle).

The model is DeepFM with Adam at --rows x --k (fm_v, fm_w, both Adam slots, the MLP 256,128,64 over 39 fields), with
its constructor's random variables; the state is every tensor of tf_names.tf_tensors.

  crc        ctr_crc32c_ranges over every tensor of the state in one call: device time from CUDA events (median of
             --crc_reps after a warm-up), GB/s, and the HBM read floor bytes / 3.35 TB/s (H100 SXM data sheet)
  save       wall clock of tf_checkpoint.save (CRC, device -> pinned -> file, index, state file) and its GB/s; the
             share of it that is the CRC's device time
  restore    wall clock of tf_checkpoint.restore (index checks, file -> pinned -> device, CRC) and its GB/s
  b200       the same save / restore through estimator.save_checkpoint / restore_checkpoint
The formats alternate for --rounds rounds; the files go to a temporary directory (--tmpdir) that is removed.  Results
depend on the disk and the page cache as much as on the GPU: the card's name and power limit are printed beside them.
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=20_000_000)
    ap.add_argument("--k", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--crc_reps", type=int, default=10)
    ap.add_argument("--tmpdir", default=None)
    ap.add_argument("--json", default=None, help="also write the result here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tf_checkpoint needs a GPU")
    from tf_repos_b200 import estimator, ops, tf_checkpoint, tf_names
    from tf_repos_b200.deepfm import DeepFM
    name, power = _card()
    model = DeepFM(39, a.rows, a.k, 1024, deep_layers="256,128,64", dropout="1.0,1.0,1.0", optimizer="Adam",
                   update_mode="exact", device="cuda:0")
    views = [t.reshape(-1).view(torch.uint8) for _, t in tf_names.tf_tensors(model)]
    nbytes = sum(v.numel() for v in views)
    ops.crc32c(views)
    torch.cuda.synchronize()
    times = []
    for _ in range(a.crc_reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ops.crc32c(views)
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1) / 1e3)
    crc_s = sorted(times)[len(times) // 2]
    res = {"card": name, "power_limit": power, "rows": a.rows, "k": a.k, "tensors": len(views), "state_bytes": nbytes,
           "crc_s": crc_s, "crc_GBps": nbytes / crc_s / 1e9, "crc_hbm_floor_s": nbytes / HBM_BYTES_PER_S,
           "crc_share_of_floor": (nbytes / HBM_BYTES_PER_S) / crc_s, "rounds": []}
    tmp = tempfile.mkdtemp(prefix="bench_tf_ckpt_", dir=a.tmpdir)
    try:
        for r in range(a.rounds):
            row = {}
            for fmt in ("tf", "b200"):
                d = os.path.join(tmp, fmt)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if fmt == "tf":
                    tf_checkpoint.save(model, d)
                else:
                    estimator.save_checkpoint(model, d)
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                if fmt == "tf":
                    tf_checkpoint.restore(model, d)
                else:
                    estimator.restore_checkpoint(model, d)
                torch.cuda.synchronize()
                t2 = time.perf_counter()
                row[fmt] = {"save_s": t1 - t0, "save_GBps": nbytes / (t1 - t0) / 1e9,
                            "restore_s": t2 - t1, "restore_GBps": nbytes / (t2 - t1) / 1e9}
                shutil.rmtree(d)
            row["tf"]["crc_share_of_save"] = crc_s / row["tf"]["save_s"]
            res["rounds"].append(row)
            print("round %d: %s" % (r, json.dumps(row)), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(res))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
