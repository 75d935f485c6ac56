#!/usr/bin/env python
"""Times the GPU Criteo feature pipeline (Feature_pipeline/get_criteo_feature.py) on a seeded synthetic raw Criteo
dataset sized like a user's (default 10 M train lines, about 3 GB; Kaggle's train.txt is 45.8 M lines / 11 GB).

Reports the device time of each pass (CUDA events around the library calls), the GB/s of raw text each pass reads over
its device time, lines/s and the wall clock of the whole preprocess() including file reads and writes, with the card's
name and power limit read in the same run.  The CPU baseline is oracle/criteo_feature.py (the pure-Python restatement
of the reference script) on the first `--cpu_lines` lines, and the sha256 of the GPU and CPU outputs on that cut must
match.  Generated data goes to --data_dir (deleted afterwards unless --keep); one JSON line is printed and, with
--json, written there."""
import argparse
import hashlib
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
    return name, power


def _digests(prefix):
    out = {}
    for n in ("tr.libsvm", "va.libsvm", "te.libsvm"):
        out[n] = hashlib.sha256(open(prefix + n, "rb").read()).hexdigest()
    fmap = b"\n".join(sorted(open(prefix + "feature_map", "rb").read().splitlines()))
    out["feature_map(sorted lines)"] = hashlib.sha256(fmap).hexdigest()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lines", type=int, default=10_000_000)
    ap.add_argument("--test_lines", type=int, default=1_500_000)
    ap.add_argument("--cpu_lines", type=int, default=200_000)
    ap.add_argument("--cutoff", type=int, default=200)
    ap.add_argument("--chunk_mb", type=int, default=64)
    ap.add_argument("--data_dir", default="")
    ap.add_argument("--keep", action="store_true")
    ap.add_argument("--json", default="")
    a = ap.parse_args()

    import torch
    from oracle import criteo_feature as ocf
    from tests.test_gpu_criteo_feature import write_raw
    from tf_repos_b200.criteo_feature import preprocess

    if not torch.cuda.is_available():
        raise SystemExit("bench_criteo_etl: needs a CUDA device")
    d = (a.data_dir or tempfile.mkdtemp(prefix="criteo_etl_")).rstrip("/") + "/"
    os.makedirs(d, exist_ok=True)
    res = {}
    try:
        small, big = d + "small/", d + "big/"
        os.makedirs(small, exist_ok=True); os.makedirs(big, exist_ok=True)
        t = time.perf_counter()
        write_raw(big + "train.txt", a.lines, seed=0)
        write_raw(big + "test.txt", a.test_lines, seed=1, test=True)
        res["generate_s"] = round(time.perf_counter() - t, 1)
        # the CPU cut: the first cpu_lines train lines and a tenth as many test lines of the same data
        for name, n in (("train.txt", a.cpu_lines), ("test.txt", max(1, a.cpu_lines // 10))):
            with open(big + name, "rb") as src, open(small + name, "wb") as dst:
                for _, line in zip(range(n), src):
                    dst.write(line)

        kw = dict(cutoff=a.cutoff, chunk_bytes=a.chunk_mb << 20)
        preprocess(small, small + "gpu_", **kw)                         # warm-up: context, module load, allocator
        t = time.perf_counter()
        preprocess(small, small + "gpu_", **kw)
        gpu_small_s = time.perf_counter() - t
        t = time.perf_counter()
        ocf.preprocess(small, small + "cpu_", cutoff=a.cutoff)
        cpu_small_s = time.perf_counter() - t
        g, c = _digests(small + "gpu_"), _digests(small + "cpu_")

        name, power = _card()
        torch.cuda.synchronize()
        t = time.perf_counter()
        info = preprocess(big, big + "gpu_", **kw)
        wall = time.perf_counter() - t
        name2, power2 = _card()
        ms = info["device_ms"]
        tr_b, te_b = info["train_bytes"], info["test_bytes"]
        n_lines = info["lines"]["tr"] + info["lines"]["va"] + info["lines"]["te"]
        read = {"stats": tr_b, "vocab": 0, "emit_train": tr_b, "emit_test": te_b}
        res.update({
            "card": name, "power_limit": power, "card_after": name2, "power_limit_after": power2,
            "train_lines": a.lines, "test_lines": a.test_lines, "train_bytes": tr_b, "test_bytes": te_b,
            "cutoff": a.cutoff, "chunk_mb": a.chunk_mb, "feature_size": info["feature_size"],
            "output_bytes": sum(os.path.getsize(big + "gpu_" + n) for n in ("tr.libsvm", "va.libsvm", "te.libsvm")),
            "device_ms": {k: round(v, 2) for k, v in ms.items()},
            "device_GBps": {k: round(read[k] / (ms[k] * 1e6), 2) for k in ms if read[k] and ms[k] > 0},
            "device_ms_total": round(sum(ms.values()), 1),
            "wall_s": round(wall, 2), "lines_per_s_wall": round(n_lines / wall),
            "text_GBps_wall": round((2 * tr_b + te_b) / wall / 1e9, 3),
            "cpu_cut_lines": a.cpu_lines, "cpu_oracle_s": round(cpu_small_s, 2), "gpu_cut_wall_s": round(gpu_small_s, 3),
            "cpu_oracle_lines_per_s": round((a.cpu_lines + max(1, a.cpu_lines // 10)) / cpu_small_s),
            "sha256_match": g == c, "sha256_gpu": g,
        })
    finally:
        if not a.keep:
            shutil.rmtree(d, ignore_errors=True)
    line = json.dumps(res)
    print(line)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        open(a.json, "w").write(line + "\n")
    if not res.get("sha256_match"):
        raise SystemExit("sha256 of the GPU and CPU outputs differ on the CPU cut")


if __name__ == "__main__":
    main()
