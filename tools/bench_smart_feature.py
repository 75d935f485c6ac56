#!/usr/bin/env python
"""Times the GPU smart and Frappe feature stages (Feature_pipeline/get_smart_feature.py --build_feature_map=True and
get_frape_feature.py) on seeded synthetic inputs: a 128-column smart CSV of about --gb GB (default 1) and a Frappe
libsvm file of about a fifth of that.

Reports the device time of each pass (CUDA events around the library calls), the GB/s of text each pass reads over
its device time, and lines/s over the wall clock of the whole call including file reads and writes, with the card's
name and power limit read in the same run.  The CPU baseline is oracle/smart_feature.py (the pure-Python restatement)
on the first --cpu_lines lines; the sha256 of the GPU and CPU outputs on that cut must match.  Generated data goes to
--data_dir (deleted afterwards unless --keep); one JSON line is printed and, with --json, written there."""
import argparse
import hashlib
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
    return name, power


def _pool(n, seed):
    """n distinct-ish smart lines, vectorised per column (continuous: %.5f; categorical: Zipf ids)."""
    from oracle.smart_feature import continuous
    rng = np.random.default_rng(seed)
    cols = [np.where(rng.random(n) < 0.3, b"1", b"0")]
    for i in range(1, 128):
        if continuous(i):
            cols.append(np.char.mod("%.5f", rng.random(n)).astype("S8"))
        else:
            vocab = 10_000 if i < 11 else 300
            cols.append(np.char.mod("%d", np.minimum(rng.zipf(1.3, n), vocab)).astype("S6"))
    return [b",".join(r) + b"\n" for r in zip(*[c.tolist() for c in cols])]


def _write_repeated(path, pool, target_bytes, seed):
    rng = np.random.default_rng(seed)
    n = 0
    with open(path, "wb") as fh:
        while n < target_bytes:
            block = b"".join(pool[i] for i in rng.permutation(len(pool)))
            fh.write(block)
            n += len(block)
    return n


def _frappe_pool(n, seed):
    rng = np.random.default_rng(seed)
    ids = np.sort(rng.integers(1, 5400, (n, 10)), axis=1)
    return [(b"-1 " if rng.random() < 0.66 else b"1 ") + b" ".join(b"%d:1" % v for v in r) + b"\n" for r in ids]


def _head(src, dst, lines):
    with open(src, "rb") as fi, open(dst, "wb") as fo:
        for k, line in enumerate(fi):
            if k == lines:
                break
            fo.write(line)


def _sha(path):
    return hashlib.sha256(open(path, "rb").read()).hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gb", type=float, default=1.0)
    ap.add_argument("--cpu_lines", type=int, default=20_000)
    ap.add_argument("--chunk_mb", type=int, default=64)
    ap.add_argument("--data_dir", default="")
    ap.add_argument("--keep", action="store_true")
    ap.add_argument("--json", default="")
    a = ap.parse_args()

    import torch
    from oracle import smart_feature as O
    from tf_repos_b200.smart_feature import frappe_feature, smart_feature

    if not torch.cuda.is_available():
        raise SystemExit("bench_smart_feature: needs a CUDA device")
    d = (a.data_dir or tempfile.mkdtemp(prefix="smartbench")).rstrip("/") + "/"
    chunk = a.chunk_mb << 20
    try:
        for sub in ("in", "out", "cut/in", "cut/gpu", "cut/ora", "fr", "frcut/gpu", "frcut/ora"):
            os.makedirs(d + sub, exist_ok=True)
        smart_in = d + "in/s_x_part_0"
        n_bytes = _write_repeated(smart_in, _pool(50_000, 1), int(a.gb * 1e9), 2)
        fr_in = d + "fr/frappe.libsvm"
        fr_bytes = _write_repeated(fr_in, _frappe_pool(200_000, 3), int(a.gb * 0.2e9), 4)

        torch.cuda.synchronize()
        t0 = time.perf_counter()
        g = smart_feature(d + "in", d + "out/", "tr", build_feature_map_first=True, chunk_bytes=chunk)
        wall = time.perf_counter() - t0
        n_lines = sum(v[0] for v in g["lines"].values())
        t0 = time.perf_counter()
        f = frappe_feature(d + "fr", chunk_bytes=chunk)
        fr_wall = time.perf_counter() - t0
        fr_lines = sum(v[0] for v in f["lines"].values())

        # CPU baseline and byte identity on a cut
        _head(smart_in, d + "cut/in/c_x_part_0", a.cpu_lines)
        gc = smart_feature(d + "cut/in", d + "cut/gpu/", "tr", build_feature_map_first=True, chunk_bytes=chunk)
        t0 = time.perf_counter()
        oc = O.smart_feature(d + "cut/in", d + "cut/ora/", "tr", build=True)
        cpu_s = time.perf_counter() - t0
        pairs = list(zip(gc["outputs"], oc["outputs"])) + [(d + "cut/gpu/feature_map", d + "cut/ora/feature_map")]
        same = len(gc["outputs"]) == len(oc["outputs"]) == 1 and all(_sha(x) == _sha(y) for x, y in pairs)
        _head(fr_in, d + "frcut/gpu/f.libsvm", a.cpu_lines * 5)
        shutil.copy(d + "frcut/gpu/f.libsvm", d + "frcut/ora/f.libsvm")
        frappe_feature(d + "frcut/gpu", chunk_bytes=chunk)
        t0 = time.perf_counter()
        O.frappe_feature(d + "frcut/ora")
        fr_cpu_s = time.perf_counter() - t0
        fr_same = _sha(d + "frcut/gpu/f_.libsvm") == _sha(d + "frcut/ora/f_.libsvm")

        name, power = _card()
        ms = g["device_ms"]
        res = {
            "card": name, "power_limit": power, "chunk_mb": a.chunk_mb,
            "smart": {"input_bytes": n_bytes, "lines": n_lines, "map_keys": g["map_keys"],
                      "device_ms": {k: round(v, 2) for k, v in ms.items()},
                      "device_GBps": {k: round(n_bytes / (v * 1e6), 2) for k, v in ms.items() if k != "map" and v > 0},
                      "wall_s": round(wall, 2), "lines_per_s": round(n_lines / wall),
                      "cpu_oracle_lines_per_s": round(a.cpu_lines / cpu_s), "cpu_cut_lines": a.cpu_lines,
                      "cut_bytes_identical": same},
            "frappe": {"input_bytes": fr_bytes, "lines": fr_lines, "device_ms": round(f["device_ms"]["frappe"], 2),
                       "device_GBps": round(fr_bytes / (f["device_ms"]["frappe"] * 1e6), 2),
                       "wall_s": round(fr_wall, 2), "lines_per_s": round(fr_lines / fr_wall),
                       "cpu_oracle_lines_per_s": round(a.cpu_lines * 5 / fr_cpu_s), "cut_bytes_identical": fr_same},
        }
        line = json.dumps(res)
        print(line)
        if a.json:
            with open(a.json, "w") as fh:
                fh.write(json.dumps(res, indent=1) + "\n")
        if not (same and fr_same):
            raise SystemExit("bench_smart_feature: GPU and CPU outputs differ on the cut")
    finally:
        if not a.keep:
            shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
