#!/usr/bin/env python
"""Times the GPU Ali-CCP TFRecord writer (Feature_pipeline/get_aliccp_tfrecord.py) on seeded synthetic joined Ali-CCP
lines shaped like DeepMTL/README.md's samples: 11 common fields, about 250 user multi-hot (fid, val) pairs over
109_14 / 110_14 / 127_14 / 150_14, the ad fields and a few dropped context fields (default 600 k lines, about 3 GB).

Reports lines/s, input and output GB/s over the wall clock of convert() (file reads and writes included), the device
time of the plan and write passes (CUDA events around the library calls) and the GB/s of text each reads over it, with
the card's name and power limit read in the same run.  The CPU baseline is oracle/aliccp_tfrecord.py on the first
`--cpu_lines` lines, whose output must match the GPU's byte for byte.  Generated data goes to --data_dir (deleted
afterwards unless --keep); one JSON line is printed and, with --json, written there."""
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

COMMON = ["101", "121", "122", "124", "125", "126", "127", "128", "129", "205", "301"]
UMH = [("109_14", 60), ("110_14", 80), ("127_14", 70), ("150_14", 40)]   # mean pairs per line
OTHER = ["206", "207", "216", "508", "509", "702", "853"]


def _card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
    return name, power


def _pool(rng, n):
    """n distinct synthetic lines (without '\\n')"""
    out = []
    for _ in range(n):
        t = ["%s:%d:1.0" % (f, rng.randint(1, 10_000_000)) for f in COMMON]
        for f, m in UMH:
            k = rng.poisson(m)
            ids = rng.randint(1, 10_000_000, k)
            vals = np.log1p(rng.randint(1, 40, k))
            t += ["%s:%d:%.5g" % (f, i, v) for i, v in zip(ids, vals)]
        t += ["%s:%d:1.0" % (f, rng.randint(1, 10_000_000)) for f in OTHER]
        t += ["210:%d:1.0" % i for i in rng.randint(1, 10_000_000, rng.randint(1, 8))]
        rng.shuffle(t)
        y = rng.rand() < 0.04
        out.append("%d,%d,%d,%s" % (rng.randint(1 << 31), y, y and rng.rand() < 0.2, " ".join(t)))
    return [s.encode() for s in out]


def write_lines(path, n, seed, pool_size=20_000):
    """n lines drawn from a seeded pool of distinct lines, in seeded order"""
    rng = np.random.RandomState(seed)
    pool = _pool(rng, min(pool_size, n))
    with open(path, "wb") as fh:
        for start in range(0, n, 100_000):
            idx = rng.randint(len(pool), size=min(100_000, n - start))
            fh.write(b"\n".join(pool[i] for i in idx) + b"\n")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lines", type=int, default=600_000)
    ap.add_argument("--cpu_lines", type=int, default=2_000)
    ap.add_argument("--chunk_mb", type=int, default=64)
    ap.add_argument("--data_dir", default="")
    ap.add_argument("--keep", action="store_true")
    ap.add_argument("--json", default="")
    a = ap.parse_args()

    import torch
    from oracle import aliccp_tfrecord as oa
    from tf_repos_b200.aliccp_tfrecord import convert

    if not torch.cuda.is_available():
        raise SystemExit("bench_aliccp_tfrecord: needs a CUDA device")
    d = a.data_dir or tempfile.mkdtemp(prefix="aliccp_tfrecord_")
    small, big = os.path.join(d, "small"), os.path.join(d, "big")
    os.makedirs(small, exist_ok=True); os.makedirs(big, exist_ok=True)
    res = {}
    try:
        t = time.perf_counter()
        write_lines(os.path.join(big, "sample-0"), a.lines, seed=0)
        res["generate_s"] = round(time.perf_counter() - t, 1)
        with open(os.path.join(big, "sample-0"), "rb") as src, open(os.path.join(small, "sample-0"), "wb") as dst:
            for _, line in zip(range(a.cpu_lines), src):
                dst.write(line)

        kw = dict(chunk_bytes=a.chunk_mb << 20)
        convert(small, small + "_gpu", **kw)                               # warm-up: context, module load, allocator
        t = time.perf_counter()
        oa.convert(small, small + "_cpu")
        cpu_s = time.perf_counter() - t
        g, c = [hashlib.sha256(open(os.path.join(x, "sample-0.tfrecord"), "rb").read()).hexdigest()
                for x in (small + "_gpu", small + "_cpu")]

        name, power = _card()
        torch.cuda.synchronize()
        t = time.perf_counter()
        info = convert(big, big + "_gpu", **kw)
        wall = time.perf_counter() - t
        name2, power2 = _card()
        st, ms = info["outputs"][0], info["device_ms"]
        res.update({
            "card": name, "power_limit": power, "card_after": name2, "power_limit_after": power2,
            "lines": st["lines"], "input_bytes": st["in_bytes"], "output_bytes": st["out_bytes"],
            "declined": st["declined"], "chunk_mb": a.chunk_mb,
            "wall_s": round(wall, 2), "lines_per_s": round(st["lines"] / wall),
            "input_GBps": round(st["in_bytes"] / wall / 1e9, 3), "output_GBps": round(st["out_bytes"] / wall / 1e9, 3),
            "device_ms": {k: round(v, 2) for k, v in ms.items()},
            "device_input_GBps": {k: round(st["in_bytes"] / (v * 1e6), 2) for k, v in ms.items() if v > 0},
            "cpu_oracle_lines": a.cpu_lines, "cpu_oracle_s": round(cpu_s, 2),
            "cpu_oracle_lines_per_s": round(a.cpu_lines / cpu_s), "sha256_match": g == c,
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
        raise SystemExit("the GPU and CPU outputs differ on the CPU cut")


if __name__ == "__main__":
    main()
