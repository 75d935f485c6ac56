#!/usr/bin/env python
"""Latency and throughput of ESMM's serving entry (serving.ESMMServable.predict) on one GPU.

The model has the DeepMTL README shape of DESIGN.md §6 (ESMM, F'=11, feature_size 4 519 540, embedding_size 16, towers
256,128, max_batch 4096) with its constructor's random variables.  Every Example of a request has the training schema of
DeepCvrMTL.py:66-83 without labels: bags of seeded ids with the lengths §6 assumes (u_shop U{1..499}, the other u_*
U{1..49}, a_int U{1..8}; 333 occurrences per Example on average), u_* with weights.  The occurrence capacity starts at
max_batch x the longest possible Example (654 occurrences), so no request grows it.

  latency     wall clock around predict (host -> device copy, kernels, device -> host copy, the one synchronise) per
              request after a warm-up of every size: median and p99 for n in --sizes
  device      parse = ESMMServable.parse (scan, one-CTA offset scan, capacity clamp, emit), model = ESMM.predict on
              the emitted batch: device time from torch.profiler (CUDA activity only, in a phase of its own) per
              slice.  ESMM.predict always runs the full max_batch rows, so the model time does not shrink with
              n; its bag sums do, with the padding slots repeating Example 0
  throughput  Examples/s of predict at each n (n / median latency)
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
BAG_MAX = {"cat": 49, "shop": 499, "brand": 49, "int": 49}
A_INT_MAX = 8


def _request(n, rng, F, N):
    from tf_repos_b200.tfrecord import encode_example
    out = []
    for _ in range(n):
        ex = {"feat_ids": rng.integers(0, N, F), "a_catids": rng.integers(0, N, 1), "a_shopids": rng.integers(0, N, 1),
              "a_brandids": rng.integers(0, N, 1), "a_intids": rng.integers(0, N, int(rng.integers(1, A_INT_MAX + 1)))}
        for u, top in BAG_MAX.items():
            ln = int(rng.integers(1, top + 1))
            ex["u_%sids" % u] = rng.integers(0, N, ln)
            ex["u_%svals" % u] = rng.random(ln, dtype=np.float32)
        out.append(encode_example(ex))
    return out


def _kernel_ms(fn, reps):
    """device time per call: the durations of the kernels fn launches, from torch.profiler (CUDA activity only)"""
    from torch.autograd import DeviceType
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if e.device_type == DeviceType.CUDA)
    return us / 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,16,256,4096")
    ap.add_argument("--requests", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default="esmm_serving.json")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_esmm_serving measures on a GPU"
    from tf_repos_b200.esmm import ESMM
    from tf_repos_b200.serving import ESMMServable

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    F, N, K, B = 11, 4_519_540, 16, 4096
    cap = B * (sum(BAG_MAX.values()) + A_INT_MAX)
    m = ESMM(F, N, K, B, cap, deep_layers="256,128", dropout="0.8,0.5", ctr_task_wgt=0.3, update_mode="lazy",
             device="cuda:0")
    s = ESMMServable(m)
    rng = np.random.default_rng(0)
    sizes = [int(t) for t in a.sizes.split(",")]
    reqs = {n: _request(n, rng, F, N) for n in sizes}
    res = {"card": smi, "device_name": torch.cuda.get_device_name(0),
           "model": f"ESMM F'={F} N={N} K={K} towers 256,128, max_batch {B}, occ_capacity {cap}; bags u_shop "
                    f"U{{1..499}}, u_cat/u_brand/u_int U{{1..49}}, a_int U{{1..8}}",
           "latency_ms": {}, "examples_per_s": {}, "device_ms": {}}
    for n in sizes:                      # every shape warmed up before any timing
        for _ in range(a.warmup):
            s.predict(reqs[n])
    assert m.cap == cap
    for n in sizes:
        count = a.requests if n <= 256 else max(a.requests // 4, 20)
        t = []
        for _ in range(count):
            t0 = time.perf_counter()
            s.predict(reqs[n])
            t.append((time.perf_counter() - t0) * 1e3)
        med = float(np.median(t))
        res["latency_ms"][str(n)] = {"median": med, "p99": float(np.percentile(t, 99)), "mean": float(np.mean(t)),
                                     "requests": count}
        res["examples_per_s"][str(n)] = n / (med / 1e3)
        print(n, res["latency_ms"][str(n)], flush=True)
    for n in sizes:
        ex = reqs[n]
        lens = np.array([len(r) for r in ex])
        off = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int64, device="cuda:0")
        data = torch.tensor(np.frombuffer(b"".join(ex), dtype=np.uint8), device="cuda:0")
        err = torch.full((1,), -1, dtype=torch.int64, device="cuda:0")
        rec = torch.zeros(8, dtype=torch.uint8, device="cuda:0")
        total = rec.view(torch.int64)                                  # the slice's occurrence total
        bt = s.parse(data, off, 0, err, rec)
        reps = 50
        d = {"parse": _kernel_ms(lambda: s.parse(data, off, 0, err, rec), reps),
             "model": _kernel_ms(lambda: m.predict(bt), reps), "request_bytes": int(lens.sum())}
        assert int(err.item()) == -1 and int(total.item()) <= cap
        d["occurrences"] = int(total.item())
        d["parse_over_model"] = d["parse"] / d["model"]
        res["device_ms"][str(n)] = d
        print(n, d, flush=True)
    print(json.dumps(res))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
