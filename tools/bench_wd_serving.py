#!/usr/bin/env python
"""Latency and throughput of wide_n_deep's serving entry (serving.WideDeepServable.classify) on one GPU.

The model is the reference's default (wide_n_deep.py:31-34: wide_n_deep, embedding_size 32, deep_layers 256,128,64)
with random variables.  A request has the shape of wide_n_deep_serving_client.cpp:45-62 -- I1..I13 one float each,
and here all 26 model columns C14..C39 with one seeded id each -- and the client's own request (quirk Q13) is timed
as well.  The reference publishes latency_ms = 0.5256*n_ads + 15.449 for TF-Serving on a CPU server, measured with
gRPC, a cache lookup and logging around the model (deep_ctr/README.md:74-81), so the two are not like for like.

  latency     wall clock around classify (host -> device copy, kernels, device -> host copy) per request, after a
              warm-up: median and p99 over --requests requests for n_ads in --sizes, and a least-squares a*n + b over
              the medians
  device      the parse + feature-column kernel (ctr_wd_serve_input) and the kernels of the MLP + head: their device
              time from torch.profiler (in a phase of its own), and CUDA events around back-to-back calls (at small n
              these measure the host's launch rate, not the device)
  throughput  Examples/s of classify at n = --big, and the kernel's bytes/s over the bytes it reads: the serialized
              Examples plus 26*(K+1)*4 B of table rows per Example
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


def _request(n, rng):
    from tests import wd_serving_oracle as so
    return [so.request_row(rng.standard_normal(13).astype(np.float32), [[int(v)] for v in rng.integers(0, 10000, 26)])
            for _ in range(n)]


def _events(fn, reps):
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def _kernel_ms(fn, reps):
    """device time per call: the durations of the kernels fn launches, from torch.profiler (CUDA activity only), so
    that the host's launch cost at small n does not count"""
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
    ap.add_argument("--sizes", default="1,2,5,10,20,50,100")
    ap.add_argument("--requests", type=int, default=600)
    ap.add_argument("--warmup", type=int, default=100)
    ap.add_argument("--big", type=int, default=8192)
    ap.add_argument("--out", default="wd_serving.json")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_wd_serving measures on a GPU"
    from tests import wd_serving_oracle as so
    from tf_repos_b200 import ops
    from tf_repos_b200.serving import WideDeepServable
    from tf_repos_b200.wide_deep import NUM_BUCKETS, WideDeep

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    K = 32
    m = WideDeep(K, a.big, "256,128,64", "wide_n_deep", device="cuda:0", seed=0)
    g = torch.Generator().manual_seed(1)
    m.load_variables({n: torch.randn(v.shape, generator=g) * 0.1 for n, v in m.variables().items()})
    s = WideDeepServable(m)
    rng = np.random.default_rng(0)
    res = {"card": smi, "device_name": torch.cuda.get_device_name(0), "model": "wide_n_deep K=32 256,128,64",
           "latency_ms": {}, "device_ms": {}}

    def wall(reqs, count):
        for _ in range(a.warmup):
            s.classify(reqs)
        t = []
        for _ in range(count):
            t0 = time.perf_counter()
            s.classify(reqs)
            t.append((time.perf_counter() - t0) * 1e3)
        return {"median": float(np.median(t)), "p99": float(np.percentile(t, 99)), "mean": float(np.mean(t)),
                "requests": count}

    def device(reqs):
        n = len(reqs)
        lens = np.array([len(r) for r in reqs])
        off = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int64, device="cuda:0")
        data = torch.tensor(np.frombuffer(b"".join(reqs), dtype=np.uint8), device="cuda:0")
        err = torch.full((1,), -1, dtype=torch.int64, device="cuda:0")
        pred = torch.empty(n, device="cuda:0")
        kern = lambda: ops.wd_serve_input(data, off, 0, m.emb.var, m.wide_cat.var, m.dense_lin["linear/numeric"],  # noqa: E731
                                          m.dense_lin["linear/linear_model/bias_weights"], m.num_perm, NUM_BUCKETS, K,
                                          m.x[:n], m.lin[:n], err)
        mlp = lambda: m._probabilities(n, m.lin[:n], m._dnn(n), pred)  # noqa: E731
        reps = 200 if n <= 1024 else 50
        out = {"kernel": _kernel_ms(kern, reps), "mlp_and_head": _kernel_ms(mlp, reps),
               "kernel_events_per_call": _events(kern, reps), "mlp_and_head_events_per_call": _events(mlp, reps),
               "bytes": int(lens.sum())}
        assert int(err.item()) == -1
        return out

    sizes = [int(t) for t in a.sizes.split(",")]
    for n in sizes:
        reqs = _request(n, rng)
        res["latency_ms"][str(n)] = wall(reqs, a.requests)
        res["device_ms"][str(n)] = device(reqs)
        print(n, res["latency_ms"][str(n)], res["device_ms"][str(n)], flush=True)
    med = np.array([res["latency_ms"][str(n)]["median"] for n in sizes])
    slope, icpt = np.polyfit(np.array(sizes, dtype=np.float64), med, 1)
    res["fit_median_ms"] = {"a_per_example": float(slope), "b": float(icpt)}
    res["client_request_ms"] = wall([so.client_request()], a.requests)

    big = _request(a.big, rng)
    w = wall(big, 30)
    d = device(big)
    rows_bytes = a.big * 26 * (K + 1) * 4
    res["throughput"] = {"n": a.big, "classify_ms_median": w["median"], "examples_per_s": a.big / (w["median"] / 1e3),
                         "kernel_ms": d["kernel"], "mlp_and_head_ms": d["mlp_and_head"],
                         "kernel_bytes_read": d["bytes"] + rows_bytes,
                         "kernel_GB_per_s": (d["bytes"] + rows_bytes) / (d["kernel"] / 1e3) / 1e9}
    print(json.dumps(res, indent=1))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
