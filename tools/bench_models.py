#!/usr/bin/env python
"""Side measurements for BASELINE.json configs[2] (DCN) and configs[3] (DIN): training samples/s on one H100
with the inputs resident in HBM, CUDA-event timed.  (bench.py is the contract benchmark: DeepFM configs[1].)"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tf_repos_b200 import synth  # noqa: E402

dev = torch.device("cuda:0")
EPOCH = 16
which = sys.argv[1:] or ["dcn", "din"]
out = {}


def timeit(step, model, steps):
    for i in range(3):
        step(i)
    while getattr(model, "update_mode", "") == "exact_deferred" and model.epoch_pos != 0:
        step(0)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        step(i)
    model.flush()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


if "dcn" in which:
    from tf_repos_b200.dcn import DCN
    B, F, N, K, L = 8192, 39, int(os.environ.get("VOCAB", 200_000_000)), 16, 6
    batches = [synth.criteo_batch(B, N, F, seed=i, device=dev) for i in range(8)]
    for mode in ("exact_deferred", "exact", "lazy"):
        m = DCN(F, N, K, B, cross_layers=L, update_mode=mode, epoch_steps=EPOCH, device=dev)
        ms = timeit(lambda i: m.train_step(*batches[i % 8]), m, EPOCH if mode != "lazy" else 32)
        out[f"dcn_{mode}"] = {"ms_per_step": ms, "samples_per_s": B / ms * 1e3,
                              "config": f"DCN B={B} F={F} N={N} K={K} cross_layers={L} Adam l2=1e-4 dropout 0.5"}
        print(f"DCN {mode:15s} {ms:8.3f} ms/step  {B / ms * 1e3 / 1e6:7.3f} M samples/s", flush=True)
        del m
        torch.cuda.empty_cache()

if "din" in which:
    from tf_repos_b200.din import DIN
    B, Fp, N, K, P = 4096, 11, int(os.environ.get("VOCAB_DIN", 100_000_000)), 32, 100
    batches = []
    for i in range(4):
        b, l = synth.din_batch(B, N, Fp, P, 8, seed=i)
        batches.append(({k: v.to(dev) for k, v in b.items()}, l.to(dev)))
    for mode in ("exact_deferred", "lazy"):
        m = DIN(Fp, N, K, B, P, max_a_int=8, update_mode=mode, epoch_steps=EPOCH, device=dev)
        ms = timeit(lambda i: m.train_step(*batches[i % 4]), m, EPOCH)
        out[f"din_{mode}"] = {"ms_per_step": ms, "samples_per_s": B / ms * 1e3,
                              "config": f"DIN B={B} F'={Fp} P={P} (lens~U[1,100]) N={N} K={K} att hidden 256, Adam l2=1e-4 dropout 0.5"}
        print(f"DIN {mode:15s} {ms:8.3f} ms/step  {B / ms * 1e3 / 1e6:7.3f} M samples/s", flush=True)
        del m
        torch.cuda.empty_cache()
print(json.dumps(out), flush=True)
