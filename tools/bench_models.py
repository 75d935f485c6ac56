#!/usr/bin/env python
"""Side measurements for BASELINE.json configs[2] (DCN) and configs[3] (DIN), and for DeepMVM (`deepmvm`, not run by
default): training samples/s on one H100 with the inputs resident in HBM, CUDA-event timed.  (bench.py is the contract
benchmark: DeepFM configs[1].)"""
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

if "deepmvm" in which:
    from tf_repos_b200 import ops
    from tf_repos_b200.deepmvm import DeepMVM
    B, F, N, K = 8192, 39, int(os.environ.get("VOCAB", 200_000_000)), 16
    batches = [synth.criteo_batch(B, N, F, seed=50 + i, device=dev) for i in range(8)]
    m = DeepMVM(F, N, K, B, update_mode="exact_deferred", epoch_steps=EPOCH, device=dev)
    for i in range(2 * EPOCH):          # a position's first visit runs eagerly, its second captures the CUDA graph
        m.train_step_graphed(*batches[i % 8])
    ms = timeit(lambda i: m.train_step_graphed(*batches[i % 8]), m, 2 * EPOCH)
    out["deepmvm_exact_deferred_graphed"] = {"ms_per_step": ms, "samples_per_s": B / ms * 1e3,
                                             "config": f"DeepMVM B={B} F={F} N={N} K={K} Adam l2=1e-4 dropout 0.5"}
    print(f"DeepMVM exact_deferred, graphed {ms:8.3f} ms/step  {B / ms * 1e3 / 1e6:7.3f} M samples/s", flush=True)
    del m
    torch.cuda.empty_cache()
    # the product kernels alone, at the same shape: algorithmic bytes fwd 4(F+1)K, bwd 4(3F+1)K per sample
    x = torch.randn(B, F * K, device=dev) * 1e-3
    mb = torch.rand(F, K, device=dev) * 0.2 + 0.9
    gx, dX = torch.randn(B, K, device=dev), torch.randn(B, F * K, device=dev)
    xm, de, db = torch.empty(B, K, device=dev), torch.empty(B, F * K, device=dev), torch.empty(F, K, device=dev)
    ws = torch.empty(ops.mvm_bwd_workspace_bytes(B, F, K), dtype=torch.uint8, device=dev)
    for name, fn, nbytes in (("fwd", lambda: ops.mvm_fwd(x, mb, xm), 4 * B * K * (F + 1)),
                             ("bwd", lambda: ops.mvm_bwd(x, mb, gx, dX, de, db, ws), 4 * B * K * (3 * F + 1))):
        for _ in range(20):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(500):
            fn()
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) / 500 * 1e3
        out[f"mvm_{name}"] = {"us": us, "algorithmic_bytes": nbytes, "GB_per_s": nbytes / us / 1e3}
        print(f"mvm_{name} {us:8.1f} us  {nbytes / us / 1e3:7.1f} GB/s", flush=True)

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
