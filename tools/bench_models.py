#!/usr/bin/env python
"""Side measurements for BASELINE.json configs[2] (DCN) and configs[3] (DIN), and for DeepMVM (`deepmvm`) and ESMM
(`esmm`, with CUDA-event times of its embedding kernels), which are not run by default: training samples/s on one H100 with the inputs resident in HBM, CUDA-event timed.  (bench.py is the contract
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

if "esmm" in which:
    # the shape of the DeepMTL README invocation; bag lengths assumed (the README only states that the largest field
    # averages 250 values): u_shop ~ U{1..499}, the other u_* ~ U{1..49}, a_int ~ U{1..8}
    from tf_repos_b200 import ops
    from tf_repos_b200.esmm import ESMM
    Fp, N, K, lens = 11, 4_519_540, 16, (49, 499, 49, 49, 8)
    kw = dict(deep_layers="256,128", dropout="0.8,0.5", ctr_task_wgt=0.3, l2_reg=0.005)
    for B in (1024, 8192):
        batches = [synth.esmm_batch(B, N, Fp, max_lens=lens, seed=70 + i, device=dev) for i in range(4)]
        cap = max(b["bag_ids"].numel() for b, _ in batches)
        for mode in ("exact_deferred", "lazy"):
            m = ESMM(Fp, N, K, B, cap, update_mode=mode, epoch_steps=EPOCH, device=dev, **kw)
            ms = timeit(lambda i: m.train_step(*batches[i % 4]), m, EPOCH)
            out[f"esmm_B{B}_{mode}"] = {"ms_per_step": ms, "samples_per_s": B / ms * 1e3,
                                        "config": f"ESMM B={B} F'={Fp} N={N} K={K} bag lens max {lens} "
                                                  f"(mean occurrences/sample {cap / B:.0f}) layers 256,128 Adam l2=0.005"}
            print(f"ESMM B={B} {mode:15s} {ms:8.3f} ms/step  {B / ms * 1e3 / 1e6:7.3f} M samples/s", flush=True)
            del m
            torch.cuda.empty_cache()
        # the embedding kernels alone; algorithmic bytes from the batch's shapes:
        #   fwd reads ids, weights, offsets and one K-row per lookup, writes x;  bwd reads dx, weights, offsets and
        #   writes one K-row per lookup slot (the capacity)
        batch, _ = batches[0]
        nnz = batch["bag_ids"].numel()
        n_w = int(batch["bag_off"][4 * B].item())
        Dx = (Fp + 8) * K
        V = torch.randn(N, K, device=dev) * 0.01
        x, dx = torch.empty(B, Dx, device=dev), torch.randn(B, Dx, device=dev)
        g = torch.empty(B * (Fp + 3) + cap, K, device=dev)
        lookups = B * (Fp + 3) + nnz
        fwd_bytes = 4 * lookups + 4 * n_w + 4 * (5 * B + 1) + 4 * K * lookups + 4 * B * Dx
        bwd_bytes = 4 * B * Dx + 4 * n_w + 4 * (5 * B + 1) + 4 * K * (B * (Fp + 3) + cap)
        for name, fn, nbytes in (
                ("fwd", lambda: ops.esmm_embed_fwd(batch["feat_ids"], batch["a_ids"], batch["bag_ids"], batch["bag_wgt"],
                                                   batch["bag_off"], V, x), fwd_bytes),
                ("bwd", lambda: ops.esmm_embed_bwd(dx, batch["bag_wgt"], batch["bag_off"], B, Fp, K, g), bwd_bytes)):
            for _ in range(20):
                fn()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(200):
                fn()
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) / 200 * 1e3
            out[f"esmm_embed_{name}_B{B}"] = {"us": us, "algorithmic_bytes": nbytes, "GB_per_s": nbytes / us / 1e3}
            print(f"esmm_embed_{name} B={B} {us:8.1f} us  {nbytes / us / 1e3:7.1f} GB/s", flush=True)
        del V, batches
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
