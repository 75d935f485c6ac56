#!/usr/bin/env python
"""Times ctr_fc_fwd / ctr_fc_bwd for the MLP and DIN-attention shapes; run with CTR_GEMM=simt to compare the
fp32 SIMT tiles against the default wgmma 3xTF32 path; prints TFLOP/s (2*M*K*N per product) and max error."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tf_repos_b200 import ops  # noqa: E402

d = torch.device("cuda:0")
print("CTR_GEMM =", os.environ.get("CTR_GEMM", "tc (default)"))
for (M, Kd, Nd) in [(8192, 624, 256), (8192, 256, 128), (8192, 128, 64), (409600, 32, 256), (4096, 608, 256)]:
    x = torch.randn(M, Kd, device=d); W = torch.randn(Kd, Nd, device=d) / Kd ** 0.5; b = torch.zeros(Nd, device=d)
    out = torch.empty(M, Nd, device=d); dO = torch.randn(M, Nd, device=d)
    dIn = torch.empty(M, Kd, device=d); dW = torch.empty(Kd, Nd, device=d); db = torch.empty(Nd, device=d)
    ws = torch.empty(ops.fc_bwd_workspace_bytes(M, Kd, Nd), dtype=torch.uint8, device=d)

    def t(fn, n=20):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record(); torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n
    tf = t(lambda: ops.fc_fwd(x, W, b, None, 1.0, 1, out))
    tb = t(lambda: ops.fc_bwd(x, W, out, None, 1.0, dO, 1, dIn, dW, db, ws))
    fl = 2.0 * M * Kd * Nd
    ref = torch.relu(x[:2048].double() @ W.double())
    err = ((out[:2048].double() - ref).abs().max() / ref.abs().max()).item()
    print(f"M={M:7d} K={Kd:4d} N={Nd:4d}: fwd {tf*1e3:8.1f} us ({fl/tf/1e9:6.1f} TF/s)  bwd(dz+dW+dIn) {tb*1e3:8.1f} us "
          f"({2*fl/tb/1e9:6.1f} TF/s)  fwd max rel err {err:.2e}", flush=True)
