#!/usr/bin/env python
"""Times ctr_epoch_sweep (Adam, config-2 fm_v: 2e8 x 16, 16 steps per pass) on table states from different phases of a
run.

  python tools/time_sweep.py [fresh early parked verylong] [--n 200000000] [--k 16]
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = r'''
import sys, json, torch
sys.path.insert(0, %(root)r)
from tf_repos_b200 import ops, engine
d = torch.device("cuda:0")
N, K, P, state = %(n)d, %(k)d, 16, %(state)r
ost = engine.OptimizerState("Adam", 5e-4, 1e-4, d)
var = torch.empty(N * K, device=d); ops.init_trunc_normal(var, (2.0 / (N + K)) ** 0.5, 1)
m = torch.zeros(N * K, device=d); v = torch.zeros(N * K, device=d)
if state in ("parked", "verylong"):
    ost.state[0] = 0.0; ost.state[1] = 0.999 ** 3000
    g = torch.Generator(device=d).manual_seed(1)
    CH = 1 << 28
    for o in range(0, N * K, CH):
        n = min(CH, N * K - o)
        u = lambda: torch.rand(n, device=d, generator=g)
        sign = lambda: torch.where(u() < 0.5, -1.0, 1.0)
        var[o:o + n] = sign() * (0.25 + 4.0 * u()) * 2.0 ** -126
        mm = sign() * u() * 4e-42
        m[o:o + n] = torch.where(u() < 0.2, torch.zeros_like(mm), mm)
        v[o:o + n] = (0.5 + u()) * 1e-24 if state == "parked" else torch.where(u() < 0.2, 0.0, 1.0) * u() * 1e-40
last = torch.zeros(N, dtype=torch.uint8, device=d)
pmax = ops.epoch_max_steps()
part = torch.zeros(pmax * ops.epoch_partials_count(), dtype=torch.float64, device=d)
ss = torch.zeros(pmax, dtype=torch.float64, device=d)
lst = torch.empty(16 * 320_000, dtype=torch.int32, device=d); cnt = torch.zeros(1, dtype=torch.int32, device=d)
touched = torch.randint(0, N, (16 * 200_000,), device=d)
lvals = torch.randint(1, P + 1, (touched.numel(),), device=d, dtype=torch.uint8)
def sweep():
    for j in range(P): ost.tick_epoch(j)
    last[touched] = lvals      # like a real epoch: ~1.6 %% of the rows were gathered and are already past some step
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    ops.epoch_sweep(ost.opt, var, m, v, last, N, K, ost.record(0), ost.lr_table, 0, P, True, part, lst, cnt, ss)
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1)
if state == "early":
    for _ in range(6): sweep()     # ~100 steps in
ts = sorted(sweep() for _ in range(4))
print(json.dumps({"state": state, "N": N, "K": K, "ms_median": ts[len(ts) // 2], "ms_best": ts[0],
                  "listed_rows": int(cnt.item()), "GBps": N * K * 24 / ts[0] / 1e6}))
'''
args = [a for a in sys.argv[1:] if not a.startswith("--")]
n = int(sys.argv[sys.argv.index("--n") + 1]) if "--n" in sys.argv else 200_000_000
k = int(sys.argv[sys.argv.index("--k") + 1]) if "--k" in sys.argv else 16
args = [a for a in args if not a.isdigit()]
for state in args or ["fresh", "early", "parked", "verylong"]:
    subprocess.run([sys.executable, "-c", CHILD % dict(root=ROOT, n=n, k=k, state=state)], check=False)
