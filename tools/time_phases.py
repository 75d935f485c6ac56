#!/usr/bin/env python
"""In-situ device time per C-ABI entry point and per kernel during DeepFM train steps at bench.py's configuration
(N = 2e8, B = 8192, F = 39, K = 16, epoch of 16 steps).

  python tools/time_phases.py [mode] [steps] [--json OUT]     mode: exact_deferred (default) | exact | lazy

Three runs of `steps` steps each (whole epochs when steps is a multiple of 16), from the same model:
  1. eager steps, CUDA events around every C-ABI call (warm caches, real step context).  The epoch sweep is keyed
     by table (K) so fm_v's and fm_w's passes are apart; sort/unique and the segment sums are their own entry points;
  2. eager steps under torch.profiler: device time per KERNEL, which splits the epoch sweep into its stages (the
     packed pass, the catch-up of the listed rows, the `last` rewrite);
  3. graphed steps (train_step_graphed, what bench.py times): whole-step time from CUDA events, and per kernel
     under torch.profiler in a separate run.
The card's name and power limit are printed with the numbers.
"""
import collections
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tf_repos_b200 import ops, synth  # noqa: E402
from tf_repos_b200.deepfm import DeepFM  # noqa: E402


class TimedLib:
    def __init__(self, lib):
        self._lib, self.records, self.on = lib, [], False

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith("ctr_") or name in ("ctr_last_error", "ctr_launch_count"):
            return fn

        def call(*a):
            if not self.on:
                return fn(*a)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = fn(*a)
            e1.record()
            key = name
            if name == "ctr_epoch_rows":   # (opt, apply, ..., K at 10, ..., j at 13)
                key = f"{name}[apply={a[1]},K={a[10]}]"
            elif name == "ctr_epoch_rows2":
                key = f"{name}[apply={a[1]}]"
            elif name == "ctr_epoch_sweep":   # (opt, var, s0, s1, w_var, w_s0, w_s1, last, n_rows, K, ...)
                key = f"{name}[K={a[9]}{'+W' if a[4] else ''}]"
            self.records.append((key, e0, e1))
            return r
        return call


def device_info(dev):
    info = {"name": torch.cuda.get_device_name(dev), "power_limit_w": None, "sm_max_mhz": None}
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(dev.index or 0)
        info["power_limit_w"] = pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
        info["sm_max_mhz"] = pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM)
    except Exception:
        pass
    return info


def kernel_table(prof, steps):
    """{kernel name: [launches per step, us per step]} from a torch.profiler run of `steps` steps."""
    agg = collections.OrderedDict()
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        t = agg.setdefault(ev.name, [0, 0.0])
        t[0] += 1
        t[1] += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
    return {k: [c / steps, us / steps] for k, (c, us) in agg.items()}


def short(name, n=96):
    name = name.replace("(anonymous namespace)::", "").replace("ctr::", "")
    return name if len(name) <= n else name[: n - 3] + "..."


def print_kernels(title, table, step_ms):
    print(f"# {title}: device time per kernel (torch.profiler), {step_ms:.3f} ms/step")
    print(f"# {'kernel':96s} {'calls/step':>10s} {'us/step':>9s} {'share':>7s}")
    acc = 0.0
    for name, (cnt, us) in sorted(table.items(), key=lambda kv: -kv[1][1]):
        acc += us
        print(f"  {short(name):96s} {cnt:10.2f} {us:9.1f} {us / (step_ms * 10):6.1f}%")
    print(f"# in kernels: {acc / 1e3:.3f} ms/step; idle / gaps: {step_ms - acc / 1e3:.3f} ms/step")


def main():
    args = [a for a in sys.argv[1:]]
    out_json = None
    if "--json" in args:
        i = args.index("--json")
        out_json = args[i + 1]
        del args[i:i + 2]
    mode = args[0] if len(args) > 0 else "exact_deferred"
    steps = int(args[1]) if len(args) > 1 else 32
    N, B, F, K = int(os.environ.get("VOCAB", 200_000_000)), 8192, 39, 16
    dev = torch.device("cuda:0")
    info = device_info(dev)
    tl = TimedLib(ops._L)
    ops._L = tl
    batches = [synth.criteo_batch(B, N, F, seed=i, device=dev) for i in range(8)]
    m = DeepFM(F, N, K, B, update_mode=mode, epoch_steps=16, device=dev)
    deferred = mode == "exact_deferred"

    def align(step):
        i = 0
        while deferred and m.epoch_pos != 0:
            step(batches[i % 8]); i += 1

    def run(step, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(n):
            step(batches[i % 8])
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    eager = lambda b: m.train_step(*b)
    graphed = lambda b: m.train_step_graphed(*b)
    for i in range(5):
        eager(batches[i % 8])
    align(eager)
    torch.cuda.synchronize()
    print(f"# device: {info['name']}, power limit {info['power_limit_w']} W, max SM clock {info['sm_max_mhz']} MHz")
    print(f"# DeepFM N={N} B={B} F={F} K={K} epoch=16, mode {mode}, {steps} steps per run")

    # 1. eager, events per entry point
    tl.on = True
    ms_events = run(eager, steps)
    tl.on = False
    agg = collections.OrderedDict()
    for name, a, b in tl.records:
        t = agg.setdefault(name, [0, 0.0])
        t[0] += 1
        t[1] += a.elapsed_time(b)
    tl.records = []
    print(f"# eager, events around every entry point: {ms_events:.3f} ms/step (with event overhead)")
    print(f"# {'entry point':40s} {'calls/step':>10s} {'us/call':>10s} {'us/step':>10s} {'share':>7s}")
    acc = 0.0
    entries = {}
    for name, (cnt, ms) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        acc += ms
        entries[name] = [cnt / steps, ms / steps * 1e3]
        print(f"  {name:40s} {cnt / steps:10.2f} {ms / cnt * 1e3:10.1f} {ms / steps * 1e3:10.1f} "
              f"{ms / (ms_events * steps) * 100:6.1f}%")
    print(f"# inside entry points: {acc / steps:.3f} ms/step; outside (torch ops, gaps): {ms_events - acc / steps:.3f} ms/step")

    # 2. eager, plain and profiled
    align(eager)
    ms_eager = run(eager, steps)
    from torch.profiler import ProfilerActivity, profile
    align(eager)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(eager, steps)
    k_eager = kernel_table(prof, steps)
    print(f"# eager (no events): {ms_eager:.3f} ms/step")
    print_kernels("eager", k_eager, ms_eager)

    # 3. graphed: warm every position (first visit eager, second captures), then time and profile
    res = {"device": info, "mode": mode, "steps": steps, "eager_ms_per_step": ms_eager,
           "entry_points_us_per_step": entries, "kernels_eager_us_per_step": k_eager}
    if deferred:
        align(eager)
        for _ in range(2 * 16):
            graphed(batches[0])
        align(graphed)
        ms_graphed = run(graphed, steps)
        align(graphed)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run(graphed, steps)
        k_graphed = kernel_table(prof, steps)
        print(f"# graphed: {ms_graphed:.3f} ms/step")
        print_kernels("graphed", k_graphed, ms_graphed)
        res.update(graphed_ms_per_step=ms_graphed, kernels_graphed_us_per_step=k_graphed)
    if out_json:
        os.makedirs(os.path.dirname(os.path.abspath(out_json)), exist_ok=True)
        with open(out_json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
