#!/usr/bin/env python
"""libsvm tokenizer throughput: GPU (ctr_parse_libsvm_device, text resident in HBM / including the H2D copy)
versus the host parser (ctr_parse_libsvm, 10 threads like the reference's num_parallel_calls, and all cores).
Criteo-layout lines (39 pairs); prints lines/s and GB/s of text, JSON on the last line.

Then input_fn end to end, device path and host path: one epoch over a file of at least INPUT_FN_BYTES (default 1 GiB;
the LINES-line file repeated, the tokenizer keeps nothing between lines), batches of 8192 dropped as they come, host
clock around a final synchronise; the file was just written and synced, so reads come from the page cache.  For the device path
also torch.cuda.max_memory_allocated over the epoch, with what was allocated before it."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tf_repos_b200 import input_fn, ops, synth  # noqa: E402

F, LINES = 39, int(os.environ.get("LINES", 200_000))
ids, vals, labels = synth.criteo_batch(LINES, 200_000_000, F, seed=3)
path = "/tmp/bench_tr.libsvm"
synth.write_libsvm(path, ids, vals, labels)
data = open(path, "rb").read()
n_bytes = len(data)
res = {"lines": LINES, "bytes": n_bytes, "bytes_per_line": n_bytes / LINES}

chunk = input_fn.CHUNK
for threads in (10, os.cpu_count() or 1):
    t0 = time.perf_counter()
    input_fn.CHUNK = max(1 << 20, n_bytes // threads + 1)
    h = input_fn.decode_libsvm_file(path, F, threads=threads)
    dt = time.perf_counter() - t0
    res[f"host_{threads}_threads"] = {"lines_per_s": LINES / dt, "GB_per_s": n_bytes / dt / 1e9}
input_fn.CHUNK = chunk

# the oracle's pure-Python decode_libsvm (what a Python-level restatement of the TF string ops costs), 5 000 lines
from oracle import libsvm as olib  # noqa: E402
sample = data.decode().splitlines()[:5000]
t0 = time.perf_counter()
for ln in sample:
    olib.decode_libsvm(ln)
dt = time.perf_counter() - t0
res["oracle_python_1_thread"] = {"lines_per_s": len(sample) / dt, "GB_per_s": sum(len(l) + 1 for l in sample) / dt / 1e9}

dev = torch.device("cuda:0")
res["card"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip().splitlines()
pinned = torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).pin_memory()
text = pinned.to(dev)
max_rows = n_bytes // (2 * F + 2)
out = ops.parse_libsvm_device(text, F, max_rows)          # warm-up + correctness
assert not out[4] and out[0].shape[0] == LINES
assert np.array_equal(out[0].cpu().numpy(), h[0]) and np.array_equal(out[1].cpu().numpy().view(np.uint32), h[1].view(np.uint32))
torch.cuda.synchronize()
for name, with_copy in (("gpu_resident", False), ("gpu_with_h2d", True)):
    ts = []
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        if with_copy:
            text.copy_(pinned, non_blocking=True)
        ops.parse_libsvm_device(text, F, max_rows)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e-3)
    dt = sorted(ts)[len(ts) // 2]
    res[name] = {"lines_per_s": LINES / dt, "GB_per_s": n_bytes / dt / 1e9, "ms": dt * 1e3}
del out, text, pinned

big = "/tmp/bench_input_fn.libsvm"
reps = -(-int(os.environ.get("INPUT_FN_BYTES", 1 << 30)) // n_bytes)
with open(big, "wb") as fh:
    for _ in range(reps):
        fh.write(data)
    fh.flush()
    os.fsync(fh.fileno())                                               # no write-back under the timed reads


def drain(p, device):
    torch.cuda.synchronize()
    t0, k = time.perf_counter(), 0
    for _, labels in input_fn.input_fn([p], batch_size=8192, field_size=F, device=device):
        k += labels.shape[0]
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return {"lines": k, "seconds": dt, "lines_per_s": k / dt}


try:
    drain(path, dev)                                                    # warm-up: pinned buffers, modules
    drain(path, None)
    torch.cuda.reset_peak_memory_stats(dev)
    before = torch.cuda.memory_allocated(dev)
    res["input_fn"] = {"bytes": reps * n_bytes, "batch_size": 8192, "device": drain(big, dev)}
    res["input_fn"]["device"].update(memory_allocated_before=before,
                                     max_memory_allocated=torch.cuda.max_memory_allocated(dev))
    res["input_fn"]["host"] = drain(big, None)
    assert res["input_fn"]["device"]["lines"] == res["input_fn"]["host"]["lines"] == reps * LINES
finally:
    os.remove(big)
for k, v in res.items():
    print(k, v)
print(json.dumps(res))
