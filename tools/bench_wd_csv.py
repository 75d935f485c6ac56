#!/usr/bin/env python
"""wide_n_deep CSV input on one GPU: the tokenizer kernel, input_fn end to end and training, device path against host path.

The file is seeded synthetic CSV in the Criteo shape of wide_n_deep.py:55-73 -- a 0/1 label, 13 floats with 6 decimals,
26 ids below 10000 -- written under --out-dir and removed afterwards: a block of --block distinct lines repeated up to
--lines lines (the tokenizer keeps nothing between lines, so repetition does not help it).

  kernel      ctr_parse_csv_device on one piece of wide_deep_main.CSV_CHUNK bytes resident in HBM: CUDA events around
              --reps back-to-back launches (line starts + the per-line kernel) -> ms per piece, lines/s, GB/s of text;
              the same with the pinned host-to-device copy of the piece queued before each launch, and the copy alone
  input_fn    one epoch over the file at --batch_size, nothing done with the batches: host clock around the generator
              and a final synchronise.  device = the whole file; host = its first --host-lines lines (the Python decoder
              takes minutes on the whole file).  The file was just written, so reads come from the page cache.
  train       WideDeep.train_step over one epoch of the first --train-lines lines, the loop of wide_deep_main.run(), at
              each of --train-batch-sizes, host and device input alternated --rounds times; samples/s by the host clock
              around the loop and a final synchronise, and the final variables of the two paths compared bit for bit.
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def csv_block(n: int, seed: int) -> bytes:
    g = np.random.default_rng(seed)
    lab = g.integers(0, 2, n)
    dense = g.random((n, 13)) * np.array([10.0 ** (k % 4) for k in range(13)])
    cat = g.integers(0, 10000, (n, 26))
    fmt = "%d," + ",".join(["%.6f"] * 13) + "," + ",".join(["%d"] * 26) + "\n"
    return "".join(fmt % ((lab[i],) + tuple(dense[i]) + tuple(cat[i])) for i in range(n)).encode()


def write_csv(path: str, block: bytes, block_lines: int, lines: int):
    """the first `lines` lines of the block repeated"""
    with open(path, "wb") as fh:
        for _ in range(lines // block_lines):
            fh.write(block)
        rest = lines % block_lines
        if rest:
            fh.write(b"".join(block.splitlines(keepends=True)[:rest]))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--lines", type=int, default=5_000_000)
    ap.add_argument("--block", type=int, default=250_000)
    ap.add_argument("--host-lines", type=int, default=200_000)
    ap.add_argument("--train-lines", type=int, default=500_000)
    ap.add_argument("--train-batch-sizes", default="128,8192")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch_size", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out-dir", default="profiles")
    ap.add_argument("--name", default="wd_csv_h100.json")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_wd_csv measures on a GPU"
    from tf_repos_b200 import ops, text_chunks
    from tf_repos_b200 import wide_deep_main as wm
    from tf_repos_b200.wide_deep import WideDeep

    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    res = {"card": smi, "device_name": torch.cuda.get_device_name(0), "lines": a.lines, "block_lines": min(a.block, a.lines),
           "chunk_bytes": wm.CSV_CHUNK}
    data_dir = os.path.join(a.out_dir, "wd_csv_data")
    os.makedirs(data_dir, exist_ok=True)
    try:
        bl = min(a.block, a.lines)
        block = csv_block(bl, seed=7)
        full, cut, tr = (os.path.join(data_dir, n) for n in ("full.csv", "host_cut.csv", "tr.csv"))
        write_csv(full, block, bl, a.lines)
        write_csv(cut, block, bl, min(a.host_lines, a.lines))
        write_csv(tr, block, bl, min(a.train_lines, a.lines))
        res["bytes"] = os.path.getsize(full)
        res["bytes_per_line"] = res["bytes"] / a.lines

        # ---- kernel: one piece ---------------------------------------------------------------------------------
        piece = next(text_chunks.pieces(full, wm.CSV_CHUNK))
        n, rows = len(piece), piece.count(b"\n")
        pinned = torch.from_numpy(np.frombuffer(piece, dtype=np.uint8).copy()).pin_memory()
        text = pinned.to(dev)
        ws = text_chunks.scratch(ops.parse_csv_device_workspace_bytes(n, rows + 1), dev)
        out = ops.parse_csv_device(text, n, 14, 26, rows + 1, ws)
        assert out[3].tolist() == [rows, n, 0, 0, 0], out[3].tolist()
        want = wm.decode_csv_bytes(b"".join(piece.splitlines(keepends=True)[:2000]), full)
        for got, w in zip(out[:3], want[:3]):
            assert np.array_equal(got[:2000].cpu().numpy().view(np.uint32), w.view(np.uint32))

        def events(fn):
            fn()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.reps):
                fn()
            e1.record()
            e1.synchronize()
            ms = e0.elapsed_time(e1) / a.reps
            return {"ms_per_piece": ms, "lines_per_s": rows / (ms * 1e-3), "GB_per_s": n / (ms * 1e-3) / 1e9}

        parse = lambda: ops.parse_csv_device(text, n, 14, 26, rows + 1, ws)  # noqa: E731
        copy = lambda: text.copy_(pinned, non_blocking=True)  # noqa: E731
        res["kernel"] = {"piece_bytes": n, "piece_lines": rows, "launches": a.reps,
                         "resident": events(parse), "with_h2d": events(lambda: (copy(), parse())), "h2d_alone": events(copy)}
        print("kernel", res["kernel"], flush=True)
        del out, text, pinned

        # ---- input_fn end to end ---------------------------------------------------------------------------------
        def drain(path, device):
            torch.cuda.synchronize()
            t0, k = time.perf_counter(), 0
            for dense, cat, labels in wm.input_fn([path], 1, a.batch_size, device=device):
                k += labels.shape[0]
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            return {"lines": k, "seconds": dt, "lines_per_s": k / dt}

        drain(cut, dev)                                                  # warm-up: pinned buffers, modules
        res["input_fn"] = {"batch_size": a.batch_size, "device_whole_file": drain(full, dev),
                           "device_host_cut": drain(cut, dev), "host_host_cut": drain(cut, None)}
        print("input_fn", res["input_fn"], flush=True)

        # ---- training ----------------------------------------------------------------------------------------------
        def train(B, device):
            m = WideDeep(32, B, "256,128,64", "wide_n_deep", device=dev, seed=0)
            torch.cuda.synchronize()
            t0, k = time.perf_counter(), 0
            for batch in wm.input_fn([tr], 1, B, device=device):
                dense, cat, labels = batch if device is not None else tuple(t.to(dev) for t in batch)
                m.train_step(dense, cat, labels)
                k += labels.shape[0]
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            return k / dt, {name: v.detach().cpu().clone() for name, v in m.variables().items()}

        res["train"] = {"model": "wide_n_deep K=32 256,128,64", "lines": min(a.train_lines, a.lines), "epochs": 1}
        for B in (int(t) for t in a.train_batch_sizes.split(",")):
            train(B, dev)                                                # warm-up at this shape
            rates = {"host": [], "device": []}
            final = {}
            for _ in range(a.rounds):
                for mode, d in (("host", None), ("device", dev)):
                    r, final[mode] = train(B, d)
                    rates[mode].append(r)
            same = all(torch.equal(final["host"][k].view(torch.int32), final["device"][k].view(torch.int32))
                       for k in final["host"])
            res["train"][str(B)] = {"samples_per_s_host_input": rates["host"], "samples_per_s_device_input": rates["device"],
                                    "final_variables_bit_identical": same}
            print("train", B, res["train"][str(B)], flush=True)
    finally:
        shutil.rmtree(data_dir, ignore_errors=True)
    print(json.dumps(res))
    with open(os.path.join(a.out_dir, a.name), "w") as fh:
        json.dump(res, fh, indent=1)
        fh.write("\n")


if __name__ == "__main__":
    main()
