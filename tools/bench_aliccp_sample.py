#!/usr/bin/env python
"""Times tf_repos_b200.aliccp_sample.prepare on seeded synthetic raw Ali-CCP data (DESIGN.md §6): pass A, the vocabulary,
the rendering of the common records, pass B and the wall clock.  The data is shaped like the Tianchi files: common
records of about 250 tokens, each shared by many samples, and samples of about 20 tokens.  The CPU oracle runs on a
cut of the same data, and the GPU's output on that cut is checked against it by sha256 in the same run.  Everything is
written under a temporary directory (or --work_dir).  Prints one JSON line.
  python tools/bench_aliccp_sample.py --samples=1000000 --records=20000"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

COMMON = [b"101", b"121", b"122", b"124", b"125", b"126", b"127", b"128", b"129", b"205", b"301", b"109_14",
          b"110_14", b"127_14", b"150_14"]
AD = [b"206", b"207", b"210", b"216", b"508", b"509", b"702", b"853"]


def _tokens(rng, fields, n, n_ids):
    f = rng.randint(len(fields), size=n)
    ids = np.minimum(rng.zipf(1.3, size=n), n_ids).astype(np.int64) + rng.randint(4) * n_ids
    return b"\x01".join(b"%s\x02%d\x03%s" % (fields[a], b, b"1.0" if a < 11 else b"0.693147")
                        for a, b in zip(f.tolist(), ids.tolist()))


def make(d, rng, n_records, n_samples, n_ids):
    os.makedirs(d, exist_ok=True)
    md5s = [b"%032x" % v for v in rng.randint(1 << 62, size=n_records, dtype=np.int64).tolist()]
    with open(os.path.join(d, "common_features.csv"), "wb") as fh:
        for m in md5s:
            fh.write(b"%s,250,%s\n" % (m, _tokens(rng, COMMON, 250, n_ids)))
    pool = [_tokens(rng, AD, 20, n_ids) for _ in range(4096)]
    with open(os.path.join(d, "sample_skeleton.csv"), "wb") as fh:
        rec = rng.randint(n_records, size=n_samples).tolist()
        feats = rng.randint(len(pool), size=n_samples).tolist()
        yz = rng.randint(4, size=n_samples).tolist()
        buf = []
        for j in range(n_samples):
            buf.append(b"%d,%d,%d,%s,20,%s\n" % (j, yz[j] >> 1, yz[j] & 1, md5s[rec[j]], pool[feats[j]]))
            if len(buf) == 65536:
                fh.write(b"".join(buf))
                buf = []
        fh.write(b"".join(buf))


def cut(src, dst, n_lines):
    for name in ("tr", "te"):
        os.makedirs(os.path.join(dst, name))
        for f in sorted(os.listdir(os.path.join(src, name))):
            with open(os.path.join(src, name, f), "rb") as a, open(os.path.join(dst, name, f), "wb") as b:
                for k, line in enumerate(a):
                    if k == n_lines:
                        break
                    b.write(line)


def digest(d, parts):
    h = hashlib.sha256()
    for rel in ["feat_cnts"] + ["%s/part-%05d" % (n, p) for n in ("tr", "te") for p in range(parts)]:
        with open(os.path.join(d, rel), "rb") as fh:
            h.update(fh.read())
    return h.hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=20_000)
    ap.add_argument("--samples", type=int, default=1_000_000)
    ap.add_argument("--ids", type=int, default=1_000_000)
    ap.add_argument("--parts", type=int, default=100)
    ap.add_argument("--cut_lines", type=int, default=3000)
    ap.add_argument("--work_dir", type=str, default=None)
    a = ap.parse_args()
    import torch
    from oracle import aliccp_sample as oa
    from tf_repos_b200 import aliccp_sample as gs
    assert torch.cuda.is_available(), "needs a GPU"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    with tempfile.TemporaryDirectory(dir=a.work_dir) as tmp:
        raw = os.path.join(tmp, "raw")
        rng = np.random.RandomState(0)
        t0 = time.time()
        make(os.path.join(raw, "tr"), rng, a.records, a.samples, a.ids)
        make(os.path.join(raw, "te"), rng, a.records // 4, a.samples // 4, a.ids)
        gen_s = time.time() - t0
        in_bytes = sum(os.path.getsize(os.path.join(raw, n, f)) for n in ("tr", "te")
                       for f in os.listdir(os.path.join(raw, n)))
        # warm-up on the cut (module load, first launches), then the cut against the oracle
        small = os.path.join(tmp, "small")
        cut(raw, small, a.cut_lines)
        gs.prepare(small, os.path.join(tmp, "warm"), parts=a.parts)
        torch.cuda.synchronize()
        gs.prepare(small, os.path.join(tmp, "gpu_cut"), parts=a.parts)
        t0 = time.time()
        ost = oa.prepare(small, os.path.join(tmp, "cpu_cut"), parts=a.parts)
        cpu_s = time.time() - t0
        cut_lines = ost["tr"]["lines"] + ost["te"]["lines"]
        same = digest(os.path.join(tmp, "gpu_cut"), a.parts) == digest(os.path.join(tmp, "cpu_cut"), a.parts)
        # the full run (the page cache holds the files just written)
        torch.cuda.synchronize()
        t0 = time.time()
        st = gs.prepare(raw, os.path.join(tmp, "out"), parts=a.parts)
        torch.cuda.synchronize()
        wall = time.time() - t0
        lines = st["tr"]["lines"] + st["te"]["lines"]
        ms = st["device_ms"]
        print(json.dumps({
            "gpu": smi, "input_bytes": in_bytes, "lines": lines, "records": a.records + a.records // 4,
            "samples_kept": st["tr"]["samples"] + st["te"]["samples"], "kept_fids": st["kept_fids"],
            "feature_size": st["feature_size"], "wall_s": round(wall, 3),
            "device_ms": {k: round(v, 2) for k, v in ms.items()},
            "pass_a_GBps": round(in_bytes / ms["pass_a"] / 1e6, 2),
            "end_to_end_MBps": round(in_bytes / wall / 1e6, 1), "lines_per_s": round(lines / wall),
            "host_share": round(1 - sum(ms.values()) / 1e3 / wall, 3),
            "cpu_oracle_lines_per_s": round(cut_lines / cpu_s), "cut_lines": cut_lines, "cut_sha256_equal": same,
            "data_gen_s": round(gen_s, 1)}))
        assert same, "GPU output differs from the oracle on the cut"


if __name__ == "__main__":
    main()
