#!/usr/bin/env python3
"""Times the GPU TFRecord input of DIN / ESMM (tf_repos_b200/tfrecord_device.py) on seeded Ali-CCP-shaped records:
20 000 distinct records from tfrecord.encode_example, tiled to --records (default 1 M) in a temporary directory.
Reports pass-1 device time and GB/s, the emit's device time per batch (ESMM B=8192, DIN B=4096) next to each model's
train-step time at that shape, the wall-clock samples/s of batches() alone and of ESMM training from files, the host
decoder on a 10 k cut as the CPU baseline, and the card name and power limit read in the same run.  One JSON line."""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# the Ali-CCP shape DESIGN.md §6 assumes for ESMM (tools/bench_models.py esmm): F'=11, N=4 519 540, K=16,
# u_shop ~ U{1..499}, the other u_* ~ U{1..49}, a_int ~ U{1..8}: ~333 occurrences and ~2.8 KB a record
F, N, K = 11, 4_519_540, 16
BAG_MAX = {"cat": 49, "shop": 499, "brand": 49, "int": 49}
ESMM_KW = dict(deep_layers="256,128", dropout="0.8,0.5", ctr_task_wgt=0.3, l2_reg=0.005, update_mode="exact_deferred")
DIN_KW = dict(deep_layers="256,128,64", dropout="0.5,0.5,0.5", attention_layers="256", update_mode="exact_deferred")


def _records(n, seed=0):
    from tf_repos_b200 import tfrecord as tfr
    rng = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        ex = {"y": np.float32(rng.rand() < 0.3), "z": np.float32(rng.rand() < 0.05),
              "feat_ids": rng.randint(1, N, F).astype(np.int64), "a_catids": np.int64(rng.randint(1, N)),
              "a_shopids": np.int64(rng.randint(1, N)), "a_brandids": np.int64(rng.randint(1, N)),
              "a_intids": rng.randint(1, N, rng.randint(1, 9)).astype(np.int64)}
        for f, m in BAG_MAX.items():
            ln = int(rng.randint(1, m + 1))
            ex["u_%sids" % f] = rng.randint(1, N, ln).astype(np.int64)
            ex["u_%svals" % f] = (rng.rand(ln) * 3).astype(np.float32)
        out.append(tfr.encode_example(ex))
    return out


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return q
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def _events(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=1_000_000)
    ap.add_argument("--distinct", type=int, default=20_000)
    args = ap.parse_args()
    from tf_repos_b200 import din_main as dm
    from tf_repos_b200 import esmm_main as em
    from tf_repos_b200 import tfrecord as tfr
    from tf_repos_b200.tfrecord_device import TFRecordIndex
    out = {"card": _card()}
    recs = _records(args.distinct)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "part0.tfrecord")
        tfr.write_records(path, recs)
        one = open(path, "rb").read()
        reps = -(-args.records // len(recs))
        with open(path, "wb") as fh:
            for _ in range(reps):
                fh.write(one)
        nbytes = os.path.getsize(path)
        out.update(records=reps * len(recs), file_gb=nbytes / 1e9, bytes_per_record=nbytes / (reps * len(recs)))
        quiet = contextlib.redirect_stdout(io.StringIO())
        with quiet:
            torch.cuda.synchronize(); t0 = time.perf_counter()
            index = TFRecordIndex.build([path], F, ("y", "z"), "cuda")
            torch.cuda.synchronize(); t1 = time.perf_counter()
        out["pass1_wall_s"] = t1 - t0
        out["pass1_gb_s_wall"] = nbytes / (t1 - t0) / 1e9
        # pass-1 device time alone: the scan over one staged 256 MB chunk
        from tf_repos_b200 import ops
        buf = np.frombuffer(one * max(1, (256 << 20) // len(one)), dtype=np.uint8)
        rec_off, consumed, _, _, _ = ops.tfrecord_frame(buf, True, len(buf) // 16 + 1)
        chunk = torch.from_numpy(buf[:consumed].copy()).cuda()
        ro = torch.from_numpy(rec_off).cuda()
        lens = torch.empty(len(rec_off), 5, dtype=torch.int32, device="cuda")
        err = torch.full((1,), -1, dtype=torch.int64, device="cuda")
        ms = _events(lambda: ops.tfrecord_scan(chunk, ro, 0, F, 3, lens, err), 5)
        out["scan_ms_per_256MB"] = ms
        out["scan_gb_s"] = consumed / ms / 1e6
        P, A = index.max_lengths()
        for layout, B in (("esmm", 8192), ("din", 4096)):
            it = index.batches(1, B, layout, P)
            torch.cuda.synchronize(); t0 = time.perf_counter(); k = 0
            for _ in range(50):
                batch, labels, n = next(it); k += n
            torch.cuda.synchronize()
            out[f"{layout}_batches_samples_per_s"] = k / (time.perf_counter() - t0)
            it.close()
        # emit alone, CUDA events over many launches of one staged batch
        for layout, B in (("esmm", 8192), ("din", 4096)):
            stage = chunk
            n_rec = len(rec_off)
            slot = torch.from_numpy((rec_off[np.arange(B) % n_rec] + 12).astype(np.int64)).cuda()
            sizes = np.diff(np.append(rec_off, consumed)) - 16
            slen = torch.from_numpy(sizes[np.arange(B) % n_rec].astype(np.int32)).cuda()
            L = lens.cpu().numpy()[np.arange(B) % n_rec].astype(np.int64)
            feat = torch.empty(B, F, dtype=torch.int32, device="cuda"); a_ids = torch.empty(3, B, dtype=torch.int32, device="cuda")
            y = torch.empty(B, device="cuda"); z = torch.empty(B, device="cuda")
            if layout == "esmm":
                off = np.zeros(5 * B + 1, np.int32); off[1:] = np.cumsum(L.T.reshape(-1))
                offd = torch.from_numpy(off).cuda()
                ids = torch.empty(int(off[-1]), dtype=torch.int32, device="cuda"); wgt = torch.empty(int(off[-1]), device="cuda")
                fn = lambda: ops.tfrecord_emit_esmm(stage, slot, slen, B, F, offd, feat, a_ids, ids, wgt, y, z)  # noqa: E731
            else:
                Pd = int(L[:, :4].max())
                off = np.zeros(B + 1, np.int32); off[1:] = np.cumsum(L[:, 4])
                offd = torch.from_numpy(off).cuda()
                ids = torch.empty(int(off[-1]), dtype=torch.int32, device="cuda")
                ui = torch.empty(4, B, Pd, dtype=torch.int32, device="cuda"); uw = torch.empty(4, B, Pd, device="cuda")
                fn = lambda: ops.tfrecord_emit_din(stage, slot, slen, B, F, Pd, offd, feat, a_ids, ids, ui, uw, y)  # noqa: E731
            out[f"{layout}_emit_ms_per_batch_B{B}"] = _events(fn, 20)
        # step times at the same shapes (CUDA-event-free wall clock over synchronised repeats), and ESMM training
        # from files
        from tf_repos_b200.din import DIN
        from tf_repos_b200.esmm import ESMM

        def step_ms(model, steps, reps=4):
            for batch, labels, n in steps:
                model.train_step(batch, labels, n_valid=n)
            torch.cuda.synchronize(); t0 = time.perf_counter()
            for _ in range(reps):
                for batch, labels, n in steps:
                    model.train_step(batch, labels, n_valid=n)
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) / (reps * len(steps)) * 1e3

        it = index.batches(1, 4096, "din", P)
        steps = [next(it) for _ in range(8)]
        it.close()
        din = DIN(F, N, K, 4096, P, max_a_int=A, device="cuda:0", **DIN_KW)
        out["din_step_ms_B4096"] = step_ms(din, steps)
        del din, steps
        B = 8192
        cap = index.max_batch_occurrences(1, B)
        model = ESMM(F, N, K, B, cap, device="cuda:0", **ESMM_KW)
        it = index.batches(1, B, "esmm")
        steps = [next(it) for _ in range(8)]
        out["esmm_step_ms_B8192"] = step_ms(model, steps)
        del steps
        torch.cuda.synchronize(); t0 = time.perf_counter(); k = 0
        for i, (batch, labels, n) in enumerate(it):
            model.train_step(batch, labels, n_valid=n); k += n
            if i == 60:
                break
        torch.cuda.synchronize()
        out["esmm_train_from_files_samples_per_s"] = k / (time.perf_counter() - t0)
        it.close()
        # where pass 2's wall time goes: the host preads of one 8192-sample batch's record ranges
        plan = index._plan(1, B, 0, 1, "esmm")
        fd = os.open(path, os.O_RDONLY)
        buf = bytearray(plan["nbytes"])
        mv = memoryview(buf)
        t0 = time.perf_counter()
        for _ in range(10):
            for _fid, off, cnt, at in plan["reads"]:
                os.preadv(fd, [mv[at:at + cnt]], off)
        os.close(fd)
        out["pread_ms_per_esmm_batch_one_thread"] = (time.perf_counter() - t0) / 10 * 1e3
        out["staged_mb_per_esmm_batch"] = plan["nbytes"] / 1e6
        # the host decoder on a 10 k cut
        cut = os.path.join(tmp, "cut.tfrecord")
        tfr.write_records(cut, recs[:10_000])
        with contextlib.redirect_stdout(io.StringIO()):
            t0 = time.perf_counter(); d = em.decode([cut], F); t1 = time.perf_counter()
            for idx in dm.index_stream(10_000, 1, 8192):
                em.make_batch(d, idx, 8192, "cpu")
            t2 = time.perf_counter()
        out["host_decode_records_per_s"] = 10_000 / (t1 - t0)
        out["host_make_batch_samples_per_s"] = 10_000 / (t2 - t1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
