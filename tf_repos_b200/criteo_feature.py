"""Criteo raw TSV -> tr.libsvm / va.libsvm / te.libsvm / feature_map on the GPU: the whole of
deep_ctr/Feature_pipeline/get_criteo_feature.py, through the ctr_criteo_* entry points (csrc/criteo_feature.cu).

The files are read in chunks cut at line ends and uploaded one at a time, so inputs may be larger than device memory;
only the count table (table_capacity slots of 16 bytes) and the vocabulary stay resident.  The output files are
byte-identical to what the reference writes under Python 2.7, except feature_map's line order (Python 2 dict order
there; here each field's ids 1..n, then <unk>).  What the reference raises on, this raises on, naming file, line and
column; the restrictions of DESIGN.md §2.4 raise the same way."""
from __future__ import annotations

import os
from typing import Dict, List

import numpy as np
import torch

from . import _lib
from ._lib import check
from .ops import _stream
from .text_chunks import Timer, chunks, scratch, upload

_L = _lib.raw()

N_INT, N_CAT = 13, 26
MAXSIZE = 2 ** 63 - 1          # Python 2's sys.maxsize on LP64: the reference's initial min / -max (:71-72)
_NONE = (1 << 64) - 1           # error word: no error
_WHAT = {
    1: "too few columns (the reference raises IndexError here)",
    2: "not an integer of the form [+-]?[0-9]+ (the only form this implementation accepts)",
    3: "integer magnitude above 2^53 (this implementation accepts |value| <= 2^53, where int and float are exact)",
    4: "categorical value longer than 8 bytes (this implementation accepts at most 8)",
    5: "categorical value contains a NUL byte (not accepted by this implementation)",
    6: "categorical value is the literal <unk>, which the reference would overwrite with id 0 and so shift every "
       "later offset (not accepted by this implementation)",
    7: "max == min for this column over train.txt and the value is not empty (the reference raises "
       "ZeroDivisionError here)",
}


class CriteoFeatureError(ValueError):
    pass


def split_decisions(n: int, state: np.random.RandomState) -> np.ndarray:
    """to tr.libsvm? for the next n train lines (:127,148).  The reference runs under Python 2, where
    random.randint(0, 9999) is int(random() * 10000) after random.seed(0); RandomState([0]) seeds MT19937 the same
    way (init_by_array([0])) and random_sample() is random()'s 53-bit draw."""
    return (np.floor(state.random_sample(n) * 10000).astype(np.int64) % 10) != 0


def _column(col: int, test: bool) -> str:
    j = col + (1 if test else 0)
    return "label" if j == 0 else (f"I{j}" if j <= N_INT else f"C{j - N_INT}")


def _raise(path: str, word: int, test: bool = False):
    line, col, code = (word >> 16) & ((1 << 46) - 1), (word >> 8) & 0xFF, word & 0xFF
    raise CriteoFeatureError(f"{path}: line {line + 1}, column {col} ({_column(col, test)}): {_WHAT[code]}")


def preprocess(input_dir: str, output_dir: str, cutoff: int = 200, device="cuda", chunk_bytes: int = 64 << 20,
               table_capacity: int = 1 << 26) -> Dict:
    """get_criteo_feature.py's preprocess(): reads input_dir + 'train.txt' and input_dir + 'test.txt' (plain string
    concatenation, as the reference builds its paths) and writes output_dir + 'feature_map', 'tr.libsvm', 'va.libsvm',
    'te.libsvm'.  table_capacity = slots of the categorical count table: at least the number of distinct
    (field, value) pairs of train.txt, better twice that (16 bytes each; it raises when too small).
    Returns dict_sizes, feature_size (= offset[26]: every emitted id is below it), offsets, min/max, line counts
    and the device milliseconds of each pass."""
    train, test = input_dir + "train.txt", input_dir + "test.txt"
    dev = torch.device(device)
    if dev.type != "cuda":
        raise _lib.CtrError("criteo_feature.preprocess runs on a CUDA device (there is no CPU path)")
    if chunk_bytes < 1 or chunk_bytes >= (1 << 30) or not (1 <= table_capacity <= (1 << 31)):
        raise ValueError("chunk_bytes must be in [1, 2^30) and table_capacity in [1, 2^31]")
    with torch.cuda.device(dev):
        return _preprocess(train, test, output_dir, int(cutoff), dev, int(chunk_bytes), int(table_capacity))


def _preprocess(train, test, output_dir, cutoff, dev, chunk_bytes, cap):
    cap_name = f"table_capacity={cap}"
    table = torch.zeros(int(_L.ctr_criteo_table_bytes(cap)), dtype=torch.uint8, device=dev)
    minmax = torch.tensor([MAXSIZE] * N_INT + [-MAXSIZE] * N_INT, dtype=torch.int64, device=dev)
    info = torch.empty(5, dtype=torch.int64, device=dev)
    timers = {k: Timer() for k in ("stats", "vocab", "emit_train", "emit_test")}

    # ---- pass 1: min/max and categorical counts (:74-85, :39-45) ----
    chunk_lines: List[int] = []
    line_base, n_bytes, first_dict_err, last = 0, 0, _NONE, b""
    for data in chunks(train, chunk_bytes):
        text = upload(data, dev)
        ws_bytes = int(_L.ctr_criteo_stats_workspace_bytes(len(data)))
        ws = scratch(ws_bytes, dev)
        timers["stats"].start()
        check(_L.ctr_criteo_stats(text.data_ptr(), len(data), line_base, table.data_ptr(), cap, minmax.data_ptr(),
                                  info.data_ptr(), ws.data_ptr(), ws_bytes, _stream()), "ctr_criteo_stats")
        timers["stats"].stop()
        n, word, dropped = info[:3].tolist()
        word &= _NONE
        if dropped:
            raise CriteoFeatureError(
                f"{train}: the categorical count table is full ({cap_name} slots; {dropped} values found no slot in "
                f"the chunk ending at line {line_base + n}): raise table_capacity (about twice the number of distinct "
                "(field, value) pairs)")
        if word != _NONE and word >> 62 == 0:
            _raise(train, word)          # the reference's min/max pass runs over the whole file before anything else
        first_dict_err = min(first_dict_err, word)
        chunk_lines.append(n)
        line_base += n
        n_bytes += len(data)
        last = data
    if first_dict_err != _NONE:
        _raise(train, first_dict_err)
    n_train = line_base

    # ---- vocabulary (:46-51) ----
    vocab_keys = torch.empty(cap, dtype=torch.int64, device=dev)
    field_counts = torch.empty(N_CAT, dtype=torch.int64, device=dev)
    ws_bytes = int(_L.ctr_criteo_vocab_workspace_bytes(cap))
    ws = scratch(ws_bytes, dev)
    timers["vocab"].start()
    check(_L.ctr_criteo_vocab(table.data_ptr(), cap, cutoff, vocab_keys.data_ptr(), field_counts.data_ptr(),
                              ws.data_ptr(), ws_bytes, _stream()), "ctr_criteo_vocab")
    timers["vocab"].stop()
    del ws
    counts = field_counts.tolist()
    for i, c in enumerate(counts):
        if c == 0:   # the reference: `vocabs, _ = list(zip(*[]))` -> ValueError (:49)
            raise CriteoFeatureError(f"{train}: column C{i + 1}: no value occurs at least cutoff={cutoff} times "
                                     "(the reference raises ValueError here)")
    keys = vocab_keys[:sum(counts)].cpu().numpy().view(np.uint64).astype(">u8").view("S8")   # trailing NULs dropped
    dict_sizes = [c + 1 for c in counts]
    offsets = [N_INT]
    for i in range(1, N_CAT + 1):
        offsets.append(offsets[i - 1] + dict_sizes[i - 1])

    # ---- feature_map (:116-125): per field ids 1..n, then <unk> ----
    fmap = [b"I%d %d\n" % (i, i) for i in range(1, N_INT + 1)]
    pos = 0
    for i in range(N_CAT):
        base = offsets[i] + 1
        fmap.extend(b"C%d|%s %d\n" % (i + 1, k, base + j + 1) for j, k in enumerate(keys[pos:pos + counts[i]].tolist()))
        fmap.append(b"C%d|<unk> %d\n" % (i + 1, base))
        pos += counts[i]
    with open(output_dir + "feature_map", "wb") as fh:
        fh.write(b"".join(fmap))

    mm = minmax.tolist()
    lo, hi = mm[:N_INT], mm[N_INT:]
    num_min = torch.tensor([float(v) for v in lo], dtype=torch.float64, device=dev)            # float - int (:91)
    num_den = torch.tensor([float(b - a) for a, b in zip(lo, hi)], dtype=torch.float64, device=dev)   # float / int
    off_dev = torch.tensor(offsets[:N_CAT], dtype=torch.int64, device=dev)
    body = last[:-1] if last.endswith(b"\n") else last
    label = body[body.rfind(b"\n") + 1:].split(b"\t")[0]     # `label` of the last train line, used by te (:147,167)
    label_dev = upload(label, dev) if label else None

    def emit(path, files, test, timer, lines_per_chunk=None):
        rs = np.random.RandomState([0])              # random.seed(0) (:127)
        line_base, n_tr, n_va = 0, 0, 0
        for k, data in enumerate(chunks(path, chunk_bytes)):
            text = upload(data, dev)
            flags = None
            if not test:
                flags = torch.from_numpy(split_decisions(lines_per_chunk[k], rs).astype(np.uint8)).to(dev)
            ws_bytes = int(_L.ctr_criteo_emit_workspace_bytes(len(data)))
            ws = scratch(ws_bytes, dev)
            common = (table.data_ptr(), cap, num_min.data_ptr(), num_den.data_ptr(), off_dev.data_ptr(),
                      label_dev.data_ptr() if (test and label_dev is not None) else None, len(label) if test else 0)
            flag_ptr = flags.data_ptr() if flags is not None and flags.numel() else None
            timer.start()
            check(_L.ctr_criteo_emit_plan(text.data_ptr(), len(data), int(test), line_base, flag_ptr, *common,
                                          info.data_ptr(), ws.data_ptr(), ws_bytes, _stream()), "ctr_criteo_emit_plan")
            timer.stop()
            n, word, tr_lines, tr_bytes, va_bytes = info.tolist()
            word &= _NONE
            if word != _NONE:
                _raise(path, word, test)
            out_tr = scratch(tr_bytes, dev)
            out_va = scratch(va_bytes, dev)
            timer.start()
            check(_L.ctr_criteo_emit_write(text.data_ptr(), len(data), int(test), flag_ptr, *common, out_tr.data_ptr(),
                                           out_va.data_ptr(), ws.data_ptr(), ws_bytes, _stream()),
                  "ctr_criteo_emit_write")
            timer.stop()
            files[0].write(out_tr[:tr_bytes].cpu().numpy().tobytes())
            if va_bytes:
                files[1].write(out_va[:va_bytes].cpu().numpy().tobytes())
            line_base += n
            n_tr += tr_lines
            n_va += n - tr_lines
        return n_tr, n_va

    # ---- pass 2: train -> tr / va (:127-151) ----
    with open(output_dir + "tr.libsvm", "wb") as f_tr, open(output_dir + "va.libsvm", "wb") as f_va:
        n_tr, n_va = emit(train, (f_tr, f_va), False, timers["emit_train"], chunk_lines)
    assert n_tr + n_va == n_train
    # ---- pass 3: test -> te (:153-167) ----
    with open(output_dir + "te.libsvm", "wb") as f_te:
        n_te, _ = emit(test, (f_te, None), True, timers["emit_test"])
    return {"dict_sizes": dict_sizes, "feature_size": offsets[N_CAT], "offsets": offsets[:N_CAT], "min": lo, "max": hi,
            "lines": {"tr": n_tr, "va": n_va, "te": n_te}, "train_bytes": n_bytes,
            "test_bytes": os.path.getsize(test), "device_ms": {k: t.ms() for k, t in timers.items()}}
