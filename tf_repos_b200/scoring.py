"""What the drop-in scripts do with the predictions of --task_type=eval and infer, on the device (DESIGN.md §2.13).

AucCounts: tf.metrics.auc (DeepFM.py:194, DeepCvrMTL.py:229-233) from per-class threshold histograms that
ctr_auc_counts accumulates on the device; auc() copies them once and evaluates estimator.auc_from_counts, the float32
arithmetic auc_200 uses, so the value is auc_200's bit for bit.

PredWriter: pred.txt (DeepFM.py:351-353) formatted by ctr_format_preds into one device text buffer at a device-resident
offset, so no batch waits for the host.  Before a batch whose worst case (rows x columns x 48 bytes) would not fit, and
at close(), the host synchronises once, copies the text to pinned memory and writes it to the file.
"""
from __future__ import annotations

from typing import Callable, List, Optional

import numpy as np
import torch

from . import ops
from .estimator import auc_from_counts, auc_thresholds

N_BINS = 201
ROW_BYTES = 48          # "%f" of a float32 is at most 47 characters, then '\t' or '\n'
BUFFER_BYTES = 64 << 20


class AucCounts:
    """One device counts tensor per AUC head.  add() only enqueues work; auc() copies the counts once."""

    def __init__(self, device, heads: int = 1):
        self.thresholds = torch.from_numpy(auc_thresholds()).to(device)
        self.counts = torch.zeros(heads, 2, N_BINS, dtype=torch.int64, device=device)
        self.rows = [0] * heads

    def add(self, pred: torch.Tensor, label: torch.Tensor, head: int = 0) -> None:
        ops.auc_counts(pred, label, self.thresholds, self.counts[head])
        self.rows[head] += pred.numel()

    def auc(self) -> List[float]:
        return [auc_of_histogram(c) for c in self.counts.cpu().numpy()]


def auc_of_histogram(c: np.ndarray) -> float:
    """tf.metrics.auc of ctr_auc_counts' int64 [2, 201] histogram (row 0: negatives, row 1: positives; bin k: k
    thresholds below the prediction)."""
    neg, pos = c
    # tp[i] = positives above threshold i = those in bins i+1 .. 200, as auc_200 counts them
    tp = np.cumsum(pos[::-1])[::-1][1:].astype(np.float32)
    fp = np.cumsum(neg[::-1])[::-1][1:].astype(np.float32)
    fn = int(pos.sum()) - tp
    tn = int(neg.sum()) - fp
    return auc_from_counts(tp, fp, fn, tn)


class PredWriter:
    """pred.txt with "%f\\n" (columns=1) or "%f\\t%f\\n" (columns=2) per row, formatted on the device.

    check: called before every write to the file (the device work is complete then), e.g. the model's check_ids, so
    that a bad id raises before the lines of its flush reach the file.  Without a check the file is opened (and
    truncated) at once, as `open(path, "w")` before the scoring loop; with one, at the first write."""

    def __init__(self, path: str, device, columns: int = 1, buffer_bytes: int = BUFFER_BYTES,
                 check: Optional[Callable[[], None]] = None):
        if columns not in (1, 2):
            raise ValueError("columns must be 1 or 2")
        if buffer_bytes < columns * ROW_BYTES:
            raise ValueError(f"buffer_bytes={buffer_bytes}: smaller than one row ({columns * ROW_BYTES} bytes)")
        self.path, self.columns, self.check = path, columns, check
        self.buf = torch.empty(buffer_bytes, dtype=torch.uint8, device=device)
        self.offset = torch.zeros(1, dtype=torch.int64, device=device)
        self.ws = torch.empty(0, dtype=torch.uint8, device=device)
        self.host: Optional[torch.Tensor] = None
        self.reserved = 0     # worst-case bytes enqueued since the last flush (>= the device offset)
        self.fo = None if check is not None else open(path, "wb")

    def add(self, a: torch.Tensor, b: Optional[torch.Tensor] = None) -> None:
        """Enqueues the rows of a (and b, columns=2); a batch larger than the buffer goes in pieces."""
        if (b is None) != (self.columns == 1):
            raise ValueError(f"PredWriter of {self.columns} columns")
        n = a.numel()
        row = self.columns * ROW_BYTES
        step = self.buf.numel() // row
        for i in range(0, n, step):
            m = min(step, n - i)
            if self.reserved + m * row > self.buf.numel():
                self.flush()
            need = ops.format_preds_workspace_bytes(m)
            if self.ws.numel() < need:
                self.ws = torch.empty(need, dtype=torch.uint8, device=self.buf.device)
            ops.format_preds(a[i:i + m], None if b is None else b[i:i + m], self.buf, self.offset, self.ws)
            self.reserved += m * row

    def flush(self) -> None:
        """One synchronisation: the text so far -> pinned memory -> the file."""
        if self.reserved == 0:
            return
        n = int(self.offset.item())
        if n > self.buf.numel():
            raise RuntimeError(f"PredWriter: {n} bytes of text in a buffer of {self.buf.numel()}")
        self._write(n)
        self.offset.zero_()
        self.reserved = 0

    def _write(self, n: int) -> None:
        if self.check is not None:
            self.check()
        if self.fo is None:
            self.fo = open(self.path, "wb")
        if n:
            if self.host is None:
                self.host = torch.empty(self.buf.numel(), dtype=torch.uint8, pin_memory=True)
            self.host[:n].copy_(self.buf[:n])
            self.fo.write(memoryview(self.host.numpy())[:n])

    def close(self) -> None:
        """Writes what is left; an input without rows leaves an empty file."""
        self.flush()
        if self.fo is None:
            self._write(0)
        self.fo.close()

    def __enter__(self):
        return self

    def __exit__(self, exc_type, exc, tb):
        if exc_type is None:
            self.close()
        elif self.fo is not None:
            self.fo.close()
        return False
