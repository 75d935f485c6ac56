"""libsvm `input_fn`, same contract as deep_ctr/Model_pipeline/DeepFM.py:63-98:

    input_fn(filenames, batch_size=32, num_epochs=1, perform_shuffle=False)
      -> iterator of ({"feat_ids": int32 [B,F,1], "feat_vals": float32 [B,F,1]}, labels float32 [B])

TextLineDataset -> decode_libsvm -> [shuffle(256)] -> repeat(num_epochs) -> batch(batch_size): `repeat`
comes BEFORE `batch`, so batches straddle file and epoch boundaries and only the very last batch may be
partial (it is kept).  Tokenising is done by the native parser in libctr_b200.so (ctr_parse_libsvm,
csrc/libsvm_host.cu) on a small thread pool (the reference uses num_parallel_calls=10).
Tensors are returned in pinned host memory when CUDA is available (ready for an async H2D copy).
"""
from __future__ import annotations

import ctypes
import random
from concurrent.futures import ThreadPoolExecutor
from typing import Dict, Iterator, List, Sequence, Tuple, Union

import numpy as np
import torch

from . import _lib, ops, text_chunks

_L = _lib.raw()
CHUNK = 32 << 20  # bytes per piece of text: a parse task of the host path, a piece of the device path


def _max_rows(n_bytes: int, F: int) -> int:
    return max(1, n_bytes // max(2 * F + 2, 1))  # every row has >= 2F+2 characters


def _parse(data: bytes, lo: int, hi: int, F: int):
    """ctr_parse_libsvm of data[lo:hi], whole lines; the row numbers in its errors count from lo."""
    view = memoryview(data)[lo:hi]
    buf = ctypes.c_char_p(bytes(view)) if lo or hi != len(data) else ctypes.c_char_p(data)
    n_bytes = hi - lo
    max_rows = _max_rows(n_bytes, F)
    ids = np.empty((max_rows, F), dtype=np.int32)
    vals = np.empty((max_rows, F), dtype=np.float32)
    labels = np.empty(max_rows, dtype=np.float32)
    consumed = ctypes.c_size_t(0)
    rows = _L.ctr_parse_libsvm(buf, n_bytes, F, max_rows, 1, ids.ctypes.data, vals.ctypes.data,
                               labels.ctypes.data, ctypes.byref(consumed))
    if rows < 0:
        raise ValueError(_lib.last_error())
    return ids[:rows], vals[:rows], labels[:rows]


def _count_fields(path: str) -> int:
    """The id:val pairs of the file's first line that is not blank (0 when there is none)."""
    for data in text_chunks.chunks(path, 1 << 16):
        if data.strip(b" \r\n"):
            return _L.ctr_libsvm_count_fields(data, len(data))
    return 0


def decode_libsvm_file(path: str, field_size: int = 0, threads: int = 10):
    """Whole file -> (ids int32 [n,F], vals f32 [n,F], labels f32 [n]).  field_size 0 = infer from line 1."""
    F = field_size or _count_fields(path)
    parts = list(text_chunks.pieces(path, CHUNK)) if F > 0 else []
    if not parts:
        return (np.empty((0, max(field_size, 0)), np.int32), np.empty((0, max(field_size, 0)), np.float32),
                np.empty(0, np.float32))
    if len(parts) == 1:
        return _parse(parts[0], 0, len(parts[0]), F)
    with ThreadPoolExecutor(max_workers=threads) as ex:
        parsed = list(ex.map(lambda data: _parse(data, 0, len(data), F), parts))
    return tuple(np.concatenate([p[k] for p in parsed]) for k in range(3))


def _device_parts(files: List[str], num_epochs: int, field_size: int, dev: torch.device, chunk_bytes: int):
    """(ids, vals, labels) CUDA tensors of every piece of every file, num_epochs times (text_chunks.device_parts):
    tokenised by ctr_parse_libsvm_device, a declined piece parsed by ctr_parse_libsvm."""
    fields = {path: field_size or _count_fields(path) for path in files}

    def tokenize(path, text, n_bytes):
        F = fields[path]
        max_rows = _max_rows(n_bytes, F)
        ws = text_chunks.scratch(ops.parse_libsvm_device_workspace_bytes(n_bytes, max_rows), text.device)
        ids, vals, labels, info = ops.parse_libsvm_device_core(text, n_bytes, F, max_rows, ws)
        return (ids, vals, labels), info

    def decode(path, data, line_base):
        return _parse(data, 0, len(data), fields[path]), data.count(b"\n") + (not data.endswith(b"\n"))

    return text_chunks.device_parts([p for p in files if fields[p] > 0], num_epochs, dev, chunk_bytes, tokenize, decode)


def _host_parts(files: List[str], num_epochs: int, field_size: int, perform_shuffle: bool):
    for _ in range(num_epochs):
        for path in files:
            ids, vals, labels = decode_libsvm_file(path, field_size)
            if perform_shuffle:  # tf.data shuffle(buffer_size=256) window semantics
                buf: List[int] = []
                order = []
                for i in range(len(labels)):
                    if len(buf) < 256:
                        buf.append(i)
                        continue
                    j = random.randrange(256)
                    order.append(buf[j]); buf[j] = i
                random.shuffle(buf)
                order.extend(buf)
                ids, vals, labels = ids[order], vals[order], labels[order]
            yield torch.from_numpy(ids), torch.from_numpy(vals), torch.from_numpy(labels)


def _pin(t: torch.Tensor) -> torch.Tensor:
    return t.pin_memory() if torch.cuda.is_available() else t


def input_fn(filenames: Union[str, Sequence[str]], batch_size: int = 32, num_epochs: int = 1,
             perform_shuffle: bool = False, field_size: int = 0, device=None,
             chunk_bytes: int = CHUNK) -> Iterator[Tuple[Dict[str, torch.Tensor], torch.Tensor]]:
    """device=None: host parser, pinned host tensors.  device="cuda[:i]": the text is streamed to the GPU in pieces of
    chunk_bytes and tokenised there (ctr_parse_libsvm_device); batches are CUDA tensors.  Identical values either way.
    perform_shuffle runs on the host parser."""
    print("Parsing", filenames)  # DeepFM.py:64
    files = [filenames] if isinstance(filenames, str) else list(filenames)
    if device is not None and not perform_shuffle:
        parts = _device_parts(files, num_epochs, field_size, torch.device(device), chunk_bytes)
        for ids, vals, labels in text_chunks.batches(parts, batch_size):
            yield {"feat_ids": ids.unsqueeze(-1), "feat_vals": vals.unsqueeze(-1)}, labels
        return
    parts = _host_parts(files, num_epochs, field_size, perform_shuffle)
    for ids, vals, labels in text_chunks.batches(parts, batch_size):
        yield {"feat_ids": _pin(ids.unsqueeze(-1)), "feat_vals": _pin(vals.unsqueeze(-1))}, _pin(labels)
