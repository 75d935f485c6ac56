"""Host side of the GPU text pipelines (criteo_feature, aliccp_tfrecord, aliccp_sample, wide_n_deep's CSV input):
input files read in pieces cut at line ends, the upload of a piece, device scratch buffers and the CUDA-event timer of
each pass."""
from __future__ import annotations

from typing import Iterator

import numpy as np
import torch


def chunks(path: str, chunk_bytes: int) -> Iterator[bytes]:
    """The file in pieces of about chunk_bytes that end at a '\\n' (the last piece: at the end of the file)."""
    with open(path, "rb") as fh:
        rest = b""
        while True:
            buf = fh.read(chunk_bytes)
            data = rest + buf
            if not buf:
                if data:
                    yield data
                return
            cut = data.rfind(b"\n") + 1
            if cut == 0:
                rest = data
                continue
            yield data[:cut]
            rest = data[cut:]


def pieces(path: str, chunk_bytes: int) -> Iterator[bytes]:
    """The file in pieces of whole lines, at most chunk_bytes each unless one line alone is longer."""
    for data in chunks(path, chunk_bytes):
        if len(data) <= chunk_bytes:
            yield data
            continue
        pos = 0
        while pos < len(data):
            end = data.rfind(b"\n", pos, pos + chunk_bytes) + 1
            if end <= pos:
                end = data.find(b"\n", pos) + 1 or len(data)
            yield data[pos:end]
            pos = end


class Timer:
    """Device time of the enqueued work between start() and stop(), summed over calls (CUDA events)."""

    def __init__(self):
        self.pairs = []

    def start(self):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        self.pairs.append([e, None])

    def stop(self):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        self.pairs[-1][1] = e

    def ms(self) -> float:
        torch.cuda.synchronize()
        return sum(a.elapsed_time(b) for a, b in self.pairs)


def scratch(nbytes: int, dev) -> torch.Tensor:
    """Uninitialised device bytes (at least one, so that data_ptr() is a real pointer)."""
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=dev)


def upload(data: bytes, dev) -> torch.Tensor:
    return torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).to(dev)
