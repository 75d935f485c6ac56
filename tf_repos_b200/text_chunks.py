"""Host side of the GPU text pipelines (criteo_feature, aliccp_tfrecord, aliccp_sample, the libsvm and CSV input_fns):
input files read in pieces cut at line ends, the upload of a piece, device scratch buffers, the CUDA-event timer of
each pass, and the streamed tokenising and "repeat before batch" batching of the two input_fns."""
from __future__ import annotations

from typing import Callable, Iterable, Iterator, Sequence, Tuple

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
    """The file in pieces of whole lines, at most chunk_bytes each unless one line alone is longer: each chunk of
    chunks() that is longer than chunk_bytes is cut at the last line end before every chunk_bytes.  The file is read
    into one reused buffer, so a piece costs one copy out of it."""
    buf, n = bytearray(max(chunk_bytes, 1)), 0                # buf[:n]: the bytes after the last line end cut so far
    with open(path, "rb") as fh:
        while True:
            if len(buf) < n + chunk_bytes:                    # no line end yet: the line is longer than a read
                buf.extend(bytes(n + chunk_bytes - len(buf)))
            with memoryview(buf) as mv:
                got = fh.readinto(mv[n:n + chunk_bytes])
            if not got:
                if n:
                    with memoryview(buf) as mv:
                        piece = bytes(mv[:n])
                    yield piece
                return
            n += got
            cut = buf.rfind(b"\n", 0, n) + 1
            if cut == 0:
                continue
            pos = 0
            while pos < cut:
                end = cut if cut - pos <= chunk_bytes else buf.rfind(b"\n", pos, pos + chunk_bytes) + 1
                if end <= pos:                                # one line longer than chunk_bytes
                    end = buf.find(b"\n", pos, cut) + 1
                with memoryview(buf) as mv:
                    piece = bytes(mv[pos:end])
                yield piece
                pos = end
            buf[:n - cut] = buf[cut:n]
            n -= cut


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


def device_parts(files: Sequence[str], num_epochs: int, dev: torch.device, chunk_bytes: int, tokenize: Callable,
                 decode: Callable) -> Iterator[Tuple[torch.Tensor, ...]]:
    """Row-aligned tuples of CUDA tensors for every piece of every file, num_epochs times, tokenised on the GPU.

    The file is read in pieces of whole lines (pieces), a piece is staged in pinned memory, copied on a side stream and
    tokenised on the current stream by the format's kernel; a piece the kernel declines is decoded on the host.
      tokenize(path, text, n_bytes) -> (outputs, info int64 [5] on the device) for text[:n_bytes], without waiting
        for the device; info = (rows, bytes consumed, blank lines, malformed lines, lines with a number for the host),
        and the first `rows` rows of the outputs are the piece's;
      decode(path, data, line_base) -> (host arrays, lines in the piece): the host decoder, which owns every error
        message; line_base = lines of the file before the piece.
    Piece i+1 is read and its copy queued before piece i's counters are read back, so the copy runs under piece i's
    kernel and under whatever the consumer queues for piece i's batches; that read-back is the only synchronise."""
    main, side = torch.cuda.current_stream(dev), torch.cuda.Stream(dev)
    copied = [torch.cuda.Event(), torch.cuda.Event()]
    host = [torch.empty(max(chunk_bytes, 1), dtype=torch.uint8, pin_memory=True) for _ in range(2)]
    text = [scratch(chunk_bytes, dev) for _ in range(2)]

    def stream():
        for _ in range(num_epochs):
            for path in files:
                line_base = [0]                               # advanced by the consumer of each piece
                for data in pieces(path, chunk_bytes):
                    yield path, line_base, data

    def stage(i: int, data: bytes):
        """stage piece i and queue its copy.  Piece i-2's counters have been read back by now, so its copy and its
        kernel, the last users of host[s] and text[s], are done."""
        s, n = i % 2, len(data)
        if host[s].numel() < n:                               # one line longer than chunk_bytes
            host[s] = torch.empty(n, dtype=torch.uint8, pin_memory=True)
            text[s] = scratch(n, dev)
            side.wait_stream(main)                            # the new block may be memory main's queue still reads
        host[s].numpy()[:n] = np.frombuffer(data, dtype=np.uint8)
        with torch.cuda.stream(side):
            text[s][:n].copy_(host[s][:n], non_blocking=True)
            copied[s].record(side)

    it = stream()
    nxt = next(it, None)
    if nxt is not None:
        stage(0, nxt[2])
    i = 0
    try:
        while nxt is not None:
            path, line_base, data = nxt
            s, n = i % 2, len(data)
            main.wait_event(copied[s])
            outputs, info = tokenize(path, text[s], n)
            nxt = next(it, None)
            if nxt is not None:
                stage(i + 1, nxt[2])
            rows, consumed, blank, bad, number = info.tolist()
            if blank or bad or number or consumed != n:
                arrays, n_lines = decode(path, data, line_base[0])
                outputs = tuple(torch.from_numpy(a).to(dev) for a in arrays)
                line_base[0] += n_lines
            else:
                outputs = tuple(t[:rows] for t in outputs)
                line_base[0] += rows
            yield outputs
            i += 1
    finally:
        side.synchronize()                                    # no copy out of the pinned buffers is left in flight


def batches(parts: Iterable[Tuple[torch.Tensor, ...]], batch_size: int) -> Iterator[Tuple[torch.Tensor, ...]]:
    """Batches of batch_size rows over a stream of row-aligned tuples of tensors, as tf.data's repeat before batch
    makes them: batches straddle parts (pieces, files and epochs), the last partial batch is kept.  A batch inside
    one part is a view into it; only the rows that straddle two parts are copied."""
    carry = None                                              # fewer than batch_size rows waiting for the next part
    for part in parts:
        n = part[0].shape[0]
        if n == 0:
            continue
        lo = 0
        if carry is not None:
            lo = min(batch_size - carry[0].shape[0], n)
            carry = tuple(torch.cat([c, p[:lo]]) for c, p in zip(carry, part))
            if carry[0].shape[0] < batch_size:
                continue
            yield carry
            carry = None
        n_full = lo + ((n - lo) // batch_size) * batch_size
        for b in range(lo, n_full, batch_size):
            yield tuple(p[b:b + batch_size] for p in part)
        if n_full < n:
            carry = tuple(p[n_full:] for p in part)
    if carry is not None:
        yield carry
