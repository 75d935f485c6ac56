"""DIN / ESMM TFRecord input decoded on the GPU (DIN.py:57-99, DeepCvrMTL.py:63-105; DESIGN.md §2.5), streamed from
disk in two passes so the data set is bounded by the disk, not by host RAM:

    index = TFRecordIndex.build(files, field_size, labels)     # pass 1: frame on the host, scan on the device
    P, A = index.max_lengths(); cap = index.max_batch_occurrences(num_epochs, B)
    for batch, labels, n in index.batches(num_epochs, B, "din", P):   # pass 2: pread, upload, emit
        ...

Pass 1 reads every file in chunks, frames the records on the host (ctr_tfrecord_frame) and scans them on the device
(ctr_tfrecord_scan: data CRC, protobuf walk, the checks of din_main.decode_tfrecord_files); it keeps each record's
file, data offset, size and five bag lengths (host numpy arrays, 40 bytes per record).  Pass 2 cuts
din_main.index_stream's order into groups of whole batches within a byte budget, preads each group's contiguous
record ranges into pinned staging, copies them on a side stream and emits every batch (ctr_tfrecord_emit_din /
_esmm) into fresh tensors: exactly din_main.make_batch / esmm_main.make_batch of decode_tfrecord_files, bit for bit.

Errors are those of the host decoder, with its messages: the device reports the first failing record and check, and
the host decoder is run on that record alone to raise its own exception (with the file's path in its message).  Three stated deviations raise where the host is
silent (DESIGN.md §2.5): a masked CRC-32C mismatch (read_records(verify_crc=True)'s message), a schema key holding the
wrong Feature kind or several, and an id outside [0, 2^31).  A protobuf the host decoder reads but protobuf itself
rejects (payload past its parent, varint > 10 bytes, a wire type that cannot hold a message) raises too.
"""
from __future__ import annotations

import contextlib
import io
import os
import struct
import tempfile
from concurrent.futures import ThreadPoolExecutor
from typing import Iterator, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import ops
from .din_main import U_FIELDS, decode_tfrecord_files, max_lengths_of
from .esmm_main import batch_occurrence_max
from .tfrecord import write_records

# schema keys in the device's numbering (include/ctr_b200.h, ctr_tfrecord_scan)
KEYS = ("y", "z", "feat_ids", "a_catids", "a_shopids", "a_brandids", "a_intids") + \
       tuple("u_%sids" % f for f in U_FIELDS) + tuple("u_%svals" % f for f in U_FIELDS)
CHECK_CRC, CHECK_MALFORMED, CHECK_REQUIRED, CHECK_COUNT, CHECK_MISMATCH, CHECK_KIND, CHECK_RANGE = range(7)
_FRAME_MSG = {1: "truncated record header", 2: "corrupted record length", 3: "truncated record"}
_ALIGN = 128          # per-batch offset arrays start on 512-byte boundaries, like fresh allocations
_NONE = (1 << 64) - 1
_READERS, _READ_PIECE = 8, 2 << 20     # pass-2 file reads: threads, bytes per piece


def plan_groups(rec_bytes: np.ndarray, num_epochs: int, B: int, budget: int) -> List[Tuple[int, int]]:
    """index_stream(n, num_epochs, B) cut into groups of whole batches whose records' bytes (rec_bytes[i] each) sum to
    at most `budget`; a batch larger than the budget is a group of its own.  -> [(first batch, end batch)]."""
    n = len(rec_bytes)
    total = n * max(num_epochs, 0)
    if total == 0:
        return []
    nb = -(-total // B)
    cum = np.concatenate([[0], np.cumsum(rec_bytes, dtype=np.int64)])
    ends = np.minimum(np.arange(1, nb + 1, dtype=np.int64) * B, total)
    at = np.concatenate([[0], (ends // n) * cum[n] + cum[ends % n]])      # stream bytes before each batch boundary
    groups, b = [], 0
    while b < nb:
        e = min(max(int(np.searchsorted(at, at[b] + budget, side="right")) - 1, b + 1), nb)
        groups.append((b, e))
        b = e
    return groups


def group_slots(n: int, num_epochs: int, B: int, b0: int, b1: int) -> Tuple[np.ndarray, np.ndarray]:
    """Sample index of every slot of batches [b0, b1) of index_stream(n, num_epochs, B) -- the padded last batch repeats
    its first sample, as make_batch pads it -- and each batch's real sample count."""
    total = n * num_epochs
    t = np.arange(b0 * B, b1 * B, dtype=np.int64)
    t = np.where(t < total, t, (t // B) * B)
    return t % n, np.minimum(total - np.arange(b0, b1, dtype=np.int64) * B, B)


def _host_error(path: str, at: int, F: int, labels) -> Optional[BaseException]:
    """The exception decode_tfrecord_files raises on the record whose header is at byte `at` of `path` (every record
    before it passed the same checks on the device), with `path` in its message; None when it raises nothing."""
    with open(path, "rb") as fh:
        fh.seek(at)
        (length,) = struct.unpack("<Q", fh.read(12)[:8])
        data = fh.read(length)
    with tempfile.TemporaryDirectory() as tmp:
        one = os.path.join(tmp, os.path.basename(path))
        write_records(one, [data])
        try:
            with contextlib.redirect_stdout(io.StringIO()):
                decode_tfrecord_files([one], F, labels)
        except Exception as e:  # noqa: BLE001 -- whatever the host raises is the answer
            e.args = tuple(a.replace(one, path) if isinstance(a, str) else a for a in e.args)
            return e
    return None


class TFRecordIndex:
    """Pass 1 over TFRecord files of tf.Example: per record its file, data offset, data size and bag lengths."""

    def __init__(self, files, field_size, labels, device, file_id, data_off, size, lens):
        self.files, self.field_size, self.labels, self.device = list(files), field_size, tuple(labels), device
        self.file_id, self.data_off, self.size, self.lens = file_id, data_off, size, lens

    def __len__(self) -> int:
        return len(self.size)

    @classmethod
    def build(cls, files: Sequence[str], field_size: int, labels: Sequence[str] = ("y",), device="cuda",
              chunk_bytes: int = 256 << 20) -> "TFRecordIndex":
        """Frames and scans `files` (decode_tfrecord_files' arguments and its "Parsing" line); raises what it raises."""
        print("Parsing", list(files))
        labels = tuple(labels)
        if labels not in (("y",), ("y", "z")):
            raise ValueError(f"labels must be ('y',) or ('y', 'z'), got {labels}")
        dev = torch.device(device)
        mask = 1 | (2 if "z" in labels else 0)
        err = torch.full((1,), -1, dtype=torch.int64, device=dev)
        file_id, data_off, size, lens = [], [], [], []
        first = []                                      # index of each file's first record
        n_rec = 0
        host = torch.empty(0, dtype=torch.uint8)
        for fi, path in enumerate(files):
            first.append(n_rec)
            with open(path, "rb") as fh:
                fsize = os.fstat(fh.fileno()).st_size
                pos, cap = 0, max(int(chunk_bytes), 16)
                while pos < fsize:
                    want = min(cap, fsize - pos)
                    if host.numel() < want:
                        host = torch.empty(want, dtype=torch.uint8, pin_memory=True)
                    buf = host.numpy()[:want]
                    fh.seek(pos)
                    got = fh.readinto(memoryview(buf))
                    if got != want:
                        raise ValueError(f"{path}: short read at byte {pos}")
                    final = pos + want >= fsize
                    rec_off, consumed, cls_, at, need = ops.tfrecord_frame(buf, final, want // 16 + 1)
                    n = len(rec_off)
                    if n:
                        chunk = host[:consumed].to(dev, non_blocking=True)
                        lens_d = torch.empty(n, 5, dtype=torch.int32, device=dev)
                        ops.tfrecord_scan(chunk, torch.from_numpy(rec_off).to(dev), n_rec, field_size, mask, lens_d, err)
                        sizes = np.diff(np.append(rec_off, consumed)) - 16
                        file_id.append(np.full(n, fi, np.int32)); data_off.append(pos + rec_off + 12)
                        size.append(sizes.astype(np.int64)); lens.append(lens_d.cpu().numpy())
                        n_rec += n
                    word = int(err.item()) & _NONE            # also orders the next read after the upload
                    if word != _NONE:
                        cls._raise_device(word, files, first, data_off, field_size, labels)
                    if cls_ == 4 and pos + at + 16 + struct.unpack_from("<Q", buf, at)[0] > fsize:
                        cls_ = 3                              # the host meets the truncation first
                    if cls_:
                        msg = _FRAME_MSG.get(cls_, "record longer than 2^31 - 17 bytes")
                        raise ValueError(f"{path}: {msg} at byte {pos + at}")
                    if consumed == 0:                         # the next record is larger than the chunk
                        cap = max(2 * cap, need)
                    pos += consumed
        cat = (lambda xs, dt: np.concatenate(xs) if xs else np.zeros(0, dt))
        return cls(files, field_size, labels, dev, cat(file_id, np.int32), cat(data_off, np.int64),
                   cat(size, np.int64), cat(lens, np.int32).reshape(-1, 5))

    @staticmethod
    def _raise_device(word, files, first, data_off, F, labels):
        rec, check, arg = word >> 16, (word >> 8) & 0xFF, word & 0xFF
        fi = int(np.searchsorted(np.asarray(first), rec, side="right")) - 1
        path, local = files[fi], rec - first[fi]
        at = int(np.concatenate(data_off)[rec]) - 12
        if check == CHECK_CRC:
            raise ValueError(f"{path}: corrupted record data at byte {at}")
        host = _host_error(path, at, F, labels)      # the host decoder's own exception, if it raises on this record
        if host is not None:
            raise host
        if check <= CHECK_MISMATCH:
            raise ValueError(f"{path}: record {local} (byte {at}): malformed tf.Example protobuf")
        key = KEYS[arg]
        if check == CHECK_KIND:
            kind = "float_list" if key in labels or key.endswith("vals") else "int64_list"
            raise ValueError(f"{path}: record {local} (byte {at}): feature {key} must hold exactly one Feature kind, "
                             f"{kind}")
        raise ValueError(f"{path}: record {local} (byte {at}): {key} holds an id outside [0, 2^31)")

    # ---- what the host functions compute from decode_tfrecord_files' dict ---------------------------------------
    def max_lengths(self) -> Tuple[int, int]:
        """din_main.max_lengths of this input"""
        return max_lengths_of(self.lens)

    def max_batch_occurrences(self, num_epochs: int, B: int) -> int:
        """esmm_main.max_batch_occurrences of this input"""
        return batch_occurrence_max(self.lens.sum(axis=1), num_epochs, B)

    # ---- pass 2 ----------------------------------------------------------------------------------------------------
    def _plan(self, num_epochs: int, B: int, b0: int, b1: int, layout: str) -> dict:
        idx, counts = group_slots(len(self), num_epochs, B, b0, b1)
        G = b1 - b0
        real = (np.arange(G * B) % B) < np.repeat(counts, B)
        seq = idx[real]
        brk = np.ones(len(seq), dtype=bool)
        brk[1:] = (seq[1:] != seq[:-1] + 1) | (self.file_id[seq[1:]] != self.file_id[seq[:-1]])
        run_of = np.cumsum(brk) - 1
        starts = np.flatnonzero(brk)
        last = np.append(starts[1:], len(seq)) - 1
        r_off = self.data_off[seq[starts]]
        r_bytes = self.data_off[seq[last]] + self.size[seq[last]] - r_off
        r_pos = np.concatenate([[0], np.cumsum(r_bytes)[:-1]]).astype(np.int64)
        slot_off = np.empty(G * B, dtype=np.int64)
        slot_off[real] = r_pos[run_of] + self.data_off[seq] - r_off[run_of]
        slot_off = slot_off.reshape(G, B)
        slot_off[:] = np.where(real.reshape(G, B), slot_off, slot_off[:, :1])
        lens = self.lens[idx].reshape(G, B, 5)
        if layout == "din":
            per = lens[:, :, 4]
        else:
            per = lens.transpose(0, 2, 1).reshape(G, 5 * B)
        W = per.shape[1] + 1
        stride = -(-W // _ALIGN) * _ALIGN
        meta32 = np.zeros((G, stride + -(-B // _ALIGN) * _ALIGN), dtype=np.int32)
        meta32[:, 1:W] = np.cumsum(per, axis=1)
        meta32[:, stride:stride + B] = self.size[idx].reshape(G, B)
        reads = list(zip(self.file_id[seq[starts]].tolist(), r_off.tolist(), r_bytes.tolist(), r_pos.tolist()))
        return {"G": G, "counts": counts.tolist(), "slot_off": slot_off, "meta32": meta32, "W": W, "stride": stride,
                "reads": reads, "nbytes": int(r_bytes.sum()), "totals": meta32[:, W - 1].tolist()}

    def batches(self, num_epochs: int, B: int, layout: str = "din", P: int = 0,
                budget_bytes: int = 256 << 20) -> Iterator[tuple]:
        """(batch dict, labels, n) of every batch of index_stream(len, num_epochs, B), as din_main.make_batch (layout
        "din", P >= the longest behaviour list) or esmm_main.make_batch (layout "esmm", labels = (y, z)) return them."""
        if layout not in ("din", "esmm"):
            raise ValueError(f"layout must be 'din' or 'esmm', got {layout!r}")
        if layout == "esmm" and self.labels != ("y", "z"):
            raise ValueError("the esmm layout needs an index built with labels=('y', 'z')")
        if layout == "din" and len(self) and P < self.max_lengths()[0]:
            raise ValueError(f"P={P} is shorter than the longest behaviour list ({self.max_lengths()[0]})")
        groups = plan_groups(self.size + 16, num_epochs, B, budget_bytes)
        if not groups:
            return
        plans = [None] * len(groups)
        dev, F = self.device, self.field_size
        main, side = torch.cuda.current_stream(dev), torch.cuda.Stream(dev)
        copied = [torch.cuda.Event(), torch.cuda.Event()]
        released = [torch.cuda.Event(), torch.cuda.Event()]
        host: List[torch.Tensor] = [torch.empty(0, dtype=torch.uint8)] * 2
        stage: List[torch.Tensor] = [torch.empty(0, dtype=torch.uint8, device=dev)] * 2
        fds = [os.open(p, os.O_RDONLY) for p in self.files]

        def load(gi: int) -> dict:
            """read group gi into host staging gi % 2 and queue its upload on the side stream"""
            s, pl = gi % 2, plans[gi]
            copied[s].synchronize()                      # the previous upload from this host buffer is done
            nb = pl["nbytes"]
            if host[s].numel() < nb:
                host[s] = torch.empty(nb, dtype=torch.uint8, pin_memory=True)
            mv = memoryview(host[s].numpy())

            def read(piece):
                fid, off, cnt, at = piece
                done = 0
                while done < cnt:
                    got = os.preadv(fds[fid], [mv[at + done:at + cnt]], off + done)
                    if got <= 0:
                        raise ValueError(f"{self.files[fid]}: short read at byte {off + done}")
                    done += got
            # one thread copies ~3.6 GB/s out of the page cache, below what a B=8192 ESMM step consumes: the group's
            # ranges are read in _READ_PIECE pieces by _READERS threads (os.preadv releases the GIL)
            pieces = [(fid, off + k, min(_READ_PIECE, cnt - k), at + k)
                      for fid, off, cnt, at in pl["reads"] for k in range(0, cnt, _READ_PIECE)]
            list(readers.map(read, pieces))
            m64 = torch.from_numpy(pl["slot_off"].reshape(-1)).pin_memory()
            m32 = torch.from_numpy(pl["meta32"].reshape(-1)).pin_memory()
            with torch.cuda.stream(side):
                side.wait_event(released[s])             # group gi - 2's emits and train steps are queued before
                if stage[s].numel() < nb:
                    stage[s] = torch.empty(nb, dtype=torch.uint8, device=dev)
                stage[s][:nb].copy_(host[s][:nb], non_blocking=True)
                pl["m64"] = m64.to(dev, non_blocking=True)
                pl["m32"] = m32.to(dev, non_blocking=True)
                copied[s].record(side)
            pl["pinned"] = (m64, m32)
            return pl

        pool = ThreadPoolExecutor(max_workers=1)
        readers = ThreadPoolExecutor(max_workers=_READERS)
        fut = None
        try:
            plans[0] = self._plan(num_epochs, B, *groups[0], layout)
            fut = pool.submit(load, 0)
            for gi in range(len(groups)):
                s = gi % 2
                pl = fut.result()
                fut = None
                main.wait_event(copied[s])
                for t in (pl["m64"], pl["m32"]):
                    t.record_stream(main)
                if gi + 1 < len(groups):
                    plans[gi + 1] = self._plan(num_epochs, B, *groups[gi + 1], layout)
                    fut = pool.submit(load, gi + 1)
                m64, m32, W, stride = pl["m64"].view(pl["G"], B), pl["m32"].view(pl["G"], -1), pl["W"], pl["stride"]
                for g in range(pl["G"]):
                    off, slot_len = m32[g, :W].clone(), m32[g, stride:stride + B]
                    total = pl["totals"][g]
                    feat_ids = torch.empty(B, F, dtype=torch.int32, device=dev)
                    a_ids = torch.empty(3, B, dtype=torch.int32, device=dev)
                    ids = torch.empty(total, dtype=torch.int32, device=dev)
                    y = torch.empty(B, dtype=torch.float32, device=dev)
                    if layout == "din":
                        u_ids = torch.empty(4, B, P, dtype=torch.int32, device=dev)
                        u_wgt = torch.empty(4, B, P, dtype=torch.float32, device=dev)
                        ops.tfrecord_emit_din(stage[s], m64[g], slot_len, B, F, P, off, feat_ids, a_ids, ids, u_ids,
                                              u_wgt, y)
                        batch = {"feat_ids": feat_ids, "a_ids": a_ids, "a_int_ids": ids, "a_int_off": off,
                                 "u_ids": u_ids, "u_wgt": u_wgt}
                        yield batch, y, pl["counts"][g]
                    else:
                        wgt = torch.empty(total, dtype=torch.float32, device=dev)
                        z = torch.empty(B, dtype=torch.float32, device=dev)
                        ops.tfrecord_emit_esmm(stage[s], m64[g], slot_len, B, F, off, feat_ids, a_ids, ids, wgt, y, z)
                        batch = {"feat_ids": feat_ids, "a_ids": a_ids, "bag_ids": ids, "bag_wgt": wgt, "bag_off": off}
                        yield batch, (y, z), pl["counts"][g]
                released[s].record(main)                 # everything that reads stage[s] is queued before this
                plans[gi] = None
        finally:
            if fut is not None:
                with contextlib.suppress(Exception):
                    fut.result()
            pool.shutdown(wait=True)
            readers.shutdown(wait=True)
            side.synchronize()
            main.synchronize()
            for fd in fds:
                os.close(fd)
