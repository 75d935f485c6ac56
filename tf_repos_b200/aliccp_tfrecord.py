"""Joined Ali-CCP samples -> DIN / ESMM TFRecords on the GPU: the whole of
deep_ctr/Feature_pipeline/get_aliccp_tfrecord.py (also DeepMTL/Feature_pipeline/get_tfrecord.py and get_ai_tfrecord.py),
through the ctr_aliccp_* entry points (csrc/aliccp_tfrecord.cu).

Each input file is read in chunks cut at line ends and uploaded one at a time, so files may be far larger than device
memory.  Per chunk: plan (record sizes, declined numbers, first error), the declined numbers converted here with
Python float(), write, copy back, append.  Every output file is byte-identical to
tfrecord.write_records(path, [tfrecord.encode_example(features) ...]) of the features the reference builds (keys
sorted; the reference's own files differ only in TensorFlow's map-entry order, DESIGN.md §2.6).  What the reference
raises on, and the restrictions of DESIGN.md §2.6, raise AliccpTFRecordError (a ValueError) naming the file, the
1-based line and the token, for the first failing line of the file; the file's partial output is removed."""
from __future__ import annotations

import glob
import os
import re
from typing import Dict, List

import numpy as np
import torch

from . import _lib
from ._lib import check
from .ops import _stream
from .text_chunks import Timer, pieces, scratch, upload

_L = _lib.raw()

MAX_LINE = 1 << 31        # a line of this many bytes or more (without its '\n') raises
_NONE = (1 << 64) - 1     # error word: no error
_NUL, _COUNT, _EMPTY, _ID, _FLOAT, _LONG = 1, 2, 3, 4, 5, 6
_WHAT = {
    _NUL: "NUL byte in the line (not accepted by this implementation)",
    _COUNT: "feature list is not (field, fid, val) triples: its token count is not a multiple of 3 (the reference's "
            "np.reshape raises ValueError here)",
    _EMPTY: "empty token in the feature list, which the reference can silently mis-align (not accepted by this "
            "implementation)",
    _ID: "fid of a kept field is not of the form [0-9]+ below 2^63 (the only form this implementation accepts; the "
         "reference raises ValueError on a non-integer fid)",
    _FLOAT: "not a number (the reference's float() raises ValueError here)",
    _LONG: "line of 2^31 bytes or more (not accepted by this implementation)",
}
_KEPT = {b"101", b"121", b"122", b"124", b"125", b"126", b"127", b"128", b"129", b"205", b"301",
         b"109_14", b"110_14", b"127_14", b"150_14", b"206", b"207", b"210", b"216"}
_DIGITS = re.compile(rb"[0-9]+\Z")


class AliccpTFRecordError(ValueError):
    pass


def to_f32(tok: bytes) -> float:
    """float32(float(tok)) under Python 2's float(): Python 3's, except that '_' digit separators are rejected."""
    if b"_" in tok:
        raise ValueError(tok)
    with np.errstate(over="ignore"):
        return np.float64(float(tok)).astype(np.float32)


def _fault_token(line: bytes, code: int) -> bytes:
    """The token the device's error code refers to: for _EMPTY / _ID the first empty token or bad kept fid."""
    s = line.strip()
    if code == _NUL:
        return s
    f3 = s.split(b",")[3]
    if code == _COUNT:
        return f3
    toks = re.split(rb"[ :]", f3)
    for i, t in enumerate(toks):
        if t == b"":
            return t
        if i % 3 == 1 and toks[i - 1] in _KEPT and not (_DIGITS.match(t) and int(t) < (1 << 63)):
            return t
    return b""


def _raise(path: str, line_no: int, code: int, token: bytes):
    shown = token if len(token) <= 80 else token[:77] + b"..."
    raise AliccpTFRecordError(f"{path}: line {line_no}: {_WHAT[code]}: {shown!r}")


def _long_line(piece: bytes):
    """index of the first line of 2^31 bytes (MAX_LINE) or more, or None"""
    pos, k = 0, 0
    while pos < len(piece):
        end = piece.find(b"\n", pos)
        end = len(piece) if end < 0 else end
        if end - pos >= MAX_LINE:
            return k
        pos, k = end + 1, k + 1
    return None


def convert_file(in_path: str, out_path: str, chunk_bytes: int = 64 << 20, device="cuda",
                 timers: Dict[str, Timer] = None) -> Dict:
    """gen_tfrecords(in_file) (:38-102) into out_path.  -> lines, input and output bytes, declined numbers."""
    dev = torch.device(device)
    if dev.type != "cuda":
        raise _lib.CtrError("aliccp_tfrecord runs on a CUDA device (there is no CPU path)")
    if not 1 <= chunk_bytes < (1 << 30):
        raise ValueError("chunk_bytes must be in [1, 2^30)")
    timers = timers if timers is not None else {"plan": Timer(), "write": Timer()}
    stats = {"lines": 0, "in_bytes": 0, "out_bytes": 0, "declined": 0}
    try:
        with torch.cuda.device(dev), open(out_path, "wb") as fo:
            _convert(in_path, fo, chunk_bytes, dev, timers, stats)
    except BaseException:
        if os.path.exists(out_path):
            os.remove(out_path)
        raise
    return stats


def _convert(path, fo, chunk_bytes, dev, timers, stats):
    info = torch.empty(4, dtype=torch.int64, device=dev)
    line_base = 0
    for piece in pieces(path, chunk_bytes):
        if len(piece) >= MAX_LINE:
            k = _long_line(piece)
            if k is not None:
                _raise(path, line_base + k + 1, _LONG, piece[:80])
        text = upload(piece, dev)
        ws_bytes = int(_L.ctr_aliccp_workspace_bytes(len(piece)))
        ws = scratch(ws_bytes, dev)
        timers["plan"].start()
        check(_L.ctr_aliccp_plan(text.data_ptr(), len(piece), line_base, info.data_ptr(), ws.data_ptr(), ws_bytes,
                                 _stream()), "ctr_aliccp_plan")
        timers["plan"].stop()
        n, word, out_bytes, n_decl = info.tolist()
        word &= _NONE
        fail = None                              # (line in the chunk, code, token)
        if word != _NONE:
            fail = ((word >> 8) - line_base, word & 0xFF, None)
        decl_vals = None
        if n_decl:
            spans = torch.empty(3 * n_decl, dtype=torch.int64, device=dev)
            check(_L.ctr_aliccp_declines(text.data_ptr(), len(piece), ws.data_ptr(), ws_bytes, spans.data_ptr(),
                                         _stream()), "ctr_aliccp_declines")
            vals = np.empty(n_decl, dtype=np.float32)
            for i, (row, s, e) in enumerate(spans.view(-1, 3).cpu().tolist()):
                if fail is not None and row >= fail[0]:
                    break                        # on the failing line itself the device's error comes first
                try:
                    vals[i] = to_f32(piece[s:e])
                except ValueError:
                    fail = (row, _FLOAT, piece[s:e])
                    break
            decl_vals = torch.from_numpy(vals).to(dev)
        if fail is not None:
            row, code, token = fail
            if token is None:
                token = _fault_token(piece.split(b"\n", row + 1)[row], code)
            _raise(path, line_base + row + 1, code, token)
        out = scratch(out_bytes, dev)
        timers["write"].start()
        check(_L.ctr_aliccp_write(text.data_ptr(), len(piece), decl_vals.data_ptr() if decl_vals is not None else None,
                                  out.data_ptr(), ws.data_ptr(), ws_bytes, _stream()), "ctr_aliccp_write")
        timers["write"].stop()
        fo.write(out[:out_bytes].cpu().numpy().tobytes())
        line_base += n
        stats["in_bytes"] += len(piece)
        stats["out_bytes"] += out_bytes
        stats["declined"] += n_decl
    stats["lines"] += line_base


def convert(input_dir: str, output_dir: str, chunk_bytes: int = 64 << 20, device="cuda") -> Dict:
    """main() (:104-113): output_dir is created with os.mkdir when missing; every file matching input_dir/*-* (the
    glob is taken once, before anything is written, so outputs in the same directory are not picked up) becomes
    output_dir/<basename>.tfrecord.  Files are converted one after another in sorted order; the first error raises and
    removes that file's partial output (files already converted stay).
    -> files, per-file stats and the device milliseconds of the plan and write passes."""
    if not os.path.exists(output_dir):
        os.mkdir(output_dir)
    files = sorted(glob.glob(os.path.join(input_dir, "*-*")))
    timers = {"plan": Timer(), "write": Timer()}
    per_file: List[Dict] = []
    for f in files:
        out = os.path.join(output_dir, os.path.basename(f) + ".tfrecord")
        per_file.append(dict(convert_file(f, out, chunk_bytes, device, timers), path=out))
    return {"files": files, "outputs": per_file, "device_ms": {k: t.ms() for k, t in timers.items()}}
