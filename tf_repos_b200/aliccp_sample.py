"""Raw Ali-CCP (Tianchi) files -> the joined, remapped, shuffled part files of the TFRecord writer's input, and feat_cnts,
on the GPU: DeepMTL/Feature_pipeline's join (get_join_mapper.py, get_join_reducer.py), stat (get_stat_mapper.py,
get_stat_reducer.py) and remap (get_remap_mapper.py) jobs, through the ctr_aliccp_sample_* entry points
(csrc/aliccp_sample.cu).  Semantics, orders and restrictions: DESIGN.md §2.7; oracle/aliccp_sample.py restates them.

Every file is read in chunks cut at line ends, so nothing about the input has to fit on the host.  Per set (tr, then
te): pass A streams the files once (classify, md5 table, counts of the samples' own tokens; common records stay resident
on the device); then the records' multiplicities, the commons' counts, the vocabulary (tr only) and each record's
remapped text; then pass B streams the chunks that hold samples again: once for the exact line sizes, then once per group
of parts that fits budget_bytes, writing output_dir/<set>/part-%05d."""
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

FIRST_ID = 20                 # get_remap_mapper.py:12
MAX_CHUNK = 1 << 30           # the kernels take chunks below 2^30 bytes
_NONE = (1 << 64) - 1
_LINES, _ERR, _FILTERED, _MALFORMED, _CNT_DROP, _MD5_DROP, _COMMONS, _CBYTES, _SAMPLES = range(9)
_BAD = re.compile(rb"[\x00-\x03\t\n\x0b\x0c\r :]")
_FID = re.compile(rb"(0|[1-9][0-9]*)\Z")
_WHAT = {
    "nul": "NUL byte in the line",
    "md5": "md5 that is empty or longer than 64 bytes",
    "text": "sample_id, y, z, md5 or val holding whitespace, ':' or a byte \\x00-\\x03",
    "field": "field that is empty, longer than 16 bytes, or holds whitespace, ':' or a byte \\x00-\\x03",
    "fid": "fid that is not 0 or [1-9][0-9]* below 2^63",
}


class AliccpSampleError(ValueError):
    pass


def _fault(line: bytes):
    """(kind, token) of the first restriction a kept line breaks (DESIGN.md §2.7), in the order NUL, sample_id, y, z,
    md5, then each token's field, fid, val; None when there is none."""
    s = line.strip()
    if b"\0" in s:
        return "nul", s
    f = s.split(b",")
    text = (f[:3] if len(f) == 6 else []) + [f[-3]]
    for t in text[:-1]:
        if _BAD.search(t):
            return "text", t
    md5 = text[-1]
    if not 1 <= len(md5) <= 64:
        return "md5", md5
    if _BAD.search(md5):
        return "text", md5
    for tok in f[-1].split(b"\x01"):
        field, rest = tok.split(b"\x02")
        fid, val = rest.split(b"\x03")
        if not 1 <= len(field) <= 16 or _BAD.search(field):
            return "field", field
        if not _FID.match(fid) or int(fid) >= (1 << 63):
            return "fid", fid
        if _BAD.search(val):
            return "text", val
    return None


def _raise_fault(path: str, line_no: int, line: bytes):
    kind, token = _fault(line) or ("nul", line)
    shown = token if len(token) <= 80 else token[:77] + b"..."
    raise AliccpSampleError(f"{path}: line {line_no}: {_WHAT[kind]} (not accepted by this implementation): {shown!r}")


def _capacity(what: str, param: str, value: int, hint: str):
    raise AliccpSampleError(f"{what} does not fit ({param}={value}): raise {param} ({hint})")


def _grow(t: torch.Tensor, need: int) -> torch.Tensor:
    if t.numel() >= need:
        return t
    n = torch.empty(max(need, 2 * t.numel()), dtype=t.dtype, device=t.device)
    n[:t.numel()].copy_(t)
    return n


class _Set:
    """The resident state of one set after pass A."""

    def __init__(self, dev):
        self.arena = torch.empty(0, dtype=torch.uint8, device=dev)
        self.rec_off = torch.empty(0, dtype=torch.int64, device=dev)
        self.rec_len = torch.empty(0, dtype=torch.int32, device=dev)
        self.rec_slot = torch.empty(0, dtype=torch.int32, device=dev)
        self.s_rec = torch.empty(0, dtype=torch.int32, device=dev)
        self.s_key = torch.empty(0, dtype=torch.int64, device=dev)
        self.n_bytes = self.n_rec = self.n_samples = 0
        self.chunks: List[tuple] = []    # (path, offset, length, lines, line_base, sample_base) of chunks with samples
        self.stats = {"lines": 0, "commons": 0, "commons_superseded": 0, "samples": 0, "filtered": 0,
                      "malformed": 0, "no_common": 0, "empty_lines": 0}


def _input_files(d: str) -> List[str]:
    return sorted(p for p in glob.glob(os.path.join(d, "*")) if os.path.isfile(p))


def _pass_a(files, mode, count_table, cap, md5_table, seed, parts, chunk_bytes, budget, dev, timer) -> _Set:
    S = _Set(dev)
    info = torch.empty(9, dtype=torch.int64, device=dev)
    line_base = 0
    for path in files:
        file_line, offset = 0, 0
        for piece in pieces(path, chunk_bytes):
            if len(piece) >= MAX_CHUNK:
                raise AliccpSampleError(f"{path}: a line near line {file_line + 1} is 2^30 bytes or longer "
                                        "(not accepted by this implementation)")
            n_lines = piece.count(b"\n") + (0 if piece.endswith(b"\n") else 1)
            text = upload(piece, dev)
            ws_bytes = int(_L.ctr_aliccp_sample_chunk_workspace_bytes(len(piece), n_lines))
            ws = scratch(ws_bytes, dev)
            timer.start()
            check(_L.ctr_aliccp_sample_classify(text.data_ptr(), len(piece), n_lines, mode,
                                                count_table.data_ptr() if mode == 2 else None, cap,
                                                md5_table.data_ptr(), cap, info.data_ptr(), ws.data_ptr(), ws_bytes,
                                                _stream()), "ctr_aliccp_sample_classify")
            timer.stop()
            v = info.tolist()
            if v[_ERR] & _NONE != _NONE:
                row = v[_ERR]
                _raise_fault(path, file_line + row + 1, piece.split(b"\n", row + 1)[row])
            if v[_CNT_DROP]:
                _capacity("the (field, fid) count table", "table_capacity", cap,
                          "about twice the number of distinct field:fid keys of tr")
            if v[_MD5_DROP]:
                _capacity("the md5 table", "table_capacity", cap, "about twice the number of distinct md5s of a set")
            nc, cb, ns = v[_COMMONS], v[_CBYTES], v[_SAMPLES]
            resident = (S.n_bytes + cb) + 16 * (S.n_rec + nc) + 12 * (S.n_samples + ns)
            if resident > budget:
                _capacity("the resident common records and sample summaries (%d bytes by %s line %d)"
                          % (resident, path, file_line + n_lines), "budget_bytes", budget, "or split the input")
            S.arena = _grow(S.arena, S.n_bytes + cb)
            S.rec_off, S.rec_len, S.rec_slot = (_grow(t, S.n_rec + nc) for t in (S.rec_off, S.rec_len, S.rec_slot))
            S.s_rec, S.s_key = (_grow(t, S.n_samples + ns) for t in (S.s_rec, S.s_key))
            timer.start()
            check(_L.ctr_aliccp_sample_place(text.data_ptr(), len(piece), n_lines, line_base, seed, parts,
                                             md5_table.data_ptr(), cap, S.arena.data_ptr(), S.n_bytes,
                                             S.rec_off.data_ptr(), S.rec_len.data_ptr(), S.rec_slot.data_ptr(), S.n_rec,
                                             S.s_rec.data_ptr(), S.s_key.data_ptr(), S.n_samples, ws.data_ptr(),
                                             ws_bytes, _stream()), "ctr_aliccp_sample_place")
            timer.stop()
            if ns:
                S.chunks.append((path, offset, len(piece), n_lines, line_base, S.n_samples))
            S.n_bytes += cb
            S.n_rec += nc
            S.n_samples += ns
            S.stats["lines"] += n_lines
            S.stats["filtered"] += v[_FILTERED]
            S.stats["malformed"] += v[_MALFORMED]
            line_base += n_lines
            file_line += n_lines
            offset += len(piece)
    S.stats["commons"], S.stats["samples"] = S.n_rec, S.n_samples
    return S


def _resolve(S: _Set, md5_table, cap, dev) -> torch.Tensor:
    info = torch.empty(2, dtype=torch.int64, device=dev)
    mult = torch.empty(max(S.n_rec, 1), dtype=torch.int32, device=dev)
    check(_L.ctr_aliccp_sample_resolve(md5_table.data_ptr(), cap, S.s_rec.data_ptr(), S.n_samples,
                                       S.rec_slot.data_ptr(), S.n_rec, mult.data_ptr(), info.data_ptr(), _stream()),
          "ctr_aliccp_sample_resolve")
    S.stats["no_common"], S.stats["commons_superseded"] = info.tolist()
    return mult


def _read(path, offset, length) -> bytes:
    with open(path, "rb") as fh:
        fh.seek(offset)
        return fh.read(length)


def _pass_b(S: _Set, mult, vocab, n_vocab, out_dir, seed, parts, budget, dev, timers) -> None:
    # each record's remapped text, once
    r_off = torch.empty(S.n_rec + 1, dtype=torch.int64, device=dev)
    args = (S.arena.data_ptr(), S.rec_off.data_ptr(), S.rec_len.data_ptr(), mult.data_ptr(), S.n_rec,
            vocab.data_ptr(), n_vocab, r_off.data_ptr())
    timers["render"].start()
    check(_L.ctr_aliccp_sample_render(*args, None, _stream()), "ctr_aliccp_sample_render")
    rendered = scratch(int(r_off[S.n_rec]), dev)
    check(_L.ctr_aliccp_sample_render(*args, rendered.data_ptr(), _stream()), "ctr_aliccp_sample_render")
    timers["render"].stop()

    # exact line sizes, then (part, r_i, line) order and offsets
    s_val = torch.empty(max(S.n_samples, 1), dtype=torch.int64, device=dev)
    info = torch.empty(1, dtype=torch.int64, device=dev)
    empty = 0

    def emit(out, lo, hi):
        nonlocal empty
        for path, offset, length, n_lines, line_base, sample_base in S.chunks:
            text = upload(_read(path, offset, length), dev)
            ws_bytes = int(_L.ctr_aliccp_sample_chunk_workspace_bytes(length, n_lines))
            ws = scratch(ws_bytes, dev)
            timers["pass_b"].start()
            check(_L.ctr_aliccp_sample_emit(text.data_ptr(), length, n_lines, line_base, seed, S.s_rec.data_ptr(),
                                            sample_base, r_off.data_ptr(), rendered.data_ptr(), vocab.data_ptr(),
                                            n_vocab, s_val.data_ptr(), lo, hi, out, info.data_ptr(), ws.data_ptr(),
                                            ws_bytes, _stream()), "ctr_aliccp_sample_emit")
            timers["pass_b"].stop()
            if out is None:
                empty += int(info.item())

    emit(None, 0, 0)
    S.stats["empty_lines"] = empty
    part_bytes = torch.empty(parts, dtype=torch.int64, device=dev)
    ws_bytes = int(_L.ctr_aliccp_sample_order_workspace_bytes(S.n_samples))
    ws = scratch(ws_bytes, dev)
    timers["pass_b"].start()
    check(_L.ctr_aliccp_sample_order(S.s_key.data_ptr(), s_val.data_ptr(), S.n_samples, parts, part_bytes.data_ptr(),
                                     ws.data_ptr(), ws_bytes, _stream()), "ctr_aliccp_sample_order")
    timers["pass_b"].stop()
    del ws
    sizes = part_bytes.tolist()
    starts = np.concatenate([[0], np.cumsum(sizes)]).tolist()

    # groups of consecutive parts that fit budget_bytes, all planned before any file is written
    groups, g0 = [], 0
    for p in range(parts):
        if sizes[p] > budget:
            _capacity("part %d of %s (%d bytes)" % (p, out_dir, sizes[p]), "budget_bytes", budget,
                      "or raise --parts")
        if starts[p + 1] - starts[g0] > budget:
            groups.append((g0, p))
            g0 = p
    groups.append((g0, parts))
    for a, b in groups:
        lo, hi = starts[a], starts[b]
        out = scratch(hi - lo, dev)
        if hi > lo:
            emit(out.data_ptr(), lo, hi)
        for p in range(a, b):
            with open(os.path.join(out_dir, "part-%05d" % p), "wb") as fh:
                out[starts[p] - lo:starts[p + 1] - lo].cpu().numpy().tofile(fh)


def prepare(input_dir: str, output_dir: str, cutoff: int = 20, parts: int = 100, seed: int = 0,
            chunk_bytes: int = 64 << 20, table_capacity: int = 1 << 25, budget_bytes: int = 16 << 30,
            device="cuda") -> Dict:
    """The join, stat and remap jobs over input_dir/tr/* and input_dir/te/* (every file, sorted by name) into
    output_dir/{tr,te}/part-%05d and output_dir/feat_cnts (directories made when missing).  te is joined with its own
    common records and remapped with tr's vocabulary; feat_cnts counts tr.
    table_capacity = slots of the (field, fid) count table (32 B each) and of the md5 table (80 B each): about twice
    the distinct keys.  budget_bytes bounds the device bytes of a set's resident common records and sample summaries,
    and of each group of part files written at once.  Running out of either raises before any part file of the set is
    written.  A restriction (DESIGN.md §2.7) raises AliccpSampleError naming file, line and token; the set's partial
    output is removed.
    -> feature_size (= 20 + kept fids), kept_fids, per-set stats and the device milliseconds of each pass."""
    dev = torch.device(device)
    if dev.type != "cuda":
        raise _lib.CtrError("aliccp_sample.prepare runs on a CUDA device (there is no CPU path)")
    if not (1 <= chunk_bytes < MAX_CHUNK and 1 <= table_capacity <= (1 << 31) and 1 <= parts <= (1 << 20)
            and 0 <= seed < (1 << 64) and budget_bytes >= 1):
        raise ValueError("chunk_bytes must be in [1, 2^30), table_capacity in [1, 2^31], parts in [1, 2^20], "
                         "seed in [0, 2^64) and budget_bytes >= 1")
    for d in ("tr", "te"):
        if not os.path.isdir(os.path.join(input_dir, d)):
            raise AliccpSampleError(f"{os.path.join(input_dir, d)}: no such directory")
    for d in (output_dir, os.path.join(output_dir, "tr"), os.path.join(output_dir, "te")):
        os.makedirs(d, exist_ok=True)
    with torch.cuda.device(dev):
        return _prepare(input_dir, output_dir, int(cutoff), int(parts), int(seed), int(chunk_bytes),
                        int(table_capacity), int(budget_bytes), dev)


def _remove(out_dir, parts, extra=()):
    for p in [os.path.join(out_dir, "part-%05d" % i) for i in range(parts)] + list(extra):
        if os.path.exists(p):
            os.remove(p)


def _prepare(input_dir, output_dir, cutoff, parts, seed, chunk_bytes, cap, budget, dev):
    timers = {k: Timer() for k in ("pass_a", "vocab", "render", "pass_b")}
    count_table = torch.zeros(int(_L.ctr_aliccp_sample_count_table_bytes(cap)), dtype=torch.uint8, device=dev)
    md5_table = torch.empty(int(_L.ctr_aliccp_sample_md5_table_bytes(cap)), dtype=torch.uint8, device=dev)
    feat_cnts = os.path.join(output_dir, "feat_cnts")
    result = {}
    vocab, n_vocab = None, 0
    for name, mode in (("tr", 2), ("te", 1)):
        out_dir = os.path.join(output_dir, name)
        md5_table[:72 * cap].zero_()
        md5_table[72 * cap:].fill_(0xFF)
        try:
            S = _pass_a(_input_files(os.path.join(input_dir, name)), mode, count_table, cap, md5_table, seed, parts,
                        chunk_bytes, budget, dev, timers["pass_a"])
            mult = _resolve(S, md5_table, cap, dev)
            if name == "tr":
                info = torch.empty(5, dtype=torch.int64, device=dev)
                timers["vocab"].start()
                check(_L.ctr_aliccp_sample_count_commons(S.arena.data_ptr(), S.rec_off.data_ptr(),
                                                         S.rec_len.data_ptr(), mult.data_ptr(), S.n_rec,
                                                         count_table.data_ptr(), cap, info.data_ptr(), _stream()),
                      "ctr_aliccp_sample_count_commons")
                if info[0].item():
                    _capacity("the (field, fid) count table", "table_capacity", cap,
                              "about twice the number of distinct field:fid keys of tr")
                vocab = torch.empty(cap, dtype=torch.int64, device=dev)
                ws_bytes = int(_L.ctr_aliccp_sample_vocab_workspace_bytes(cap))
                ws = scratch(ws_bytes, dev)
                check(_L.ctr_aliccp_sample_vocab(count_table.data_ptr(), cap, cutoff, vocab.data_ptr(),
                                                 info.data_ptr(), ws.data_ptr(), ws_bytes, _stream()),
                      "ctr_aliccp_sample_vocab")
                _, _, n_vocab, _, fc_bytes = info.tolist()
                text = scratch(fc_bytes, dev)
                check(_L.ctr_aliccp_sample_feat_cnts(text.data_ptr(), ws.data_ptr(), ws_bytes, cap, _stream()),
                      "ctr_aliccp_sample_feat_cnts")
                timers["vocab"].stop()
                del ws
                with open(feat_cnts, "wb") as fh:
                    fh.write(text[:fc_bytes].cpu().numpy().tobytes())
                del text
                count_table = None
            _pass_b(S, mult, vocab, n_vocab, out_dir, seed, parts, budget, dev, timers)
        except BaseException:
            _remove(out_dir, parts, [feat_cnts] if name == "tr" else [])
            raise
        result[name] = S.stats
        del S, mult
    return {"feature_size": FIRST_ID + n_vocab, "kept_fids": n_vocab, **result,
            "device_ms": {k: t.ms() for k, t in timers.items()}}
