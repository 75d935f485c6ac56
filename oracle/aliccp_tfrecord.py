"""Pure-Python restatement of deep_ctr/Feature_pipeline/get_aliccp_tfrecord.py's gen_tfrecords (:38-102), the test
oracle of tf_repos_b200.aliccp_tfrecord.  Written from the script's semantics (DESIGN.md §2.6), under Python 3:

- every line of a file (Python 2 file iteration: split after each '\\n') is `line.strip().split(',')`; lines without
  exactly 4 fields are skipped;
- y = float(fields[1]), z = float(fields[2]) (Python 2 float(), then float32 as the FloatList stores them);
- fields[3] is `re.split('[ :]', ...)` reshaped to (field, fid, val) triples (a token count that is not a multiple of 3
  raises);
- feat_ids: for each of the 11 common fields, in the iteration order of the Common_Fileds dict literal under Python
  2.7 (derived below, not run on Python 2), every fid of that field in line order, or its default id;
- u_{cat,shop,brand,int}{ids,vals}: every (fid, val) of 109_14 / 110_14 / 127_14 / 150_14 in line order, or
  ([default], [1.0]); a_{cat,shop,int,brand}ids: every fid of 206 / 207 / 210 / 216, or [default];
- every other field is dropped.

The features are encoded with tfrecord.encode_example (keys sorted) and framed with tfrecord.write_records.  The
implementation's restrictions are part of the contract too and raise OracleError here in the same order: a NUL byte in
the line, the token count, then the first of an empty token / a kept field's fid that is not [0-9]+ below 2^63, then
the first y, z or user multi-hot value that float() rejects.
"""
from __future__ import annotations

import glob
import os
import re
from typing import Dict, Iterator, List, Optional, Tuple

import numpy as np

from tf_repos_b200 import tfrecord

# ---- Python 2.7 dict iteration order of the Common_Fileds literal (:33) -----------------------------------------
COMMON_LITERAL = [("101", 1), ("121", 2), ("122", 3), ("124", 4), ("125", 5), ("126", 6), ("127", 7), ("128", 8),
                  ("129", 9), ("205", 10), ("301", 11)]
_M64 = (1 << 64) - 1


def py2_str_hash(s: bytes) -> int:
    """CPython 2.7 string_hash without hash randomisation (prefix = suffix = 0), as a C long."""
    if not s:
        return 0
    x = (s[0] << 7) & _M64
    for c in s:
        x = ((1000003 * x) & _M64) ^ c
    x ^= len(s)
    x = x - (1 << 64) if x >> 63 else x
    return -2 if x == -1 else x


def _insert_clean(table: List, key: bytes, h: int) -> None:
    """insertdict_clean / lookdict_string's probe: i = hash & mask, then i = 5i + perturb + 1, perturb >>= 5."""
    mask = len(table) - 1
    i = h & _M64
    perturb = h & _M64
    slot = i & mask
    while table[slot] is not None:
        i = (5 * i + perturb + 1) & _M64
        slot = i & mask
        perturb >>= 5
    table[slot] = key


def py2_dict_order(keys: List[bytes]) -> List[bytes]:
    """Iteration order of a Python 2.7 dict display with these distinct str keys: BUILD_MAP presizes the table with
    dictresize(n) (n > 5: the smallest power of two above n, from 8), STORE_MAP inserts in source order, and after an
    insert that leaves fill * 3 >= size * 2 the table is resized to the smallest power of two above 4 * used and the
    old slots are reinserted in slot order.  Iteration walks the slots."""
    def size_above(n):
        size = 8
        while size <= n:
            size <<= 1
        return size

    table: List[Optional[bytes]] = [None] * (size_above(len(keys)) if len(keys) > 5 else 8)
    used = 0
    for k in keys:
        _insert_clean(table, k, py2_str_hash(k))
        used += 1
        if used * 3 >= len(table) * 2:
            old, table = table, [None] * size_above(4 * used)
            for o in old:
                if o is not None:
                    _insert_clean(table, o, py2_str_hash(o))
    return [k for k in table if k is not None]


_DEFAULT = {k.encode(): v for k, v in COMMON_LITERAL}
COMMON: List[Tuple[bytes, int]] = [(k, _DEFAULT[k]) for k in py2_dict_order([k.encode() for k, _ in COMMON_LITERAL])]
UMH = {b"109_14": ("u_cat", 12), b"110_14": ("u_shop", 13), b"127_14": ("u_brand", 14), b"150_14": ("u_int", 15)}
AD = {b"206": ("a_cat", 16), b"207": ("a_shop", 17), b"210": ("a_int", 18), b"216": ("a_brand", 19)}
KEPT = set(_DEFAULT) | set(UMH) | set(AD)


# ---- numbers -------------------------------------------------------------------------------------------------------
def py2_float(tok: bytes) -> float:
    """Python 2's float() of a str: Python 3's float() of the bytes, except that '_' digit separators (new in 3.6)
    are rejected."""
    if b"_" in tok:
        raise ValueError(f"could not convert string to float: {tok!r}")
    return float(tok)


def to_f32(x: float) -> np.float32:
    """The FloatList's double -> float (round to nearest; overflow gives inf)."""
    with np.errstate(over="ignore"):
        return np.float64(x).astype(np.float32)


_ID = re.compile(rb"[0-9]+\Z")


def fid(tok: bytes) -> Optional[int]:
    """astype(np.int) of a kept field's fid, restricted to [0-9]+ below 2^63; None = raises."""
    if not _ID.match(tok):
        return None
    v = int(tok)
    return v if v < (1 << 63) else None


class OracleError(ValueError):
    def __init__(self, line: int, kind: str, token: bytes):
        super().__init__(f"line {line}: {kind}: {token!r}")
        self.line, self.kind, self.token = line, kind, token


# ---- one line ------------------------------------------------------------------------------------------------------
def line_fault(line: bytes) -> Optional[Tuple[str, bytes]]:
    """(kind, token) of the first fault of a 4-field line before any number is converted, or None.  kind: 'nul',
    'count', 'empty' or 'id'."""
    s = line.strip()
    f3 = s.split(b",")[3]
    if b"\0" in s:
        return "nul", s
    toks = re.split(rb"[ :]", f3)
    if len(toks) % 3:
        return "count", f3
    for i, t in enumerate(toks):
        if t == b"":
            return "empty", t
        if i % 3 == 1 and toks[i - 1] in KEPT and fid(t) is None:
            return "id", t
    return None


def parse_line(line: bytes, line_no: int = 0) -> Optional[Dict[str, np.ndarray]]:
    """The features gen_tfrecords builds for one line (None = skipped); raises OracleError."""
    fields = line.strip().split(b",")
    if len(fields) != 4:
        return None
    fault = line_fault(line)
    if fault:
        raise OracleError(line_no, *fault)

    def num(tok):
        try:
            return to_f32(py2_float(tok))
        except ValueError:
            raise OracleError(line_no, "float", tok) from None

    y, z = num(fields[1]), num(fields[2])
    ffv = re.split(rb"[ :]", fields[3])
    triples = [(ffv[i], ffv[i + 1], ffv[i + 2]) for i in range(0, len(ffv), 3)]
    umh_vals = {f: [num(v) for g, _, v in triples if g == f] for f in UMH}
    feat = {"y": np.array([y], np.float32), "z": np.array([z], np.float32)}
    ids: List[int] = []
    for f, default in COMMON:
        got = [fid(i) for g, i, _ in triples if g == f]
        ids.extend(got if got else [default])
    feat["feat_ids"] = np.array(ids, np.int64)
    for f, (name, default) in UMH.items():
        got = [fid(i) for g, i, _ in triples if g == f]
        feat[name + "ids"] = np.array(got if got else [default], np.int64)
        feat[name + "vals"] = np.array(umh_vals[f] if got else [1.0], np.float32)
    for f, (name, default) in AD.items():
        got = [fid(i) for g, i, _ in triples if g == f]
        feat[name + "ids"] = np.array(got if got else [default], np.int64)
    return feat


def lines_of(data: bytes) -> List[bytes]:
    """Python 2 file iteration: each line ends after its '\\n'; a last line without one still counts."""
    parts = data.split(b"\n")
    if parts and parts[-1] == b"":
        parts.pop()
    return parts


def examples(data: bytes) -> Iterator[Dict[str, np.ndarray]]:
    for n, line in enumerate(lines_of(data), 1):
        feat = parse_line(line, n)
        if feat is not None:
            yield feat


def records(data: bytes) -> List[bytes]:
    return [tfrecord.encode_example(f) for f in examples(data)]


def convert_file(in_path: str, out_path: str) -> None:
    with open(in_path, "rb") as fh:
        data = fh.read()
    tfrecord.write_records(out_path, records(data))


def convert(input_dir: str, output_dir: str) -> List[str]:
    """main(): mkdir, glob input_dir/*-*, one <basename>.tfrecord per file."""
    if not os.path.exists(output_dir):
        os.mkdir(output_dir)
    files = sorted(glob.glob(os.path.join(input_dir, "*-*")))
    for f in files:
        convert_file(f, os.path.join(output_dir, os.path.basename(f) + ".tfrecord"))
    return files
