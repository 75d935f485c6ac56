"""CPU restatement of wide_n_deep's serving input (wide_n_deep.py:233-242: build_parsing_serving_input_receiver_fn over
make_parse_example_spec(columns)) on top of oracle/wide_deep.py.  Test infrastructure, like oracle/: the GPU tests
compare csrc/wd_serving.cu and serving.WideDeepServable against it, and test_oracle_wide_deep_serving.py pins it with
known answers.  Each rule is [TF-sem] with the lower confidence of SURVEY.md A.8 (DESIGN.md §2.8):

  parse spec   I1..I13 FixedLenFeature([1], float32), no default: present, a FloatList, exactly one value
               C14..C39 VarLenFeature(int64): missing, empty or any number of values
               any other key is ignored (its Feature must still be well formed: the host parser reads them all)
  map entries  the last entry of a key wins; an entry without a key is skipped; a Feature with no kind set is an
               empty list; a Feature's kind is its first field numbered 1..3, a later one is "several kinds"
  identity     an int64 outside [0, 10000) (all 64 bits) becomes bucket 0
  combiners    embedding_column 'mean' = rows summed in value order / bag length; linear_model 'sum'; an empty bag
               gives a zero row and adds 0 (safe_embedding_lookup_sparse); duplicate ids count each time
  errors       "example <i>: ..." for the first rejected Example; inside one Example a malformed protobuf first, then
               keys I1..I13, C14..C39 in that order, each: missing (I), several kinds / wrong kind, count != 1 (I)
  outputs      scores [n,2] = [1-p, p], classes [n,2] = b"0", b"1"
"""
from __future__ import annotations

import re
import struct
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from oracle import tf_semantics as tfs
from oracle import wide_deep as owd

KEYS = owd.NUM_NAMES + owd.CAT_NAMES            # key index 0..12 = I1..I13, 13..38 = C14..C39
MALFORMED, MISSING, KIND, COUNT = 1, 2, 3, 4
MESSAGES = {MALFORMED: "malformed tf.Example protobuf", MISSING: "required key {key!r} is missing",
            KIND: "key {key!r} holds several kinds or the wrong kind (I*: FloatList, C*: Int64List)",
            COUNT: "key {key!r} must hold exactly one float"}
NONE, BYTES, FLOAT, INT = 0, 1, 2, 3
_KEY = re.compile(r"^([IC])([1-9][0-9]?)$")


class Rejected(ValueError):
    def __init__(self, index: int, check: int, key: int = 0):
        super().__init__(f"example {index}: " + MESSAGES[check].format(key=KEYS[key]))
        self.index, self.check, self.key = index, check, key


class _Malformed(Exception):
    pass


# ---- protobuf wire format, strict ---------------------------------------------------------------------------------
def _varint(b: bytes, p: int, e: int) -> Tuple[int, int]:
    v = 0
    for i in range(10):
        if p >= e:
            raise _Malformed
        c = b[p]; p += 1
        if i == 9 and c > 1:
            raise _Malformed
        v |= (c & 0x7F) << (7 * i)
        if not c & 0x80:
            return v, p
    raise _Malformed


def _fields(b: bytes, s: int, e: int):
    """(num, wire type, value or (start, end)) of the message b[s:e]"""
    p = s
    while p < e:
        key, p = _varint(b, p, e)
        num, wt = key >> 3, key & 7
        if wt == 0:
            v, p = _varint(b, p, e)
            yield num, wt, v
        elif wt in (1, 5):
            n = 8 if wt == 1 else 4
            if e - p < n:
                raise _Malformed
            yield num, wt, (p, p + n)
            p += n
        elif wt == 2:
            ln, p = _varint(b, p, e)
            if ln > e - p:
                raise _Malformed
            yield num, wt, (p, p + ln)
            p += ln
        else:
            raise _Malformed


def _feature(b: bytes, s: int, e: int):
    """-> (kind, values, several kinds)"""
    kind, vals, multi = NONE, [], False
    for num, wt, v in _fields(b, s, e):
        if not 1 <= num <= 3:
            continue
        if kind != NONE:
            multi = True
            continue
        if wt != 2:
            raise _Malformed
        kind = num
        for n2, w2, x in _fields(b, *v):
            if n2 != 1:
                continue
            if kind == BYTES:
                vals.append(bytes(b[x[0]:x[1]]) if w2 in (1, 2, 5) else x)
            elif kind == FLOAT:
                if w2 == 2:
                    if (x[1] - x[0]) % 4:
                        raise _Malformed
                    vals.extend(struct.unpack("<%df" % ((x[1] - x[0]) // 4), b[x[0]:x[1]]))
                elif w2 == 5:
                    vals.append(struct.unpack("<f", b[x[0]:x[1]])[0])
            else:
                if w2 == 2:
                    q = x[0]
                    while q < x[1]:
                        t, q = _varint(b, q, x[1])
                        vals.append(t)
                elif w2 == 0:
                    vals.append(x)
    return kind, vals, multi


def key_index(key: str) -> int:
    """0..38 for I1..I13 / C14..C39, -1 for any other key"""
    m = _KEY.match(key)
    if not m:
        return -1
    num = int(m.group(2))
    if m.group(1) == "I":
        return num - 1 if num <= 13 else -1
    return num - 1 if 13 < num <= 39 else -1


def parse(data: bytes, index: int = 0) -> Tuple[List[float], List[List[int]]]:
    """one serialized Example -> (I1..I13 as float32 values, the C14..C39 bags as raw uint64 values); Rejected"""
    slots: Dict[int, Tuple[int, list, bool]] = {}
    try:
        for num, wt, v in _fields(data, 0, len(data)):
            if num != 1:
                continue
            if wt != 2:
                raise _Malformed
            for n2, w2, entry in _fields(data, *v):
                if n2 != 1:
                    continue
                if w2 != 2:
                    raise _Malformed
                key, feat = None, (0, 0)
                for n3, w3, x in _fields(data, *entry):
                    if n3 in (1, 2) and w3 != 2:
                        raise _Malformed
                    if n3 == 1:
                        key = x
                    elif n3 == 2:
                        feat = x
                if key is None:
                    continue
                try:
                    name = bytes(data[key[0]:key[1]]).decode("utf-8")
                except UnicodeDecodeError:
                    raise _Malformed from None
                f = _feature(data, *feat)
                k = key_index(name)
                if k >= 0:
                    slots[k] = f
    except _Malformed:
        raise Rejected(index, MALFORMED) from None
    for k in range(len(KEYS)):
        num = k < owd.N_NUM
        if k not in slots:
            if num:
                raise Rejected(index, MISSING, k)
            continue
        kind, vals, multi = slots[k]
        if multi or (kind != NONE and kind != (FLOAT if num else INT)):
            raise Rejected(index, KIND, k)
        if num and len(vals) != 1:
            raise Rejected(index, COUNT, k)
    dense = [slots[k][1][0] for k in range(owd.N_NUM)]
    bags = [list(slots[k][1]) if k in slots else [] for k in range(owd.N_NUM, len(KEYS))]
    return dense, bags


def bucket(v: int) -> int:
    """categorical_column_with_identity(10000, default_value=0) on the int64 value (raw uint64 bits here)"""
    return v if v < owd.NUM_BUCKETS else 0


def columns(model: owd.WideDeep, examples: Sequence[bytes]):
    """-> (rows {C: [n,K]} mean embeddings, lin_rows {C: [n,1]} summed linear weights, dense [n,13]) in model.dtype"""
    parsed = [parse(e, i) for i, e in enumerate(examples)]
    n, dt = len(parsed), model.dtype
    dense = torch.tensor([p[0] for p in parsed], dtype=dt).reshape(n, owd.N_NUM)
    rows, lin_rows = {}, {}
    for f, c in enumerate(owd.CAT_NAMES):
        ids = [[bucket(v) for v in p[1][f]] for p in parsed]
        if model.has_dnn:
            t = model.params[model.emb_name(c)]
            rows[c] = torch.stack([t[i].sum(0) / len(i) if i else torch.zeros(model.K, dtype=dt) for i in ids]) \
                if n else torch.zeros(0, model.K, dtype=dt)
        if model.has_linear:
            w = model.params[f"linear/linear_model/{c}/weights"].reshape(-1)
            lin_rows[c] = torch.tensor([[float(w[i].sum()) if i else 0.0] for i in ids], dtype=dt).reshape(n, 1)
    return rows, lin_rows, dense


def classify(model: owd.WideDeep, examples: Sequence[bytes]) -> Dict[str, np.ndarray]:
    """serving_default: {"scores": [n,2] = [1-p, p], "classes": [n,2]}, p = sigmoid(logits) in model.dtype"""
    rows, lin_rows, dense = columns(model, examples)
    with torch.no_grad():
        p = tfs.sigmoid(model._forward(model.params, rows, lin_rows, dense)).numpy()
    return {"scores": np.stack([1 - p, p], axis=1),
            "classes": np.tile(np.array([b"0", b"1"], dtype="S1"), (len(examples), 1))}


# ---- building requests ------------------------------------------------------------------------------------------
def _enc_varint(v: int) -> bytes:
    v &= (1 << 64) - 1
    out = bytearray()
    while True:
        b, v = v & 0x7F, v >> 7
        out.append(b | (0x80 if v else 0))
        if not v:
            return bytes(out)


def _ld(num: int, payload: bytes) -> bytes:
    return _enc_varint(num << 3 | 2) + _enc_varint(len(payload)) + payload


def float_feature(values, packed: bool = True) -> bytes:
    vals = [struct.pack("<f", float(np.float32(v))) for v in values]
    body = (_ld(1, b"".join(vals)) if vals else b"") if packed else b"".join(b"\x0d" + x for x in vals)
    return _ld(2, body)


def int64_feature(values, packed: bool = True) -> bytes:
    vals = [_enc_varint(int(v)) for v in values]
    body = (_ld(1, b"".join(vals)) if vals else b"") if packed else b"".join(b"\x08" + x for x in vals)
    return _ld(3, body)


def bytes_feature(values) -> bytes:
    return _ld(1, b"".join(_ld(1, v) for v in values))


def example(entries: Sequence[Tuple[Optional[str], Optional[bytes]]]) -> bytes:
    """Example{Features{map entries in the given order}}; key None = an entry without key, feature None = without
    value (an empty Feature)"""
    out = b""
    for key, feat in entries:
        e = (b"" if key is None else _ld(1, key.encode() if isinstance(key, str) else key)) + \
            (b"" if feat is None else _ld(2, feat))
        out += _ld(1, e)
    return _ld(1, out)


def request_row(dense: Sequence[float], bags: Sequence[Sequence[int]], packed: bool = True) -> bytes:
    """I1..I13 = dense, C14..C39 = bags (an empty bag is sent as an empty Int64List)"""
    return example([(owd.NUM_NAMES[j], float_feature([dense[j]], packed)) for j in range(owd.N_NUM)] +
                   [(c, int64_feature(bags[f], packed)) for f, c in enumerate(owd.CAT_NAMES)])


def client_request() -> bytes:
    """wide_n_deep_serving_client.cpp:45-50 verbatim: I1..I13 = 0.5, C1..C26 = 123, in the client's insertion order.
    The model reads C14..C39, so C14..C26 hold 123, C27..C39 are empty and C1..C13 are ignored (quirk Q13)."""
    return example([("I%d" % (i + 1), float_feature([0.5])) for i in range(13)] +
                   [("C%d" % (i + 1), int64_feature([123])) for i in range(26)])
