"""CPU restatement of DIN's serving input (DIN.py:385-397 served with the training schema of DIN.py:60-77 without
labels; DESIGN.md §2.10): the host parser tfrecord.parse_example plus din_main.decode_tfrecord_files' checks with
labels=(), the stated deviations of §2.5, and an id check against feature_size.  Test infrastructure: the GPU tests
compare csrc/tfrecord_device.cu's ctr_din_serve_scan and serving.DINServable against it, and
test_oracle_din_serving.py pins it on hand-built requests.

  map entries  as §2.5 (the protobuf walk of wd_serving_oracle): the last entry of a key wins; an entry without a key is
               skipped; every keyed entry's Feature must be well formed, unknown keys and y / z included; a key that is
               not UTF-8 is malformed; packed and unpacked lists are both read
  y, z         parsed, then dropped: neither required nor kind-checked
  checks       per Example in this order: malformed protobuf; feat_ids, a_catids, a_shopids, a_brandids missing or
               empty; feat_ids count != field_size; u_*ids / u_*vals lengths differ; a model key holding several kinds
               or the wrong kind; a read id outside [0, 2^31); a read id >= feature_size.  Read ids: all of feat_ids,
               a_intids and u_*ids, the first value of a_*ids
  errors       "example <i>: ..." for the first rejected Example of the request
  values       an id keeps its low 32 bits, a float its float32 bits with a signalling NaN quieted
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np

from tests import wd_serving_oracle as wo
from tests.wd_serving_oracle import BYTES, FLOAT, INT, NONE, example, float_feature, int64_feature, bytes_feature  # noqa: F401

U = ("cat", "shop", "brand", "int")
KEYS = ("y", "z", "feat_ids", "a_catids", "a_shopids", "a_brandids", "a_intids") + \
    tuple("u_%sids" % u for u in U) + tuple("u_%svals" % u for u in U)
MALFORMED, REQUIRED, COUNT, MISMATCH, KIND, RANGE, VOCAB = 1, 2, 3, 4, 5, 6, 7
# value count each key's read ids are cut to (None = all); keys without an entry hold no ids
READ = {"feat_ids": None, "a_catids": 1, "a_shopids": 1, "a_brandids": 1, "a_intids": None,
        **{"u_%sids" % u: None for u in U}}


class Rejected(ValueError):
    def __init__(self, index: int, check: int, arg: int = 0, F: int = 0, N: int = 0):
        key = KEYS[arg]
        msg = {MALFORMED: "malformed tf.Example protobuf",
               REQUIRED: f"required key {key!r} is missing or empty",
               COUNT: f"feat_ids must hold exactly field_size={F} values",
               MISMATCH: f"u_{U[arg % 4]}ids and u_{U[arg % 4]}vals differ in length",
               KIND: f"key {key!r} holds several kinds or the wrong kind "
                     f"({'float_list' if key.endswith('vals') else 'int64_list'})",
               RANGE: f"key {key!r} holds an id outside [0, 2^31)",
               VOCAB: f"key {key!r} holds an id outside [0, feature_size={N})"}[check]
        super().__init__(f"example {index}: {msg}")
        self.index, self.check, self.arg = index, check, arg


def parse(data: bytes, index: int, F: int, N: Optional[int] = None) -> Dict[str, list]:
    """one serialized Example -> {model key: values} (ids as raw uint64, floats as Python floats); Rejected"""
    slots = {}
    try:
        for num, wt, v in wo._fields(data, 0, len(data)):
            if num != 1:
                continue
            if wt != 2:
                raise wo._Malformed
            for n2, w2, entry in wo._fields(data, *v):
                if n2 != 1:
                    continue
                if w2 != 2:
                    raise wo._Malformed
                key, feat = None, (0, 0)
                for n3, w3, x in wo._fields(data, *entry):
                    if n3 in (1, 2) and w3 != 2:
                        raise wo._Malformed
                    if n3 == 1:
                        key = x
                    elif n3 == 2:
                        feat = x
                if key is None:
                    continue
                try:
                    name = bytes(data[key[0]:key[1]]).decode("utf-8")
                except UnicodeDecodeError:
                    raise wo._Malformed from None
                f = wo._feature(data, *feat)
                if name in KEYS[2:]:
                    slots[name] = f
    except wo._Malformed:
        raise Rejected(index, MALFORMED) from None
    count = {k: len(slots[k][1]) if k in slots else 0 for k in KEYS}
    for k in ("feat_ids", "a_catids", "a_shopids", "a_brandids"):
        if count[k] == 0:
            raise Rejected(index, REQUIRED, KEYS.index(k))
    if count["feat_ids"] != F:
        raise Rejected(index, COUNT, 0, F=F)
    for f, u in enumerate(U):
        if count["u_%sids" % u] != count["u_%svals" % u]:
            raise Rejected(index, MISMATCH, f)
    for k in KEYS[2:]:
        if k in slots:
            kind, _, multi = slots[k]
            if multi or (kind != NONE and kind != (FLOAT if k.endswith("vals") else INT)):
                raise Rejected(index, KIND, KEYS.index(k))
    read = {k: slots[k][1][:n] if k in slots else [] for k, n in READ.items()}
    for k in KEYS:
        if any(v >> 31 for v in read.get(k, [])):
            raise Rejected(index, RANGE, KEYS.index(k))
    if N is not None:
        for k in READ:
            if any(v >= N for v in read[k]):
                raise Rejected(index, VOCAB, KEYS.index(k), N=N)
    return {k: slots[k][1] if k in slots else [] for k in KEYS[2:]}


def decode(examples: Sequence[bytes], F: int, N: Optional[int] = None) -> Dict[str, List]:
    """the request as decode_tfrecord_files' dict (labels=(); "y" = 0.0 so that din_main.make_batch takes it)"""
    d: Dict[str, List] = {k: [] for k in ("y", "feat_ids", "a_cat", "a_shop", "a_brand", "a_int")}
    for u in U:
        d["u_%sids" % u], d["u_%svals" % u] = [], []
    ids = (lambda v: np.asarray([x & 0xFFFFFFFF for x in v], dtype=np.int64))
    for i, data in enumerate(examples):
        ex = parse(data, i, F, N)
        d["y"].append(0.0)
        d["feat_ids"].append(ids(ex["feat_ids"]))
        d["a_cat"].append(int(ex["a_catids"][0])); d["a_shop"].append(int(ex["a_shopids"][0]))
        d["a_brand"].append(int(ex["a_brandids"][0]))
        d["a_int"].append(ids(ex["a_intids"]))
        for u in U:
            d["u_%sids" % u].append(ids(ex["u_%sids" % u]))
            d["u_%svals" % u].append(np.asarray(ex["u_%svals" % u], dtype=np.float64).astype(np.float32))
    return d


def din_example(feat_ids, a, a_int=(), u_ids=((),) * 4, u_vals=((),) * 4, packed: bool = True, extra=()) -> bytes:
    """an Example with DIN's schema: a = (a_cat, a_shop, a_brand); extra = more (key, Feature bytes) entries, last"""
    entries = [("feat_ids", int64_feature(feat_ids, packed))]
    entries += [(k, int64_feature([v], packed)) for k, v in zip(("a_catids", "a_shopids", "a_brandids"), a)]
    entries.append(("a_intids", int64_feature(a_int, packed)))
    for f, u in enumerate(U):
        entries.append(("u_%sids" % u, int64_feature(u_ids[f], packed)))
        entries.append(("u_%svals" % u, float_feature(u_vals[f], packed)))
    return example(entries + list(extra))
