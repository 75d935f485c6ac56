"""Serving entry for an exported model (SURVEY.md 8f-4): answers the request the reference's TF-Serving clients send
(`Serving_pipeline/deep_fm_serving_client.cpp:42-60`: signature `serving_default`, inputs `feat_ids` int64 [n,F] and
`feat_vals` float32 [n,F], output `prob` float32 [n]; export definition DeepFM.py:354-366) from the files that
`--task_type=export` writes (`<servable_model_dir>/<timestamp>/{variables.pt, signature.json}`).

    s = Servable.load("./servable/1700000000")
    prob = s.predict(feat_ids, feat_vals)        # torch / numpy, host or device, any n

No training state is created (update_mode='lazy': no `last` bytes, no sweeps); requests larger than the configured
batch are served in slices.  The gather kernel reads int64 ids directly (ctr_fm_embed_fwd id_bits = 64).

wide_n_deep's export (`--task_type=export_model`, `<servable_model_dir>/saved_model.pt`) answers the other client,
`Serving_pipeline/wide_n_deep_serving_client.cpp:45-62`: its `inputs` tensor is a batch of serialized tf.Examples
(export definition wide_n_deep.py:233-242, DESIGN.md §2.8), and the output is the classification signature.

    s = Servable.load("./servable")
    out = s.classify([example_bytes, ...])       # {"scores": float32 [n,2] = [1-p, p], "classes": [n,2] b"0", b"1"}

DIN's export (`DIN.py --task_type=export`, `<servable_model_dir>/<timestamp>/`) is a parsing receiver too (DIN.py:385-397);
its request is serialized tf.Examples with the training schema of DIN.py:60-77 (DESIGN.md §2.10: the feat_ids /
feat_vals spec its signature.json declares cannot feed DIN, quirk Q6).

    s = Servable.load("./servable/1700000000")
    prob = s.predict([example_bytes, ...])       # float32 [n]

ESMM (DeepCvrMTL.py) declares the serving signature PredictOutput({"pcvr", "pctr", "pctcvr"}) (:210-217), but its
`--task_type=export` is a stub that writes nothing, so there is no export directory: a servable is built from the
`model_dir` that `--task_type=train` leaves, with the hyperparameters passed as the reference's export would read them
from its flags (DESIGN.md §2.14).  The request is serialized tf.Examples with the training schema of DeepCvrMTL.py:66-83
(labels not read).

    s = ESMMServable.load("./model_ckpt/20260922", field_size=11, feature_size=4519540, embedding_size=16,
                          deep_layers="256,128")        # checkpoint_format="tf": a bundle from tf_checkpoint.save
    out = s.predict([example_bytes, ...])        # {"pctr", "pcvr", "pctcvr"}: float32 [n] each
"""
from __future__ import annotations

import json
import os
from typing import Dict, Optional

import numpy as np
import torch

from . import ops


def _build(model_name: str, p: Dict, batch_size: int, device):
    common = dict(dropout=p.get("dropout", "0.5,0.5,0.5"), l2_reg=p.get("l2_reg", 1e-4), learning_rate=p.get("learning_rate", 5e-4),
                  optimizer=p.get("optimizer", "Adam"), update_mode="lazy", device=device)
    F, N, K = int(p["field_size"]), int(p["feature_size"]), int(p["embedding_size"])
    if model_name == "DeepFM":
        from .deepfm import DeepFM
        return DeepFM(F, N, K, batch_size, deep_layers=p["deep_layers"], **common)
    if model_name == "DCN":
        from .dcn import DCN
        return DCN(F, N, K, batch_size, deep_layers=p["deep_layers"], cross_layers=int(p["cross_layers"]), **common)
    if model_name == "DeepMVM":
        from .deepmvm import DeepMVM
        return DeepMVM(F, N, K, batch_size, deep_layers=p["deep_layers"], batch_norm=bool(p.get("batch_norm", False)),
                       **common)
    if model_name == "NFM":
        from .nfm import NFM
        return NFM(F, N, K, batch_size, deep_layers=p["deep_layers"], **common)
    if model_name == "PNN":
        from .pnn import PNN
        return PNN(F, N, K, batch_size, model_type=p["model_type"], deep_layers=p["deep_layers"], **common)
    if model_name == "AFM":
        from .afm import AFM
        return AFM(F, N, K, batch_size, attention_layers=p["attention_layers"], **common)
    raise ValueError(f"unknown exported model {model_name!r}")


class _Requests:
    """The staging of a request of n serialized tf.Examples for the device parsers, in a pinned host buffer and a device
    buffer that only grow:  prob f32 [outputs * n] (padded to 8 bytes) | error word | `extra` bytes | offsets int64
    [n+1] | bytes.  `send` writes the error word ~0, zeroes the extra bytes and copies error word..bytes in one
    transfer; `receive` copies prob..extra back in one transfer and waits for it."""

    def __init__(self, device):
        self.device = device
        self._host = self._dev = None

    def send(self, examples, extra: int = 0, outputs: int = 1):
        """examples: n >= 1 serialized Examples -> their device views (prob f32 [outputs * n], err int64 [1], extra
        uint8, offsets int64 [n+1], data uint8).  Raises ValueError for an Example of 2^31 bytes or more."""
        n = len(examples)
        lens = np.fromiter(map(len, examples), dtype=np.int64, count=n)
        if int(lens.max()) >= 1 << 31:
            raise ValueError(f"example {int(np.argmax(lens >= 1 << 31))}: an Example of 2^31 bytes or more")
        self._n, self._e = outputs * n, (4 * outputs * n + 7) & ~7
        self._back = self._e + 8 + extra
        head = self._back + 8 * (n + 1)
        total = head + int(lens.sum())
        if self._host is None or self._host.numel() < total:
            cap = max(total, 1 << 16)
            self._host = torch.empty(cap, dtype=torch.uint8, pin_memory=True)
            self._dev = torch.empty(cap, dtype=torch.uint8, device=self.device)
        e, h, dev = self._e, self._host.numpy(), self._dev
        h[e:e + 8].view(np.int64)[0] = -1
        h[e + 8:self._back] = 0
        off = h[self._back:head].view(np.int64)
        off[0] = 0
        np.cumsum(lens, out=off[1:])
        h[head:total] = np.frombuffer(b"".join(examples), dtype=np.uint8)
        dev[e:total].copy_(self._host[e:total], non_blocking=True)
        return (dev[:4 * self._n].view(torch.float32), dev[e:e + 8].view(torch.int64), dev[e + 8:self._back],
                dev[self._back:head].view(torch.int64), dev[head:total])

    def receive(self):
        """-> (prob f32 [outputs * n], the error word's (example, check, arg) or None, extra uint8), host views valid
        until the next send"""
        self._host[:self._back].copy_(self._dev[:self._back], non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        h, e = self._host.numpy(), self._e
        word = int(h[e:e + 8].view(np.int64)[0])        # (example << 16) | (check << 8) | arg, ~0 = none
        error = None if word == -1 else (word >> 16, (word >> 8) & 0xFF, word & 0xFF)
        return h[:4 * self._n].view(np.float32), error, h[e + 8:self._back]


_WD_KEYS = ["I%d" % i for i in range(1, 14)] + ["C%d" % i for i in range(14, 40)]
_WD_CHECKS = {1: "malformed tf.Example protobuf", 2: "required key {key!r} is missing",
              3: "key {key!r} holds several kinds or the wrong kind (I*: FloatList, C*: Int64List)",
              4: "key {key!r} must hold exactly one float"}


class WideDeepServable:
    """serving_default of an exported wide_n_deep: serialized tf.Examples in, the binary head's classification out.
    Per request: one pinned host->device copy (error word, offsets and bytes), the parse + feature-column kernel and
    the MLP per slice of at most max_batch Examples, one device->host copy (probabilities and error word).  It keeps
    its own loop: the columns map every id into range and its buffers never grow, so it has none of the out-of-range
    counter, per-slice records and growth that _DINSchemaServable's loop is built around."""

    def __init__(self, model):
        self.model = model
        self._requests = _Requests(model.device)

    @classmethod
    def load(cls, export_dir: str, max_batch: int = 4096, device="cuda") -> "WideDeepServable":
        from .wide_deep import WideDeep
        st = torch.load(os.path.join(export_dir, "saved_model.pt"), map_location="cpu")
        v = st["variables"]
        emb = v.get("dnn/input_from_feature_columns/input_layer/C14_embedding/embedding_weights")
        layers, i = [], 0
        while f"dnn/hiddenlayer_{i}/kernel" in v:
            layers.append(int(v[f"dnn/hiddenlayer_{i}/kernel"].shape[1]))
            i += 1
        model = WideDeep(int(emb.shape[1]) if emb is not None else 1, max_batch, layers, st["model_type"], device=device)
        model.load_variables(v)
        return cls(model)

    def classify(self, examples) -> Dict[str, np.ndarray]:
        """examples: the string_vals of the request's `inputs` tensor (a sequence of bytes).  Raises ValueError naming
        the first rejected Example (its index in the whole request) and the key."""
        n = len(examples)
        if n == 0:
            return {"scores": np.zeros((0, 2), dtype=np.float32), "classes": np.zeros((0, 2), dtype="S1")}
        pred, err, _, off, data = self._requests.send(examples)
        B = self.model.B
        for lo in range(0, n, B):
            hi = min(lo + B, n)
            self.model.predict_examples(data, off[lo:hi + 1], err, pred[lo:hi], example_base=lo)
        p, error, _ = self._requests.receive()
        if error is not None:
            ex, check, key = error
            raise ValueError(f"example {ex}: " + _WD_CHECKS[check].format(key=_WD_KEYS[key]))
        p = p.copy()
        return {"scores": np.stack([np.float32(1) - p, p], axis=1),
                "classes": np.tile(np.array([b"0", b"1"], dtype="S1"), (n, 1))}


_DIN_KEYS = ("y", "z", "feat_ids", "a_catids", "a_shopids", "a_brandids", "a_intids", "u_catids", "u_shopids",
             "u_brandids", "u_intids", "u_catvals", "u_shopvals", "u_brandvals", "u_intvals")
_DIN_U = ("cat", "shop", "brand", "int")
_DIN_CHECKS = {1: "malformed tf.Example protobuf", 2: "required key {key!r} is missing or empty",
               3: "feat_ids must hold exactly field_size={F} values",
               4: "u_{u}ids and u_{u}vals differ in length",
               5: "key {key!r} holds several kinds or the wrong kind ({kind})",
               6: "key {key!r} holds an id outside [0, 2^31)"}
# the ids DIN reads, in check order: all of feat_ids, the first value of a_*ids, all of a_intids and u_*ids
_DIN_ID_KEYS = (("feat_ids", None), ("a_catids", 1), ("a_shopids", 1), ("a_brandids", 1), ("a_intids", None)) + \
    tuple(("u_%sids" % u, None) for u in _DIN_U)


class _DINSchemaServable:
    """The request loop of DINServable and ESMMServable, whose requests are serialized tf.Examples with DIN's training
    schema (ESMM's adds the label z, and serving reads neither label), so the checks and their messages are the same
    (DESIGN.md §2.10).  Per request: one pinned host->device copy (error word, extra, offsets, bytes); per slice of at
    most max_batch Examples `parse` and the model's predict; one device->host copy (outputs, error word, extra) after
    the only synchronisation.  extra is the model's out-of-range id counter int32 [2], then one 8-byte record per slice
    from the scan.  A slice whose record (`_need`) exceeds the model's `_capacity()` is run again after `_grow`, a
    second round trip.  Growth is permanent; a failed growth (out of memory) raises and leaves the servable as it was.

    A subclass supplies OUTPUTS, `_capacity`, `_alloc`, `parse`, `_predict`, `_need` (host records uint8 [S, 8] -> each
    slice's sizes [S, len(_capacity())]) and `_result` (host outputs float32 [OUTPUTS * n] -> predict's value)."""

    OUTPUTS = 1                 # float32 outputs per Example

    def __init__(self, model):
        self.model = model
        self._requests = _Requests(model.device)
        self._scratch, self._batch = self._alloc(*self._capacity())

    def _grow(self, need):
        """model and emit buffers for the sizes `need`, or neither: the emit buffers are allocated first, and the
        model's grow changes nothing until all of its own allocations succeeded"""
        bufs = self._alloc(*map(max, need, self._capacity()))
        self.model.grow(*need)
        self._scratch, self._batch = bufs

    def _rejection(self, examples, error) -> str:
        """error: the device's first error word as (example, check, arg), or None when only the model's out-of-range
        counter is set -> the ValueError text.  An id >= feature_size is found by the host parser among the Examples
        before the device's first error, so the text names the first rejected Example of the whole request."""
        from .tfrecord import parse_example
        m = self.model
        for i in range(len(examples) if error is None else error[0]):
            ex = parse_example(examples[i])
            for key, first in _DIN_ID_KEYS:
                v = np.asarray(ex.get(key, []), dtype=np.int64)[:first]
                if len(v) and int(v.max()) >= m.N:
                    return f"example {i}: key {key!r} holds an id outside [0, feature_size={m.N})"
        if error is None:
            return f"an id outside [0, feature_size={m.N})"
        index, check, arg = error
        key = _DIN_KEYS[arg]
        kind = "float_list" if key.endswith("vals") else "int64_list"
        return f"example {index}: " + _DIN_CHECKS[check].format(key=key, F=m.Fp, u=_DIN_U[arg % 4], kind=kind)

    def predict(self, examples):
        """examples: the serialized tf.Examples of the request (a sequence of bytes) -> DIN: prob float32 [n]; ESMM:
        {"pctr", "pcvr", "pctcvr"}, each float32 [n].  Raises ValueError naming the first rejected Example (its index
        in the whole request) and the check."""
        n, m, k = len(examples), self.model, self.OUTPUTS
        if n == 0:
            return self._result(np.zeros(0, dtype=np.float32))
        slices = [(lo, min(lo + m.B, n)) for lo in range(0, n, m.B)]
        S = len(slices)
        out, err, extra, off, data = self._requests.send(examples, 8 + 8 * S, outputs=k)
        oob, rec = extra[:8].view(torch.int32), extra[8:].view(S, 8)
        todo = range(S)
        while True:
            for s in todo:
                lo, hi = slices[s]
                for i, y in enumerate(self._predict(self.parse(data, off[lo:hi + 1], lo, err, rec[s]))):
                    out[i * n + lo:i * n + hi].copy_(y[:hi - lo])
            oob.copy_(m.oob)
            p, error, h_extra = self._requests.receive()
            if error is not None or int(h_extra[:4].view(np.int32)[0]):
                m.oob.zero_()
                raise ValueError(self._rejection(examples, error))
            need, cap = self._need(h_extra[8:].reshape(S, 8), slices).tolist(), self._capacity()
            todo = [s for s in todo if any(a > c for a, c in zip(need[s], cap))]
            if not todo:
                return self._result(p)
            self._grow([max(sizes) for sizes in zip(*(need[s] for s in todo))])


class DINServable(_DINSchemaServable):
    """serving_default of an exported DIN (DIN.py:385-397, DESIGN.md §2.10): serialized tf.Examples with the training
    schema of DIN.py:60-77 (labels not read) in, prob out, through ctr_din_serve_scan, ctr_tfrecord_emit_din and
    DIN.predict per slice.  A slice's record is int32 (longest behaviour list, longest a_int bag); a slice whose lists
    or bags outgrow the model's P / max_a_int is run again after DIN.grow.  Later requests run the forward at the
    larger P."""

    @classmethod
    def load(cls, export_dir: str, max_batch: int = 4096, device="cuda", max_len: int = 64,
             max_a_int: int = 8) -> "DINServable":
        """export_dir as `DIN.py --task_type=export` writes it; max_len / max_a_int: the starting buffer lengths"""
        from .din import DIN
        p = json.load(open(os.path.join(export_dir, "signature.json")))["params"]
        model = DIN(int(p["field_size"]), int(p["feature_size"]), int(p["embedding_size"]), max_batch, max_len,
                    max_a_int=max_a_int, deep_layers=p.get("deep_layers", "256,128,64"),
                    dropout=p.get("dropout", "0.5,0.5,0.5"), attention_layers=p.get("attention_layers", "256"),
                    attention_pooling=bool(p.get("attention_pooling", True)), l2_reg=p.get("l2_reg", 1e-4),
                    learning_rate=p.get("learning_rate", 5e-4), optimizer=p.get("optimizer", "Adam"),
                    update_mode="lazy", device=device, batch_norm=bool(p.get("batch_norm", False)),
                    batch_norm_decay=p.get("batch_norm_decay", 0.9))
        model.load_variables(torch.load(os.path.join(export_dir, "variables.pt"), map_location="cpu"))
        return cls(model)

    def _capacity(self):
        return self.model.P, self.model.max_a_int

    def _alloc(self, P: int, A: int):
        """(scan scratch, batch): the buffers for behaviour lists up to P and a_int bags up to A"""
        m = self.model
        B, F, dev = m.B, m.Fp, m.device
        i32 = dict(dtype=torch.int32, device=dev)
        return ({"slot_off": torch.empty(B, dtype=torch.int64, device=dev), "slot_len": torch.empty(B, **i32),
                 "y": torch.empty(B, dtype=torch.float32, device=dev)},         # absorbs the emit's label
                {"feat_ids": torch.empty(B, F, **i32), "a_ids": torch.empty(3, B, **i32),
                 "a_int_ids": torch.empty(B * A, **i32), "a_int_off": torch.empty(B + 1, **i32),
                 "u_ids": torch.empty(4, B, P, **i32), "u_wgt": torch.empty(4, B, P, dtype=torch.float32, device=dev)})

    def parse(self, data, off, lo: int, err, rec) -> Dict[str, torch.Tensor]:
        """One slice: the serialized Examples data[off[b], off[b+1]) (uint8, off int64 [n+1], n <= max_batch),
        Example lo + b of the request -> DIN.predict's batch, in the servable's buffers.  err int64 [1] (~0 = none)
        and rec uint8 [8] (int32 longest behaviour list, longest a_int bag; zeroed by the caller) are folded into."""
        m, sc, bt = self.model, self._scratch, self._batch
        # the emit writes u_ids / u_wgt at stride P and up to B * max_a_int a_int ids: never past these tensors
        if bt["u_ids"].shape[2] != m.P or bt["a_int_ids"].numel() != m.B * m.max_a_int:
            raise RuntimeError(f"DINServable: batch buffers {tuple(bt['u_ids'].shape)} / {bt['a_int_ids'].numel()} do "
                               f"not match the model's P={m.P}, max_a_int={m.max_a_int}")
        ops.din_serve_scan(data, off, lo, m.Fp, m.B, m.max_a_int, sc["slot_off"], sc["slot_len"], bt["a_int_off"],
                           rec.view(torch.int32), err)
        ops.tfrecord_emit_din(data, sc["slot_off"], sc["slot_len"], m.B, m.Fp, m.P, bt["a_int_off"], bt["feat_ids"],
                              bt["a_ids"], bt["a_int_ids"], bt["u_ids"], bt["u_wgt"], sc["y"])
        return bt

    def _predict(self, batch):
        return (self.model.predict(batch),)

    def _need(self, rec, slices):
        return rec.view(np.int32)

    def _result(self, p):
        return p.copy()


ESMM_OUTPUTS = ("pctr", "pcvr", "pctcvr")       # PredictOutput of DeepCvrMTL.py:210-217


class ESMMServable(_DINSchemaServable):
    """serving_default of a trained ESMM (DeepCvrMTL.py:210-217, DESIGN.md §2.14): serialized tf.Examples with the
    training schema of DeepCvrMTL.py:66-83 (labels not read) in, pctr / pcvr / pctcvr out, through
    ctr_esmm_serve_scan, ctr_tfrecord_emit_esmm and ESMM.predict per slice.  A slice's record is its int64 bag
    occurrence total; a slice past the occurrence capacity is run again after ESMM.grow."""

    OUTPUTS = len(ESMM_OUTPUTS)

    @classmethod
    def load(cls, model_dir: str, field_size: int, feature_size: int, embedding_size: int,
             deep_layers: str = "256,128,64", batch_norm: bool = False, batch_norm_decay: float = 0.9,
             max_batch: int = 4096, device="cuda", occ_capacity: Optional[int] = None,
             checkpoint_format: str = "b200") -> "ESMMServable":
        """model_dir as `DeepCvrMTL.py --task_type=train` leaves it (ctr_b200.ckpt), or with checkpoint_format="tf" a
        TensorFlow bundle written by tf_checkpoint.save.  The hyperparameters are DeepCvrMTL.py's flags of the same
        names.  occ_capacity: the starting bag-occurrence capacity per slice; default the one esmm_shapes.json in
        model_dir records."""
        from .esmm import ESMM
        from .estimator import _ckpt_path
        if checkpoint_format not in ("b200", "tf"):
            raise ValueError(f"checkpoint_format={checkpoint_format!r}: must be one of {{b200, tf}}")
        if occ_capacity is None:
            meta = os.path.join(model_dir, "esmm_shapes.json")
            if not os.path.exists(meta):
                raise ValueError(f"{meta} does not exist: pass occ_capacity")
            occ_capacity = int(json.load(open(meta))["occ_capacity"])
        model = ESMM(field_size, feature_size, embedding_size, max_batch, occ_capacity, deep_layers=deep_layers,
                     update_mode="lazy", device=device, batch_norm=batch_norm, batch_norm_decay=batch_norm_decay)
        if checkpoint_format == "tf":
            from . import tf_checkpoint
            tf_checkpoint.restore(model, model_dir, variables_only=True)
        else:
            path = _ckpt_path(model_dir)
            if not os.path.exists(path):
                raise FileNotFoundError(f"{path} does not exist")
            model.load_variables(torch.load(path, map_location="cpu")["variables"])
        return cls(model)

    def _capacity(self):
        return (self.model.cap,)

    def _alloc(self, cap: int):
        """(scan scratch, batch): the buffers for slices of up to cap bag occurrences; ESMM.grow allocates nothing"""
        m = self.model
        B, F, dev = m.B, m.Fp, m.device
        i32 = dict(dtype=torch.int32, device=dev)
        return ({"slot_off": torch.empty(B, dtype=torch.int64, device=dev), "slot_len": torch.empty(B, **i32),
                 "labels": torch.empty(2, B, dtype=torch.float32, device=dev)},    # absorbs the emit's y and z
                {"feat_ids": torch.empty(B, F, **i32), "a_ids": torch.empty(3, B, **i32),
                 "bag_ids": torch.empty(cap, **i32), "bag_wgt": torch.empty(cap, dtype=torch.float32, device=dev),
                 "bag_off": torch.empty(5 * B + 1, **i32)})

    def parse(self, data, off, lo: int, err, rec) -> Dict[str, torch.Tensor]:
        """One slice: the serialized Examples data[off[b], off[b+1]) (uint8, off int64 [n+1], n <= max_batch),
        Example lo + b of the request -> ESMM.predict's batch, in the servable's buffers.  err int64 [1] (~0 = none)
        is folded into; rec uint8 [8] receives the slice's int64 occurrence total (its bags are empty past the
        capacity)."""
        m, sc, bt = self.model, self._scratch, self._batch
        # the emit writes up to m.cap occurrences (the scan empties a slice's bags past it): never past these tensors
        if bt["bag_ids"].numel() != m.cap or bt["bag_wgt"].numel() != m.cap:
            raise RuntimeError(f"ESMMServable: occurrence buffers of {bt['bag_ids'].numel()} do not match the model's "
                               f"occ_capacity={m.cap}")
        ops.esmm_serve_scan(data, off, lo, m.Fp, m.B, m.cap, sc["slot_off"], sc["slot_len"], bt["bag_off"],
                            rec.view(torch.int64), err)
        ops.tfrecord_emit_esmm(data, sc["slot_off"], sc["slot_len"], m.B, m.Fp, bt["bag_off"], bt["feat_ids"],
                               bt["a_ids"], bt["bag_ids"], bt["bag_wgt"], sc["labels"][0], sc["labels"][1])
        return bt

    def _predict(self, batch):
        return self.model.predict(batch)

    def _need(self, rec, slices):
        tot = rec.view(np.int64)
        s = int(np.argmax(tot))
        if tot[s, 0] > max(self.model.cap, (1 << 31) - 1):        # outgrown, and past the int32 CSR offsets
            raise ValueError(f"examples {slices[s][0]}..{slices[s][1] - 1}: {int(tot[s, 0])} bag occurrences in one "
                             f"slice of max_batch={self.model.B} Examples, more than 2^31 - 1")
        return tot

    def _result(self, p):
        p = p.reshape(len(ESMM_OUTPUTS), -1)
        return {k: p[i].copy() for i, k in enumerate(ESMM_OUTPUTS)}


class Servable:
    def __init__(self, model, signature: Dict):
        self.model, self.signature = model, signature
        self.F = int(signature["inputs"]["feat_ids"]["shape"][1])

    @classmethod
    def load(cls, export_dir: str, max_batch: int = 4096, device="cuda"):
        """the directory `--task_type=export` writes (DeepFM family) -> Servable, (DIN) -> DINServable; the one
        wide_n_deep's `--task_type=export_model` writes (saved_model.pt) -> WideDeepServable"""
        if os.path.exists(os.path.join(export_dir, "saved_model.pt")):
            return WideDeepServable.load(export_dir, max_batch, device)
        sig = json.load(open(os.path.join(export_dir, "signature.json")))
        if sig["model"] == "DIN":
            return DINServable.load(export_dir, max_batch, device)
        model = _build(sig["model"], sig["params"], max_batch, torch.device(device))
        model.load_variables(torch.load(os.path.join(export_dir, "variables.pt"), map_location="cpu"))
        return cls(model, sig)

    def predict(self, feat_ids, feat_vals) -> torch.Tensor:
        """feat_ids int64|int32 [n,F] (or [n,F,1]), feat_vals float32 [n,F]; returns prob float32 [n] on the host."""
        dev = self.model.device
        ids = torch.as_tensor(np.asarray(feat_ids) if not torch.is_tensor(feat_ids) else feat_ids)
        vals = torch.as_tensor(np.asarray(feat_vals) if not torch.is_tensor(feat_vals) else feat_vals)
        ids = ids.reshape(-1, self.F)
        vals = vals.reshape(-1, self.F).to(torch.float32)
        if ids.dtype not in (torch.int32, torch.int64):
            ids = ids.to(torch.int64)
        ids, vals = ids.to(dev).contiguous(), vals.to(dev).contiguous()
        out = torch.empty(ids.shape[0], dtype=torch.float32)
        B = self.model.B
        for lo in range(0, ids.shape[0], B):
            hi = min(lo + B, ids.shape[0])
            out[lo:hi] = self.model.predict(ids[lo:hi], vals[lo:hi]).cpu()
        self.model.check_ids()
        return out
