"""The GPU TFRecord input (csrc/tfrecord_device.cu through tf_repos_b200/tfrecord_device.py) against the host decoder:
every batch bit for bit equal to make_batch(decode_tfrecord_files(...)) on seeded adversarial encodings, and every
error raised with the host's message (plus the three stated deviations of DESIGN.md §2.5)."""
import contextlib
import io
import os
import struct

import numpy as np
import pytest
import torch

from tf_repos_b200 import tfrecord as tfr
from tf_repos_b200.tfrecord import _enc_varint, _ld

pytestmark = pytest.mark.gpu
F = 5
U = ("cat", "shop", "brand", "int")
FLOAT_BITS = [0x7FC00000, 0x7F800001, 0xFFBFFFFF, 0x7FA5A5A5, 0x80000000, 0x00000001, 0x807FFFFF, 0x7F800000,
              0xFF800000, 0x3F800000, 0x00000000]


def _varint(v, rng):
    """v as a varint of its canonical length up to 10 bytes (non-canonical zero continuation bytes)"""
    enc = bytearray(_enc_varint(v))
    pad = int(rng.randint(0, 11 - len(enc))) if rng.rand() < 0.3 else 0
    if pad:
        enc[-1] |= 0x80
        enc += b"\x80" * (pad - 1) + b"\x00"
    return bytes(enc)


def _runs(n, rng):
    cuts = sorted(rng.randint(0, n + 1, rng.randint(0, 3)).tolist()) if n else []
    bounds = [0] + cuts + [n]
    return [(a, b) for a, b in zip(bounds[:-1], bounds[1:])]


def _int_list(vals, rng):
    out = b""
    for a, b in _runs(len(vals), rng):
        if rng.rand() < 0.5:
            out += _ld(1, b"".join(_varint(int(v), rng) for v in vals[a:b])) if b > a or rng.rand() < 0.5 else b""
        else:
            out += b"".join(b"\x08" + _varint(int(v), rng) for v in vals[a:b])
    if rng.rand() < 0.2:
        out += b"\x10\x05"                                   # an unknown field inside the list is skipped
    return _ld(3, out)


def _float_list(bits, rng):
    out = b""
    for a, b in _runs(len(bits), rng):
        raw = [struct.pack("<I", int(x)) for x in bits[a:b]]
        if rng.rand() < 0.5:
            out += _ld(1, b"".join(raw))
        else:
            out += b"".join(b"\x0d" + r for r in raw)
    return _ld(2, out)


def _example(rng, maxlen=7):
    def fbits(n):
        return [FLOAT_BITS[i] if rng.rand() < 0.3 else int(np.float32(rng.rand() * 3).view(np.uint32))
                for i in rng.randint(0, len(FLOAT_BITS), n)]
    ents = [("y", _float_list(fbits(1 + (rng.rand() < 0.2)), rng)), ("z", _float_list(fbits(1), rng)),
            ("feat_ids", _int_list(rng.randint(0, 2 ** 31, F) if rng.rand() < 0.3 else rng.randint(0, 300, F), rng))]
    for k in ("a_catids", "a_shopids", "a_brandids"):
        ents.append((k, _int_list(rng.randint(0, 2 ** 31, 1 + (rng.rand() < 0.2)), rng)))
    if rng.rand() < 0.8:
        ents.append(("a_intids", _int_list(rng.randint(0, 1000, rng.randint(0, 5)), rng)))
    for f in U:
        if rng.rand() < 0.85:
            ln = int(rng.randint(0, maxlen + 1))
            ents.append(("u_%sids" % f, _int_list(rng.randint(0, 2 ** 20, ln), rng)))
            ents.append(("u_%svals" % f, _float_list(fbits(ln), rng)))
    extra = []
    for j in range(rng.randint(0, 3)):                       # unknown keys, BytesList among them
        extra.append(("x%d" % j, _ld(1, _ld(1, b"abc") + _ld(1, b"")) if j == 0 else _int_list([1, 2], rng)))
    for k, _ in list(ents):                                  # an earlier occurrence the last one overrides
        if rng.rand() < 0.1:
            extra.append((k, _int_list([7, 8, 9], rng) if k not in ("y", "z") and "vals" not in k else
                          _float_list([0x40000000], rng)))
    order = rng.permutation(len(ents)).tolist()

    def entry(k, v):
        """one map entry; sometimes value first, sometimes with earlier key / value fields the last ones override"""
        body = _ld(2, v) + _ld(1, k.encode()) if rng.rand() < 0.2 else _ld(1, k.encode()) + _ld(2, v)
        if rng.rand() < 0.15:
            body = _ld(1, b"a_catids") + _ld(2, _float_list([0x7F800001], rng)) + body
        if rng.rand() < 0.15:
            body = _ld(1, k.encode()) + _ld(2, b"\x1a\x03\x08\x01\x02") + b"\x18\x07" + body
        return _ld(1, body)
    entries = [entry(k, v) for k, v in extra] + [entry(*ents[i]) for i in order]
    cut = int(rng.randint(0, len(entries) + 1))              # the map split over two Features fields
    return _ld(1, b"".join(entries[:cut])) + b"\x10\x01" + _ld(1, b"".join(entries[cut:]))


def _write_set(tmp_path, sizes, seed):
    rng = np.random.RandomState(seed)
    paths = []
    for i, n in enumerate(sizes):
        p = os.path.join(tmp_path, "part%d.tfrecord" % i)
        tfr.write_records(p, [_example(rng) for _ in range(n)])
        paths.append(p)
    return paths


def _host(paths, labels):
    from tf_repos_b200 import din_main as dm
    with contextlib.redirect_stdout(io.StringIO()):
        return dm.decode_tfrecord_files(paths, F, labels)


def _same(a, b):
    assert a.dtype == b.dtype and a.shape == b.shape, (a.dtype, b.dtype, a.shape, b.shape)
    if a.dtype == torch.float32:
        a, b = a.view(torch.int32), b.view(torch.int32)
    assert torch.equal(a.cpu(), b.cpu())


@pytest.mark.parametrize("layout", ["din", "esmm"])
def test_batches_equal_host_make_batch(tmp_path, layout):
    from tf_repos_b200 import din_main as dm
    from tf_repos_b200 import esmm_main as em
    from tf_repos_b200.tfrecord_device import TFRecordIndex, plan_groups
    labels = ("y",) if layout == "din" else ("y", "z")
    paths = _write_set(str(tmp_path), [23, 0, 31, 9], seed=7 if layout == "din" else 8)
    d = _host(paths, labels)
    n = len(d["y"])
    index = TFRecordIndex.build(paths, F, labels, "cuda", chunk_bytes=300)
    assert len(index) == n
    P, A = index.max_lengths()
    assert (P, A) == dm.max_lengths(d)
    budget = 2500
    for epochs in (1, 3):
        for B in (1, 3, 64, n, n + 5):
            if layout == "esmm":
                assert index.max_batch_occurrences(epochs, B) == em.max_batch_occurrences(d, epochs, B)
            if B == 3 and epochs == 3:
                assert len(plan_groups(index.size + 16, epochs, B, budget)) >= 10
            want = list(dm.index_stream(n, epochs, B))
            got = list(index.batches(epochs, B, layout, P, budget_bytes=budget))
            assert len(got) == len(want)
            for (batch, lab, cnt), idx in zip(got, want):
                if layout == "din":
                    wb, wl, wn = dm.make_batch(d, idx, B, P, "cpu")
                    _same(lab, wl)
                else:
                    wb, (wy, wz), wn = em.make_batch(d, idx, B, "cpu")
                    _same(lab[0], wy); _same(lab[1], wz)
                assert cnt == wn and batch.keys() == wb.keys()
                for k in wb:
                    _same(batch[k], wb[k])


def _rec(**over):
    """one valid Example (F = 5) with `over` replacing / removing (None) features; values are raw Feature bytes"""
    rng = np.random.RandomState(0)
    feats = {"y": _ld(2, _ld(1, struct.pack("<f", 1.0))), "z": _ld(2, _ld(1, struct.pack("<f", 0.0))),
             "feat_ids": _ld(3, _ld(1, bytes(range(1, 6)))), "a_catids": _ld(3, _ld(1, b"\x03")),
             "a_shopids": _ld(3, _ld(1, b"\x04")), "a_brandids": _ld(3, _ld(1, b"\x05")),
             "u_catids": _int_list([1, 2], rng), "u_catvals": _float_list([0x3F800000] * 2, rng)}
    feats.update(over)
    return _ld(1, b"".join(_ld(1, _ld(1, k.encode()) + _ld(2, v)) for k, v in feats.items() if v is not None))


def _files(tmp_path, *recs_per_file):
    paths = []
    for i, recs in enumerate(recs_per_file):
        p = os.path.join(str(tmp_path), "f%d.tfrecord" % i)
        tfr.write_records(p, recs)
        paths.append(p)
    return paths


def _host_error(paths, labels):
    with pytest.raises(Exception) as e:
        _host(paths, labels)
    return e.value


def _device_error(paths, labels, **kw):
    from tf_repos_b200.tfrecord_device import TFRecordIndex
    with pytest.raises(ValueError) as e:
        with contextlib.redirect_stdout(io.StringIO()):
            TFRecordIndex.build(paths, F, labels, "cuda", **kw)
    return e.value


@pytest.mark.parametrize("case", ["missing", "empty", "missing_z", "count", "mismatch", "malformed", "second_file",
                                  "truncated_record", "truncated_header"])
def test_host_errors_raise_the_host_message(tmp_path, case):
    good = _rec()
    labels = ("y", "z")
    if case == "missing":
        paths = _files(tmp_path, [good, good, _rec(a_shopids=None, feat_ids=None), _rec(y=None)])
    elif case == "empty":
        paths = _files(tmp_path, [good, _rec(a_brandids=_ld(3, b""))])
    elif case == "missing_z":
        paths = _files(tmp_path, [good, _rec(z=_ld(2, _ld(1, b"")))])
    elif case == "count":
        paths = _files(tmp_path, [good, _rec(feat_ids=_ld(3, _ld(1, b"\x01\x02")), u_catvals=None)])
    elif case == "mismatch":
        paths = _files(tmp_path, [good, _rec(u_shopids=_ld(3, b"\x08\x01"), u_catvals=None)])
    elif case == "malformed":
        paths = _files(tmp_path, [good, _ld(1, b"\x0b\x01")])       # wire type 3 inside Features
    elif case == "second_file":
        paths = _files(tmp_path, [good, good], [good, _rec(a_catids=None)], [_rec(feat_ids=None)])
    else:
        paths = _files(tmp_path, [good, good, good])
        raw = open(paths[0], "rb").read()
        cut = len(raw) - 3 if case == "truncated_record" else 2 * (len(good) + 16) + 5
        open(paths[0], "wb").write(raw[:cut])
    want = _host_error(paths, labels)
    got = _device_error(paths, labels, chunk_bytes=64)
    assert type(got) is type(want) and str(got) == str(want)


def test_din_does_not_require_z(tmp_path):
    from tf_repos_b200.tfrecord_device import TFRecordIndex
    paths = _files(tmp_path, [_rec(z=None), _rec(z=_ld(3, _ld(1, b"\x01")))])  # z absent / of the wrong kind: unused
    with contextlib.redirect_stdout(io.StringIO()):
        assert len(TFRecordIndex.build(paths, F, ("y",), "cuda")) == 2


def test_crc_mismatches_raise_read_records_messages(tmp_path):
    good = _rec()
    for byte in (16 + len(good) + 3, 2 * (16 + len(good)) + 12 + 7, 2 * (16 + len(good)) - 2):
        paths = _files(tmp_path, [good, good, good])
        raw = bytearray(open(paths[0], "rb").read())
        raw[byte] ^= 0x40
        open(paths[0], "wb").write(bytes(raw))
        with pytest.raises(ValueError) as e:
            list(tfr.read_records(paths[0], verify_crc=True))
        assert str(_device_error(paths, ("y",))) == str(e.value)


@pytest.mark.parametrize("over, what", [
    ({"y": _ld(3, _ld(1, b"\x01"))}, "feature y must hold exactly one Feature kind, float_list"),
    ({"u_catvals": _ld(3, _ld(1, b"\x01\x02"))}, "feature u_catvals must hold exactly one Feature kind, float_list"),
    ({"a_catids": _ld(3, _ld(1, b"\x03")) + _ld(2, b"")}, "feature a_catids must hold exactly one Feature kind"),
    ({"feat_ids": _ld(3, _ld(1, b"\x01\x02\x03\x04" + _enc_varint(2 ** 31)))}, "feat_ids holds an id outside"),
    ({"a_shopids": _ld(3, _ld(1, _enc_varint(-1)))}, "a_shopids holds an id outside"),
    ({"u_catids": _ld(3, b"\x08\x01\x08" + _enc_varint(-5))}, "u_catids holds an id outside"),
    ({"feat_ids": _ld(3, _ld(1, b"\x01\x02\x03\x04\x05")) + _ld(3, _ld(1, b"\x06"))},      # the kind field twice
     "feature feat_ids must hold exactly one Feature kind, int64_list"),
])
def test_stated_deviations_raise(tmp_path, over, what):
    paths = _files(tmp_path, [_rec(), _rec(**over)])
    with contextlib.redirect_stdout(io.StringIO()):
        _host(paths, ("y", "z"))                                     # the host decoder is silent here
    msg = str(_device_error(paths, ("y", "z")))
    assert msg.startswith(paths[0] + ": record 1 (byte ") and what in msg, msg


def test_a_kind_deviation_the_host_raises_on_raises_the_host_error(tmp_path):
    """a FloatList a_catids holding NaN: the host's int(nan) raises before the device's kind deviation would"""
    paths = _files(tmp_path, [_rec(), _rec(a_catids=_ld(2, _ld(1, struct.pack("<I", 0x7FC00000))))])
    want = _host_error(paths, ("y",))
    got = _device_error(paths, ("y",))
    assert type(got) is type(want) and str(got) == str(want)


def test_truncated_record_claiming_2gb_raises_the_host_message(tmp_path):
    hdr = struct.pack("<Q", 3 << 30)
    paths = _files(tmp_path, [_rec()])
    with open(paths[0], "ab") as fh:
        fh.write(hdr + struct.pack("<I", tfr.masked_crc(hdr)) + b"\x00" * 40)
    want = _host_error(paths, ("y",))
    assert "truncated record at byte" in str(want)
    assert str(_device_error(paths, ("y",), chunk_bytes=64)) == str(want)


def _din_model(P, A, B):
    from tf_repos_b200.din import DIN
    return DIN(F, 3000, 8, B, P, max_a_int=A, deep_layers="16,8", dropout="1,1", attention_layers="16",
               device="cuda:0")


def _esmm_model(cap, B):
    from tf_repos_b200.esmm import ESMM
    return ESMM(F, 3000, 8, B, cap, deep_layers="16,8", dropout="1,1", device="cuda:0")


@pytest.mark.parametrize("layout", ["din", "esmm"])
def test_training_on_streamed_batches_equals_host_batches(tmp_path, layout):
    """train steps queued while later groups load on the side stream (a small budget forces many groups) leave the
    same variables, bit for bit, as training on host make_batch batches"""
    from tf_repos_b200 import din_main as dm
    from tf_repos_b200 import esmm_main as em
    from tf_repos_b200.tfrecord_device import TFRecordIndex, plan_groups
    labels = ("y",) if layout == "din" else ("y", "z")
    rng = np.random.RandomState(11)
    recs = []
    for _ in range(150):
        ex = {"y": np.float32(rng.rand() < 0.4), "z": np.float32(rng.rand() < 0.2),
              "feat_ids": rng.randint(0, 3000, F).astype(np.int64), "a_catids": np.int64(rng.randint(0, 3000)),
              "a_shopids": np.int64(rng.randint(0, 3000)), "a_brandids": np.int64(rng.randint(0, 3000)),
              "a_intids": rng.randint(0, 3000, rng.randint(0, 4)).astype(np.int64)}
        for f in U:
            ln = rng.randint(0, 9)
            ex["u_%sids" % f] = rng.randint(0, 3000, ln).astype(np.int64)
            ex["u_%svals" % f] = rng.rand(ln).astype(np.float32)
        recs.append(tfr.encode_example(ex))
    paths = _files(tmp_path, recs[:90], recs[90:])
    d = _host(paths, labels)
    with contextlib.redirect_stdout(io.StringIO()):
        index = TFRecordIndex.build(paths, F, labels, "cuda")
    epochs, B, budget = 3, 32, 4000
    assert len(plan_groups(index.size + 16, epochs, B, budget)) >= 10
    P, A = dm.max_lengths(d)
    if layout == "din":
        a, b = _din_model(P, A, B), _din_model(P, A, B)
        host = (dm.make_batch(d, idx, B, P, "cuda:0") for idx in dm.index_stream(150, epochs, B))
    else:
        cap = em.max_batch_occurrences(d, epochs, B)
        a, b = _esmm_model(cap, B), _esmm_model(cap, B)
        host = (em.make_batch(d, idx, B, "cuda:0") for idx in dm.index_stream(150, epochs, B))
    for batch, lab, n in host:
        a.train_step(batch, lab, n_valid=n)
    for batch, lab, n in index.batches(epochs, B, layout, P, budget_bytes=budget):
        b.train_step(batch, lab, n_valid=n)
    va, vb = a.variables(), b.variables()
    assert va.keys() == vb.keys() and all(torch.equal(va[k], vb[k]) for k in va)
