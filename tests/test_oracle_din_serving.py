"""Pins the CPU restatement of DIN's serving input (tests/din_serving_oracle.py, DESIGN.md §2.10) on hand-built requests:
what it accepts decodes as tfrecord.parse_example + din_main.decode_tfrecord_files(labels=()) decode it, and each
rejection names the right Example and check."""
import struct

import numpy as np
import pytest

from tests import din_serving_oracle as so
from tf_repos_b200 import din_main as dm
from tf_repos_b200 import tfrecord as tfr

F, N = 3, 1000


def _good(i=0, **kw):
    args = dict(feat_ids=[1 + i, 2, 3], a=(4, 5, 6), a_int=[7, 8], u_ids=([9], [], [10, 11], []),
                u_vals=([0.5], [], [1.5, -2.0], []))
    args.update(kw)
    return so.din_example(**args)


def _host_decode(tmp_path, examples):
    path = str(tmp_path / "req.tfrecord")
    tfr.write_records(path, examples)
    return dm.decode_tfrecord_files([path], F, labels=())


def _same(a, b):
    assert a.keys() - {"y"} == b.keys() - {"y"}
    for k in a.keys() - {"y"}:
        assert len(a[k]) == len(b[k]), k
        for x, y in zip(a[k], b[k]):
            x, y = np.asarray(x), np.asarray(y)
            assert x.dtype == y.dtype and x.shape == y.shape, k
            assert x.tobytes() == y.tobytes(), k


def test_accepted_requests_decode_as_the_host_decoder(tmp_path):
    reqs = [_good(i) for i in range(4)] + [_good(9, a_int=[], u_ids=((),) * 4, u_vals=((),) * 4)]
    _same(so.decode(reqs, F, N), _host_decode(tmp_path, reqs))


def test_packed_and_unpacked_lists_decode_alike(tmp_path):
    packed, unpacked = _good(packed=True), _good(packed=False)
    assert packed != unpacked
    _same(so.decode([packed], F), so.decode([unpacked], F))
    _same(so.decode([unpacked], F), _host_decode(tmp_path, [unpacked]))


def test_a_repeated_key_keeps_its_last_entry(tmp_path):
    ex = _good(extra=[("a_intids", so.int64_feature([42, 43, 44])), ("u_catvals", so.float_feature([9.0]))])
    d = so.decode([ex], F)
    assert d["a_int"][0].tolist() == [42, 43, 44] and d["u_catvals"][0].tolist() == [9.0]
    _same(d, _host_decode(tmp_path, [ex]))


@pytest.mark.parametrize("feat", [so.float_feature([1.0]), so.int64_feature([1 << 40]), so.bytes_feature([b"x"]),
                                  so.float_feature([1.0]) + so.int64_feature([2]), b"", None])
@pytest.mark.parametrize("key", ["y", "z"])
def test_labels_of_any_kind_are_ignored(tmp_path, key, feat):
    ex = _good(extra=[(key, feat)])
    _same(so.decode([ex], F), so.decode([_good()], F))
    _same(so.decode([ex], F), _host_decode(tmp_path, [ex]))


def test_a_malformed_label_is_still_malformed():
    ex = _good(extra=[("y", b"\x12\x05\x0d")])          # FloatList payload runs past its Feature
    with pytest.raises(so.Rejected, match=r"^example 0: malformed tf.Example protobuf$"):
        so.decode([ex], F)


def test_nan_payloads_keep_their_bits_and_signalling_nans_come_out_quiet():
    bits = [0x7FC00001, 0xFFC12345, 0x7F800001, 0x00000001, 0x80000000]
    floats = [struct.unpack("<f", struct.pack("<I", b))[0] for b in bits]
    ex = _good(u_ids=([1] * 5, [], [], []), u_vals=(floats, [], [], []))
    got = so.decode([ex], F)["u_catvals"][0].view(np.uint32).tolist()
    assert got == [0x7FC00001, 0xFFC12345, 0x7FC00001, 0x00000001, 0x80000000]


def test_ids_keep_their_low_32_bits_below_2_31():
    d = so.decode([_good(feat_ids=[(1 << 31) - 1, 0, 5])], F)
    assert d["feat_ids"][0].tolist() == [(1 << 31) - 1, 0, 5]


def _with(**over):
    return _good(**over)


_TRUNC = so.example([("feat_ids", b"\x1a\x03\x0a\x01\x81")])     # a packed varint cut short
CASES = [
    ("truncated varint", so.example([]) + b"\x0a\x81", so.MALFORMED, 0),
    ("truncated packed varint", _TRUNC, so.MALFORMED, 0),
    ("11-byte varint", so.example([("a_intids", b"\x1a\x0d\x0a\x0b" + b"\xff" * 10 + b"\x01")]), so.MALFORMED, 0),
    ("non-UTF-8 key", _good(extra=[(b"\xff\xfe", so.float_feature([1.0]))]), so.MALFORMED, 0),
    ("unknown key malformed", _good(extra=[("other", b"\x1a\x02\x0a\x05")]), so.MALFORMED, 0),
    ("feat_ids missing", so.example([("a_catids", so.int64_feature([1]))]), so.REQUIRED, 2),
    ("a_shopids empty", _good(extra=[("a_shopids", so.int64_feature([]))]), so.REQUIRED, 4),
    ("a_brandids no kind", _good(extra=[("a_brandids", None)]), so.REQUIRED, 5),
    ("feat_ids count", _with(feat_ids=[1, 2]), so.COUNT, 0),
    ("u_brand mismatch", _with(u_ids=([], [], [1], []), u_vals=([], [], [], [])), so.MISMATCH, 2),
    ("multi-kind feature", _good(extra=[("a_intids", so.int64_feature([1]) + so.float_feature([1.0]))]), so.KIND, 6),
    ("same kind twice", _good(extra=[("u_catids", so.int64_feature([1]) + so.int64_feature([2]))]), so.KIND, 7),
    ("float ids", _good(extra=[("feat_ids", so.float_feature([1.0, 2.0, 3.0]))]), so.KIND, 2),
    ("int vals", _good(extra=[("u_intvals", so.int64_feature([]))]), so.KIND, 14),
    ("negative id", _with(a_int=[-1]), so.RANGE, 6),
    ("id 2^31", _with(u_ids=([], [], [], [1 << 31]), u_vals=([], [], [], [1.0])), so.RANGE, 10),
    ("id >= feature_size", _with(feat_ids=[1, N, 2]), so.VOCAB, 2),
    ("a_catids first id >= feature_size", _with(a=(N + 5, 1, 1)), so.VOCAB, 3),
]


@pytest.mark.parametrize("what,bad,check,arg", CASES, ids=[c[0] for c in CASES])
@pytest.mark.parametrize("at", [0, 2])
def test_errors_name_the_first_bad_example_and_the_check(what, bad, check, arg, at):
    reqs = [_good(i) for i in range(4)]
    reqs[at] = bad
    reqs.append(so.example([]))                         # a later bad Example never wins
    with pytest.raises(so.Rejected) as e:
        so.decode(reqs, F, N)
    assert (e.value.index, e.value.check, e.value.arg) == (at, check, arg)
    assert str(e.value).startswith(f"example {at}: ")


def test_only_the_first_value_of_a_star_ids_is_read():
    d = so.decode([_good(a=(1, 2, 3), extra=[("a_catids", so.int64_feature([7, 1 << 40, N]))])], F, N)
    assert d["a_cat"] == [7]


def test_messages():
    assert str(so.Rejected(3, so.REQUIRED, 4)) == "example 3: required key 'a_shopids' is missing or empty"
    assert str(so.Rejected(0, so.COUNT, 0, F=11)) == "example 0: feat_ids must hold exactly field_size=11 values"
    assert str(so.Rejected(1, so.MISMATCH, 3)) == "example 1: u_intids and u_intvals differ in length"
    assert str(so.Rejected(2, so.KIND, 12)) == \
        "example 2: key 'u_shopvals' holds several kinds or the wrong kind (float_list)"
    assert str(so.Rejected(5, so.RANGE, 7)) == "example 5: key 'u_catids' holds an id outside [0, 2^31)"
    assert str(so.Rejected(6, so.VOCAB, 2, N=10)) == "example 6: key 'feat_ids' holds an id outside [0, feature_size=10)"
