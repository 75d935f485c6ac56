"""The shared tf.Example walk (csrc/example_wire.cuh, DESIGN.md §2.5) seen through both of its serving consumers:
ctr_wd_serve_input (wide_n_deep) and ctr_din_serve_scan (DIN) must call exactly the same requests malformed (check 1).

Each case takes a valid request for each parser and adds one map entry under a key neither schema knows, carrying one
encoding; cases at the Example and Features level wrap the base instead.  Every case states its verdict, and both
parsers must reach it."""
import numpy as np
import pytest
import torch

from tests import wd_serving_oracle as wo

pytestmark = pytest.mark.gpu
F = 5


def _varint(v: int) -> bytes:
    out = bytearray()
    while True:
        b, v = v & 0x7F, v >> 7
        out.append(b | (0x80 if v else 0))
        if not v:
            return bytes(out)


def _ld(num: int, payload: bytes) -> bytes:
    return _varint(num << 3 | 2) + _varint(len(payload)) + payload


def _entry(key: bytes, feature: bytes) -> bytes:
    return _ld(1, _ld(1, key) + _ld(2, feature))


# Features bodies of a valid request for each parser
WD_BASE = b"".join(_entry(k.encode(), wo.float_feature([1.0]) if k[0] == "I" else wo.int64_feature([1]))
                   for k in wo.KEYS)
DIN_BASE = _entry(b"feat_ids", wo.int64_feature(range(1, F + 1))) + \
    b"".join(_entry(k, wo.int64_feature([1])) for k in (b"a_catids", b"a_shopids", b"a_brandids"))

KEY = _ld(1, b"xkey")                  # the key field of a key neither schema knows
INTS = _ld(3, _ld(1, b"\x05"))         # an Int64List Feature holding 5
VARINT10 = b"\x80" * 9 + b"\x01"       # 2^63, the largest 10-byte varint


def _entry_of(body: bytes):
    """the base plus one map entry whose bytes are body"""
    return lambda feats: _ld(1, feats + _ld(1, body))


CASES = [   # (name, malformed, Features body of the base -> serialized Example)
    ("base", False, lambda f: _ld(1, f)),
    ("keyless entry, its Feature not parsed", False, _entry_of(_ld(2, b"\x0f"))),
    ("entry without value field", False, _entry_of(KEY)),
    ("empty Feature", False, _entry_of(KEY + _ld(2, b""))),
    ("unknown fields in the Example", False, lambda f: _ld(1, f) + b"\x28\x01" + _ld(6, b"x") + b"\x3d\0\0\0\0"),
    ("two Features messages", False, lambda f: _ld(1, f) + _ld(1, _entry(b"xkey", INTS))),
    ("unknown fields in Features", False, lambda f: _ld(1, f + b"\x10\x07" + _ld(3, b"\xff"))),
    ("unknown fields in an entry", False, _entry_of(KEY + b"\x18\x05" + b"\x21" + b"\0" * 8 + _ld(2, INTS))),
    ("unknown fields in a Feature", False, _entry_of(KEY + _ld(2, b"\x20\x01" + _ld(9, b"") + INTS))),
    ("unknown fields in a list", False, _entry_of(KEY + _ld(2, _ld(3, b"\x10\x01" + _ld(1, b"\x05") + _ld(4, b"z"))))),
    ("10-byte varint ending in 1", False, _entry_of(KEY + b"\x18" + VARINT10 + _ld(2, INTS))),
    ("10-byte packed varint ending in 1", False, _entry_of(KEY + _ld(2, _ld(3, _ld(1, VARINT10))))),
    ("two kinds", False, _entry_of(KEY + _ld(2, INTS + _ld(2, _ld(1, b"\0" * 4))))),
    ("a later kind field is not read", False, _entry_of(KEY + _ld(2, INTS + b"\x10\x01" + _ld(2, _ld(1, b"abc"))))),
    ("UTF-8 key", False, _entry_of(_ld(1, "xké€𝄞".encode()) + _ld(2, INTS))),
    ("BytesList", False, _entry_of(KEY + _ld(2, _ld(1, _ld(1, b"ab") + _ld(1, b""))))),
    ("floats packed and not", False, _entry_of(KEY + _ld(2, _ld(2, b"\x0d\0\0\x80\x3f" + _ld(1, b"\0" * 8))))),
    ("unpacked ints", False, _entry_of(KEY + _ld(2, _ld(3, b"\x08\x05\x08" + VARINT10)))),
    ("Example field 1 not length-delimited", True, lambda f: _ld(1, f) + b"\x08\x01"),
    ("Features past the Example", True, lambda f: b"\x0a" + _varint(len(f) + 1) + f),
    ("map entry not length-delimited", True, lambda f: _ld(1, f + b"\x08\x01")),
    ("key not length-delimited", True, _entry_of(b"\x08\x01" + _ld(2, INTS))),
    ("value not length-delimited", True, _entry_of(KEY + b"\x15\0\0\0\0")),
    *[(f"wire type {wt} in an entry", True, _entry_of(KEY + bytes([3 << 3 | wt]) + _ld(2, INTS))) for wt in (3, 4, 6, 7)],
    *[(f"wire type {wt} in a list", True, _entry_of(KEY + _ld(2, _ld(3, bytes([1 << 3 | wt]))))) for wt in (3, 4, 6, 7)],
    ("value past its entry", True, _entry_of(KEY + b"\x12\x05\x1a")),
    ("list past its Feature", True, _entry_of(KEY + _ld(2, b"\x1a\x05\x0a"))),
    ("fixed64 past its entry", True, _entry_of(KEY + b"\x19\0\0\0")),
    ("11-byte varint", True, _entry_of(KEY + b"\x18" + b"\x80" * 10 + b"\x01" + _ld(2, INTS))),
    ("10-byte varint ending above 1", True, _entry_of(KEY + b"\x18" + b"\x80" * 9 + b"\x02" + _ld(2, INTS))),
    ("11-byte field key", True, _entry_of(KEY + b"\x98" + b"\x80" * 9 + b"\x01\x00" + _ld(2, INTS))),
    ("key not UTF-8", True, _entry_of(_ld(1, b"\xc3\x28") + _ld(2, INTS))),
    ("key an encoded surrogate", True, _entry_of(_ld(1, b"x\xed\xa0\x80") + _ld(2, INTS))),
    ("key cut inside a character", True, _entry_of(_ld(1, b"x\xe2\x82") + _ld(2, INTS))),
    ("kind field not length-delimited", True, _entry_of(KEY + _ld(2, b"\x18\x05" + INTS))),
    ("packed floats not a multiple of 4", True, _entry_of(KEY + _ld(2, _ld(2, _ld(1, b"abc"))))),
    ("unterminated packed varint", True, _entry_of(KEY + _ld(2, _ld(3, _ld(1, b"\x05\x80"))))),
    ("11-byte packed varint", True, _entry_of(KEY + _ld(2, _ld(3, _ld(1, b"\x80" * 10 + b"\x01"))))),
    ("10-byte packed varint ending above 1", True, _entry_of(KEY + _ld(2, _ld(3, _ld(1, b"\x80" * 9 + b"\x7f"))))),
]


def _stage(example: bytes):
    off = torch.tensor([0, len(example)], dtype=torch.int64, device="cuda:0")
    data = torch.tensor(np.frombuffer(example, dtype=np.uint8), device="cuda:0")
    return data, off, torch.full((1,), -1, dtype=torch.int64, device="cuda:0")


def _wd_check(example: bytes) -> int:
    """ctr_wd_serve_input's check on one Example (parse and checks only): 0 = accepted"""
    from tf_repos_b200 import ops
    from tf_repos_b200.wide_deep import NUM_BUCKETS
    data, off, err = _stage(example)
    ops.wd_serve_input(data, off, 0, None, None, None, None, None, NUM_BUCKETS, 8, None, None, err)
    word = int(err.item())
    return 0 if word == -1 else (word >> 8) & 0xFF


def _din_check(example: bytes) -> int:
    """ctr_din_serve_scan's check on one Example: 0 = accepted"""
    from tf_repos_b200 import ops
    data, off, err = _stage(example)
    i32 = dict(dtype=torch.int32, device="cuda:0")
    slot_off = torch.empty(1, dtype=torch.int64, device="cuda:0")
    ops.din_serve_scan(data, off, 0, F, 1, 4, slot_off, torch.empty(1, **i32), torch.empty(2, **i32),
                       torch.zeros(2, **i32), err)
    word = int(err.item())
    return 0 if word == -1 else (word >> 8) & 0xFF


@pytest.mark.parametrize("name,malformed,build", CASES, ids=[c[0] for c in CASES])
def test_both_serving_parsers_reach_the_stated_verdict(name, malformed, build):
    want = 1 if malformed else 0
    got = {"wide_n_deep": _wd_check(build(WD_BASE)), "DIN": _din_check(build(DIN_BASE))}
    assert got == {"wide_n_deep": want, "DIN": want}, name
