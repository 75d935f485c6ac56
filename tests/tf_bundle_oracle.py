"""An independent restatement of TensorFlow's V2 checkpoint format (tensor bundle + LevelDB table), written from the
format description in DESIGN.md §2.11 and not from tf_repos_b200/tf_checkpoint.py.  Pure Python with its own CRC-32C.

The writer takes the layout knobs the engine's writer never varies (block size, restart interval, shard count) and a
few deliberate defects for the rejection tests; the reader verifies every block and every tensor checksum on the host.
"""
from __future__ import annotations

import os
import struct
from typing import Dict, List, Optional, Tuple

import numpy as np

_P = 0x82F63B78
_T = [0] * 256
for _b in range(256):
    _r = _b
    for _ in range(8):
        _r = (_r >> 1) ^ (_P & -(_r & 1))
    _T[_b] = _r


def crc32c(data, crc: int = 0) -> int:
    c = crc ^ 0xFFFFFFFF
    t = _T
    for b in bytes(data):
        c = t[(c ^ b) & 0xFF] ^ (c >> 8)
    return c ^ 0xFFFFFFFF


def mask(c: int) -> int:
    return ((((c >> 15) | (c << 17)) & 0xFFFFFFFF) + 0xA282EAD8) & 0xFFFFFFFF


def _gf_mul(a: int, b: int) -> int:      # reflected polynomials mod P: bit 31 is x^0
    p = 0
    for _ in range(32):
        if a & 0x80000000:
            p ^= b
        a = (a << 1) & 0xFFFFFFFF
        b = (b >> 1) ^ _P if b & 1 else b >> 1
    return p


def _x_pow_8n(n: int) -> int:
    r, sq = 0x80000000, 0x00800000     # 1, x^8
    while n:
        if n & 1:
            r = _gf_mul(r, sq)
        sq = _gf_mul(sq, sq)
        n >>= 1
    return r


def crc32c_combine(c1: int, c2: int, len2: int) -> int:
    """CRC-32C of A + B from crc(A), crc(B) and len(B)."""
    return _gf_mul(c1, _x_pow_8n(len2)) ^ c2


def crc32c_repeat(c: int, n_bytes: int, times: int) -> int:
    """CRC-32C of a pattern of n_bytes bytes (CRC c) repeated `times` times, by doubling."""
    out, out_len, blk, blk_len = None, 0, c, n_bytes
    while times:
        if times & 1:
            out = blk if out is None else crc32c_combine(out, blk, blk_len)
            out_len += blk_len
        blk, blk_len = crc32c_combine(blk, blk, blk_len), 2 * blk_len
        times >>= 1
    return crc32c(b"") if out is None else out


def _uv(x: int) -> bytes:
    x &= 0xFFFFFFFFFFFFFFFF
    b = bytearray()
    while x > 0x7F:
        b.append(0x80 | (x & 0x7F))
        x >>= 7
    b.append(x)
    return bytes(b)


def _rv(b: bytes, i: int) -> Tuple[int, int]:
    x, s = 0, 0
    while True:
        c = b[i]
        x |= (c & 0x7F) << s
        i, s = i + 1, s + 7
        if c < 0x80:
            return x, i


def _msg(fields: List[Tuple[int, object]]) -> bytes:
    """fields: (number, int -> varint | ('f32', int) -> fixed32 | bytes -> length-delimited)."""
    out = b""
    for n, v in fields:
        if isinstance(v, bytes):
            out += _uv(n << 3 | 2) + _uv(len(v)) + v
        elif isinstance(v, tuple):
            out += _uv(n << 3 | 5) + struct.pack("<I", v[1])
        else:
            out += _uv(n << 3) + _uv(v)
    return out


def _parse(b: bytes) -> Dict[int, list]:
    out: Dict[int, list] = {}
    i = 0
    while i < len(b):
        k, i = _rv(b, i)
        n, w = k >> 3, k & 7
        if w == 0:
            v, i = _rv(b, i)
        elif w == 1:
            v, i = b[i:i + 8], i + 8
        elif w == 2:
            ln, i = _rv(b, i)
            v, i = b[i:i + ln], i + ln
        elif w == 5:
            v, i = struct.unpack("<I", b[i:i + 4])[0], i + 4
        else:
            raise ValueError("wire type %d" % w)
        out.setdefault(n, []).append(v)
    return out


_DT = {np.dtype(np.float32): 1, np.dtype(np.int64): 9, np.dtype(np.float64): 2, np.dtype(np.int32): 3}
_NP = {v: k for k, v in _DT.items()}


def _block(entries: List[Tuple[bytes, bytes]], interval: int) -> bytes:
    body, restarts, prev = b"", [], b""
    for i, (k, v) in enumerate(entries):
        if i % interval == 0:
            restarts.append(len(body))
            s = 0
        else:
            s = 0
            while s < min(len(k), len(prev)) and k[s] == prev[s]:
                s += 1
        body += _uv(s) + _uv(len(k) - s) + _uv(len(v)) + k[s:] + v
        prev = k
    if not restarts:
        restarts = [0]
    return body + b"".join(struct.pack("<I", r) for r in restarts) + struct.pack("<I", len(restarts))


def write_bundle(prefix: str, tensors: Dict[str, np.ndarray], block_size: int = 4096, restart_interval: int = 16,
                 num_shards: int = 1, block_type: int = 0, endianness: int = 0, min_consumer: int = 0,
                 sliced: Tuple[str, ...] = ()):
    """Writes `tensors` as <prefix>.index + <prefix>.data-*; tensors go round-robin to the shards by sorted name.
    block_type, endianness, min_consumer and sliced write the defects the reader must reject."""
    shards = [bytearray() for _ in range(num_shards)]
    kv = []
    for i, name in enumerate(sorted(tensors, key=lambda s: s.encode())):
        a = np.asarray(tensors[name])
        raw = a.tobytes()
        sh = i % num_shards
        dims = b"".join(_msg([(2, _msg([(1, d)]))]) for d in a.shape)
        # explicit zero shard_id / offset, crc before the offset, and an unknown field 15: all legal protobuf
        fields = [(1, _DT[a.dtype]), (2, dims), (3, sh), (6, ("f32", mask(crc32c(raw)))), (4, len(shards[sh])),
                  (5, len(raw)), (15, 7)]
        if name in sliced:
            fields.append((7, _msg([(1, _msg([(1, 0), (2, 1)]))])))
        kv.append((name.encode(), _msg(fields)))
        shards[sh] += raw
    version = [(1, 1)] + ([(2, min_consumer)] if min_consumer else [])
    header = _msg([(1, num_shards), (2, endianness), (3, _msg(version))])
    kv = [(b"", header)] + kv
    out = bytearray()

    def emit(blk):
        h = _uv(len(out)) + _uv(len(blk))
        out.extend(blk + bytes([block_type]) + struct.pack("<I", mask(crc32c(blk + bytes([block_type])))))
        return h

    index, cur, size, pending = [], [], 0, None
    for k, v in kv:
        if pending is not None:           # LevelDB's shortest separator: last <= sep < k
            last, h = pending
            d = 0
            while d < min(len(last), len(k)) and last[d] == k[d]:
                d += 1
            sep = last
            if d < min(len(last), len(k)) and last[d] < 0xFF and last[d] + 1 < k[d]:
                sep = last[:d] + bytes([last[d] + 1])
            index.append((sep, h))
            pending = None
        cur.append((k, v))
        size += len(k) + len(v) + 3
        if size >= block_size:
            pending = (k, emit(_block(cur, restart_interval)))
            cur, size = [], 0
    if pending is not None:
        index.append(pending)
    if cur:
        index.append((cur[-1][0], emit(_block(cur, restart_interval))))
    meta = emit(_block([], 1))
    idx = emit(_block(index, 1))
    out.extend((meta + idx).ljust(40, b"\0") + struct.pack("<Q", 0xDB4775248B80FB57))
    with open(prefix + ".index", "wb") as f:
        f.write(out)
    for s in range(num_shards):
        with open("%s.data-%05d-of-%05d" % (prefix, s, num_shards), "wb") as f:
            f.write(shards[s])


def _read_block(buf: bytes, off: int, size: int) -> List[Tuple[bytes, bytes]]:
    blk, t = buf[off:off + size], buf[off + size]
    assert t == 0, "compressed block"
    assert struct.unpack("<I", buf[off + size + 1:off + size + 5])[0] == mask(crc32c(buf[off:off + size + 1])), "block crc"
    n = struct.unpack("<I", blk[-4:])[0]
    lim, i, prev, out = len(blk) - 4 - 4 * n, 0, b"", []
    while i < lim:
        s, i = _rv(blk, i)
        ns, i = _rv(blk, i)
        vl, i = _rv(blk, i)
        k = prev[:s] + blk[i:i + ns]
        out.append((k, blk[i + ns:i + ns + vl]))
        i, prev = i + ns + vl, k
    return out


def read_bundle(prefix: str, names_only: bool = False) -> Dict[str, Optional[np.ndarray]]:
    """{name: array} of a bundle, every block and tensor checksum verified (AssertionError on a mismatch)."""
    buf = open(prefix + ".index", "rb").read()
    foot = buf[-48:]
    assert struct.unpack("<Q", foot[40:])[0] == 0xDB4775248B80FB57, "magic"
    i = 0
    _, i = _rv(foot, i)
    _, i = _rv(foot, i)
    io, i = _rv(foot, i)
    isz, i = _rv(foot, i)
    kv = []
    for _, h in _read_block(buf, io, isz):
        o, j = _rv(h, 0)
        s, _ = _rv(h, j)
        kv += _read_block(buf, o, s)
    hdr = _parse(kv[0][1])
    assert kv[0][0] == b"" and hdr.get(2, [0])[0] == 0
    nsh = hdr.get(1, [1])[0]
    out: Dict[str, Optional[np.ndarray]] = {}
    files: Dict[int, bytes] = {}
    for k, v in kv[1:]:
        e = _parse(v)
        dt = _NP[e[1][0]]
        shape = tuple(_parse(d).get(1, [0])[0] for d in _parse(e[2][0]).get(2, [])) if 2 in e else ()
        if names_only:
            out[k.decode()] = None
            continue
        sh, off, size = e.get(3, [0])[0], e.get(4, [0])[0], e.get(5, [0])[0]
        if sh not in files:
            files[sh] = open("%s.data-%05d-of-%05d" % (prefix, sh, nsh), "rb").read()
        raw = files[sh][off:off + size]
        assert len(raw) == size, "truncated data"
        assert mask(crc32c(raw)) == e.get(6, [mask(0)])[0], "tensor crc: " + k.decode()
        out[k.decode()] = np.frombuffer(raw, dtype=dt).reshape(shape).copy()
    return out


def write_state(model_dir: str, prefixes: List[str]):
    """The directory's `checkpoint` file naming prefixes (the last is the latest), written as given."""
    with open(os.path.join(model_dir, "checkpoint"), "w") as f:
        f.write('model_checkpoint_path: "%s"\n' % prefixes[-1])
        for p in prefixes:
            f.write('all_model_checkpoint_paths: "%s"\n' % p)
