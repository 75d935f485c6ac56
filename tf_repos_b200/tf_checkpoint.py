"""TensorFlow V2 checkpoints (`tf.train.Saver` / `tf.estimator` model_dir) read and written without TensorFlow.

A checkpoint is a tensor bundle `<prefix>.index` + `<prefix>.data-%05d-of-%05d` plus the `checkpoint` state file of
the directory [TF-sem, tensorflow/core/util/tensor_bundle, core/lib/io/table, core/protobuf/tensor_bundle.proto]:

    .index   a LevelDB-format table: data blocks, an (empty) metaindex block, an index block, a 48-byte footer
             footer   = varint64 offset/size of the metaindex and of the index block, zero-padded to 40 bytes,
                        fixed64 magic 0xdb4775248b80fb57 (little-endian)
             block    = entries {varint32 shared, varint32 non_shared, varint32 value_len, key suffix, value}, keys
                        prefix-compressed between restart points, fixed32 restart offsets, fixed32 restart count;
                        stored with a 5-byte trailer {type byte (0 = uncompressed), fixed32 masked CRC-32C of the
                        contents + type byte}; a block handle's size excludes the trailer
             index    = per data block: a key >= its last key (here: the last key), value = the block's handle
             keys     sorted bytewise; "" -> BundleHeaderProto {num_shards = 1, endianness = 2 (LITTLE = 0),
                        version = 3 (VersionDef: producer = 1, min_consumer = 2, bad_consumers = 3)}; a tensor name ->
                        BundleEntryProto {dtype = 1 (DT_FLOAT = 1, DT_INT64 = 9), shape = 2 (TensorShapeProto: dim = 2
                        of {size = 1}), shard_id = 3, offset = 4, size = 5, crc32c = 6 (fixed32, masked CRC-32C of
                        the tensor's bytes), slices = 7}
    .data    the tensors' raw row-major little-endian bytes at `offset` in shard `shard_id`, no alignment
    checkpoint  text proto: `model_checkpoint_path: "..."`, `all_model_checkpoint_paths: "..."` lines

The names are tf_names.tf_tensors'.  save() / restore() stream between HBM and the files through two pinned buffers;
the CRC-32C of every tensor runs on the device (ops.crc32c, csrc/crc32c_bulk.cu).  The small host CRC of the index
blocks is tfrecord.crc32c.  Contract and deviations: DESIGN.md §2.11.
"""
from __future__ import annotations

import codecs
import glob
import os
import re
import struct
from typing import Dict, Iterator, List, NamedTuple, Optional, Sequence, Tuple

import torch

from . import tf_names
from .tfrecord import masked_crc

MAGIC = 0xDB4775248B80FB57
FOOTER_BYTES = 48
BLOCK_SIZE = 262144          # TensorFlow's table_options.h block_size
RESTART_INTERVAL = 16
KEEP_CHECKPOINT_MAX = 5      # RunConfig / Saver default max_to_keep
CHUNK_BYTES = 64 << 20       # each of the two pinned staging buffers

DT_FLOAT, DT_INT64 = 1, 9
_DTYPE_OF = {torch.float32: DT_FLOAT, torch.int64: DT_INT64}
_DTYPE_NAME = {1: "float32", 2: "float64", 3: "int32", 4: "uint8", 5: "int16", 6: "int8", 7: "string", 9: "int64",
               10: "bool", 19: "float16", 14: "bfloat16"}
_ITEMSIZE = {DT_FLOAT: 4, DT_INT64: 8}


class MissingTensorError(KeyError, ValueError):
    """A tensor the model needs is not in the bundle (a KeyError like tf_names.load_state_dict_tf's, and a
    ValueError like every other rejection of a bundle)."""


# ---- protobuf wire format ------------------------------------------------------------------------------------
def _varint(v: int) -> bytes:
    v &= (1 << 64) - 1
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _get_varint(buf: bytes, pos: int, end: int, what: str) -> Tuple[int, int]:
    v = shift = 0
    while True:
        if pos >= end or shift > 63:
            raise ValueError(f"{what}: bad varint")
        b = buf[pos]
        pos += 1
        v |= (b & 0x7F) << shift
        shift += 7
        if not b & 0x80:
            return v, pos


def _fields(buf: bytes, what: str) -> Iterator[Tuple[int, int, object]]:
    """(field number, wire type, value) of a serialized message; unknown fields are the caller's to skip."""
    pos, end = 0, len(buf)
    while pos < end:
        key, pos = _get_varint(buf, pos, end, what)
        f, wt = key >> 3, key & 7
        if wt == 0:
            v, pos = _get_varint(buf, pos, end, what)
        elif wt == 1:
            if pos + 8 > end:
                raise ValueError(f"{what}: truncated field {f}")
            v, pos = struct.unpack_from("<Q", buf, pos)[0], pos + 8
        elif wt == 2:
            n, pos = _get_varint(buf, pos, end, what)
            if pos + n > end:
                raise ValueError(f"{what}: truncated field {f}")
            v, pos = buf[pos:pos + n], pos + n
        elif wt == 5:
            if pos + 4 > end:
                raise ValueError(f"{what}: truncated field {f}")
            v, pos = struct.unpack_from("<I", buf, pos)[0], pos + 4
        else:
            raise ValueError(f"{what}: unsupported wire type {wt} (field {f})")
        yield f, wt, v


def _int64(v: int) -> int:
    return v - (1 << 64) if v >= 1 << 63 else v


def _tag(f: int, wt: int) -> bytes:
    return _varint(f << 3 | wt)


def _len_field(f: int, payload: bytes) -> bytes:
    return _tag(f, 2) + _varint(len(payload)) + payload


class Entry(NamedTuple):
    """BundleEntryProto: where a tensor lives and what it is."""
    dtype: int
    shape: Tuple[int, ...]
    shard_id: int
    offset: int
    size: int
    crc32c: int          # masked CRC-32C of the tensor's bytes
    sliced: bool = False


def encode_entry(e: Entry) -> bytes:
    shape = b"".join(_len_field(2, (_tag(1, 0) + _varint(d)) if d else b"") for d in e.shape)
    out = _tag(1, 0) + _varint(e.dtype) + _len_field(2, shape)
    for f, v in ((3, e.shard_id), (4, e.offset), (5, e.size)):
        if v:
            out += _tag(f, 0) + _varint(v)
    if e.crc32c:
        out += _tag(6, 5) + struct.pack("<I", e.crc32c)
    return out


def decode_entry(buf: bytes, what: str) -> Entry:
    v = dict(dtype=0, shape=(), shard_id=0, offset=0, size=0, crc32c=0, sliced=False)
    for f, wt, x in _fields(buf, what):
        if f == 1 and wt == 0:
            v["dtype"] = x
        elif f == 2 and wt == 2:
            dims = []
            for df, dwt, dx in _fields(x, what):
                if df == 2 and dwt == 2:
                    size = 0
                    for sf, swt, sx in _fields(dx, what):
                        if sf == 1 and swt == 0:
                            size = _int64(sx)
                    dims.append(size)
                elif df == 3 and dwt == 0 and dx:
                    raise ValueError(f"{what}: unknown-rank shape")
            v["shape"] = tuple(dims)
        elif f in (3, 4, 5) and wt == 0:
            v[{3: "shard_id", 4: "offset", 5: "size"}[f]] = _int64(x)
        elif f == 6 and wt == 5:
            v["crc32c"] = x
        elif f == 7:
            v["sliced"] = True
    return Entry(**v)


def encode_header(num_shards: int = 1) -> bytes:
    return _tag(1, 0) + _varint(num_shards) + _len_field(3, _tag(1, 0) + _varint(1))


def decode_header(buf: bytes, what: str) -> int:
    """Checks a BundleHeaderProto the way TensorFlow's BundleReader does; returns num_shards."""
    num_shards, endianness, min_consumer, bad = 0, 0, 0, []
    for f, wt, x in _fields(buf, what):
        if f == 1 and wt == 0:
            num_shards = _int64(x)
        elif f == 2 and wt == 0:
            endianness = x
        elif f == 3 and wt == 2:
            for vf, vwt, vx in _fields(x, what):
                if vf == 2 and vwt == 0:
                    min_consumer = _int64(vx)
                elif vf == 3 and vwt == 0:
                    bad.append(_int64(vx))
                elif vf == 3 and vwt == 2:          # packed
                    p = 0
                    while p < len(vx):
                        b, p = _get_varint(vx, p, len(vx), what)
                        bad.append(_int64(b))
    if endianness != 0:
        raise ValueError(f"{what}: big-endian bundle (endianness {endianness}); only little-endian is supported")
    if min_consumer > 1 or 1 in bad:
        raise ValueError(f"{what}: bundle version needs a newer reader (min_consumer {min_consumer}, "
                         f"bad_consumers {bad})")
    if num_shards < 1:
        raise ValueError(f"{what}: num_shards {num_shards}")
    return num_shards


# ---- LevelDB table -------------------------------------------------------------------------------------------
class _BlockBuilder:
    def __init__(self, restart_interval: int):
        self.ri, self.out, self.restarts, self.last, self.count = restart_interval, bytearray(), [0], b"", 0

    def add(self, k: bytes, v: bytes):
        shared = 0
        if self.count < self.ri:
            n = min(len(self.last), len(k))
            while shared < n and self.last[shared] == k[shared]:
                shared += 1
        else:
            self.restarts.append(len(self.out))
            self.count = 0
        self.out += _varint(shared) + _varint(len(k) - shared) + _varint(len(v)) + k[shared:] + v
        self.last, self.count = k, self.count + 1

    def size(self) -> int:
        return len(self.out) + 4 * len(self.restarts) + 4

    def finish(self) -> bytes:
        return bytes(self.out) + b"".join(struct.pack("<I", r) for r in self.restarts) + struct.pack("<I", len(self.restarts))


def _trailer(contents: bytes) -> bytes:
    return b"\x00" + struct.pack("<I", masked_crc(contents + b"\x00"))


def write_table(path: str, items: Sequence[Tuple[bytes, bytes]], block_size: int = BLOCK_SIZE,
                restart_interval: int = RESTART_INTERVAL):
    """items sorted bytewise by key.  A data block is closed once its size reaches block_size (TensorFlow's rule);
    the index block has restart interval 1 and keys each block's last key."""
    out, index = bytearray(), _BlockBuilder(1)

    def put(blk: bytes) -> bytes:
        handle = _varint(len(out)) + _varint(len(blk))
        out.extend(blk + _trailer(blk))
        return handle

    cur = _BlockBuilder(restart_interval)
    for k, v in items:
        cur.add(k, v)
        if cur.size() >= block_size:
            index.add(k, put(cur.finish()))
            cur = _BlockBuilder(restart_interval)
    if cur.out:
        index.add(cur.last, put(cur.finish()))
    meta_handle = put(_BlockBuilder(restart_interval).finish())
    idx_handle = put(index.finish())
    out.extend((meta_handle + idx_handle).ljust(40, b"\x00") + struct.pack("<Q", MAGIC))
    with open(path, "wb") as f:
        f.write(out)
        f.flush()
        os.fsync(f.fileno())


def _read_block(buf: bytes, handle: bytes, path: str) -> List[Tuple[bytes, bytes]]:
    off, p = _get_varint(handle, 0, len(handle), path)
    size, _ = _get_varint(handle, p, len(handle), path)
    if off + size + 5 > len(buf):
        raise ValueError(f"{path}: truncated file (block at {off} of {size} bytes, file {len(buf)} bytes)")
    contents, typ = buf[off:off + size], buf[off + size]
    if typ == 1:
        raise ValueError(f"{path}: snappy-compressed block at {off} (only uncompressed bundles are supported)")
    if typ != 0:
        raise ValueError(f"{path}: unknown block compression type {typ} at {off}")
    if struct.unpack_from("<I", buf, off + size + 1)[0] != masked_crc(buf[off:off + size + 1]):
        raise ValueError(f"{path}: block checksum mismatch at {off}")
    if size < 4:
        raise ValueError(f"{path}: block at {off} too short")
    (nr,) = struct.unpack_from("<I", contents, size - 4)
    end = size - 4 - 4 * nr
    if nr < 1 or end < 0:
        raise ValueError(f"{path}: bad restart array in block at {off}")
    items, pos, last = [], 0, b""
    while pos < end:
        shared, pos = _get_varint(contents, pos, end, path)
        non_shared, pos = _get_varint(contents, pos, end, path)
        vlen, pos = _get_varint(contents, pos, end, path)
        if shared > len(last) or pos + non_shared + vlen > end:
            raise ValueError(f"{path}: corrupt entry in block at {off}")
        key = last[:shared] + contents[pos:pos + non_shared]
        pos += non_shared
        items.append((key, contents[pos:pos + vlen]))
        pos += vlen
        last = key
    return items


def read_table(path: str) -> List[Tuple[bytes, bytes]]:
    """Every (key, value) of a table file, in key order; ValueError names the file on any defect."""
    with open(path, "rb") as f:
        buf = f.read()
    if len(buf) < FOOTER_BYTES:
        raise ValueError(f"{path}: truncated file ({len(buf)} bytes, a footer alone is {FOOTER_BYTES})")
    foot = buf[-FOOTER_BYTES:]
    if struct.unpack_from("<Q", foot, 40)[0] != MAGIC:
        raise ValueError(f"{path}: bad table magic (not a TensorFlow checkpoint index)")
    p = 0
    for _ in range(2):                      # skip the metaindex handle
        _, p = _get_varint(foot, p, 40, path)
    idx_off, p = _get_varint(foot, p, 40, path)
    idx_size, p = _get_varint(foot, p, 40, path)
    items: List[Tuple[bytes, bytes]] = []
    for _, handle in _read_block(buf, _varint(idx_off) + _varint(idx_size), path):
        for k, v in _read_block(buf, handle, path):
            if items and k <= items[-1][0]:
                raise ValueError(f"{path}: keys out of order at {k!r}")
            items.append((k, v))
    return items


# ---- bundles -------------------------------------------------------------------------------------------------
def data_path(prefix: str, shard: int, num_shards: int) -> str:
    return "%s.data-%05d-of-%05d" % (prefix, shard, num_shards)


def read_index(prefix: str) -> Tuple[int, Dict[str, Entry]]:
    """(num_shards, {tensor name: Entry}) of `<prefix>.index`, header checked."""
    path = prefix + ".index"
    items = read_table(path)
    if not items or items[0][0] != b"":
        raise ValueError(f"{path}: no bundle header")
    num_shards = decode_header(items[0][1], path)
    entries = {}
    for k, v in items[1:]:
        name = k.decode("utf-8")
        entries[name] = decode_entry(v, f"{path}: tensor {name!r}")
    return num_shards, entries


def write_index(path: str, entries: Dict[str, Entry], block_size: int = BLOCK_SIZE):
    items = [(b"", encode_header(1))] + sorted((k.encode("utf-8"), encode_entry(e)) for k, e in entries.items())
    write_table(path, items, block_size)


def list_variables(path: str) -> List[Tuple[str, Tuple[int, ...], str]]:
    """(name, shape, dtype) of every tensor of a bundle (a prefix or a model_dir), from the index alone."""
    prefix = _resolve(path)
    _, entries = read_index(prefix)
    return [(k, e.shape, _DTYPE_NAME.get(e.dtype, "dtype%d" % e.dtype)) for k, e in sorted(entries.items())]


# ---- the `checkpoint` state file -----------------------------------------------------------------------------
_STATE_LINE = re.compile(r'^\s*(model_checkpoint_path|all_model_checkpoint_paths)\s*:\s*"((?:[^"\\]|\\.)*)"\s*$')


def read_state(model_dir: str) -> Tuple[Optional[str], List[str]]:
    """(model_checkpoint_path, all_model_checkpoint_paths) of model_dir/checkpoint as written, or (None, [])."""
    path = os.path.join(model_dir, "checkpoint")
    if not os.path.exists(path):
        return None, []
    latest, all_paths = None, []
    with open(path, encoding="utf-8") as f:
        for line in f:
            m = _STATE_LINE.match(line)
            if not m:
                continue
            val = codecs.escape_decode(m.group(2).encode("utf-8"))[0].decode("utf-8")
            if m.group(1) == "model_checkpoint_path":
                latest = val
            else:
                all_paths.append(val)
    return latest, all_paths


def _locate(model_dir: str, p: str) -> Optional[str]:
    """A prefix of the state file as an existing bundle: relative to model_dir, else its basename there (a moved
    directory)."""
    cand = p if os.path.isabs(p) else os.path.join(model_dir, p)
    if os.path.exists(cand + ".index"):
        return cand
    moved = os.path.join(model_dir, os.path.basename(p))
    return moved if os.path.exists(moved + ".index") else None


def latest_checkpoint(model_dir: str) -> Optional[str]:
    """The bundle prefix model_dir/checkpoint names, or None (no state file, or its bundle is gone)."""
    latest, _ = read_state(model_dir)
    return _locate(model_dir, latest) if latest else None


def _resolve(path: str) -> str:
    if os.path.isdir(path):
        p = latest_checkpoint(path)
        if p is None:
            raise FileNotFoundError(f"{path}: no checkpoint (no `checkpoint` file naming an existing bundle)")
        return p
    if path.endswith(".index"):
        path = path[:-len(".index")]
    if not os.path.exists(path + ".index"):
        raise FileNotFoundError(f"{path}.index: no such bundle")
    return path


def _quote(s: str) -> str:
    return '"' + s.replace("\\", "\\\\").replace('"', '\\"') + '"'


def _write_state(model_dir: str, latest: str, all_paths: Sequence[str]):
    text = "model_checkpoint_path: %s\n" % _quote(latest)
    text += "".join("all_model_checkpoint_paths: %s\n" % _quote(p) for p in all_paths)
    tmp = os.path.join(model_dir, "checkpoint.tmp%d" % os.getpid())
    with open(tmp, "w", encoding="utf-8") as f:
        f.write(text)
        f.flush()
        os.fsync(f.fileno())
    os.replace(tmp, os.path.join(model_dir, "checkpoint"))


def _delete_bundle(prefix: str):
    for p in [prefix + ".index", prefix + ".meta"] + glob.glob(glob.escape(prefix) + ".data-?????-of-?????"):
        if os.path.exists(p):
            os.remove(p)


# ---- streaming between HBM and the files ---------------------------------------------------------------------
def _pieces(sizes: Sequence[int], chunk: int) -> List[List[Tuple[int, int, int, int]]]:
    """Cuts the concatenation of `sizes` bytes into chunks of <= chunk bytes: per chunk, the pieces
    (item, byte offset in the item, byte offset in the chunk, bytes)."""
    out, cur, used = [], [], 0
    for k, n in enumerate(sizes):
        o = 0
        while o < n:
            take = min(n - o, chunk - used)
            cur.append((k, o, used, take))
            o, used = o + take, used + take
            if used == chunk:
                out.append(cur)
                cur, used = [], 0
    if cur:
        out.append(cur)
    return out


def _bytes_of(t: torch.Tensor) -> torch.Tensor:
    return t.detach().reshape(-1).view(torch.uint8)


class _Staging:
    """Two pinned host buffers, each reused once the device copy that last touched it has completed."""

    def __init__(self, chunk: int):
        self.buf = [torch.empty(chunk, dtype=torch.uint8, pin_memory=True) for _ in range(2)]
        self.np = [b.numpy() for b in self.buf]
        self.done: List[Optional[torch.cuda.Event]] = [None, None]

    def wait(self, i: int):
        if self.done[i % 2] is not None:
            self.done[i % 2].synchronize()

    def record(self, i: int):
        ev = torch.cuda.Event()
        ev.record()
        self.done[i % 2] = ev


def save(model, model_dir: str, chunk_bytes: int = CHUNK_BYTES, keep: int = KEEP_CHECKPOINT_MAX) -> str:
    """Writes the model's whole training state (tf_names.tf_tensors) as the bundle model_dir/model.ckpt-<global_step>
    and names it in model_dir/checkpoint; keeps the newest `keep` bundles.  The data file and the index are written
    under temporary names, the index renamed last, then the state file replaced.  Returns the prefix."""
    from . import ops
    os.makedirs(model_dir, exist_ok=True)
    pairs = sorted(tf_names.tf_tensors(model), key=lambda p: p[0].encode("utf-8"))
    for name, t in pairs:
        if t.dtype not in _DTYPE_OF:
            raise TypeError(f"{name}: dtype {t.dtype} has no bundle encoding here")
    views = [_bytes_of(t) for _, t in pairs]
    _, masked = ops.crc32c(views)
    sizes = [v.numel() for v in views]
    base = "model.ckpt-%d" % model.global_step
    prefix = os.path.join(model_dir, base)
    tmp_sfx = ".tmp%d" % os.getpid()
    data_final = data_path(prefix, 0, 1)
    chunks = _pieces(sizes, chunk_bytes)
    st = _Staging(min(chunk_bytes, max(sum(sizes), 1)))

    def issue(i):
        for k, src, dst, n in chunks[i]:
            st.buf[i % 2][dst:dst + n].copy_(views[k][src:src + n], non_blocking=True)
        st.record(i)

    with open(data_final + tmp_sfx, "wb") as f:
        for i in range(min(2, len(chunks))):
            issue(i)
        for i in range(len(chunks)):
            st.wait(i)
            last = chunks[i][-1]
            f.write(st.np[i % 2][:last[2] + last[3]])
            if i + 2 < len(chunks):
                issue(i + 2)
        f.flush()
        os.fsync(f.fileno())
    crcs = [c & 0xFFFFFFFF for c in masked.cpu().tolist()]
    entries, off = {}, 0
    for (name, t), n, c in zip(pairs, sizes, crcs):
        entries[name] = Entry(_DTYPE_OF[t.dtype], tuple(t.shape), 0, off, n, c)
        off += n
    write_index(prefix + ".index" + tmp_sfx, entries)
    os.replace(data_final + tmp_sfx, data_final)
    os.replace(prefix + ".index" + tmp_sfx, prefix + ".index")
    _, old = read_state(model_dir)
    kept = [p for p in old if os.path.basename(p) != base] + [base]
    for p in kept[:-keep] if keep > 0 else []:
        _delete_bundle(os.path.join(model_dir, os.path.basename(p)))     # only bundles of this directory
    _write_state(model_dir, base, kept[-keep:] if keep > 0 else kept)
    return prefix


def check_against(prefix: str, num_shards: int, entries: Dict[str, Entry],
                  wanted: Sequence[Tuple[str, torch.dtype, Tuple[int, ...], bool]]) -> List[Optional[Entry]]:
    """Host-side check of a bundle against what a model needs, before anything is read: for each (name, dtype, shape,
    required) the Entry to restore, or None for an optional name the bundle lacks.  Names the model does not have
    are ignored.  Raises MissingTensorError for required names the bundle lacks, ValueError for everything else."""
    path = prefix + ".index"
    missing = [name for name, _, _, req in wanted if req and name not in entries]
    if missing:
        raise MissingTensorError(f"{path}: missing tensors {missing[:8]}{' ...' if len(missing) > 8 else ''}")
    out = []
    shard_bytes: Dict[int, int] = {}
    for name, dtype, shape, _ in wanted:
        e = entries.get(name)
        out.append(e)
        if e is None:
            continue
        if e.sliced:
            raise ValueError(f"{path}: tensor {name!r} is saved in slices (a partitioned variable); not supported")
        if e.dtype != _DTYPE_OF[dtype]:
            raise ValueError(f"{path}: tensor {name!r} has dtype {_DTYPE_NAME.get(e.dtype, e.dtype)}, "
                             f"the model's variable is {dtype}")
        if tuple(e.shape) != tuple(shape):
            raise ValueError(f"{path}: tensor {name!r} has shape {list(e.shape)}, the model's variable is {list(shape)}")
        n = _ITEMSIZE[e.dtype]
        for d in shape:
            n *= d
        if e.size != n:
            raise ValueError(f"{path}: tensor {name!r} has {e.size} bytes, its shape needs {n}")
        if not 0 <= e.shard_id < num_shards or e.offset < 0:
            raise ValueError(f"{path}: tensor {name!r} has shard {e.shard_id} / offset {e.offset} "
                             f"({num_shards} shards)")
        shard_bytes[e.shard_id] = max(shard_bytes.get(e.shard_id, 0), e.offset + e.size)
    for s, need in shard_bytes.items():
        p = data_path(prefix, s, num_shards)
        if not os.path.exists(p):
            raise ValueError(f"{p}: missing data file")
        if os.path.getsize(p) < need:
            raise ValueError(f"{p}: truncated file ({os.path.getsize(p)} bytes, the index needs {need})")
    return out


def restore(model, path_or_model_dir: str, variables_only: bool = False, chunk_bytes: int = CHUNK_BYTES) -> str:
    """Restores a bundle (a prefix, or the latest one of a model_dir) into the model in place.

    variables_only=False (training) needs every name of tf_names.tf_tensors(model), optimizer state included;
    variables_only=True (eval / infer / export: a PREDICT graph has no optimizer) needs only the model's variables
    and takes `global_step` when the bundle has it.  Names the model does not have are ignored.  The index is checked
    against the model (names, dtypes, shapes, data file sizes) before any tensor is written: a bundle that fails
    there raises and leaves the model as it was.  Then the data streams file -> pinned -> device, and the device
    CRC-32C of every restored tensor is compared with the index.  A mismatch raises ValueError naming the tensors;
    the model's state is then partly overwritten and the model must not be used.  Returns the prefix."""
    from . import ops
    prefix = _resolve(path_or_model_dir)
    num_shards, entries = read_index(prefix)
    pairs = list(tf_names.tf_tensors(model, optimizer=not variables_only))
    n_vars = len(model.variables())
    wanted = [(name, t.dtype, tuple(t.shape), i < n_vars or not variables_only) for i, (name, t) in enumerate(pairs)]
    found = check_against(prefix, num_shards, entries, wanted)
    todo = [(name, t, e) for (name, t), e in zip(pairs, found) if e is not None]
    views = [_bytes_of(t) for _, t, _ in todo]
    for s in range(num_shards):
        mine = sorted((e.offset, k) for k, (_, _, e) in enumerate(todo) if e.shard_id == s)
        if not mine:
            continue
        chunks = _pieces([todo[k][2].size for _, k in mine], chunk_bytes)
        st = _Staging(min(chunk_bytes, max(sum(todo[k][2].size for _, k in mine), 1)))
        p = data_path(prefix, s, num_shards)
        with open(p, "rb") as f:
            for i, ch in enumerate(chunks):
                st.wait(i)
                for j, src, dst, n in ch:
                    k = mine[j][1]
                    f.seek(todo[k][2].offset + src)
                    if f.readinto(memoryview(st.np[i % 2])[dst:dst + n]) != n:
                        raise ValueError(f"{p}: truncated file while reading tensor {todo[k][0]!r}")
                for j, src, dst, n in ch:
                    views[mine[j][1]][src:src + n].copy_(st.buf[i % 2][dst:dst + n], non_blocking=True)
                st.record(i)
    if todo:
        _, masked = ops.crc32c(views)
        bad = [name for (name, _, e), c in zip(todo, masked.cpu().tolist()) if (c & 0xFFFFFFFF) != e.crc32c]
        if bad:
            raise ValueError(f"{prefix}: data checksum mismatch for tensor(s) {bad[:8]}; the model's state is now "
                             "partly overwritten and must not be used")
    for name, t, _ in todo:
        if name == "global_step":
            tf_names.set_global_step(model, int(t.item()))
    return prefix
