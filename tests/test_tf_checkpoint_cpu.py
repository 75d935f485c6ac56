"""The TensorFlow checkpoint codec of tf_repos_b200/tf_checkpoint.py on the host: its index files and those of the
independent oracle (tests/tf_bundle_oracle.py) read each other across block sizes, restart intervals and shard
counts; every defect a bundle can carry is rejected with a ValueError naming the file (and the tensor); the
`checkpoint` state file resolves relative, absolute and moved paths.  (The streaming save / restore and the device
CRC: tests/test_gpu_tf_checkpoint.py.)"""
import importlib.util
import os

import numpy as np
import pytest
import torch

from tests import tf_bundle_oracle as tb
from tf_repos_b200 import tf_checkpoint as tc
from tf_repos_b200.tfrecord import crc32c

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

NAMES = ["fm_bias", "fm_v", "fm_v/Adam", "fm_v/Adam_1", "fm_w", "global_step", "beta1_power", "beta2_power"] + [
    f"Deep-part/mlp{i}/{w}{s}" for i in range(4) for w in ("weights", "biases") for s in ("", "/Adam", "/Adam_1")]


def _tensors(seed=0):
    rng = np.random.RandomState(seed)
    out = {}
    for k, n in enumerate(NAMES):
        if n == "global_step":
            out[n] = np.array(1234567, dtype=np.int64)
        elif n.startswith("beta"):
            out[n] = np.array(0.9 ** 7, dtype=np.float32)
        else:
            out[n] = rng.randn(*((k % 5 + 1, 3) if "weights" in n or "fm_v" in n else (k % 7 + 1,))).astype(np.float32)
    return out


LAYOUTS = [dict(block_size=64, restart_interval=1, num_shards=1), dict(block_size=64, restart_interval=16, num_shards=2),
           dict(block_size=300, restart_interval=3, num_shards=2), dict(block_size=1 << 18, restart_interval=16, num_shards=1)]


@pytest.mark.parametrize("layout", LAYOUTS, ids=lambda l: "bs%d-ri%d-sh%d" % tuple(l.values()))
def test_engine_reads_oracle_bundles(tmp_path, layout):
    t = _tensors()
    prefix = str(tmp_path / "model.ckpt-3")
    tb.write_bundle(prefix, t, **layout)
    assert len(tc.read_table(prefix + ".index")) == len(t) + 1
    num_shards, entries = tc.read_index(prefix)
    assert num_shards == layout["num_shards"] and set(entries) == set(t)
    for name, a in t.items():
        e = entries[name]
        assert e.shape == a.shape and e.dtype == (9 if a.dtype == np.int64 else 1) and e.size == a.nbytes
        assert e.crc32c == tb.mask(crc32c(a.tobytes())) and not e.sliced
        with open(tc.data_path(prefix, e.shard_id, num_shards), "rb") as f:
            f.seek(e.offset)
            assert f.read(e.size) == a.tobytes()
    assert tc.list_variables(prefix) == sorted(((n, a.shape, str(a.dtype)) for n, a in t.items()),
                                               key=lambda r: r[0].encode())


@pytest.mark.parametrize("block_size", [64, 200, tc.BLOCK_SIZE])
def test_oracle_reads_engine_index(tmp_path, block_size):
    t = _tensors(1)
    entries, off = {}, 0
    for name in sorted(t):
        a = t[name]
        entries[name] = tc.Entry(9 if a.dtype == np.int64 else 1, a.shape, 0, off, a.nbytes, tb.mask(crc32c(a.tobytes())))
        off += a.nbytes
    prefix = str(tmp_path / "e")
    tc.write_index(prefix + ".index", entries, block_size=block_size)
    with open(tc.data_path(prefix, 0, 1), "wb") as f:
        f.write(b"".join(t[n].tobytes() for n in sorted(t)))
    got = tb.read_bundle(prefix)
    assert set(got) == set(t) and all(got[n].tobytes() == t[n].tobytes() and got[n].shape == t[n].shape for n in t)
    assert tc.read_index(prefix) == (1, entries)


def test_block_layout_follows_the_size_threshold(tmp_path):
    """Many data blocks and index entries with a small threshold, one data block at TensorFlow's default."""
    items = [(b""), *(n.encode() for n in sorted(NAMES))]
    items = [(k, b"v" * 20) for k in items]
    for bs in (64, tc.BLOCK_SIZE):
        p = str(tmp_path / ("t%d" % bs))
        tc.write_table(p, items, block_size=bs)
        idx = tb._read_block(open(p, "rb").read(), *_index_handle(p))
        assert len(idx) > len(items) // 3 if bs == 64 else len(idx) == 1
        assert [k for k, _ in idx][-1] == items[-1][0]
        assert tc.read_table(p) == items


def _index_handle(path):
    foot = open(path, "rb").read()[-48:]
    i = 0
    for _ in range(2):
        _, i = tb._rv(foot, i)
    off, i = tb._rv(foot, i)
    size, _ = tb._rv(foot, i)
    return off, size


def _bundle(tmp_path, **kw):
    prefix = str(tmp_path / "model.ckpt-1")
    tb.write_bundle(prefix, _tensors(), block_size=128, **kw)
    return prefix


def test_reject_bad_magic_truncation_and_flipped_byte(tmp_path):
    prefix = _bundle(tmp_path)
    idx = prefix + ".index"
    good = open(idx, "rb").read()
    open(idx, "wb").write(good[:-1] + bytes([good[-1] ^ 1]))
    with pytest.raises(ValueError, match="magic") as e:
        tc.read_index(prefix)
    assert idx in str(e.value)
    for cut in (30, len(good) // 2):
        open(idx, "wb").write(good[cut:])        # footer intact, blocks cut away from the front
        with pytest.raises(ValueError, match=r"truncated|checksum|corrupt|bad") as e:
            tc.read_index(prefix)
        assert idx in str(e.value)
    open(idx, "wb").write(good[:40])
    with pytest.raises(ValueError, match="truncated"):
        tc.read_index(prefix)
    bad = bytearray(good)
    bad[10] ^= 0x40                              # inside the first data block
    open(idx, "wb").write(bytes(bad))
    with pytest.raises(ValueError, match="checksum") as e:
        tc.read_index(prefix)
    assert idx in str(e.value)


@pytest.mark.parametrize("defect,match", [(dict(block_type=1), "snappy"), (dict(endianness=1), "big-endian"),
                                          (dict(min_consumer=2), "min_consumer")])
def test_reject_header_and_compression(tmp_path, defect, match):
    prefix = _bundle(tmp_path, **defect)
    with pytest.raises(ValueError, match=match) as e:
        tc.read_index(prefix)
    assert prefix + ".index" in str(e.value)


def _wanted(t, drop=(), reshape=None, retype=None):
    out = []
    for n, a in t.items():
        if n in drop:
            continue
        dtype = torch.int64 if a.dtype == np.int64 else torch.float32
        shape = reshape[1] if reshape and reshape[0] == n else a.shape
        out.append((n, retype[1] if retype and retype[0] == n else dtype, tuple(shape), True))
    return out


def test_check_against_the_model(tmp_path):
    t = _tensors()
    prefix = _bundle(tmp_path, num_shards=2)
    ns, entries = tc.read_index(prefix)
    found = tc.check_against(prefix, ns, entries, _wanted(t, drop=("fm_v/Adam",)))    # extra names are ignored
    assert [e.size for e in found] == [a.nbytes for n, a in t.items() if n != "fm_v/Adam"]
    with pytest.raises(ValueError, match="'fm_v'.*shape") as e:
        tc.check_against(prefix, ns, entries, _wanted(t, reshape=("fm_v", (4, 3))))
    assert prefix in str(e.value)
    with pytest.raises(ValueError, match="'global_step'.*dtype"):
        tc.check_against(prefix, ns, entries, _wanted(t, retype=("global_step", torch.float32)))
    want = _wanted(t) + [("fm_v/Ftrl", torch.float32, (1, 3), True), ("opt_only", torch.float32, (1,), False)]
    with pytest.raises(KeyError, match="fm_v/Ftrl") as e:
        tc.check_against(prefix, ns, entries, want)
    assert isinstance(e.value, ValueError) and "opt_only" not in str(e.value)
    assert tc.check_against(prefix, ns, entries, want[:-2] + want[-1:])[-1] is None
    data1 = tc.data_path(prefix, 1, 2)
    open(data1, "r+b").truncate(3)
    with pytest.raises(ValueError, match="truncated") as e:
        tc.check_against(prefix, ns, entries, _wanted(t))
    assert data1 in str(e.value)


def test_reject_sliced_tensor(tmp_path):
    t = _tensors()
    prefix = _bundle(tmp_path, sliced=("fm_w",))
    ns, entries = tc.read_index(prefix)
    assert entries["fm_w"].sliced and not entries["fm_v"].sliced
    with pytest.raises(ValueError, match="'fm_w'.*slices"):
        tc.check_against(prefix, ns, entries, _wanted(t))


def test_checkpoint_state_paths(tmp_path):
    d = str(tmp_path / "run")
    os.makedirs(d)
    assert tc.latest_checkpoint(d) is None
    tb.write_bundle(d + "/model.ckpt-8", _tensors())
    tb.write_bundle(d + "/model.ckpt-16", _tensors())
    tb.write_state(d, ["model.ckpt-8", "model.ckpt-16"])                       # relative
    assert tc.latest_checkpoint(d) == d + "/model.ckpt-16"
    assert tc.read_state(d) == ("model.ckpt-16", ["model.ckpt-8", "model.ckpt-16"])
    tb.write_state(d, [d + "/model.ckpt-8"])                                    # absolute
    assert tc.latest_checkpoint(d) == d + "/model.ckpt-8"
    tb.write_state(d, ["/gone/train_dir/model.ckpt-16"])                       # moved: same basename here
    assert tc.latest_checkpoint(d) == d + "/model.ckpt-16"
    assert [n for n, _, _ in tc.list_variables(d)] == sorted(NAMES, key=str.encode)
    tb.write_state(d, ["model.ckpt-99"])                                        # names a bundle that is not there
    assert tc.latest_checkpoint(d) is None
    with pytest.raises(FileNotFoundError):
        tc.list_variables(d)
    with open(os.path.join(d, "checkpoint"), "w") as f:                         # escapes of the text format
        f.write('model_checkpoint_path: "model.ckpt-\\0608"\nall_model_checkpoint_paths: "a\\"b"\n')
    assert tc.read_state(d) == ("model.ckpt-08", ['a"b'])
    tc._write_state(d, 'we"ird\\name', ["x", 'we"ird\\name'])
    assert tc.read_state(d) == ('we"ird\\name', ["x", 'we"ird\\name'])


@pytest.mark.parametrize("script,has_flag", [("DeepFM.py", True), ("DCN.py", True), ("DIN.py", True),
                                             ("DeepCvrMTL.py", False)])
def test_checkpoint_format_flag(script, has_flag):
    """--checkpoint_format (default b200) on the libsvm scripts and DIN; DeepCvrMTL.py keeps its flag surface."""
    import importlib
    from tf_repos_b200 import flags
    importlib.reload(flags)
    try:
        spec = importlib.util.spec_from_file_location("script", os.path.join(ROOT, "Model_pipeline", script))
        spec.loader.exec_module(importlib.util.module_from_spec(spec))
        F = flags.FLAGS
        assert ("checkpoint_format" in F._items()) == has_flag
        if has_flag:
            assert F.checkpoint_format == "b200"
            F._parse(["--checkpoint_format=tf"])
            assert F.checkpoint_format == "tf"
        else:
            with pytest.raises(SystemExit, match="checkpoint_format"):
                F._parse(["--checkpoint_format=tf"])
    finally:
        importlib.reload(flags)
