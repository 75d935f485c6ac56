"""TensorFlow V2 checkpoints on the GPU (tf_repos_b200/tf_checkpoint.py, csrc/crc32c_bulk.cu): the device CRC-32C
against host CRCs and a CRC-combine oracle, bit-exact save / restore / continue for every model and optimizer,
bundles of the independent oracle (tests/tf_bundle_oracle.py) both ways, corruption and mismatch rejection, and the
drop-in scripts' --checkpoint_format=tf (DeepFM, DIN)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import tf_bundle_oracle as tb

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"


def _crc(tensors):
    from tf_repos_b200 import ops
    raw, masked = ops.crc32c(tensors)
    return [c & 0xFFFFFFFF for c in raw.cpu().tolist()], [c & 0xFFFFFFFF for c in masked.cpu().tolist()]


# ---- the device CRC --------------------------------------------------------------------------------------------
def test_crc_check_value_and_mask():
    t = torch.tensor(list(b"123456789"), dtype=torch.uint8, device=DEV)
    raw, masked = _crc([t])
    assert raw == [0xE3069283] and masked == [tb.mask(0xE3069283)]


def test_crc_every_short_length_and_offset_in_one_batch():
    rng = np.random.RandomState(0)
    host = rng.randint(0, 256, 4096).astype(np.uint8)
    buf = torch.from_numpy(host).to(DEV)
    spans = [(off, n) for off in (0, 4, 8, 12) for n in range(0, 1025)]
    raw, masked = _crc([buf[o:o + n] for o, n in spans])
    for (o, n), r, m in zip(spans, raw, masked):
        want = tb.crc32c(host[o:o + n].tobytes())
        assert r == want and m == tb.mask(want), (o, n)


def test_crc_batch_equals_single_ranges():
    """Ranges of many chunks, odd tails and 4-byte aligned starts: the same bits together as alone, and the host's."""
    rng = np.random.RandomState(1)
    host = rng.randint(0, 256, 3 << 20).astype(np.uint8)
    buf = torch.from_numpy(host).to(DEV)
    spans = [(4, (1 << 20) + 13), (0, 131072), (12, 131072 * 3 - 4), (8, 0), (2 << 20, 777), (20, 5), (1 << 20, 1 << 21)]
    views = [buf[o:o + n] for o, n in spans]
    together = _crc(views)
    for k, v in enumerate(views):
        alone = _crc([v])
        assert (alone[0][0], alone[1][0]) == (together[0][k], together[1][k]), spans[k]
    for (o, n), r in zip(spans, together[0]):
        assert r == tb.crc32c(host[o:o + n].tobytes()), (o, n)
    # the same call twice: deterministic
    assert _crc(views) == together


def test_crc_range_longer_than_4gib():
    m, times = 1 << 20, 4097                           # 4097 MiB > 2^32 bytes
    rng = np.random.RandomState(2)
    pat = rng.randint(0, 256, m).astype(np.uint8)
    big = torch.empty(m * times, dtype=torch.uint8, device=DEV)
    big.view(times, m).copy_(torch.from_numpy(pat).to(DEV).expand(times, m))
    c = tb.crc32c(pat.tobytes())
    want_full = tb.crc32c_repeat(c, m, times)
    want_off = tb.crc32c_combine(tb.crc32c(pat[4:].tobytes()), tb.crc32c_repeat(c, m, times - 1), m * (times - 1))
    raw, _ = _crc([big, big[4:]])
    assert raw == [want_full, want_off]
    del big
    torch.cuda.empty_cache()


# ---- models ---------------------------------------------------------------------------------------------------
F, N, K, B, FP, P = 16, 3000, 8, 64, 5, 7
LENS = (5, 9, 5, 5, 3)
MODELS = ["DeepFM", "DCN", "DeepMVM", "NFM", "PNN", "AFM", "DIN", "ESMM"]
OPTS = ["Adam", "Adagrad", "Momentum", "ftrl"]
CHUNK = 40_000       # smaller than fm_v / embeddings (96 000 bytes) and not a divisor of it


def _batches(kind, n, seed=70):
    from tf_repos_b200 import synth
    out = []
    for s in range(n):
        if kind == "DIN":
            out.append(synth.din_batch(B, N, FP, P, 4, seed=seed + s, device=DEV))
        elif kind == "ESMM":
            out.append(synth.esmm_batch(B, N, FP, max_lens=LENS, min_len=0, seed=seed + s, device=DEV))
        else:
            ids, vals, labels = synth.criteo_batch(B, N, F, seed=seed + s, device=DEV)
            out.append(((ids, vals), labels))
    return out


def _model(kind, opt, feature_size=N, **over):
    from tf_repos_b200.afm import AFM
    from tf_repos_b200.dcn import DCN
    from tf_repos_b200.deepfm import DeepFM
    from tf_repos_b200.deepmvm import DeepMVM
    from tf_repos_b200.din import DIN
    from tf_repos_b200.esmm import ESMM
    from tf_repos_b200.nfm import NFM
    from tf_repos_b200.pnn import PNN
    kw = dict(optimizer=opt, learning_rate=(5e-4 if opt == "Adam" else 0.01), update_mode="exact_deferred",
              epoch_steps=4, device=DEV, seed=3)
    kw.update(over)
    bn = dict(batch_norm=True)
    if kind == "DeepFM":
        return DeepFM(F, feature_size, K, B, deep_layers="16,8", dropout="0.9,0.9", **bn, **kw)
    if kind == "DCN":
        return DCN(F, feature_size, K, B, deep_layers="16,8", cross_layers=2, dropout="0.9,0.9", **bn, **kw)
    if kind == "DeepMVM":
        return DeepMVM(F, feature_size, K, B, deep_layers="16,8", dropout="0.9,0.9", **bn, **kw)
    if kind == "NFM":
        return NFM(F, feature_size, K, B, deep_layers="16,8", dropout="0.9,0.9,0.9", **bn, **kw)
    if kind == "PNN":
        return PNN(F, feature_size, K, B, model_type="Inner", deep_layers="16,8", dropout="0.9,0.9", **bn, **kw)
    if kind == "AFM":
        return AFM(F, feature_size, K, B, attention_layers="16", dropout="1.0,0.9", **kw)
    if kind == "DIN":
        # batch norm with attention pooling raises NameError in the reference (DIN.py:166, quirk Q5)
        return DIN(FP, feature_size, K, B, P, max_a_int=4, deep_layers="16,8", dropout="0.9,0.9", **kw)
    return ESMM(FP, feature_size, K, B, 64 * sum(LENS), deep_layers="16,8", dropout="0.9,0.9", **bn, **kw)


def _step(model, batch):
    x, labels = batch
    out = model.train_step(*x, labels) if isinstance(x, tuple) else model.train_step(x, labels)
    return out.clone()


def _same_state(a, b):
    assert a.keys() == b.keys()
    for k in a:
        x, y = np.asarray(a[k]), np.asarray(b[k])
        assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), k


@pytest.mark.parametrize("opt", OPTS)
@pytest.mark.parametrize("kind", MODELS)
def test_save_restore_continue_bit_exact(tmp_path, kind, opt):
    from tf_repos_b200 import tf_checkpoint as tc
    from tf_repos_b200 import tf_names
    batches = _batches(kind, 8)
    a = _model(kind, opt)
    for b in batches[:5]:                     # 5 steps of 4-step epochs: the save is taken mid-epoch
        _step(a, b)
    d = str(tmp_path / "m")
    prefix = tc.save(a, d, chunk_bytes=CHUNK)
    assert prefix == os.path.join(d, "model.ckpt-5") and tc.latest_checkpoint(d) == prefix
    sd = tf_names.state_dict_tf(a)
    # the oracle reads the engine's bundle and verifies every CRC on the host
    _same_state(sd, tb.read_bundle(prefix))
    assert [(n, s, t) for n, s, t in tc.list_variables(d)] == sorted(
        ((k, np.asarray(v).shape, str(np.asarray(v).dtype)) for k, v in sd.items()), key=lambda r: r[0].encode())
    b = _model(kind, opt)
    tc.restore(b, d, chunk_bytes=CHUNK)
    _same_state(sd, tf_names.state_dict_tf(b))
    assert b.global_step == 5
    for batch in batches[5:]:
        la, lb = _step(a, batch), _step(b, batch)
        assert torch.equal(la, lb)
    _same_state(tf_names.state_dict_tf(a), tf_names.state_dict_tf(b))


@pytest.mark.parametrize("kind", ["DeepFM", "DIN", "ESMM"])
def test_restore_oracle_bundles(tmp_path, kind):
    """Multi-block, two-shard bundles of the oracle with extra names: whole state for training, variables only for
    inference; a variables-only bundle cannot resume training."""
    from tf_repos_b200 import tf_checkpoint as tc
    from tf_repos_b200 import tf_names
    batches = _batches(kind, 3)
    a = _model(kind, "Adam")
    for b in batches:
        _step(a, b)
    sd = tf_names.state_dict_tf(a)
    extra = {"OptimizeLoss/learning_rate": np.float32(0.1), "zz_unknown/var": np.arange(5, dtype=np.float32)}
    full = str(tmp_path / "full")
    tb.write_bundle(full, {**sd, **extra}, block_size=300, restart_interval=1, num_shards=2)
    b = _model(kind, "Adam")
    tc.restore(b, full, chunk_bytes=CHUNK)
    _same_state(sd, tf_names.state_dict_tf(b))
    var_names = list(a.variables())
    vonly = str(tmp_path / "vars")
    tb.write_bundle(vonly, {**{k: sd[k] for k in var_names}, **extra, "global_step": sd["global_step"]},
                    block_size=512, restart_interval=16, num_shards=2)
    c = _model(kind, "Adam")
    with pytest.raises(KeyError, match="Adam"):
        tc.restore(c, vonly)
    tc.restore(c, vonly, variables_only=True)
    vc, va = c.variables(), a.variables()
    assert all(torch.equal(vc[k], va[k]) for k in va) and c.global_step == a.global_step


def test_corrupt_data_and_wrong_shape(tmp_path):
    from tf_repos_b200 import tf_checkpoint as tc
    from tf_repos_b200 import tf_names
    a = _model("DeepFM", "Adam")
    for b in _batches("DeepFM", 2):
        _step(a, b)
    d = str(tmp_path / "m")
    prefix = tc.save(a, d, chunk_bytes=CHUNK)
    # a model with another feature_size: rejected from the index, before any tensor is written
    c = _model("DeepFM", "Adam", feature_size=N + 1)
    before = tf_names.state_dict_tf(c)
    with pytest.raises(ValueError, match="fm_v"):
        tc.restore(c, d)
    _same_state(before, tf_names.state_dict_tf(c))
    # one flipped byte inside fm_v's data
    _, entries = tc.read_index(prefix)
    e = entries["fm_v/Adam_1"]
    path = tc.data_path(prefix, 0, 1)
    raw = bytearray(open(path, "rb").read())
    raw[e.offset + e.size // 2] ^= 0x10
    open(path, "wb").write(bytes(raw))
    with pytest.raises(ValueError, match="fm_v/Adam_1"):
        tc.restore(_model("DeepFM", "Adam"), d, chunk_bytes=CHUNK)


def test_retention_keeps_five(tmp_path):
    from tf_repos_b200 import tf_checkpoint as tc
    from tf_repos_b200 import tf_names
    a = _model("DeepFM", "Adagrad")
    d = str(tmp_path / "m")
    for step in (1, 2, 3, 4, 5, 6, 7):
        tf_names.set_global_step(a, step)
        tc.save(a, d)
    latest, all_paths = tc.read_state(d)
    assert latest == "model.ckpt-7" and all_paths == ["model.ckpt-%d" % s for s in (3, 4, 5, 6, 7)]
    assert sorted(f for f in os.listdir(d) if f.endswith(".index")) == ["model.ckpt-%d.index" % s for s in (3, 4, 5, 6, 7)]
    assert not any(f.startswith(("model.ckpt-1.", "model.ckpt-2.")) or ".tmp" in f for f in os.listdir(d))


# ---- the drop-in scripts ----------------------------------------------------------------------------------------
def _libsvm(tmp, name, rows, seed, Nv=10_000):
    from tf_repos_b200 import synth
    ids, vals, labels = synth.criteo_batch(rows, Nv, 39, seed=seed)
    synth.write_libsvm(os.path.join(tmp, name), ids, vals, labels)


def _runner(common):
    def run(*args):
        r = subprocess.run(common + list(args), capture_output=True, text=True, timeout=280)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        return r.stdout
    return run


def test_deepfm_cli_tf_format(tmp_path):
    from tf_repos_b200 import tf_checkpoint as tc
    tmp = str(tmp_path)
    os.makedirs(tmp + "/data")
    # one training file: the script shuffles the file list (DeepFM.py:311), and the two formats' runs must see one order
    for name, rows, seed in (("tr0.libsvm", 1000, 1), ("va.libsvm", 200, 3), ("te.libsvm", 150, 4)):
        _libsvm(tmp + "/data", name, rows, seed)
    base = [sys.executable, os.path.join(ROOT, "Model_pipeline", "DeepFM.py"), "--field_size=39", "--feature_size=10000",
            "--embedding_size=8", "--batch_size=128", "--deep_layers=32,16", "--dropout=0.8,0.8", "--log_steps=5",
            "--num_epochs=1", "--data_dir=" + tmp + "/data", "--dt_dir=20261017"]
    preds = {}
    for fmt in ("b200", "tf"):
        run = _runner(base + ["--model_dir=%s/%s/m_" % (tmp, fmt), "--checkpoint_format=" + fmt])
        run("--task_type=train")
        assert "restored checkpoint" in run("--task_type=train")
        assert json.loads(run("--task_type=eval").strip().splitlines()[-1])["global_step"] == 16
        run("--task_type=infer")
        preds[fmt] = open(tmp + "/data/pred.txt").read()
    assert preds["tf"] == preds["b200"]
    mdir = tmp + "/tf/m_20261017"
    files = set(os.listdir(mdir))
    assert {"checkpoint", "model.ckpt-16.index", "model.ckpt-16.data-00000-of-00001"} <= files
    assert "ctr_b200.ckpt" not in files and tc.latest_checkpoint(mdir) == mdir + "/model.ckpt-16"
    run = _runner(base + ["--model_dir=%s/tf/m_" % tmp, "--checkpoint_format=tf"])
    run("--task_type=export", "--servable_model_dir=" + tmp + "/export")
    assert os.listdir(tmp + "/export")
    # infer from a directory holding only an oracle-written, variables-only bundle == the same values via import_npz
    from tf_repos_b200 import tf_names
    from tf_repos_b200.deepfm import DeepFM
    from tf_repos_b200.input_fn import decode_libsvm_file
    m = DeepFM(39, 10_000, 8, 128, deep_layers="32,16", dropout="0.8,0.8", device=DEV)
    vals = {k: v for k, v in tb.read_bundle(mdir + "/model.ckpt-16").items() if k in m.variables()}
    vals = {k: (v * np.float32(1.5) if v.dtype == np.float32 else v) for k, v in vals.items()}   # not the trained state
    odir = tmp + "/ora/m_20261017"
    os.makedirs(odir)
    tb.write_bundle(odir + "/model.ckpt-3", vals, block_size=200, restart_interval=1, num_shards=2)
    tb.write_state(odir, ["/elsewhere/moved/model.ckpt-3"])           # a moved directory: found by basename
    _runner(base + ["--model_dir=%s/ora/m_" % tmp, "--checkpoint_format=tf"])("--task_type=infer")
    got = open(tmp + "/data/pred.txt").read()
    np.savez(tmp + "/v.npz", **{k.replace("/", "|"): v for k, v in vals.items()})
    tf_names.import_npz(m, tmp + "/v.npz", strict=False)
    ids, fv, _ = decode_libsvm_file(tmp + "/data/te.libsvm", 39)
    ids, fv = torch.as_tensor(np.asarray(ids)), torch.as_tensor(np.asarray(fv))
    want = []
    for s in range(0, ids.shape[0], 128):
        want += ["%f\n" % p for p in m.predict(ids[s:s + 128].int().to(DEV), fv[s:s + 128].to(DEV)).cpu().tolist()]
    assert got == "".join(want)


def test_din_cli_tf_format_resume(tmp_path):
    """DIN.py through din_main.  (DeepCvrMTL.py has no --checkpoint_format; ESMM bundles go through
    tf_checkpoint.save / restore, test_save_restore_continue_bit_exact.)"""
    from tests.test_gpu_din_cli import _write_din as write
    script = "DIN.py"
    tmp = str(tmp_path)
    os.makedirs(tmp + "/data/tr"); os.makedirs(tmp + "/data/te")
    write(tmp + "/data/tr/part0.tfrecord", 120, 1); write(tmp + "/data/tr/part1.tfrecord", 80, 2)
    write(tmp + "/data/te/part0.tfrecord", 70, 3)
    run = _runner([sys.executable, os.path.join(ROOT, "Model_pipeline", script), "--field_size=11",
                   "--feature_size=5000", "--embedding_size=8", "--batch_size=64", "--deep_layers=16,8",
                   "--dropout=0.9,0.9", "--log_steps=1", "--num_epochs=1", "--data_dir=" + tmp + "/data",
                   "--model_dir=" + tmp + "/ckpt/m_", "--dt_dir=20261017", "--checkpoint_format=tf"])
    run("--task_type=train")
    assert "restored checkpoint" in run("--task_type=train")
    assert json.loads(run("--task_type=eval").strip().splitlines()[-1])["global_step"] == 8
    mdir = tmp + "/ckpt/m_20261017"
    assert {"model.ckpt-4.index", "model.ckpt-8.index", "checkpoint"} <= set(os.listdir(mdir))
    run("--task_type=infer")
    assert len(open(tmp + "/data/pred.txt").read().split("\n")) == 71
