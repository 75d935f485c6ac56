"""The capacity boundary of every lock-free key table of the text pipelines (csrc/key_table.cuh): with exactly as many
slots as distinct keys, the output is byte-identical to a run with a large table (the last keys in walk across the
wrap from slot cap - 1 to slot 0); with one slot fewer, the run raises the error that names the capacity parameter.
Tables: Criteo's count table, Ali-CCP's (field, fid) count table and md5 table, the smart feature_map table and the
smart builder's key table."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _files(d):
    """every file under d (relative path -> bytes)"""
    out = {}
    for root, _, names in os.walk(d):
        for n in names:
            p = os.path.join(root, n)
            out[os.path.relpath(p, d)] = open(p, "rb").read()
    return out


# ---- Criteo: the (field, key) count table -------------------------------------------------------------------------
def _criteo_run(d, out, cap):
    from tf_repos_b200.criteo_feature import preprocess
    os.makedirs(out, exist_ok=True)
    preprocess(d, out + "/", cutoff=1, table_capacity=cap)
    return _files(out)


def test_criteo_count_table_exactly_full(tmp_path):
    from tf_repos_b200.criteo_feature import CriteoFeatureError
    rng = np.random.default_rng(21)
    keys = 7                                                   # distinct values of every categorical column
    lines = []
    for r in range(300):
        ints = [str(int(v)) for v in rng.integers(0, 20, 13)]
        ints[0] = str(r % 20)                                  # no column is constant
        cats = ["%x" % ((f * 1000 + (r + f) % keys) * 2654435761 % (1 << 32)) for f in range(26)]
        lines.append("\t".join([str(r % 2)] + ints + cats))
    d = str(tmp_path) + "/"
    open(d + "train.txt", "w").write("\n".join(lines) + "\n")
    open(d + "test.txt", "w").write("\n".join(l.split("\t", 1)[1] for l in lines[:50]) + "\n")
    want = _criteo_run(d, d + "big", 1 << 16)
    assert _criteo_run(d, d + "full", 26 * keys) == want
    with pytest.raises(CriteoFeatureError, match=r"table_capacity=%d slots.*raise table_capacity" % (26 * keys - 1)):
        _criteo_run(d, d + "short", 26 * keys - 1)


# ---- Ali-CCP sample: the (field, fid) count table and the md5 table, which share table_capacity -------------------
def _aliccp_raw(d, commons, samples_of, tokens_of):
    """commons = md5s with a common record each; samples_of(set) = [(md5, [(field, fid)])] -> raw/{tr,te}/a.csv"""
    for name in ("tr", "te"):
        os.makedirs(os.path.join(d, name))
        lines = [b"%s,1,%s" % (m, tokens_of(m)) for m in commons[name]]
        for j, (m, toks) in enumerate(samples_of[name]):
            feats = b"\x01".join(b"%s\x02%d\x031.0" % t for t in toks)
            lines.append(b"%d,1,0,%s,%d,%s" % (j, m, len(toks), feats))
        with open(os.path.join(d, name, "a.csv"), "wb") as fh:
            fh.write(b"\n".join(lines) + b"\n")


def _aliccp_run(raw, out, cap):
    from tf_repos_b200 import aliccp_sample as gs
    gs.prepare(raw, out, cutoff=1, parts=3, chunk_bytes=4096, table_capacity=cap)
    return _files(out)


def _aliccp_boundary(raw, tmp_path, n_keys):
    from tf_repos_b200 import aliccp_sample as gs
    want = _aliccp_run(raw, str(tmp_path / "big"), 1 << 12)
    assert _aliccp_run(raw, str(tmp_path / "full"), n_keys) == want
    with pytest.raises(gs.AliccpSampleError, match="raise table_capacity"):
        _aliccp_run(raw, str(tmp_path / "short"), n_keys - 1)


def test_aliccp_md5_table_exactly_full(tmp_path):
    # 300 md5s in tr (each a common record and a sample), 40 in te; 2 (field, fid) keys
    md5 = lambda s, i: b"%s%015x" % (s, (i * 2654435761) % (1 << 60))
    commons = {"tr": [md5(b"t", i) for i in range(300)], "te": [md5(b"e", i) for i in range(40)]}
    samples = {k: [(m, [(b"206", 7)]) for m in v] for k, v in commons.items()}
    raw = str(tmp_path / "raw")
    _aliccp_raw(raw, commons, samples, lambda m: b"101\x025\x031.0")
    _aliccp_boundary(raw, tmp_path, 300)


def test_aliccp_count_table_exactly_full(tmp_path):
    # 3 md5s; tr's samples and the common records they join hold 120 + 90 distinct (field, fid) keys
    rng = np.random.default_rng(5)
    commons = {"tr": [b"m%d" % i for i in range(3)], "te": [b"m%d" % i for i in range(3)]}
    common_keys = {m: [(b"1%02d" % (i % 7), 1000 + 30 * i + k) for k in range(30)] for i, m in enumerate(commons["tr"])}
    fids = rng.permutation(1 << 20)[:120]
    samples = {"tr": [(commons["tr"][j % 3], [(b"206", int(f)) for f in fids[8 * j: 8 * j + 8]]) for j in range(15)],
               "te": [(b"m0", [(b"206", 1)])]}
    raw = str(tmp_path / "raw")
    _aliccp_raw(raw, commons, samples, lambda m: b"\x01".join(b"%s\x02%d\x031" % t for t in common_keys[m]))
    _aliccp_boundary(raw, tmp_path, 120 + 90)


# ---- smart: the feature_map table (table_capacity) and the builder's key table (build_capacity) -------------------
def _smart_csv(path, n, seed, vocab):
    rng = np.random.default_rng(seed)
    rows = []
    for _ in range(n):
        f = [b"1" if rng.random() < 0.3 else b"0"]
        for i in range(1, 128):
            f.append(b"%.4f" % rng.random() if 11 <= i <= 27 else b"v%d" % rng.integers(vocab))
        rows.append(b",".join(f))
    with open(path, "wb") as fh:
        fh.write(b"\n".join(rows) + b"\n")


def test_smart_map_table_exactly_full(tmp_path):
    from tf_repos_b200.smart_feature import CSV_COLUMNS, SmartFeatureError, smart_feature
    d = str(tmp_path) + "/"
    _smart_csv(d + "x.verify", 200, 3, vocab=6)
    # one line per key, no key twice: the UNK key and 4 of the 6 values of every categorical column, the continuous
    # names but the first two
    keys = [b"%s|%s" % (CSV_COLUMNS[i], v) for i in range(1, 128) if not 11 <= i <= 27
            for v in [b"UNK", b"v0", b"v2", b"v3", b"v5"]] + [CSV_COLUMNS[i] for i in range(13, 28)]
    open(d + "feature_map", "wb").write(b"".join(b"%s %d\n" % (k, j + 1) for j, k in enumerate(keys)))

    def run(cap):
        g = smart_feature(d, d, "va", table_capacity=cap)
        return g["map_keys"], open(d + "va.libsvm", "rb").read()

    n_keys, want = run(1 << 12)
    assert n_keys == len(keys)
    assert run(n_keys) == (n_keys, want)
    os.remove(d + "va.libsvm")
    with pytest.raises(SmartFeatureError, match="table_capacity=%d slots" % (n_keys - 1)):
        run(n_keys - 1)
    assert not os.path.exists(d + "va.libsvm")


def test_smart_builder_table_exactly_full(tmp_path):
    from tf_repos_b200.smart_feature import SmartFeatureError, smart_feature
    d = str(tmp_path) + "/"
    _smart_csv(d + "a_part_0", 300, 4, vocab=5)
    _smart_csv(d + "x.verify", 20, 6, vocab=5)
    # the builder keys columns 1 .. len - 2 (here 1..126) but the continuous ones: 109 columns of 5 values each
    n_keys = sum(1 for i in range(1, 127) if not 11 <= i <= 27) * 5

    def run(cap):
        smart_feature(d, d, "va", build_feature_map_first=True, build_capacity=cap)
        return open(d + "feature_map", "rb").read(), open(d + "va.libsvm", "rb").read()

    want = run(1 << 12)
    assert want[0].count(b"\n") == 128 + 17 + n_keys            # name|UNK lines, the continuous names, the keys
    assert run(n_keys) == want
    for p in ("feature_map", "va.libsvm"):
        os.remove(d + p)
    with pytest.raises(SmartFeatureError, match="build_capacity=%d slots" % (n_keys - 1)):
        run(n_keys - 1)
    assert not os.path.exists(d + "feature_map")
