"""The GPU Criteo feature pipeline (csrc/criteo_feature.cu through tf_repos_b200/criteo_feature.py) against the CPU
restatement oracle/criteo_feature.py: tr/va/te.libsvm byte for byte, feature_map as a set of lines, on seeded raw
data built to hit the hard cases (Zipf keys with count ties, empties in every column, negative ints, ints above the
clip, denominators that make %.6f rounding ties); chunking; every error the reference raises and every restriction;
the table-capacity check; and the drop-in script's output training DeepFM."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CLIP = np.array([20, 600, 100, 50, 64000, 500, 100, 50, 500, 10, 10, 10, 50])
# max - min of each integer column over train: powers of two (and 5 * 128) put k/den on exact %.6f ties; 1 and 3 give
# integer and repeating results
DEN = np.array([128, 64, 1, 640, 256, 3, 1024, 2, 200, 10, 8, 5, 32])
LO = CLIP - DEN
VOCAB = [4, 100, 100_000, 3000, 50, 20_000, 7, 100_000, 1000, 10, 5000, 100_000, 300,
         2, 100_000, 40, 800, 100_000, 12, 60_000, 9, 100_000, 250, 100_000, 30, 100_000]
_INT_BASE = -2000
_INT_TOKENS = np.char.mod("%d", np.arange(_INT_BASE, 66_000)).astype("S6")
_SPECIAL = np.array([b"-0", b"+3", b"007", b"-00"], dtype="S6")


def _key_tokens(f, v):
    idx = np.arange(v, dtype=np.uint64)
    if f % 5 == 4:                                               # short keys: 1..5 bytes
        return np.char.mod("%x", idx).astype("S8")
    h = (idx * np.uint64(2654435761) + np.uint64(40503 * (f + 1))) % np.uint64(1 << 32)
    return np.char.mod("%08x", h).astype("S8")


_KEYS = None


def write_raw(path, n, seed, test=False, final_newline=True, block=250_000, zipf=1.25):
    """n seeded raw Criteo lines (train: label, I1..I13, C1..C26; test: no label) -> path.  Vectorised: every token is
    a fixed-width NUL-padded byte row, the padding is dropped at the end."""
    global _KEYS
    if _KEYS is None:
        _KEYS = [_key_tokens(f, v) for f, v in enumerate(VOCAB)]
    rng = np.random.default_rng(seed)
    with open(path, "wb") as fh:
        for b0 in range(0, n, block):
            nb = min(block, n - b0)
            cols = []
            if not test:
                cols.append(np.where(rng.random(nb) < 0.25, b"1", b"0").astype("S1"))
            hi = CLIP + (500 if test else 30)
            lo = LO - (60 if test else 0)
            for i in range(13):
                v = rng.integers(lo[i], hi[i] + 1, nb)
                if b0 == 0 and not test:
                    v[0], v[1] = LO[i], CLIP[i] + 7                # min and (clipped) max of every column
                tok = _INT_TOKENS[v - _INT_BASE]
                tok[rng.random(nb) < 0.08] = b""
                if test:
                    sp = rng.random(nb) < 0.01
                    tok[sp] = _SPECIAL[rng.integers(0, len(_SPECIAL), int(sp.sum()))]
                if b0 == 0 and not test:
                    tok[:2] = _INT_TOKENS[v[:2] - _INT_BASE]
                cols.append(tok)
            for f in range(26):
                k = (rng.zipf(zipf, nb) - 1) % VOCAB[f]
                tok = _KEYS[f][k]
                tok[rng.random(nb) < 0.04] = b""
                cols.append(tok)
            parts = []
            for j, c in enumerate(cols):
                parts.append(c.view(np.uint8).reshape(nb, -1))
                parts.append(np.full((nb, 1), ord("\t" if j < len(cols) - 1 else "\n"), np.uint8))
            arr = np.concatenate(parts, axis=1)
            data = arr[arr != 0].tobytes()
            if not final_newline and b0 + nb == n:
                data = data[:-1]
            fh.write(data)


def _dataset(tmp_path, n_train, n_test, seed=0, final_newline=True):
    d = str(tmp_path) + "/"
    write_raw(d + "train.txt", n_train, seed)
    write_raw(d + "test.txt", n_test, seed + 1, test=True, final_newline=final_newline)
    return d


def _outputs(d):
    rd = lambda n: open(d + n, "rb").read()
    return rd("tr.libsvm"), rd("va.libsvm"), rd("te.libsvm"), sorted(rd("feature_map").splitlines())


def _oracle(d, cutoff):
    from oracle import criteo_feature as ocf
    o = d + "oracle_"
    info = ocf.preprocess(d, o, cutoff=cutoff)
    return info, _outputs(o)


def _gpu(d, cutoff, **kw):
    from tf_repos_b200.criteo_feature import preprocess
    out = d + "gpu_"
    info = preprocess(d, out, cutoff=cutoff, **kw)
    return info, _outputs(out)


@pytest.fixture(scope="module")
def data50k(tmp_path_factory):
    return _dataset(tmp_path_factory.mktemp("criteo50k"), 50_000, 5_000)


@pytest.mark.parametrize("cutoff", [1, 20, 200])
def test_byte_identical_to_oracle(data50k, cutoff):
    ref_info, ref = _oracle(data50k, cutoff)
    info, got = _gpu(data50k, cutoff)
    for name, a, b in zip(("tr.libsvm", "va.libsvm", "te.libsvm", "feature_map"), got, ref):
        assert a == b, f"{name} differs (cutoff={cutoff})"
    assert info["dict_sizes"] == ref_info["dict_sizes"] and info["feature_size"] == ref_info["feature_size"]
    assert info["lines"] == ref_info["lines"] and info["min"] == ref_info["min"] and info["max"] == ref_info["max"]
    # the data reaches what it is meant to: ties, values above 1 and below 0, -0, empties
    tr, te = got[0], got[2]
    assert b"1:0.007812 " in tr and b"1:0.023438 " in tr                  # k/128 ties, to even
    assert b" 10:-0 " in te and b":-0." in te                              # "-0" input; negative results
    te_vals = [float(t.split(b":")[1]) for l in te.splitlines()[:500] for t in l.split()[1:14]]
    assert max(te_vals) > 1 and min(te_vals) < 0 and b" 3:1 " in tr and b" 3:0 " in tr
    # a second run gives the same bytes
    assert _gpu(data50k, cutoff)[1] == got


@pytest.mark.parametrize("final_newline", [True, False])
def test_chunk_independence(tmp_path, final_newline):
    d = _dataset(tmp_path, 3000, 700, seed=5, final_newline=final_newline)
    _, ref = _oracle(d, 3)
    for chunk in (4096, 4093, 64 << 20):
        _, got = _gpu(d, 3, chunk_bytes=chunk)
        assert got == ref, chunk


def _train_lines(n=40, seed=9):
    from oracle.criteo_feature import CONTINUOUS_CLIP
    rng = np.random.default_rng(seed)
    lines = []
    for r in range(n):
        ints = [str(int(rng.integers(-5, c + 3))) for c in CONTINUOUS_CLIP]
        cats = ["%08x" % int(rng.integers(0, 3)) for _ in range(26)]
        lines.append(["1" if r % 3 == 0 else "0"] + ints + cats)
    return lines


def _run_lines(tmp_path, train, test=None, cutoff=1, **kw):
    from tf_repos_b200.criteo_feature import preprocess
    d = str(tmp_path) + "/"
    open(d + "train.txt", "wb").write(b"".join(b"\t".join(c.encode() if isinstance(c, str) else c for c in l) + b"\n"
                                             for l in train))
    test = test if test is not None else [l[1:] for l in _train_lines(5, 3)]
    open(d + "test.txt", "wb").write(b"".join(b"\t".join(c.encode() if isinstance(c, str) else c for c in l) + b"\n"
                                            for l in test))
    return preprocess(d, d, cutoff=cutoff, **kw)


def _expect(tmp_path, train, match, test=None, cutoff=1, **kw):
    from tf_repos_b200.criteo_feature import CriteoFeatureError
    with pytest.raises(CriteoFeatureError, match=match):
        _run_lines(tmp_path, train, test, cutoff, **kw)


def test_errors_name_file_line_and_column(tmp_path):
    L = _train_lines()
    bad = [l[:] for l in L]; bad[6] = bad[6][:21]                 # IndexError in the dictionary pass
    _expect(tmp_path, bad, r"train\.txt: line 7, column 21 \(C8\): too few columns")
    bad[30] = bad[30][:5]                                          # ... but the min/max pass fails first, later
    _expect(tmp_path, bad, r"train\.txt: line 31, column 5 \(I5\): too few columns")
    bad = [l[:] for l in L]; bad[3][2] = "1.5"
    _expect(tmp_path, bad, r"line 4, column 2 \(I2\): not an integer")
    bad = [l[:] for l in L]; bad[3][2] = " 7"
    _expect(tmp_path, bad, r"line 4, column 2 \(I2\): not an integer")
    bad = [l[:] for l in L]; bad[12][4] = "9007199254740993"
    _expect(tmp_path, bad, r"line 13, column 4 \(I4\): integer magnitude above 2\^53")
    bad = [l[:] for l in L]
    for l in bad:
        l[5] = "7"                                                  # I5 constant: max == min
    bad[0][5] = ""
    _expect(tmp_path, bad, r"train\.txt: line 2, column 5 \(I5\): max == min")
    bad = [l[:] for l in L]; bad[8][20] = "123456789"
    _expect(tmp_path, bad, r"line 9, column 20 \(C7\): categorical value longer than 8 bytes")
    bad = [l[:] for l in L]; bad[8][20] = b"ab\x00c"
    _expect(tmp_path, bad, r"line 9, column 20 \(C7\): categorical value contains a NUL")
    bad = [l[:] for l in L]; bad[9][39] = "<unk>"
    _expect(tmp_path, bad, r"line 10, column 39 \(C26\): categorical value is the literal <unk>")
    _expect(tmp_path, L, r"column C1: no value occurs at least cutoff=1000 times", cutoff=1000)
    te = [l[1:] for l in _train_lines(6, 4)]
    te[4] = te[4][:30]
    _expect(tmp_path, L, r"test\.txt: line 5, column 30 \(C18\): too few columns", test=te)
    te = [l[1:] for l in _train_lines(6, 4)]
    te[2][0] = "1e3"
    _expect(tmp_path, L, r"test\.txt: line 3, column 0 \(I1\): not an integer", test=te)
    # accepted at the edge of the restrictions: 2^53, 8-byte keys, and 41+ columns
    ok = [l[:] for l in L]; ok[0][4] = "-9007199254740992"; ok[1][20] = "ffffffff"; ok[2] = ok[2] + ["extra"]
    _run_lines(tmp_path, ok)


def test_too_small_table_raises_before_writing(tmp_path):
    _expect(tmp_path, _train_lines(), r"table_capacity=8 slots.*raise table_capacity", table_capacity=8)
    assert not os.path.exists(str(tmp_path) + "/tr.libsvm")
    info = _run_lines(tmp_path, _train_lines(), table_capacity=26 * 3)   # exactly full still works
    assert info["dict_sizes"] == [4] * 26


def test_script_output_trains_deepfm(tmp_path):
    d = _dataset(tmp_path, 6000, 700, seed=11)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "Feature_pipeline", "get_criteo_feature.py"), "--threads=4",
                        "--input_dir=" + d, "--output_dir=" + d, "--cutoff=20"], capture_output=True, text=True,
                       timeout=280)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    out = r.stdout.strip().splitlines()
    assert out[:4] == ["threads  4", "input_dir  " + d, "output_dir  " + d, "cutoff  20"]
    fs = int(out[-1].split("--feature_size=")[1].rstrip(")"))
    ids = [int(t.split(b":")[0]) for l in open(d + "tr.libsvm", "rb").read().splitlines() for t in l.split()[1:]]
    assert max(ids) < fs and min(ids) >= 1
    common = [sys.executable, os.path.join(ROOT, "Model_pipeline", "DeepFM.py"), "--field_size=39",
              f"--feature_size={fs}", "--embedding_size=8", "--batch_size=256", "--deep_layers=32,16",
              "--dropout=0.8,0.8", "--log_steps=5", "--num_epochs=1", "--data_dir=" + d, "--model_dir=" + d + "ckpt/m_",
              "--dt_dir=1"]
    for task in ("train", "infer"):
        r = subprocess.run(common + ["--task_type=" + task], capture_output=True, text=True, timeout=280)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    n_te = len(open(d + "te.libsvm", "rb").read().splitlines())
    assert n_te == 700 and len(open(d + "pred.txt").read().splitlines()) == n_te
