"""The GPU Ali-CCP sample stage (tf_repos_b200.aliccp_sample) against oracle/aliccp_sample.py: every part file and
feat_cnts byte for byte at several chunk sizes, part counts and pass-B groupings, the returned stats, determinism, every
restriction and capacity error, the drop-in's flags and layout, and the whole chain raw CSVs -> part files ->
TFRecords -> DeepCvrMTL.py / DIN.py."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import aliccp_sample as oa

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

COMMON = [b"101", b"121", b"122", b"124", b"125", b"126", b"127", b"128", b"129", b"205", b"301"]
USER = [b"109_14", b"110_14", b"127_14", b"150_14"]
AD = [b"206", b"207", b"210", b"216"]
FIELDS = COMMON + USER + AD + [b"508", b"853", b"abcdefghijklmnop", b"x"]


def _feats(toks):
    return b"\x01".join(b"%s\x02%s\x03%s" % t for t in toks)


def _tok(rng, fields, hot):
    fid = rng.randint(hot) if rng.rand() < 0.8 else rng.randint(1 << 40)
    return (fields[rng.randint(len(fields))], b"%d" % fid, [b"1.0", b"0.693147", b"", b"2.5e-3"][rng.randint(4)])


def _raw(rng, n_common, n_sample, hot=60, junk=True):
    """Raw lines: common records (some md5s repeated), samples (some without a record, some y=0/z=1), and, with junk,
    every line class the mapper skips."""
    md5s = [b"%016x" % rng.randint(1 << 62) for _ in range(n_common)]
    lines = []
    for m in md5s:
        lines.append((m, b"%d" % 3, _feats([_tok(rng, COMMON + USER, hot) for _ in range(rng.randint(1, 40))])))
        if rng.rand() < 0.1:   # a later record for the same md5
            lines.append((m, b"1", _feats([_tok(rng, COMMON, hot)])))
    lines = [b",".join(x) for x in lines]
    for j in range(n_sample):
        md5 = md5s[rng.randint(len(md5s))] if rng.rand() < 0.9 else b"nomatch%d" % j
        y, z = [(b"1", b"1"), (b"1", b"0"), (b"0", b"0"), (b"0", b"1")][rng.randint(4)]
        toks = [_tok(rng, AD + FIELDS[-4:], hot) for _ in range(rng.randint(1, 8))]
        lines.append(b"%d,%s,%s,%s,%d,%s" % (j, y, z, md5, len(toks), _feats(toks)))
    if junk:
        lines += [b"", b"  ", b"a,b", b"1,1,0,m,2,3,4", b"m,1,101\x025", b"m,1,101\x025\x031\x036", b"m,1,",
                  b"1,1,0,m,1,101\x02\x025\x031", b"9,0,1,m,1,bad\x00"]
    order = rng.permutation(len(lines))
    out = [lines[i] for i in order]
    for i in range(0, len(out), 7):
        out[i] = b" " + out[i] + b"\r"    # strip() removes both
    return out


def _write(path, lines, last_newline=True):
    with open(path, "wb") as fh:
        fh.write(b"\n".join(lines) + (b"\n" if last_newline else b""))


def _dataset(tmp_path, seed=0, n_common=40, n_sample=1500, hot=60):
    rng = np.random.RandomState(seed)
    d = tmp_path / "raw"
    for name in ("tr", "te"):
        (d / name).mkdir(parents=True)
        lines = _raw(rng, n_common, n_sample if name == "tr" else n_sample // 3, hot)
        cut = len(lines) // 2
        # two files per set, read in name order; the second without a final newline
        _write(str(d / name / "sample_skeleton.csv"), lines[cut:], last_newline=False)
        _write(str(d / name / "common_features.csv"), lines[:cut])
    return str(d)


def _read_out(d, parts):
    files = {"feat_cnts": open(os.path.join(d, "feat_cnts"), "rb").read()}
    for name in ("tr", "te"):
        assert sorted(os.listdir(os.path.join(d, name))) == ["part-%05d" % p for p in range(parts)]
        for p in range(parts):
            files["%s/%d" % (name, p)] = open(os.path.join(d, name, "part-%05d" % p), "rb").read()
    return files


_ORACLE = {}


def _oracle(tmp_path_factory, raw, parts, seed=0, cutoff=20):
    key = (raw, parts, seed, cutoff)
    if key not in _ORACLE:
        out = str(tmp_path_factory.mktemp("oracle"))
        stats = oa.prepare(raw, out, cutoff=cutoff, parts=parts, seed=seed)
        _ORACLE[key] = (_read_out(out, parts), stats)
    return _ORACLE[key]


def _strip(stats):
    return {k: v for k, v in stats.items() if k != "device_ms"}


@pytest.fixture(scope="module")
def raw(tmp_path_factory):
    return _dataset(tmp_path_factory.mktemp("ds"))


@pytest.mark.parametrize("chunk_bytes", [37, 4096, 1 << 20])
@pytest.mark.parametrize("parts", [1, 7, 100])
def test_byte_identity_with_the_oracle(tmp_path, tmp_path_factory, raw, chunk_bytes, parts):
    from tf_repos_b200 import aliccp_sample as gs
    want, want_stats = _oracle(tmp_path_factory, raw, parts)
    out = str(tmp_path / "a" / "b")          # made, with tr/ and te/, when missing
    stats = gs.prepare(raw, out, parts=parts, chunk_bytes=chunk_bytes, table_capacity=1 << 14)
    got = _read_out(out, parts)
    assert got.keys() == want.keys()
    for k in want:
        assert got[k] == want[k], k
    assert _strip(stats) == want_stats
    assert want_stats["tr"]["filtered"] and want_stats["tr"]["malformed"] and want_stats["tr"]["no_common"]
    assert want_stats["tr"]["commons_superseded"] and want_stats["tr"]["empty_lines"]


def test_budget_forces_several_groups(tmp_path, tmp_path_factory, raw):
    from tf_repos_b200 import aliccp_sample as gs
    want, want_stats = _oracle(tmp_path_factory, raw, 7)
    biggest = max(len(v) for k, v in want.items() if k != "feat_cnts")
    total = sum(len(v) for k, v in want.items() if k.startswith("tr/"))
    # the resident records and summaries of a set: feat_list bytes + 16 B per record + 12 B per sample
    resident = 0
    for name in ("tr", "te"):
        d = os.path.join(raw, name)
        lines = [l for f in sorted(os.listdir(d)) for l in oa.lines_of(open(os.path.join(d, f), "rb").read())]
        m = [oa.join_map(l) for l in lines]
        resident = max(resident, sum(len(l.strip().split(b",")[2]) + 16 for l, x in zip(lines, m) if x[0] == "common")
                       + 12 * sum(x[0] == "sample" for x in m))
    budget = max(biggest, resident) + 1
    assert total > 3 * budget          # at least four groups for tr
    out = str(tmp_path / "o")
    stats = gs.prepare(raw, out, parts=7, chunk_bytes=1000, table_capacity=1 << 14, budget_bytes=budget)
    got = _read_out(out, 7)
    for k in want:
        assert got[k] == want[k], k
    assert _strip(stats) == want_stats
    # the same budget holds every set's records, but not tr's single part
    out = tmp_path / "one"
    with pytest.raises(gs.AliccpSampleError, match="part 0 .* raise budget_bytes"):
        gs.prepare(raw, str(out), parts=1, chunk_bytes=1000, table_capacity=1 << 14, budget_bytes=budget)
    assert os.listdir(out / "tr") == [] and not os.path.exists(out / "feat_cnts")


def test_two_runs_identical_and_seed_changes_only_the_order(tmp_path, raw):
    from tf_repos_b200 import aliccp_sample as gs
    runs = []
    for i, seed in enumerate([5, 5, 6]):
        out = str(tmp_path / str(i))
        gs.prepare(raw, out, parts=7, seed=seed, chunk_bytes=8192, table_capacity=1 << 14)
        runs.append(_read_out(out, 7))
    assert runs[0] == runs[1]
    for name in ("tr", "te"):
        def lines(r):
            return sorted(l.split(b"\t", 1)[1] for k, v in r.items() if k.startswith(name + "/") for l in v.splitlines())
        assert lines(runs[0]) == lines(runs[2])
        assert [runs[0][k] for k in runs[0] if k.startswith(name)] != [runs[2][k] for k in runs[2] if k.startswith(name)]
    assert runs[0]["feat_cnts"] == runs[2]["feat_cnts"]


BAD = [
    (b"7,1,0,m1,1,101\x025\x031\x00", b"7,1,0,m1,1,101\x025\x031\x00"),
    (b"7,1,0,m 1,1,101\x025\x031", b"m 1"),
    (b"7,1 ,0,m1,1,101\x025\x031", b"1 "),
    (b"s:7,1,0,m1,1,101\x025\x031", b"s:7"),
    (b"7,1,0,,1,101\x025\x031", b""),
    (b"m" * 65 + b",1,101\x025\x031", b"m" * 65),
    (b"m1,1,101\x025\x031\x01\x025\x031", b""),
    (b"m1,1,abcdefghijklmnopq\x025\x031", b"abcdefghijklmnopq"),
    (b"m1,1,1\x030\x025\x031", b"1\x030"),
    (b"m1,1,101\x0205\x031", b"05"),
    (b"m1,1,101\x029223372036854775808\x031", b"9223372036854775808"),
    (b"m1,1,101\x025\x031:2", b"1:2"),
    (b"m1,1,101\x025\x031\x0cx", b"1\x0cx"),
]


@pytest.mark.parametrize("bad, token", BAD)
@pytest.mark.parametrize("where", ["tr", "te"])
def test_restrictions_raise_with_line_and_token_and_remove_the_set(tmp_path, bad, token, where):
    from tf_repos_b200 import aliccp_sample as gs
    rng = np.random.RandomState(3)
    d = tmp_path / "raw"
    for name in ("tr", "te"):
        (d / name).mkdir(parents=True)
        lines = _raw(rng, 5, 60, junk=False)
        if name == where:
            lines.insert(41, bad)
            lines.insert(50, bad)
        _write(str(d / name / "a.csv"), lines)
    out = tmp_path / "out"
    with pytest.raises(gs.AliccpSampleError) as e:
        gs.prepare(str(d), str(out), parts=3, chunk_bytes=300, table_capacity=1 << 12)
    msg = str(e.value)
    assert msg.startswith("%s: line 42: " % (d / where / "a.csv")) and msg.endswith(repr(token)), msg
    with pytest.raises(oa.OracleError) as o:
        oa.prepare(str(d), str(tmp_path / "oracle"), parts=3)
    assert o.value.line == 42 and o.value.token == token
    assert os.listdir(out / where) == []
    assert sorted(os.listdir(out / "tr")) == ([] if where == "tr" else ["part-00000", "part-00001", "part-00002"])
    assert os.path.exists(out / "feat_cnts") == (where == "te")


def test_capacities_raise_before_any_part_file(tmp_path):
    from tf_repos_b200 import aliccp_sample as gs
    raw = _dataset(tmp_path, seed=4, n_common=30, n_sample=600, hot=500)
    for kw, param in ((dict(table_capacity=64), "table_capacity"), (dict(table_capacity=600), "table_capacity"),
                      (dict(budget_bytes=2000), "budget_bytes")):
        out = tmp_path / ("out_" + param + str(len(os.listdir(tmp_path))))
        with pytest.raises(gs.AliccpSampleError, match="raise " + param):
            gs.prepare(raw, str(out), parts=5, chunk_bytes=4096, **kw)
        assert os.listdir(out / "tr") == [] and not os.path.exists(out / "feat_cnts")


def _run(args, cwd=ROOT):
    r = subprocess.run([sys.executable] + args, capture_output=True, text=True, timeout=280, cwd=cwd)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout


def test_script_flags_layout_and_mkdir(tmp_path, tmp_path_factory, raw):
    want, stats = _oracle(tmp_path_factory, raw, 3, seed=9, cutoff=5)
    out = tmp_path / "new" / "dir"
    stdout = _run([os.path.join(ROOT, "Feature_pipeline", "get_aliccp_sample.py"), "--input_dir=" + raw,
                   "--output_dir=%s" % out, "--cutoff=5", "--parts=3", "--seed=9"])
    assert stdout.strip().splitlines()[-1] == "feature_size %d  (train with --feature_size=%d)" % (
        stats["feature_size"], stats["feature_size"])
    assert sorted(os.listdir(out)) == ["feat_cnts", "te", "tr"]
    assert _read_out(str(out), 3) == want


def _e2e_raw(d, rng):
    """Ali-CCP-shaped raw lines every sample of which keeps features at cutoff 20."""
    for name, n in (("tr", 400), ("te", 150)):
        (d / name).mkdir(parents=True)
        md5s = [b"%032x" % rng.randint(1 << 62) for _ in range(12)]
        commons = [b"%s,1,%s" % (m, _feats([(f, b"%d" % rng.randint(20), b"1.0") for f in COMMON[:9]] +
                                           [(f, b"%d" % rng.randint(8), b"0.5") for f in USER for _ in range(2)]))
                   for m in md5s]
        samples = []
        for j in range(n):
            toks = [(f, b"%d" % rng.randint(25), b"1") for f in AD] + [(b"301", b"%d" % rng.randint(3), b"1"),
                                                                       (b"205", b"%d" % rng.randint(40), b"1")]
            samples.append(b"%d,%d,%d,%s,6,%s" % (j, rng.randint(2), rng.randint(2), md5s[rng.randint(12)],
                                                   _feats(toks)))
        _write(str(d / name / "sample_skeleton.csv"), samples)
        _write(str(d / name / "common_features.csv"), commons)


@pytest.mark.parametrize("script, extra", [
    ("DIN.py", ["--deep_layers=16,8", "--dropout=1,1", "--attention_layers=16"]),
    ("DeepCvrMTL.py", ["--deep_layers=16,8", "--dropout=1,1", "--ctr_task_wgt=0.3"]),
])
def test_raw_csvs_to_trained_models(tmp_path, script, extra):
    from oracle import aliccp_tfrecord as ot
    from tests.test_gpu_tfrecord_cli import REFERENCE
    tmp = str(tmp_path)
    _e2e_raw(tmp_path / "raw", np.random.RandomState(21))
    stdout = _run([os.path.join(ROOT, "Feature_pipeline", "get_aliccp_sample.py"), "--input_dir=%s/raw" % tmp,
                   "--output_dir=%s/sample" % tmp, "--parts=1"])
    feature_size = int(stdout.strip().splitlines()[-1].split()[1])
    os.makedirs(tmp + "/data")
    for part in ("tr", "te"):
        _run([os.path.join(ROOT, "Feature_pipeline", "get_aliccp_tfrecord.py"), "--input_dir=%s/sample/%s" % (tmp, part),
              "--output_dir=%s/data/%s" % (tmp, part)])
    # the oracle's chain: part files -> TFRecords -> host batches in-process
    st = oa.prepare(tmp + "/raw", tmp + "/osample", parts=1)
    assert st["feature_size"] == feature_size and st["tr"]["empty_lines"] == st["te"]["empty_lines"] == 0
    os.makedirs(tmp + "/odata")
    for part in ("tr", "te"):
        ot.convert(tmp + "/osample/" + part, tmp + "/odata/" + part)
    flags = ["--field_size=11", "--feature_size=%d" % feature_size, "--embedding_size=8", "--batch_size=32",
             "--num_epochs=2", "--log_steps=1000", "--data_dir=" + tmp + "/data", "--model_dir=" + tmp + "/ckpt/m_",
             "--dt_dir=20261016"] + extra
    script_path = os.path.join(ROOT, "Model_pipeline", script)
    _run([script_path, "--task_type=train"] + flags)
    _run([script_path, "--task_type=infer"] + flags)
    os.makedirs(tmp + "/ref")
    _run(["-c", REFERENCE, ROOT, script, tmp + "/odata/tr/part-00000.tfrecord", tmp + "/odata/te/part-00000.tfrecord",
          tmp + "/ref"] + flags)
    got = torch.load(tmp + "/ckpt/m_20261016/ctr_b200.ckpt", map_location="cpu")
    want = torch.load(tmp + "/ref/ctr_b200.ckpt", map_location="cpu")
    assert got["global_step"] == want["global_step"] > 0
    for k in want["variables"]:
        assert torch.equal(got["variables"][k], want["variables"][k]), k
    pred = open(tmp + "/data/pred.txt").read()
    assert pred.count("\n") == st["te"]["samples"] and pred == open(tmp + "/ref/pred.txt").read()
