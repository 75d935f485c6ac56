"""The GPU smart and Frappe feature stages (csrc/smart_feature.cu through tf_repos_b200/smart_feature.py) against the
CPU restatement oracle/smart_feature.py, byte for byte, on seeded data with every edge case of DESIGN.md §2.12 mixed
in; chunking down to one line a piece; the table-capacity check; the builder; run-to-run identity; the drop-in scripts;
and their outputs training DeepFM."""
import glob
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from oracle import smart_feature as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_ODD = [b"", b"UNK", b"a b", b"\xff\xfe", b"|", b"x|y", b" pad", b"tab\t", b"\x1c"]


def _line(rng, vocab=12, odd=True):
    f = [b"1" if rng.random() < 0.3 else b"0"]
    for i in range(1, 128):
        if O.continuous(i):
            f.append(b"" if odd and rng.random() < 0.05 else b"%.5f" % rng.random())
        elif odd and rng.random() < 0.05:
            f.append(_ODD[rng.integers(len(_ODD))])
        else:
            f.append(b"v%d" % rng.zipf(1.6) if i < 11 else b"%d" % rng.integers(vocab))
    return b",".join(f)


def write_csv(path, n, seed, edge=True):
    """n seeded 128-column lines; with edge, the rule-breaking lines of DESIGN.md §2.12 are mixed in."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        ln = _line(rng, odd=edge)
        if edge and k % 50 == 7:
            case = (k // 50) % 9
            ln = [b"", b"0", b"1,v1", ln + b",extra,more",                      # 130 fields: dropped
                  ln + b",extra", b"  " + ln + b"\r", b"\t" + ln + b" \x0b\x0c", # 129 fields, CRLF, edge whitespace
                  b",".join(ln.split(b",")[:40]), b"\x1c" + ln][case]
        out.append(ln)
    text = b"\n".join(out) + (b"" if edge else b"\n")                           # edge: no final newline
    with open(path, "wb") as fh:
        fh.write(text)


def _map_with_edges(tr_files):
    """The builder's map, then the load rules: a repeated key (the later line wins), a one-token line, an empty fid,
    a non-numeric fid, keys no lookup can reach, and a few continuous names and UNK keys removed (None / fallback)."""
    lines = O.feature_map_text(tr_files).splitlines()
    drop = {b"u_ctr", b"c_q_t_sim", b"u_de|UNK", b"xgbf_3|UNK"}
    lines = [l for l in lines if l.split(b" ")[0] not in drop]
    lines += [b"u_pl|v1 999", b"u_pl|v2", b"u_pl|v3  7", b"u_os|v1 abc", b"is_click|1 5", b"u_ctr|x 6",
              b"u_pl 8", b"nope|v1 9", b"  c_h|v1 77  \r", b"", b"xgbf_07|1 3"]
    return b"\n".join(lines)                                                    # no final newline


def _dataset(tmp_path, monkeypatch, n=4000, seed=0):
    """in_d/ under tmp_path, which becomes the current directory (relative paths keep the '_' pieces of the tr names
    known): two tr inputs, two va inputs and a test input."""
    monkeypatch.chdir(tmp_path)
    d = "in_d/"             # 'in_d//a_part_0'.rsplit('_') = ['in', 'd//a', 'part', '0']: tr_0.libsvm
    os.makedirs(d)
    write_csv(d + "a_part_0", n, seed)
    write_csv(d + "a_part_1", n // 3, seed + 1)
    write_csv(d + "x.verify", n // 4, seed + 2)
    write_csv(d + "w.verify", 100, seed + 3)
    write_csv(d + "z.test", n // 5, seed + 4)
    return d


def _run_both(d, task, build=False, **kw):
    from tf_repos_b200.smart_feature import smart_feature
    go, oo = d + "gpu/", d + "ora/"
    for o in (go, oo):
        os.makedirs(o, exist_ok=True)
    if not build:
        fmap = _map_with_edges(sorted(glob.glob(d + "/*part*")))
        for o in (go, oo):
            open(o + "feature_map", "wb").write(fmap)
    g = smart_feature(d, go, task, build_feature_map_first=build, **kw)
    r = O.smart_feature(d, oo, task, build=build)
    assert [os.path.basename(p) for p in g["outputs"]] == [os.path.basename(p) for p in r["outputs"]]
    assert g["outputs"], "no output"
    for a, b in zip(g["outputs"], r["outputs"]):
        assert open(a, "rb").read() == open(b, "rb").read(), a
        assert g["lines"][a] == r["lines"][b]
    return g


@pytest.mark.parametrize("task", ["tr", "va", "te"])
def test_emit_matches_oracle(tmp_path, monkeypatch, task):
    d = _dataset(tmp_path, monkeypatch)
    g = _run_both(d, task)
    names = {"tr": ["tr_0.libsvm", "tr_1.libsvm"], "va": ["va.libsvm"], "te": ["te.libsvm"]}[task]
    assert [os.path.basename(p) for p in g["outputs"]] == names
    out = open(g["outputs"][0], "rb").read()
    assert b" None:" in out and b"\n \n" in out and b"\n0 \n" in out     # absent fids, an empty and a short line
    n_in, n_out = g["lines"][g["outputs"][0]]
    assert n_out < n_in                                                  # the 130-field lines are dropped


@pytest.mark.parametrize("chunk_bytes", [1, 997, 1 << 16])
def test_chunk_sizes(tmp_path, monkeypatch, chunk_bytes):
    d = _dataset(tmp_path, monkeypatch, n=600 if chunk_bytes == 1 else 3000, seed=5)
    _run_both(d, "va", chunk_bytes=chunk_bytes)


def test_small_table_raises_and_writes_nothing(tmp_path, monkeypatch):
    from tf_repos_b200.smart_feature import SmartFeatureError, smart_feature
    d = _dataset(tmp_path, monkeypatch, n=500)
    open(d + "feature_map", "wb").write(_map_with_edges(sorted(glob.glob(d + "/*part*"))))
    with pytest.raises(SmartFeatureError, match="table_capacity"):
        smart_feature(d, d, "va", table_capacity=16)
    assert not os.path.exists(d + "va.libsvm")
    os.remove(d + "feature_map")
    with pytest.raises(FileNotFoundError):
        smart_feature(d, d, "va")
    assert not os.path.exists(d + "va.libsvm")


def test_builder_parity_and_build_then_emit(tmp_path, monkeypatch):
    d = _dataset(tmp_path, monkeypatch, n=3000, seed=9)
    g = _run_both(d, "tr", build=True, chunk_bytes=50_000)
    built = open(d + "gpu/feature_map", "rb").read()
    assert built == open(d + "ora/feature_map", "rb").read()       # both in fid order
    assert g["device_ms"]["build"] > 0


def test_builder_capacity_checks(tmp_path, monkeypatch):
    from tf_repos_b200.smart_feature import SmartFeatureError, smart_feature
    d = _dataset(tmp_path, monkeypatch, n=400)
    with pytest.raises(SmartFeatureError, match="build_capacity"):
        smart_feature(d, d, "tr", build_feature_map_first=True, build_capacity=64)
    with pytest.raises(SmartFeatureError, match="build_arena_bytes"):
        smart_feature(d, d, "tr", build_feature_map_first=True, build_arena_bytes=64)
    assert not os.path.exists(d + "feature_map")


def test_two_runs_give_identical_bytes(tmp_path, monkeypatch):
    from tf_repos_b200.smart_feature import frappe_feature, smart_feature
    d = _dataset(tmp_path, monkeypatch, n=2000, seed=3)
    outs = []
    for k in range(2):
        o = d + f"run{k}/"
        os.makedirs(o)
        smart_feature(d, o, "tr", build_feature_map_first=True, chunk_bytes=100_000)
        outs.append([open(o + n, "rb").read() for n in sorted(os.listdir(o))])
    assert outs[0] == outs[1]
    f = "fr"
    os.makedirs(f)
    _write_frappe(f + "/a.libsvm", 3000, 1, edge=True)
    first = open(frappe_feature(f)["outputs"][0], "rb").read()
    assert first == open(frappe_feature(f)["outputs"][0], "rb").read()


def _write_frappe(path, n, seed, edge):
    rng = np.random.default_rng(seed)
    lines = []
    for k in range(n):
        ids = np.sort(rng.choice(5000, 10, replace=False)) + 1
        lab = [b"-1", b"1"][rng.integers(2)]
        ln = lab + b" " + b" ".join(b"%d:1" % i for i in ids)
        if edge and k % 40 == 3:
            ln = [b"-1.0 3:1", b"+1 5:1", b"nospace", b"-1 ", b"1  2:1   3:1\r", b"", b"\t-1 4:1 ", b"-10 1:1",
                  b"-1"][(k // 40) % 9]
        lines.append(ln)
    open(path, "wb").write(b"\n".join(lines) + (b"" if edge else b"\n"))


@pytest.mark.parametrize("chunk_bytes", [1, 4096, 64 << 20])
def test_frappe_matches_oracle(tmp_path, monkeypatch, chunk_bytes):
    from tf_repos_b200.smart_feature import frappe_feature
    monkeypatch.chdir(tmp_path)
    for who in ("gpu", "ora"):
        os.makedirs(who + "/data")
        _write_frappe(who + "/data/b.libsvm", 300 if chunk_bytes == 1 else 5000, 2, edge=True)
        _write_frappe(who + "/data/a.libsvm", 200, 3, edge=True)
    g = frappe_feature("gpu/data", chunk_bytes=chunk_bytes)
    r = O.frappe_feature("ora/data")
    assert g["outputs"] == ["gpu/data/a_.libsvm", "gpu/data/b_.libsvm"]
    for a, b in zip(g["outputs"], r["outputs"]):
        assert open(a, "rb").read() == open(b, "rb").read()
        assert g["lines"][a] == r["lines"][b]
    # the reference's './' quirk: './data/x.libsvm' -> '_.libsvm' in the current directory
    os.makedirs("data")
    shutil.copy("ora/data/a.libsvm", "data/x.libsvm")
    assert frappe_feature("./data", chunk_bytes=chunk_bytes)["outputs"] == ["_.libsvm"]
    assert open("_.libsvm", "rb").read() == open("ora/data/a_.libsvm", "rb").read()


def _script(cwd, name, *args):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "Feature_pipeline", name), "--threads=4", *args],
                       capture_output=True, text=True, timeout=280, cwd=cwd)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout.strip().splitlines()


def _train(cwd, data_dir, field_size, feature_size):
    common = [sys.executable, os.path.join(ROOT, "Model_pipeline", "DeepFM.py"), f"--field_size={field_size}",
              f"--feature_size={feature_size}", "--embedding_size=8", "--batch_size=128", "--deep_layers=32,16",
              "--dropout=0.8,0.8", "--log_steps=5", "--num_epochs=1", "--data_dir=" + data_dir,
              "--model_dir=" + data_dir + "/ckpt/m_", "--dt_dir=1", "--task_type=train"]
    r = subprocess.run(common, capture_output=True, text=True, timeout=280, cwd=cwd)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "loss = " in r.stdout


def test_scripts_run_and_their_output_trains_deepfm(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    cwd, d = str(tmp_path), "smart/"
    os.makedirs(d)
    write_csv(d + "s_x_part_0", 1500, 21, edge=False)
    write_csv(d + "s_x_part_1", 700, 22, edge=False)
    out = _script(cwd, "get_smart_feature.py", "--input_dir=" + d, "--output_dir=" + d, "--task_type=tr",
                  "--build_feature_map=True")
    assert out[:5] == ["threads  4", "input_dir  " + d, "output_dir  " + d, "task_type  tr", "file_list size  2"]
    fs = int(out[-1].split("--feature_size=")[1].rstrip(")"))
    tr = open(d + "tr_0.libsvm", "rb").read().splitlines()
    assert len(tr) == 1500 and all(len(l.split(b" ")) == 127 for l in tr) and b"None" not in b"".join(tr)
    ids = [int(t.split(b":")[0]) for l in tr for t in l.split()[1:]]
    assert 1 <= min(ids) and max(ids) < fs
    _train(cwd, d, 126, fs)

    f = "frappe"
    os.makedirs(f)
    _write_frappe(f + "/frappe.tr.libsvm", 2000, 5, edge=False)
    out = _script(cwd, "get_frape_feature.py", "--input_dir=" + f, "--output_dir=/unused")
    assert out == ["threads  4", "input_dir  " + f, "output_dir  /unused", "file_list size  1"]
    fr = f + "/frappe_.libsvm"        # path.split('.')[0] + '_.libsvm'
    labels = {l.split(b" ")[0] for l in open(fr, "rb").read().splitlines()}
    assert labels == {b"0", b"1"}
    os.makedirs("ft")
    shutil.copy(fr, "ft/tr.libsvm")
    _train(cwd, "ft", 10, 5001)
