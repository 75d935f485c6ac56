"""Known answers for oracle/criteo_feature.py, the CPU restatement of get_criteo_feature.py that the GPU pipeline is
compared with: dictionary order, <unk> and the offsets, feature_map's +1, the %.6f formatting, the te label and the
Python 2 train/valid split."""
import random

import numpy as np
import pytest

from oracle import criteo_feature as ocf


def _line(label, ints, cats):
    return "\t".join([label] + ints + cats) + "\n"


def _write(tmp_path, train, test):
    (tmp_path / "train.txt").write_text("".join(train))
    (tmp_path / "test.txt").write_text("".join(test))
    return str(tmp_path) + "/"


CATS = ["a%d" % i for i in range(25)]   # C2..C26 hold one value each


@pytest.fixture()
def run(tmp_path):
    # I1 (clip 20) over train: min -2, max 20; I2 (clip 600): min 0, max 200
    ints = lambda i1, i2: [i1, i2] + ["5"] * 11
    train = [
        _line("0", ints("3", "0"), ["bb"] + CATS),
        _line("1", ints("1", "128"), ["aa"] + CATS),
        _line("0", ints("", "1"), ["bb"] + CATS),
        _line("1", ints("50", "3"), ["aa"] + CATS),       # I1 clipped to 20
        _line("0", ints("-2", "200"), ["cc"] + CATS),
        _line("1", ints("0", ""), ["cc"] + CATS),
        _line("0", ints("7", "12"), ["d"] + CATS),
        _line("7", ints("4", "5"), ["", ] + CATS),       # last label "7": te uses it
    ]
    # make every I3..I13 column non-constant
    train[0] = train[0].replace("\t5\t5\t5\t5\t5\t5\t5\t5\t5\t5\t5\t", "\t6\t6\t6\t6\t6\t6\t6\t6\t6\t6\t6\t")
    test = [
        "\t".join(["2", "0"] + ["5"] * 11 + ["aa"] + CATS) + "\n",
        "\t".join(["-1", "400"] + ["5"] * 11 + ["zz"] + CATS) + "\n",
        "\t".join(["-0", ""] + ["6"] * 11 + [""] + CATS) + "\n",
    ]
    d = _write(tmp_path, train, test)
    out = ocf.preprocess(d, d, cutoff=2)
    read = lambda n: (tmp_path / n).read_bytes()
    return out, read


def test_dictionary_order_unk_and_offsets(run):
    out, read = run
    # C1 counts: aa 2, bb 2, cc 2, d 1 -> cutoff 2 keeps aa, bb, cc; ties broken bytewise by key
    fmap = read("feature_map").decode().splitlines()
    c1 = [l for l in fmap if l.startswith("C1|")]
    assert c1 == ["C1|aa 15", "C1|bb 16", "C1|cc 17", "C1|<unk> 14"]   # offset 13 + id + 1 (the +1 quirk)
    assert fmap[:13] == ["I%d %d" % (i, i) for i in range(1, 14)]
    assert out["dict_sizes"][0] == 4 and out["dict_sizes"][1:] == [2] * 25
    assert out["offsets"][:3] == [13, 17, 19]
    assert out["feature_size"] == 13 + 4 + 25 * 2
    assert "C2|a0 19" in fmap and "C2|<unk> 18" in fmap


def test_lines_unk_collides_with_I13_and_formatting(run):
    out, read = run
    lines = (read("tr.libsvm") + read("va.libsvm")).decode().splitlines()
    assert len(lines) == 8 and out["lines"]["tr"] + out["lines"]["va"] == 8
    last = [l for l in lines if l.startswith("7 ")][0].split()
    assert last[14] == "13:1"          # C1 empty -> <unk> 0 + offset 13, the same id as I13
    # I2: 128 / 200, 1 / 200, 0 / 200; I1 (3 + 2) / 22 = 0.2272727..
    assert any(" 2:0.64 " in l for l in lines)
    assert any(" 2:0.005 " in l for l in lines) and any(" 2:0 " in l for l in lines)
    assert any(l.startswith("0 1:0.227273 ") for l in lines)


def test_fixed6_rounding():
    assert ocf.fixed6(1 / 128) == b"0.007812"     # exact binary 0.0078125: tie, to even
    assert ocf.fixed6(3 / 128) == b"0.023438"     # 0.0234375: tie, to even
    assert ocf.fixed6(-1e-7) == b"-0"
    assert ocf.fixed6(-0.0) == b"-0"
    assert ocf.fixed6(0.0) == b"0"
    assert ocf.fixed6(1.0) == b"1"
    assert ocf.fixed6(2.5) == b"2.5"
    assert ocf.fixed6(1e6 / 3) == b"333333.333333"


def test_te_uses_the_last_train_label_and_shifts_columns(run):
    out, read = run
    te = read("te.libsvm").decode().splitlines()
    assert out["lines"]["te"] == 3 and all(l.startswith("7 ") for l in te)
    # I1 over train: values 3, 1, 20 (50 clipped), -2, 0, 7, 4 -> min -2, max 20, den 22
    f = te[0].split()
    assert f[1] == "1:0.181818"       # (2 + 2) / 22
    assert f[2] == "2:0"              # (0 - 0) / 200
    assert f[14] == "14:1"            # C1 "aa" -> id 1 + offset 13, read from the shifted column
    f = te[1].split()
    assert f[1] == "1:0.045455"       # (-1 + 2) / 22 = 0.0454545..
    assert f[2] == "2:2"              # 400 / 200: not clipped, above 1
    assert f[14] == "13:1"            # unknown -> <unk>
    f = te[2].split()
    assert f[1] == "1:0.090909"       # -0 -> (-0.0 + 2) / 22
    assert f[2] == "2:0"              # empty


def test_negative_zero_survives():
    # (float("-0") - 0) / den = -0.0 -> "-0", as Python prints it
    assert ocf.fixed6((float("-0") - 0) / 5) == b"-0"


def test_split_decisions_are_python2_randint():
    r = random.Random(0)
    loop = [int(r.random() * 10000) % 10 != 0 for _ in range(1000)]
    assert ocf.split_decisions_loop(1000) == loop
    assert ocf.split_decisions(1000).tolist() == loop
    rs = np.random.RandomState([0])
    assert np.concatenate([ocf.split_decisions(300, rs), ocf.split_decisions(700, rs)]).tolist() == loop
    assert 0.85 < np.mean(loop) < 0.95


def test_nothing_above_cutoff_raises(tmp_path):
    d = _write(tmp_path, [_line("0", ["1"] * 13, ["x"] + CATS)], [])
    with pytest.raises(ValueError):
        ocf.preprocess(d, d, cutoff=2)
