"""The GPU Ali-CCP TFRecord writer (tf_repos_b200.aliccp_tfrecord) against oracle/aliccp_tfrecord.py: byte identity
per output file at several chunk sizes, every declined-number class, every error and restriction, and the round trip
through the GPU reader and the DIN / ESMM scripts."""
import contextlib
import io
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

COMMON = ["101", "121", "122", "124", "125", "126", "127", "128", "129", "205", "301"]
UMH = ["109_14", "110_14", "127_14", "150_14"]
AD = ["206", "207", "210", "216"]
UNKNOWN = ["508", "509", "702", "853", "12", "1010", "127_15", "2055"]
# values the device declines (converted on the host) and plain ones it converts itself
DECLINED = ["1.0000001788139343", "1e30", "1e-30", "nan", "-inf", "inf", "Infinity", "1e39", "1e-50", "1e23",
            "9007199254740993", "0.000000000000000000000000123", "123456789012345678901", "1.5\t", "\t-2.25",
            "3.4028235e38", "4.9406564584124654e-324", "-nan", "1" * 70]
PLAIN = ["1.0", "2.3979", "0.693147", "0.1", "+.5", "5.", "-0", "1E5", "1e22", "9007199254740992", "00012.50",
         "-3.25e-7", "7e-22", "0e999", "2.30259"]


def _value(rng):
    return DECLINED[rng.randint(len(DECLINED))] if rng.rand() < 0.05 else PLAIN[rng.randint(len(PLAIN))]


def _id(rng):
    r = rng.rand()
    return str(rng.randint(20, 5000)) if r < 0.9 else ("007" if r < 0.95 else "9223372036854775807")


def _line(rng, heavy=False):
    triples = []
    for f in COMMON:
        for _ in range(rng.choice([0, 1, 1, 1, 2])):
            triples.append((f, _id(rng), "1.0"))
    for f in UMH:
        for _ in range(rng.randint(0, 60 if heavy else 5)):
            triples.append((f, _id(rng), _value(rng)))
    for f in AD + UNKNOWN:
        for _ in range(rng.choice([0, 1, 1, 3])):
            triples.append((f, _id(rng), _value(rng)))
    rng.shuffle(triples)
    sid = "%d" % rng.randint(1 << 30) if rng.rand() < 0.5 else "%d\t%d" % (rng.randint(100), rng.randint(1 << 30))
    y = ["0", "1", " 1", "1.0 ", "-0.0", "1e400"][rng.randint(6)] if rng.rand() < 0.2 else str(rng.randint(2))
    z = str(rng.randint(2))
    return ("%s,%s,%s,%s" % (sid, y, z, " ".join(":".join(t) for t in triples))).encode()


def _file(rng, n, heavy=False, last_newline=True):
    out = []
    for i in range(n):
        r = rng.rand()
        if r < 0.04:
            out.append(b"")
        elif r < 0.06:
            out.append(b"  \t ")
        elif r < 0.09:
            out.append(b"1,2,3")
        elif r < 0.11:
            out.append(_line(rng) + b",extra")
        else:
            ln = _line(rng, heavy)
            if rng.rand() < 0.1:
                ln = b"  " + ln + b" \t"
            out.append(ln + (b"\r" if rng.rand() < 0.2 else b""))
    data = b"\n".join(out)
    return data + b"\n" if last_newline else data


def _dataset(tmp_path, seed=0):
    rng = np.random.RandomState(seed)
    d = tmp_path / "in"
    d.mkdir()
    (d / "part-0").write_bytes(_file(rng, 300))
    (d / "part-1").write_bytes(_file(rng, 40, heavy=True))
    (d / "part-2").write_bytes(b"")
    (d / "part-3").write_bytes(_file(rng, 25, last_newline=False))
    (d / "nodash").write_bytes(_file(rng, 5))             # not matched by *-*
    return d


def _ref(d, out):
    from oracle import aliccp_tfrecord as oa
    oa.convert(str(d), str(out))
    return {p: (out / p).read_bytes() for p in sorted(os.listdir(out))}


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("aliccp")
    d = _dataset(tmp)
    return tmp, d, _ref(d, tmp / "ref")


@pytest.mark.parametrize("chunk", [1 << 20, 4099, 64])    # 64: smaller than almost every line
def test_byte_identical_to_oracle(data, chunk):
    from tf_repos_b200.aliccp_tfrecord import convert
    tmp, d, want = data
    out = tmp / ("out%d" % chunk)
    res = convert(str(d), str(out), chunk_bytes=chunk)
    assert sorted(want) == ["part-0.tfrecord", "part-1.tfrecord", "part-2.tfrecord", "part-3.tfrecord"]
    assert sorted(os.listdir(out)) == sorted(want)
    for name, b in want.items():
        assert (out / name).read_bytes() == b, name
    assert want["part-2.tfrecord"] == b""
    assert sum(o["declined"] for o in res["outputs"]) > 0


def test_every_declined_class_matches_the_oracle(tmp_path):
    from oracle import aliccp_tfrecord as oa
    from tf_repos_b200.aliccp_tfrecord import convert_file
    lines = []
    for i, v in enumerate(DECLINED + PLAIN):
        lines.append(b"%d,%s,%s,101:%d:1 127_14:5:%s 150_14:%d:%s 508:1:1" % (i, v.encode(), v.encode(), i,
                                                                               v.encode(), i, v.encode()))
    src, dst = tmp_path / "v-0", tmp_path / "v-0.tfrecord"
    src.write_bytes(b"\n".join(lines) + b"\n")
    st = convert_file(str(src), str(dst))
    assert dst.read_bytes() == b"".join(_framed(oa.records(src.read_bytes())))
    assert st["declined"] == 4 * len(DECLINED)            # y, z and both user multi-hot values of each such line


def _framed(recs):
    import struct
    from tf_repos_b200 import tfrecord as tfr
    for r in recs:
        hdr = struct.pack("<Q", len(r))
        yield hdr + struct.pack("<I", tfr.masked_crc(hdr)) + r + struct.pack("<I", tfr.masked_crc(r))


def _expect(tmp_path, lines, line_no, match, **kw):
    from tf_repos_b200.aliccp_tfrecord import AliccpTFRecordError, convert_file
    src, dst = tmp_path / "e-0", tmp_path / "e-0.tfrecord"
    src.write_bytes(b"\n".join(lines) + b"\n")
    with pytest.raises(AliccpTFRecordError) as e:
        convert_file(str(src), str(dst), **kw)
    msg = str(e.value)
    assert msg.startswith("%s: line %d: " % (src, line_no)), msg
    assert match in msg, msg
    assert not dst.exists()
    return msg


OK = b"1,0,1,101:5:1 127_14:6:1.5"


@pytest.mark.parametrize("chunk", [1 << 20, 40])
def test_errors_name_file_line_and_token_and_remove_the_output(tmp_path, chunk):
    kw = {"chunk_bytes": chunk}
    cases = [
        (b"1,0,1,101:5", "multiple of 3", "b'101:5'"),
        (b"1,0,1,", "multiple of 3", "b''"),
        (b"1,0,1,101:5:1  121:6:1", "multiple of 3", "b'101:5:1  121:6:1'"),
        (b"1,0,1,101:5:1    121:6:1", "empty token", "b''"),
        (b"1,0,1,508:x:y 101:5x:1", "[0-9]+", "b'5x'"),
        (b"1,0,1,101:-5:1", "[0-9]+", "b'-5'"),
        (b"1,0,1,206:9223372036854775808:1", "[0-9]+", "b'9223372036854775808'"),
        (b"1,0,1,101:5:1 109_14:1:abc", "float()", "b'abc'"),
        (b"1,x,1,101:5:1", "float()", "b'x'"),
        (b"1,0,1_0,101:5:1", "float()", "b'1_0'"),
        (b"1,0,1,101:5:1 110_14:1:0x1p3", "float()", "b'0x1p3'"),
        (b"1,0,1,101:5:1\0", "NUL", ""),
    ]
    for bad, what, tok in cases:
        msg = _expect(tmp_path, [OK] * 4 + [b"1,1e99999,1,101:7:1"] + [bad, OK, bad], 6, what, **kw)
        assert tok in msg, msg
    # the first failing line wins, whether the device or the host finds it; on one line the device's fault comes first
    _expect(tmp_path, [OK, b"1,0,1,101:5:1 150_14:1:bad", b"1,0,1,101:x:1"], 2, "float()", **kw)
    _expect(tmp_path, [OK, b"1,0,1,101:5:1 150_14:1:1", b"1,bad,1,101:x:1"], 3, "[0-9]+", **kw)
    _expect(tmp_path, [OK, b"1,bad,1,101:x:1 150_14:1:bad"], 2, "[0-9]+", **kw)
    _expect(tmp_path, [OK, b"1,bad,1,101:1:1 150_14:1:bad 1"], 2, "multiple of 3", **kw)


def test_long_line_restriction(tmp_path, monkeypatch):
    from tf_repos_b200 import aliccp_tfrecord as at
    monkeypatch.setattr(at, "MAX_LINE", 60)
    _expect(tmp_path, [OK, OK, OK + b" 101:6:1" * 5, OK], 3, "2^31 bytes", chunk_bytes=32)
    _expect(tmp_path, [OK, OK + b" 101:6:1" * 7], 2, "2^31 bytes", chunk_bytes=1000)


def test_failing_file_leaves_earlier_files(tmp_path):
    from tf_repos_b200.aliccp_tfrecord import AliccpTFRecordError, convert
    d = tmp_path / "in"
    d.mkdir()
    (d / "a-0").write_bytes(OK + b"\n")
    (d / "b-0").write_bytes(OK + b"\n1,0,1,101:x:1\n")
    with pytest.raises(AliccpTFRecordError, match="b-0: line 2"):
        convert(str(d), str(tmp_path / "out"))
    assert sorted(os.listdir(tmp_path / "out")) == ["a-0.tfrecord"]


def _clean(rng, n):
    """lines whose records the model readers accept: every common field at most once (feat_ids has 11 values)"""
    lines = []
    for _ in range(n):
        t = [(f, str(rng.randint(20, 5000)), "1.0") for f in COMMON if rng.rand() < 0.85]
        for f in UMH:
            t += [(f, str(rng.randint(20, 5000)), "%.5f" % (rng.rand() * 3)) for _ in range(rng.randint(0, 9))]
        t += [(f, str(rng.randint(20, 5000)), "1.0") for f in AD for _ in range(rng.choice([0, 1, 1, 4]))]
        t += [("508", "1", "2.30259")]
        rng.shuffle(t)
        y = rng.rand() < 0.4
        lines.append(("%d,%d,%d,%s" % (rng.randint(1 << 30), y, y and rng.rand() < 0.5,
                                       " ".join(":".join(x) for x in t))).encode())
    return b"\n".join(lines) + b"\n"


@pytest.mark.parametrize("layout", ["din", "esmm"])
def test_round_trip_through_the_gpu_reader(tmp_path, layout):
    from tf_repos_b200 import din_main as dm
    from tf_repos_b200 import esmm_main as em
    from tf_repos_b200.aliccp_tfrecord import convert
    from tf_repos_b200.tfrecord_device import TFRecordIndex
    from tests.test_gpu_tfrecord_device import _same
    d = tmp_path / "in"
    d.mkdir()
    rng = np.random.RandomState(3)
    for i in range(3):
        (d / ("part-%d" % i)).write_bytes(_clean(rng, 40 + 17 * i))
    convert(str(d), str(tmp_path / "out"), chunk_bytes=2000)
    paths = [str(tmp_path / "out" / ("part-%d.tfrecord" % i)) for i in range(3)]
    labels = ("y",) if layout == "din" else ("y", "z")
    with contextlib.redirect_stdout(io.StringIO()):
        host = dm.decode_tfrecord_files(paths, 11, labels)
    index = TFRecordIndex.build(paths, 11, labels, "cuda")
    n = len(host["y"])
    assert len(index) == n == 40 + 57 + 74
    P, _ = index.max_lengths()
    for B in (7, 64):
        want = list(dm.index_stream(n, 2, B))
        got = list(index.batches(2, B, layout, P))
        assert len(got) == len(want)
        for (batch, lab, cnt), idx in zip(got, want):
            if layout == "din":
                wb, wl, wn = dm.make_batch(host, idx, B, P, "cpu")
                _same(lab, wl)
            else:
                wb, (wy, wz), wn = em.make_batch(host, idx, B, "cpu")
                _same(lab[0], wy); _same(lab[1], wz)
            assert cnt == wn and batch.keys() == wb.keys()
            for k in wb:
                _same(batch[k], wb[k])


def _run(args):
    r = subprocess.run([sys.executable] + args, capture_output=True, text=True, timeout=280, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout


def test_script_flags_naming_glob_and_mkdir(tmp_path):
    from oracle import aliccp_tfrecord as oa
    d = tmp_path / "raw"
    d.mkdir()
    rng = np.random.RandomState(5)
    (d / "sample-a").write_bytes(_clean(rng, 12))
    (d / "sample-b").write_bytes(_clean(rng, 9))
    (d / "README").write_bytes(b"not an input\n")
    out = _run([os.path.join(ROOT, "Feature_pipeline", "get_aliccp_tfrecord.py"), "--input_dir=%s" % d,
                "--output_dir=%s" % d, "--threads=4"])
    assert "total files: 2" in out and out.strip().splitlines()[-1].startswith("field_size 11")
    assert sorted(os.listdir(d)) == ["README", "sample-a", "sample-a.tfrecord", "sample-b", "sample-b.tfrecord"]
    for f in ("sample-a", "sample-b"):
        assert (d / (f + ".tfrecord")).read_bytes() == b"".join(_framed(oa.records((d / f).read_bytes())))
    d2 = tmp_path / "raw2"
    d2.mkdir()
    (d2 / "x-1").write_bytes(_clean(rng, 3))
    _run([os.path.join(ROOT, "Feature_pipeline", "get_aliccp_tfrecord.py"), "--input_dir=%s" % d2,
          "--output_dir=%s" % (tmp_path / "new")])
    assert sorted(os.listdir(tmp_path / "new")) == ["x-1.tfrecord"]


@pytest.mark.parametrize("script, extra", [
    ("DIN.py", ["--deep_layers=16,8", "--dropout=1,1", "--attention_layers=16"]),
    ("DeepCvrMTL.py", ["--deep_layers=16,8", "--dropout=1,1", "--ctr_task_wgt=0.3"]),
])
def test_models_train_and_infer_on_the_script_output(tmp_path, script, extra):
    from tests.test_gpu_tfrecord_cli import REFERENCE
    tmp = str(tmp_path)
    rng = np.random.RandomState(11)
    os.makedirs(tmp + "/data")                            # the script makes output_dir only, with os.mkdir
    for part, n in (("tr", 150), ("te", 70)):
        os.makedirs("%s/raw/%s" % (tmp, part))
        with open("%s/raw/%s/part-0" % (tmp, part), "wb") as fh:
            fh.write(_clean(rng, n))
        _run([os.path.join(ROOT, "Feature_pipeline", "get_aliccp_tfrecord.py"), "--input_dir=%s/raw/%s" % (tmp, part),
              "--output_dir=%s/data/%s" % (tmp, part)])
    os.makedirs(tmp + "/ref")
    flags = ["--field_size=11", "--feature_size=5000", "--embedding_size=8", "--batch_size=32", "--num_epochs=3",
             "--log_steps=1000", "--data_dir=" + tmp + "/data", "--model_dir=" + tmp + "/ckpt/m_",
             "--dt_dir=20261016"] + extra
    script_path = os.path.join(ROOT, "Model_pipeline", script)
    _run([script_path, "--task_type=train"] + flags)
    _run([script_path, "--task_type=infer"] + flags)
    tr, te = tmp + "/data/tr/part-0.tfrecord", tmp + "/data/te/part-0.tfrecord"
    _run(["-c", REFERENCE, ROOT, script, tr, te, tmp + "/ref"] + flags)
    got = torch.load(tmp + "/ckpt/m_20261016/ctr_b200.ckpt", map_location="cpu")
    want = torch.load(tmp + "/ref/ctr_b200.ckpt", map_location="cpu")
    assert got["global_step"] == want["global_step"] == 15
    for k in want["variables"]:
        assert torch.equal(got["variables"][k], want["variables"][k]), k
    pred = open(tmp + "/data/pred.txt").read()
    assert pred.count("\n") == 70 and pred == open(tmp + "/ref/pred.txt").read()
