"""Known answers of oracle/aliccp_tfrecord.py, the restatement of get_aliccp_tfrecord.py's gen_tfrecords that the GPU
writer is checked against byte for byte, and its records through the TFRecord readers."""
import contextlib
import ctypes
import io

import numpy as np
import pytest

from oracle import aliccp_tfrecord as oa

DERIVED = [b"205", b"301", b"121", b"122", b"124", b"125", b"126", b"127", b"128", b"129", b"101"]


def test_python2_hash_and_common_field_order():
    assert oa.py2_str_hash(b"") == 0
    assert oa.py2_str_hash(b"a") == 12416037344            # hash('a') of a 64-bit CPython 2.7
    keys = [k.encode() for k, _ in oa.COMMON_LITERAL]
    assert oa.py2_dict_order(keys) == DERIVED
    assert [k for k, _ in oa.COMMON] == DERIVED
    assert [d for _, d in oa.COMMON] == [10, 11, 2, 3, 4, 5, 6, 7, 8, 9, 1]


def _line(feats, y="1", z="0", sid="7"):
    return (",".join([sid, y, z, " ".join(feats)])).encode()


def test_defaults_repeats_and_dropped_fields():
    f = oa.parse_line(_line(["508:99:2.3", "101:5:1", "206:41:1", "101:6:1", "127_14:300:2.5", "853:1:1",
                             "127_14:301:0.5", "210:7:1", "210:8:1"]))
    assert f["feat_ids"].tolist() == [10, 11, 2, 3, 4, 5, 6, 7, 8, 9, 5, 6]       # 101 last, repeated in line order
    assert f["u_brandids"].tolist() == [300, 301] and f["u_brandvals"].tolist() == [2.5, 0.5]
    for name, d in (("u_cat", 12), ("u_shop", 13), ("u_int", 15)):
        assert f[name + "ids"].tolist() == [d] and f[name + "vals"].tolist() == [1.0]
    assert f["a_catids"].tolist() == [41] and f["a_intids"].tolist() == [7, 8]
    assert f["a_shopids"].tolist() == [17] and f["a_brandids"].tolist() == [19]
    assert f["y"].dtype == np.float32 and f["y"].tolist() == [1.0] and f["z"].tolist() == [0.0]
    assert sorted(f) == sorted(["y", "z", "feat_ids", "u_catids", "u_catvals", "u_shopids", "u_shopvals",
                                "u_brandids", "u_brandvals", "u_intids", "u_intvals", "a_catids", "a_shopids",
                                "a_intids", "a_brandids"])


def test_lines_without_four_fields_are_skipped():
    data = b"\n" + _line(["101:1:1"]) + b",x\n  \r\n" + _line(["101:2:1"]) + b"\r\n1,2,3\n" + _line(["101:3:1"])
    got = list(oa.examples(data))
    assert [int(f["feat_ids"][-1]) for f in got] == [2, 3]


def test_double_rounding_of_values():
    assert oa.to_f32(oa.py2_float(b"1.0000001788139343")).view(np.uint32) == 0x3F800002
    strtof = ctypes.CDLL(None).strtof                     # a direct decimal -> float32 rounding differs
    strtof.restype, strtof.argtypes = ctypes.c_float, [ctypes.c_char_p, ctypes.c_void_p]
    assert np.float32(strtof(b"1.0000001788139343", None)).view(np.uint32) == 0x3F800001
    f = oa.parse_line(_line(["150_14:9:1.0000001788139343"], y="1.0000001788139343"))
    assert f["u_intvals"].view(np.uint32).tolist() == [0x3F800002] and f["y"].view(np.uint32).tolist() == [0x3F800002]
    assert oa.to_f32(1e39) == np.inf
    with pytest.raises(ValueError):
        oa.py2_float(b"1_0")                              # Python 3 only


@pytest.mark.parametrize("feats, kind", [
    (["101:1"], "count"), ([], "count"), (["101:1:1:2"], "count"),
    (["101:1:1", "", "", "", "121:2:1"], "empty"), (["101:x:1"], "id"), (["101:-1:1"], "id"),
    (["101:9223372036854775808:1"], "id"), (["127_14:1:abc"], "float"),
])
def test_faults_raise(feats, kind):
    with pytest.raises(oa.OracleError) as e:
        oa.parse_line(_line(feats), 3)
    assert e.value.kind == kind and e.value.line == 3
    assert oa.parse_line(_line(["508:x:y"])) is not None                    # dropped fields are not parsed


def test_fault_order_within_a_line():
    with pytest.raises(oa.OracleError, match="count"):
        oa.parse_line(_line(["101:x:1", "1"], y="bad"))
    with pytest.raises(oa.OracleError, match="id"):
        oa.parse_line(_line(["101:x:1", "127_14:1:bad"], y="bad"))
    with pytest.raises(oa.OracleError) as e:
        oa.parse_line(_line(["127_14:1:bad"], y="bad"))
    assert e.value.token == b"bad" and e.value.kind == "float"
    assert oa.parse_line(_line(["101:0000000000000000000000005:1"]))["feat_ids"][-1] == 5
    assert oa.parse_line(_line(["101:5:1"], y=" 1 "))["y"].tolist() == [1.0]


def _sample(rng, n_lines):
    lines = []
    for _ in range(n_lines):
        feats = ["%s:%d:1.0" % (f, rng.randint(1, 1000)) for f in ("101", "121", "205", "301") if rng.rand() < 0.8]
        for f in ("109_14", "150_14", "210"):
            feats += ["%s:%d:%.4f" % (f, rng.randint(1, 1000), rng.rand() * 3) for _ in range(rng.randint(0, 4))]
        feats.append("508:1:2.30259")
        lines.append(_line(feats, y=str(rng.randint(2)), z=str(rng.randint(2))))
    return b"\n".join(lines) + b"\n"


def test_records_read_back_through_every_decoder(tmp_path):
    from tf_repos_b200 import din_main as dm
    from tf_repos_b200 import esmm_main as em
    from tf_repos_b200 import tfrecord as tfr
    data = _sample(np.random.RandomState(0), 40)
    src = tmp_path / "part-0"
    src.write_bytes(data)
    oa.convert(str(tmp_path), str(tmp_path / "out"))
    path = str(tmp_path / "out" / "part-0.tfrecord")
    recs = list(tfr.read_records(path, verify_crc=True))
    feats = list(oa.examples(data))
    assert len(recs) == len(feats) == 40
    for r, f in zip(recs, feats):
        ex = tfr.parse_example(r)
        assert sorted(ex) == sorted(f)
        for k in f:
            assert ex[k].dtype == (np.float32 if f[k].dtype == np.float32 else np.int64)
            assert ex[k].tolist() == f[k].tolist(), k
    with contextlib.redirect_stdout(io.StringIO()):
        d = dm.decode_tfrecord_files([path], 11)
        e = em.decode([path], 11)
    assert len(d["y"]) == len(e["z"]) == 40
    assert [list(x) for x in d["feat_ids"]] == [f["feat_ids"].tolist() for f in feats]
