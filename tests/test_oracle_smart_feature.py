"""Known answers for oracle/smart_feature.py, the restatement of get_smart_feature.py (with its builder) and
get_frape_feature.py that the GPU stage is compared against: every rule of DESIGN.md §2.12 with hand-written bytes."""
import os

import pytest

from oracle import smart_feature as O

MAP = (b"u_pl|a 5\n"
       b"u_pl|a 6\n"              # a repeated key: the later line wins
       b"u_pl|UNK 7\n"
       b"u_pl|b\n"                # one token: skipped
       b"u_pl|c  9\n"             # split on single spaces: the fid is the empty string
       b"u_pl|\xff\xfe 11\n"      # not UTF-8
       b"u_ctr 12\n"              # a continuous column's bare name
       b"\t u_de|x 13 extra \r\n"  # stripped; a third token is ignored
       b"\n"
       b"c_al|q 14")              # no final newline


def _emit(tmp_path, lines, fmap=MAP):
    d = str(tmp_path) + "/"
    os.makedirs(d + "in", exist_ok=True)
    with open(d + "feature_map", "wb") as fh:
        fh.write(fmap)
    with open(d + "in/x.verify", "wb") as fh:
        fh.write(lines)
    O.smart_feature(d + "in", d, "va")
    return open(d + "va.libsvm", "rb").read()


def test_map_load_rules(tmp_path):
    p = str(tmp_path / "m")
    open(p, "wb").write(MAP)
    assert O.load_map(p) == {b"u_pl|a": b"6", b"u_pl|UNK": b"7", b"u_pl|c": b"", b"u_pl|\xff\xfe": b"11",
                             b"u_ctr": b"12", b"u_de|x": b"13", b"c_al|q": b"14"}


def test_range_quirk_none_and_unk_fallback(tmp_path):
    # the last field is never emitted; u_ppvn has no key and no UNK key: None
    assert _emit(tmp_path, b"1,a,zz,x\n") == b"1 6:1 None:1\n"
    # u_pl|zz is absent: u_pl|UNK; u_de|x found
    assert _emit(tmp_path, b"0,zz,w,x,last\n") == b"0 7:1 None:1 13:1\n"
    # an empty fid and non-UTF-8 bytes
    assert _emit(tmp_path, b"1,c,w\n1,\xff\xfe,w\n") == b"1 :1\n1 11:1\n"


def test_continuous_values_are_copied_verbatim(tmp_path):
    f = [b"1"] + [b"a"] + [b"k"] * 9 + [b" 0.5e-3 x"] + [b"v"] * 2
    # i = 11 is u_ctr (fid 12) with its value as written; i = 12 (a_a_ctr) has no key: None
    want = b"1 6:1 " + b"None:1 " * 8 + b"None:1 12: 0.5e-3 x None:v\n"
    assert _emit(tmp_path, b",".join(f) + b"\n") == want


def test_long_lines_are_dropped(tmp_path):
    ok = b",".join([b"1"] + [b"a"] * 128) + b"\n"            # 129 fields: 127 features
    long = b",".join([b"0"] + [b"a"] * 129) + b"\n"          # 130 fields: CSV_COLUMNS[128] raises
    out = _emit(tmp_path, ok + long + ok)
    lines = out.splitlines()
    assert len(lines) == 2 and lines[0] == lines[1]
    assert len(lines[0].split(b" ")) == 128 and lines[0].startswith(b"1 6:1 None:1 ")


def test_empty_short_crlf_and_whitespace_lines(tmp_path):
    text = (b"\n"                      # empty: " \n"
            b"0\n"                     # one field
            b"1,a\n"                   # two fields: range(1, 1) is empty
            b"1,a,b\r\n"               # \r is stripped
            b"  1,a,b \t\x0b\x0c\n"    # Python 2 whitespace at both ends
            b"\x1c1,a,b\x1c\n"         # \x1c is not Python 2 whitespace
            b"1,a b,c\n"               # a value with a space: no map key can hold it
            b"0,a,b")                  # no final newline
    assert _emit(tmp_path, text) == (b" \n0 \n1 \n1 6:1\n1 6:1\n\x1c1 6:1\n1 7:1\n0 6:1\n")


def test_tr_naming_collisions_and_short_paths(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    os.makedirs("d_x/in")
    open("feature_map", "wb").write(MAP)
    open("d_x/in/a_part_7", "wb").write(b"1,a,b\n")
    open("d_x/in/b_part_8", "wb").write(b"0,zz,b\n")
    r = O.smart_feature("d_x/in", "", "tr")
    # 'd_x/in/a_part_7'.rsplit('_') = ['d', 'x/in/a', 'part', '7']: the underscore in the directory shifts the index
    assert r["outputs"] == ["tr_7.libsvm", "tr_8.libsvm"]
    assert open("tr_7.libsvm", "rb").read() == b"1 6:1\n" and open("tr_8.libsvm", "rb").read() == b"0 7:1\n"
    os.makedirs("e_y/in")
    open("e_y/in/p_part_1", "wb").write(b"1,a,b\n")
    open("e_y/in/q_part_1", "wb").write(b"1,a,b\n")
    with pytest.raises(O.OracleError):
        O.smart_feature("e_y/in", "out_", "tr")
    os.makedirs("f/in")
    open("f/in/part_1", "wb").write(b"1,a,b\n")
    with pytest.raises(O.OracleError):
        O.smart_feature("f/in", "out_", "tr")
    assert not any(n.startswith("out_") for n in os.listdir("."))


def test_va_inputs_concatenate_in_sorted_order_and_missing_map_raises(tmp_path):
    d = str(tmp_path) + "/"
    os.makedirs(d + "in")
    open(d + "in/b.verify", "wb").write(b"0,a,b\n")
    open(d + "in/a.verify", "wb").write(b"1,a,b\n")
    with pytest.raises(FileNotFoundError):
        O.smart_feature(d + "in", d, "va")
    assert not os.path.exists(d + "va.libsvm")
    open(d + "feature_map", "wb").write(MAP)
    O.smart_feature(d + "in", d, "va")
    assert open(d + "va.libsvm", "rb").read() == b"1 6:1\n0 6:1\n"


def test_builder_order_unk_hit_and_partial_long_lines(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)                                 # relative paths: no '_' before the file names
    d = "o/"
    os.makedirs(d + "in")
    open(d + "in/x_y_part_0", "wb").write(b"1,p,UNK,c,0.5,e\n" + b"0," + b",".join([b"p"] * 10) + b",0.25,z\n")
    long = b",".join([b"1"] + [b"v%d" % i for i in range(1, 130)])   # 130 fields, no final newline
    open(d + "in/x_y_part_1", "wb").write(long)
    seeded = [b"%s|UNK %d" % (n, i + 1) for i, n in enumerate(O.COLUMNS)]
    want = [b"u_pl|p 129", b"u_de|c 130", b"u_os|0.5 131",     # u_ppvn|UNK hits the seeded key
            b"u_ppvn|p 132", b"u_de|p 133", b"u_os|p 134", b"u_t|p 135", b"a_m_w|p 136", b"a_b_w|p 137",
            b"c_h|p 138", b"c_w|p 139", b"c_al|p 140", b"u_ctr 141"]
    fid = 142
    for i in range(1, 128):                                     # columns 1..127 of the long line, then IndexError
        key = O.COLUMNS[i] if O.continuous(i) else O.COLUMNS[i] + b"|v%d" % i
        if key != b"u_ctr":
            want.append(key + b" %d" % fid)
            fid += 1
    text = O.feature_map_text(sorted([d + "in/x_y_part_0", d + "in/x_y_part_1"]))
    assert text.splitlines() == seeded + want
    r = O.smart_feature(d + "in", d, "tr", build=True)
    assert open(d + "feature_map", "rb").read() == text
    assert open(d + "tr_0.libsvm", "rb").read() == b"1 129:1 3:1 130:1 131:1\n0 129:1 " + b" ".join(
        b"%d:1" % f for f in range(132, 141)) + b" 141:0.25\n"
    assert open(d + "tr_1.libsvm", "rb").read() == b""                  # the long line is dropped by the emit
    assert r["lines"][d + "tr_1.libsvm"] == (1, 0)


def test_frappe_rules(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    os.makedirs("data")
    open("data/x.libsvm", "wb").write(b"-1 451:1 4149:1\n"
                                      b"-1.0 3:1\n"
                                      b"+1 5:1\n"
                                      b"nospace\n"
                                      b"-1 \n"                  # stripped to one token: skipped
                                      b"1  2:1   3:1\r\n"       # repeated spaces kept, \r stripped
                                      b"\n"
                                      b"-1 7:1")
    r = O.frappe_feature("./data")
    # './data/x.libsvm'.split('.')[0] == '': the output lands in the current directory as '_.libsvm'
    assert r["outputs"] == ["_.libsvm"]
    assert open("_.libsvm", "rb").read() == b"0 451:1 4149:1\n-1.0 3:1\n+1 5:1\n1  2:1   3:1\n0 7:1\n"
    assert r["lines"]["_.libsvm"] == (8, 5)
    open("data/y.libsvm", "wb").write(b"1 1:1\n")
    with pytest.raises(O.OracleError):                          # both would write ./_.libsvm
        O.frappe_feature("./data")
    os.makedirs("e")
    open("e/y.libsvm", "wb").write(b"-1 1:1\n")
    assert O.frappe_feature("e")["outputs"] == ["e/y_.libsvm"]
    assert open("e/y_.libsvm", "rb").read() == b"0 1:1\n"
