"""Known answers for oracle/aliccp_sample.py, the restatement of DeepMTL's join / stat / remap jobs: the y=0 / z=1
filter, every silent-skip class, the join with and without a common record, last-wins md5s, counts through shared
records, the cutoff boundary, the id order, the shuffle rule and the reference's remap quirk."""
import os

import pytest

from oracle import aliccp_sample as oa
from oracle import aliccp_tfrecord as ot


def _feats(*toks):
    return b"\x01".join(b"%s\x02%s\x03%s" % t for t in toks)


def _sample(sid, y, z, md5, *toks):
    return b"%s,%s,%s,%s,%d,%s" % (sid, y, z, md5, len(toks), _feats(*toks))


def _common(md5, *toks):
    return b"%s,%d,%s" % (md5, len(toks), _feats(*toks))


def test_splitmix64_known_answers():
    # SplitMix64 seeded with 0: its first three outputs
    assert [oa.splitmix64(0, i) for i in range(3)] == [0xE220A8397B1DCDAF, 0x6E789E6AA1B965F4, 0x06C45D188009454F]
    assert oa.shuffle_key(0, 0) == 0xE220A8397B1DCDAF >> 33
    assert all(0 <= oa.shuffle_key(7, i) < (1 << 31) for i in range(1000))
    assert oa.splitmix64(1, 0) != oa.splitmix64(0, 0)


def test_filter_and_silent_skips():
    t = (b"101", b"5", b"1.0")
    assert oa.join_map(_sample(b"s", b"0", b"1", b"m", t)) == ("filtered",)
    # the filter compares strings and runs before the feature list is parsed
    assert oa.join_map(b"s,0,1,m,1,garbage") == ("filtered",)
    assert oa.join_map(_sample(b"s", b"0.0", b"1", b"m", t))[0] == "sample"
    assert oa.join_map(_sample(b"s", b"1", b"1", b"m", t))[0] == "sample"
    for line in (b"", b"   ", b"a,b", b"a,b,c,d", b"a,b,c,d,e,f,g", _sample(b"s", b"1", b"0", b"m", t) + b",x"):
        assert oa.join_map(line) == ("malformed",), line
    bad_splits = [b"m,1,101\x025", b"m,1,101\x025\x031\x02x", b"m,1,101\x025\x031\x036", b"m,1,",
                  b"m,2," + _feats(t) + b"\x01", b"m,1,101\x02\x025\x031"]
    for line in bad_splits:
        assert oa.join_map(line) == ("malformed",), line
    # \x03 before the \x02 splits fine in the mapper; the field then breaks a restriction
    with pytest.raises(oa.OracleError) as e:
        oa.join_map(b"m,1,1\x030\x025\x031", 4)
    assert e.value.line == 4 and e.value.kind == "field"


def test_restrictions():
    t = (b"101", b"5", b"1.0")
    cases = [
        (_sample(b"s\0", b"1", b"0", b"m", t), "nul"),
        (_sample(b"s:1", b"1", b"0", b"m", t), "text"),
        (_sample(b"s", b"1 1", b"0", b"m", t), "text"),
        (_sample(b"s", b"1", b"0", b"", t), "md5"),
        (_sample(b"s", b"1", b"0", b"m" * 65, t), "md5"),
        (_common(b"m\x0b1", t), "text"),
        (_common(b"m", (b"", b"5", b"1")), "field"),
        (_common(b"m", (b"f" * 17, b"5", b"1")), "field"),
        (_common(b"m", (b"f:g", b"5", b"1")), "field"),
        (_common(b"m", (b"101", b"05", b"1")), "fid"),
        (_common(b"m", (b"101", b"", b"1")), "fid"),
        (_common(b"m", (b"101", b"-5", b"1")), "fid"),
        (_common(b"m", (b"101", b"9223372036854775808", b"1")), "fid"),
        (_common(b"m", (b"101", b"5", b"1:2")), "text"),
        (_common(b"m", (b"101", b"5", b"a b")), "text"),
    ]
    for line, kind in cases:
        with pytest.raises(oa.OracleError) as e:
            oa.join_map(line, 9)
        assert e.value.kind == kind, line
    assert oa.join_map(_common(b"m" * 64, (b"f" * 16, b"9223372036854775807", b"")))[0] == "common"
    assert oa.join_map(_common(b"m", (b"101", b"0", b"x")))[0] == "common"
    # not a kept line: no restriction applies
    assert oa.join_map(b"s\0,0,1,m,1,x") == ("filtered",)
    assert oa.join_map(b"m\0,1,101\x025") == ("malformed",)


def _mapped(lines):
    return [(i, oa.join_map(l)) for i, l in enumerate(lines)]


def test_join_last_wins_no_common_and_shared_counts():
    lines = [
        _common(b"A", (b"301", b"7", b"1")),
        _sample(b"s0", b"1", b"0", b"A", (b"205", b"3", b"1")),
        _common(b"A", (b"301", b"8", b"1"), (b"302", b"9", b"2")),      # supersedes the first A
        _sample(b"s1", b"0", b"0", b"A", (b"205", b"4", b"1")),
        _sample(b"s2", b"1", b"1", b"B", (b"205", b"3", b"0.5")),         # no record
        _sample(b"s3", b"0", b"1", b"A", (b"205", b"3", b"1")),           # filtered
    ]
    joined, st = oa.join_reduce(_mapped(lines))
    assert st == {"commons": 2, "commons_superseded": 1, "no_common": 1, "samples": 3, "filtered": 1, "malformed": 0}
    assert [oa.joined_text(*j[1:]) for j in joined] == [
        b"s0,1,0,205:3:1 301:8:1 302:9:2", b"s1,0,0,205:4:1 301:8:1 302:9:2", b"s2,1,1,205:3:0.5"]
    cnt = oa.stat(joined)
    assert cnt == {(b"205", 3): 2, (b"205", 4): 1, (b"301", 8): 2, (b"302", 9): 2}
    assert oa.feat_cnts(cnt) == b"205:3\t2\n205:4\t1\n301:8\t2\n302:9\t2\n"


def test_common_record_shared_by_k_samples_counts_k_times():
    k = 23
    lines = [_common(b"C", (b"301", b"11", b"1"), (b"301", b"11", b"1"))]
    lines += [_sample(b"s%d" % j, b"1", b"0", b"C", (b"205", b"%d" % j, b"1")) for j in range(k)]
    joined, _ = oa.join_reduce(_mapped(lines))
    assert oa.stat(joined)[(b"301", 11)] == 2 * k


def test_cutoff_boundary_and_id_order():
    cnt = {(b"205", 100): 19, (b"205", 7): 20, (b"301", 100): 1, (b"301", 3): 19, (b"129", 12): 25,
           (b"129", 5): 19, (b"301", 5): 1}
    assert oa.vocabulary(cnt, 20) == {7: 20, 12: 21}
    assert oa.vocabulary(cnt, 19) == {3: 20, 5: 21, 7: 22, 12: 23, 100: 24}
    # a fid kept through one field keeps every field's token of it
    vocab = oa.vocabulary(cnt, 20)
    line = oa.remap_line(5, b"s", b"1", b"0", [(b"301", b"7", b"a"), (b"205", b"100", b"b"), (b"1", b"12", b"c")],
                         vocab)
    assert line == b"5\ts,1,0,301:20:a 1:21:c\n"
    assert oa.remap_line(1, b"s", b"1", b"0", [(b"205", b"100", b"b")], vocab) == b"1\ts,1,0,\n"
    # feat_cnts: field bytes, then the numeric fid
    assert oa.feat_cnts({(b"30", 9): 1, (b"205", 10): 1, (b"205", 9): 2, (b"2055", 1): 3}) == \
        b"205:9\t2\n205:10\t1\n2055:1\t3\n30:9\t1\n"


def _write_set(d, files):
    os.makedirs(d)
    for name, lines in files.items():
        with open(os.path.join(d, name), "wb") as fh:
            fh.write(b"\n".join(lines) + b"\n")


def test_prepare_orders_te_uses_tr_vocabulary_and_the_writer_reads_it(tmp_path):
    tr = [_common(b"M%d" % m, (b"301", b"%d" % (1000 + m % 3), b"1"), (b"216", b"%d" % (50 + m), b"1"))
          for m in range(4)]
    tr += [_sample(b"t%d" % j, b"%d" % (j % 2), b"0", b"M%d" % (j % 5), (b"205", b"%d" % (j % 4), b"1"),
                   (b"109_14", b"%d" % (j % 2), b"0.5")) for j in range(120)]
    te = [_common(b"M1", (b"301", b"1001", b"1"), (b"301", b"999999", b"1"))]
    te += [_sample(b"e%d" % j, b"1", b"%d" % (j % 2), b"M1", (b"205", b"%d" % j, b"1")) for j in range(30)]
    _write_set(str(tmp_path / "in" / "tr"), {"b_sample": tr[4:], "a_common": tr[:4]})
    _write_set(str(tmp_path / "in" / "te"), {"x": te})
    out = str(tmp_path / "out")
    stats = oa.prepare(str(tmp_path / "in"), out, parts=7, seed=3)
    assert stats["tr"]["lines"] == 124 and stats["tr"]["samples"] == 120 and stats["tr"]["no_common"] == 24
    assert stats["te"]["lines"] == 31 and stats["te"]["samples"] == 30
    vocab = oa.vocabulary(oa.stat(oa.join_reduce(oa.read_set(str(tmp_path / "in" / "tr"))[0])[0]))
    assert stats["feature_size"] == 20 + len(vocab) and sorted(vocab.values()) == list(range(20, 20 + len(vocab)))
    assert vocab == {0: 20, 1: 21, 2: 22, 3: 23, 50: 24, 51: 25, 52: 26, 53: 27, 1000: 28, 1001: 29, 1002: 30}
    # te: 205:j is kept for j < 4 only (tr's vocabulary), 999999 never
    te_lines = b"".join(open(os.path.join(out, "te", "part-%05d" % p), "rb").read() for p in range(7)).splitlines()
    assert len(te_lines) == 30 and all(b"999999" not in l for l in te_lines)
    assert sum(l.endswith(b"301:29:1") for l in te_lines) == 30
    for name, n in (("tr", 120), ("te", 30)):
        keys = []
        for p in range(7):
            data = open(os.path.join(out, name, "part-%05d" % p), "rb").read()
            rs = [int(l.split(b"\t")[0]) for l in data.splitlines()]
            assert all(r % 7 == p for r in rs) and rs == sorted(rs)
            keys += rs
        assert len(keys) == n
        # the TFRecord writer's restatement reads every part file
        ot.convert(os.path.join(out, name), str(tmp_path / ("tfr_" + name)))
    # r_i of line i is splitmix64(seed, i) >> 33, lines counted over the set's files in name order
    first = oa.shuffle_key(3, 4)           # a_common holds lines 0-3: the first sample is line 4
    assert any(l.startswith(b"%d\tt0,0,0," % first) for l in
               open(os.path.join(out, "tr", "part-%05d" % (first % 7)), "rb").read().splitlines())


def test_reference_remap_quirk_drops_everything():
    cnt = {(b"205", 3): 40, (b"301", 8): 25}
    fc = oa.feat_cnts(cnt)
    d = oa.load_fcnts_literal(fc)
    assert d == {b"205:3": 20, b"301:8": 21}
    joined = b"s0,1,0,205:3:1 301:8:1"
    assert oa.remap_literal(joined, d) == b"s0,1,0,"
    tokens = [(b"205", b"3", b"1"), (b"301", b"8", b"1")]
    assert oa.remap_line(9, b"s0", b"1", b"0", tokens, oa.vocabulary(cnt)) == b"9\ts0,1,0,205:20:1 301:21:1\n"
