"""Pure-Python restatement of DeepMTL/Feature_pipeline's Ali-CCP sample stage, the test oracle of
tf_repos_b200.aliccp_sample: the join (get_join_mapper.py, get_join_reducer.py), stat (get_stat_mapper.py,
get_stat_reducer.py) and remap (get_remap_mapper.py) jobs, one pure function per mapper and reducer, under Python 3 on
bytes (DESIGN.md §2.7):

- join_map: `line.strip().split(',')`; 3 fields = a common record `md5,feat_num,feat_list`, 6 fields = a sample
  `sample_id,y,z,md5,feat_num,feat_list`, else skipped.  A sample with y == '0' and z == '1' is dropped.  feat_list is
  split on \\x01; each token must split on \\x02 into 2 parts and the second on \\x03 into 2, or the whole line is skipped
  (the mapper's bare except); an empty list is skipped too.  feat_num is ignored.
- join_reduce: each sample `sample_id,y,z,<tokens as f:fid:val joined by ' '>`, then ' ' and the tokens of the common
  record with its md5, when there is one.  Of several records with one md5 the last in input order wins (in Hadoop the
  reducer's input order decides).
- stat: every token of every joined tr line counts 1 for its key `field:fid`; feat_cnts lines `field:fid\\t<count>`
  sorted by field bytes, then numeric fid (Hadoop's order is not fixed).
- remap: a fid is kept when any of its field:fid counts reaches cutoff; kept fids get ids 20, 21, ... in ascending
  numeric order; the tokens of dropped fids are dropped.  The shipped mapper looks its dict up by the bare fid while the
  keys are `field:fid` (get_remap_mapper.py:15,35-36), so literally it drops every feature: remap_literal restates that.
- shuffle: line i (0-based over all lines of the set's files, skipped ones included) gets r_i = splitmix64(seed, i) >> 33
  and goes to part r_i % parts, ordered by (r_i, i) within the part.

The implementation's restrictions raise OracleError, in the order NUL byte, sample_id, y, z, md5, then each token's
field, fid, val, for lines the reference keeps (not skipped, not filtered)."""
from __future__ import annotations

import os
import re
from typing import Dict, List, Optional, Tuple

FIRST_ID = 20
CUTOFF = 20
PARTS = 100
_M64 = (1 << 64) - 1
_BAD = re.compile(rb"[\x00-\x03\t\n\x0b\x0c\r :]")
_FID = re.compile(rb"(0|[1-9][0-9]*)\Z")


def splitmix64(seed: int, i: int) -> int:
    """The (i+1)-th output of SplitMix64 seeded with `seed`: z = seed + (i+1)*0x9E3779B97F4A7C15 mod 2^64, then
    z = (z ^ z>>30) * 0xBF58476D1CE4E5B9, z = (z ^ z>>27) * 0x94D049BB133111EB, z ^ z>>31 (all mod 2^64)."""
    z = (seed + (i + 1) * 0x9E3779B97F4A7C15) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def shuffle_key(seed: int, i: int) -> int:
    return splitmix64(seed, i) >> 33


class OracleError(ValueError):
    def __init__(self, line: int, kind: str, token: bytes):
        super().__init__(f"line {line}: {kind}: {token!r}")
        self.line, self.kind, self.token = line, kind, token


Token = Tuple[bytes, bytes, bytes]


def split_tokens(feat_list: bytes) -> Optional[List[Token]]:
    """get_join_mapper.py:21-24 / 34-37: (field, fid, val) per \\x01 token, or None where the mapper's except skips."""
    out = []
    for fstr in feat_list.split(b"\x01"):
        a = fstr.split(b"\x02")
        if len(a) != 2:
            return None
        b = a[1].split(b"\x03")
        if len(b) != 2:
            return None
        out.append((a[0], b[0], b[1]))
    return out


def restriction(stripped: bytes, fields: List[bytes], tokens: List[Token]) -> Optional[Tuple[str, bytes]]:
    if b"\0" in stripped:
        return "nul", stripped
    text = (fields[:3] if len(fields) == 6 else []) + [fields[-3]]
    for t in text[:-1]:
        if _BAD.search(t):
            return "text", t
    md5 = text[-1]
    if not 1 <= len(md5) <= 64:
        return "md5", md5
    if _BAD.search(md5):
        return "text", md5
    for field, fid, val in tokens:
        if not 1 <= len(field) <= 16 or _BAD.search(field):
            return "field", field
        if not _FID.match(fid) or int(fid) >= (1 << 63):
            return "fid", fid
        if _BAD.search(val):
            return "text", val
    return None


def join_map(line: bytes, line_no: int = 0):
    """One raw line -> ('common', md5, tokens) | ('sample', md5, (sample_id, y, z), tokens) | ('filtered',) |
    ('malformed',).  Raises OracleError for a kept line that breaks a restriction."""
    s = line.strip()
    f = s.split(b",")
    if len(f) == 6 and f[1] == b"0" and f[2] == b"1":
        return ("filtered",)
    if len(f) not in (3, 6):
        return ("malformed",)
    tokens = split_tokens(f[-1])
    if tokens is None:
        return ("malformed",)
    bad = restriction(s, f, tokens)
    if bad:
        raise OracleError(line_no, *bad)
    if len(f) == 3:
        return ("common", f[0], tokens)
    return ("sample", f[3], (f[0], f[1], f[2]), tokens)


def join_reduce(mapped: List[tuple]) -> Tuple[List[Tuple[int, bytes, bytes, bytes, List[Token]]], Dict]:
    """-> joined samples (line index, sample_id, y, z, tokens incl. the common ones) in line order, and stats."""
    common: Dict[bytes, List[Token]] = {}
    n_common = 0
    for m in mapped:
        if m[1][0] == "common":
            common[m[1][1]] = m[1][2]      # the last record of an md5 wins
            n_common += 1
    joined, no_common = [], 0
    for i, m in mapped:
        if m[0] == "sample":
            c = common.get(m[1])
            no_common += c is None
            joined.append((i, *m[2], m[3] + (c or [])))
    stats = {"commons": n_common, "commons_superseded": n_common - len(common), "no_common": no_common,
             "samples": len(joined), "filtered": sum(m[0] == "filtered" for _, m in mapped),
             "malformed": sum(m[0] == "malformed" for _, m in mapped)}
    return joined, stats


def stat(joined) -> Dict[Tuple[bytes, int], int]:
    """get_stat_mapper.py + get_stat_reducer.py: count per field:fid (fid as its number: its text is canonical)."""
    cnt: Dict[Tuple[bytes, int], int] = {}
    for *_, tokens in joined:
        for field, fid, _ in tokens:
            k = (field, int(fid))
            cnt[k] = cnt.get(k, 0) + 1
    return cnt


def feat_cnts(cnt) -> bytes:
    return b"".join(b"%s:%d\t%d\n" % (f, fid, c) for (f, fid), c in sorted(cnt.items()))


def vocabulary(cnt, cutoff: int = CUTOFF) -> Dict[int, int]:
    kept = sorted({fid for (_, fid), c in cnt.items() if c >= cutoff})
    return {fid: FIRST_ID + j for j, fid in enumerate(kept)}


def remap_line(r: int, sid: bytes, y: bytes, z: bytes, tokens: List[Token], vocab: Dict[int, int]) -> bytes:
    kept = [b"%s:%d:%s" % (f, vocab[int(fid)], v) for f, fid, v in tokens if int(fid) in vocab]
    return b"%d\t%s,%s,%s,%s\n" % (r, sid, y, z, b" ".join(kept))


def load_fcnts_literal(feat_cnts_text: bytes) -> Dict[bytes, int]:
    """get_remap_mapper.py:10-21 as shipped: keys are the `field:fid` of each line, ids from 20 in file order."""
    d: Dict[bytes, int] = {}
    new_id = FIRST_ID
    for line in feat_cnts_text.splitlines():
        fid, cnts = line.strip().split(b"\t")
        if d.get(fid):
            continue
        if int(cnts) >= CUTOFF:
            d[fid] = new_id
            new_id += 1
    return d


def remap_literal(joined_line: bytes, d: Dict[bytes, int]) -> Optional[bytes]:
    """get_remap_mapper.py:28-40 as shipped, without the random key: it looks up the bare fid, which is never a key."""
    try:
        splits = joined_line.strip().split(b",")
        if splits[1] == b"0" and splits[2] == b"1":
            return None
        feat_lists = []
        for fstr in splits[3].split(b" "):
            f, fid, val = fstr.split(b":")
            new_id = d.get(fid)
            if new_id:
                feat_lists.append(b"%s:%d:%s" % (f, new_id, val))
        return b"%s,%s,%s,%s" % (splits[0], splits[1], splits[2], b" ".join(feat_lists))
    except (ValueError, IndexError):
        return None


def joined_text(sid, y, z, tokens) -> bytes:
    """The join reducer's output line for one sample (without the Hadoop key)."""
    return b"%s,%s,%s,%s" % (sid, y, z, b" ".join(b":".join(t) for t in tokens))


def lines_of(data: bytes) -> List[bytes]:
    parts = data.split(b"\n")
    if parts and parts[-1] == b"":
        parts.pop()
    return parts


def read_set(d: str):
    """Every file of d in sorted name order -> [(line index, join_map)], raising OracleError with the file's name."""
    mapped, i = [], 0
    for name in sorted(os.listdir(d)):
        path = os.path.join(d, name)
        if not os.path.isfile(path):
            continue
        with open(path, "rb") as fh:
            for n, line in enumerate(lines_of(fh.read()), 1):
                try:
                    mapped.append((i, join_map(line, n)))
                except OracleError as e:
                    e.path = path
                    raise
                i += 1
    return mapped, i


def shuffle(joined, vocab, seed: int, parts: int) -> Tuple[List[bytes], int]:
    """-> the text of each part file, and the lines left with an empty feature field."""
    out = [[] for _ in range(parts)]
    empty = 0
    for i, sid, y, z, tokens in joined:
        r = shuffle_key(seed, i)
        line = remap_line(r, sid, y, z, tokens, vocab)
        empty += line.endswith(b",\n")
        out[r % parts].append((r, i, line))
    return [b"".join(l for _, _, l in sorted(p)) for p in out], empty


def prepare(input_dir: str, output_dir: str, cutoff: int = CUTOFF, parts: int = PARTS, seed: int = 0) -> Dict:
    """The whole stage: output_dir/{tr,te}/part-%05d and output_dir/feat_cnts; -> the same stats as the product."""
    result = {}
    vocab = None
    for name in ("tr", "te"):
        mapped, n_lines = read_set(os.path.join(input_dir, name))
        joined, st = join_reduce(mapped)
        if name == "tr":
            cnt = stat(joined)
            vocab = vocabulary(cnt, cutoff)
            os.makedirs(output_dir, exist_ok=True)
            with open(os.path.join(output_dir, "feat_cnts"), "wb") as fh:
                fh.write(feat_cnts(cnt))
        texts, empty = shuffle(joined, vocab, seed, parts)
        os.makedirs(os.path.join(output_dir, name), exist_ok=True)
        for p, t in enumerate(texts):
            with open(os.path.join(output_dir, name, "part-%05d" % p), "wb") as fh:
                fh.write(t)
        result[name] = dict(st, lines=n_lines, empty_lines=empty)
    return {"feature_size": FIRST_ID + len(vocab), "kept_fids": len(vocab), **result}
