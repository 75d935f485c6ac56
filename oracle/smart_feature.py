"""Pure-Python restatement of deep_ctr/Feature_pipeline/get_smart_feature.py (CSV -> libsvm through feature_map, and
its get_feature_map builder) and get_frape_feature.py (the Frappe label rewrite).
TEST INFRASTRUCTURE ONLY (small files, one thread).  Python 2 semantics where they differ from Python 3:
  * lines are byte strings that end at b'\\n' only; strip() removes Python 2's whitespace b' \\t\\n\\r\\x0b\\x0c' and
    nothing else (Python 3's str.strip() would also remove \\x1c-\\x1f);
  * get_feature_map is run with its NameError fixed (CSV_COLUMNS[i] at :32 read as fname).
Written to the deviations of DESIGN.md §2.12: sorted input order, several va / te inputs concatenated into one file,
colliding output names and short tr paths raise before anything is written, and the builder's feature_map in fid
order (compare it as a set of lines)."""
from __future__ import annotations

import glob
from typing import Dict, List, Optional

WS = b" \t\n\r\x0b\x0c"
NAMED = [b"is_click", b"u_pl", b"u_ppvn", b"u_de", b"u_os", b"u_t", b"a_m_w", b"a_b_w", b"c_h", b"c_w", b"c_al",
         b"u_ctr", b"a_a_ctr", b"a_t_ctr", b"c_q_ctr", b"c_al_ctr", b"c_n_ctr", b"c_t_ctr", b"c_t_n_ctr",
         b"u_a_city_ctr", b"u_a_age_ctr", b"u_a_x_ctr", b"u_a_g_ctr", b"u_a_c_ctr", b"c_q_a_ctr", b"c_q_t_sim",
         b"c_q_adtype_ctr", b"c_mw_a_ctr"]
COLUMNS = NAMED + [b"xgbf_%d" % i for i in range(100)]


class OracleError(ValueError):
    pass


def continuous(i: int) -> bool:
    return 11 <= i <= 27


def _lines(path: str):
    with open(path, "rb") as fh:
        yield from fh                                   # binary files split after each b'\n' only


def load_map(path: str) -> Dict[bytes, bytes]:
    fmap = {}
    for line in _lines(path):
        s = line.strip(WS).split(b" ")
        if len(s) < 2:                                  # splits[1] raises IndexError: the line is skipped
            continue
        fmap[s[0]] = s[1]
    return fmap


def smart_line(line: bytes, fmap: Dict[bytes, bytes]) -> Optional[bytes]:
    """The output line, or None where the reference's try block swallows an IndexError."""
    s = line.strip(WS).split(b",")
    feats = []
    for i in range(1, len(s) - 1):
        if i >= len(COLUMNS):
            return None
        if continuous(i):
            fid = fmap.get(COLUMNS[i])
            feats.append((b"None" if fid is None else fid) + b":" + s[i])
        else:
            fid = fmap.get(COLUMNS[i] + b"|" + s[i])
            if fid is None:
                fid = fmap.get(COLUMNS[i] + b"|UNK")
            feats.append((b"None" if fid is None else fid) + b":1")
    return s[0] + b" " + b" ".join(feats) + b"\n"


def feature_map_text(files: List[str]) -> bytes:
    fmap, fid = {}, 1
    for name in COLUMNS:
        fmap[name + b"|UNK"] = fid
        fid += 1
    for path in files:
        for line in _lines(path):
            s = line.strip(WS).split(b",")
            for i in range(1, len(s) - 1):
                if i >= len(COLUMNS):                   # IndexError: the rest of this line is skipped
                    break
                key = COLUMNS[i] if continuous(i) else COLUMNS[i] + b"|" + s[i]
                if key not in fmap:
                    fmap[key] = fid
                    fid += 1
    return b"".join(b"%s %d\n" % kv for kv in fmap.items())   # insertion order is fid order


def _unique(outs):
    names = [o for o, _ in outs]
    if len(set(names)) != len(names):
        raise OracleError("two inputs write the same output")
    return outs


def smart_feature(input_dir: str, output_dir: str, task_type: str = "tr", build: bool = False) -> Dict:
    pattern = {"tr": "/*part*", "va": "/*verify", "te": "/*test"}[task_type]
    files = sorted(glob.glob(input_dir + pattern))
    if task_type == "tr":
        outs = []
        for p in files:
            parts = p.rsplit("_")
            if len(parts) < 4:
                raise OracleError(p + ": fewer than 4 '_' pieces")
            outs.append((output_dir + "tr_" + parts[3] + ".libsvm", [p]))
        outs = _unique(outs)
    else:
        outs = [(output_dir + task_type + ".libsvm", files)] if files else []
    if build:
        with open(output_dir + "feature_map", "wb") as fh:
            fh.write(feature_map_text(sorted(glob.glob(input_dir + "/*part*"))))
    fmap = load_map(output_dir + "feature_map")
    lines = {}
    for out, ins in outs:
        n_in = n_out = 0
        with open(out, "wb") as fh:
            for p in ins:
                for line in _lines(p):
                    n_in += 1
                    o = smart_line(line, fmap)
                    if o is not None:
                        fh.write(o)
                        n_out += 1
        lines[out] = (n_in, n_out)
    return {"outputs": [o for o, _ in outs], "lines": lines}


def frappe_line(line: bytes) -> Optional[bytes]:
    s = line.strip(WS).split(b" ", 1)
    if len(s) != 2:                                     # ValueError on unpacking: the line is skipped
        return None
    label = b"0" if s[0] == b"-1" else s[0]
    return label + b" " + s[1] + b"\n"


def frappe_feature(input_dir: str) -> Dict:
    outs = _unique([(p.split(".")[0] + "_.libsvm", [p]) for p in sorted(glob.glob(input_dir + "/*libsvm"))])
    lines = {}
    for out, (p,) in outs:
        n_in = n_out = 0
        with open(out, "wb") as fh:
            for line in _lines(p):
                n_in += 1
                o = frappe_line(line)
                if o is not None:
                    fh.write(o)
                    n_out += 1
        lines[out] = (n_in, n_out)
    return {"outputs": [o for o, _ in outs], "lines": lines}
