"""Pure-Python restatement of deep_ctr/Feature_pipeline/get_criteo_feature.py (Criteo raw TSV -> libsvm).
TEST INFRASTRUCTURE ONLY (small files).  Python 2 semantics where they differ from Python 3:
  * lines are byte strings split on b'\\t' after dropping the b'\\n' (Python 2 `str`, :42,77,135,156);
  * random.randint(0, 9999) is int(random() * 10000) (Python 2's randrange), with random.seed(0) (:127,148);
  * feature_map is written in a defined order -- per field the ids 1..n, then <unk> -- where the reference writes
    Python 2 dict order; compare it as a set of lines."""
from __future__ import annotations

import random
import sys
from typing import Dict, List

import numpy as np

CONTINUOUS_CLIP = [20, 600, 100, 50, 64000, 500, 100, 50, 500, 10, 10, 10, 50]   # :25
N_INT, N_CAT = 13, 26
MAXSIZE = 2 ** 63 - 1   # Python 2's sys.maxsize on LP64 (:71-72)


def split_decisions_loop(n: int) -> List[bool]:
    """to tr.libsvm? for the first n train lines: Python 2's random.seed(0); randint(0, 9999) % 10 != 0."""
    r = random.Random(0)
    return [int(r.random() * 10000) % 10 != 0 for _ in range(n)]


def split_decisions(n: int, state: np.random.RandomState = None) -> np.ndarray:
    """The same decisions vectorised: RandomState([0]) seeds MT19937 by init_by_array([0]) as random.seed(0) does,
    and random_sample() is random()'s 53-bit draw.  Pass `state` to continue a stream."""
    rs = np.random.RandomState([0]) if state is None else state
    return (np.floor(rs.random_sample(n) * 10000).astype(np.int64) % 10) != 0


def fixed6(val: float) -> bytes:
    return "{0:.6f}".format(val).rstrip("0").rstrip(".").encode()   # :141


def _lines(path: str):
    with open(path, "rb") as fh:
        for line in fh:
            yield line.rstrip(b"\n").split(b"\t")


def preprocess(input_dir: str, output_dir: str, cutoff: int = 200) -> Dict:
    train, test = input_dir + "train.txt", input_dir + "test.txt"
    lo, hi = [MAXSIZE] * N_INT, [-MAXSIZE] * N_INT                              # :69-85
    for features in _lines(train):
        for i in range(N_INT):
            val = features[1 + i]
            if val != b"":
                val = min(int(val), CONTINUOUS_CLIP[i])
                lo[i], hi[i] = min(lo[i], val), max(hi[i], val)

    counts = [dict() for _ in range(N_CAT)]                                     # :39-45
    for features in _lines(train):
        for i in range(N_CAT):
            key = features[14 + i]
            if key != b"":
                counts[i][key] = counts[i].get(key, 0) + 1
    vocab = []                                                                   # :46-51
    for i in range(N_CAT):
        kept = sorted((kv for kv in counts[i].items() if kv[1] >= cutoff), key=lambda x: (-x[1], x[0]))
        keys, _ = list(zip(*kept))                                               # ValueError when nothing is kept
        vocab.append({k: j + 1 for j, k in enumerate(keys)})

    dict_sizes = [len(v) + 1 for v in vocab]                                     # + <unk>
    offset = [N_INT]
    fmap = [b"I%d %d\n" % (i, i) for i in range(1, N_INT + 1)]                    # :116-125
    for i in range(1, N_CAT + 1):
        offset.append(offset[i - 1] + dict_sizes[i - 1])
        for key, val in list(vocab[i - 1].items()) + [(b"<unk>", 0)]:
            fmap.append(b"C%d|%s %d\n" % (i, key, offset[i - 1] + val + 1))
    with open(output_dir + "feature_map", "wb") as fh:
        fh.write(b"".join(fmap))

    def row(features, shift):
        feats = []
        for i in range(N_INT):                                                   # :138-141, :159-161
            val = features[1 + i - shift]
            val = 0.0 if val == b"" else (float(val) - lo[i]) / (hi[i] - lo[i])
            feats.append(b"%d:%s" % (1 + i, fixed6(val)))
        for i in range(N_CAT):                                                   # :143-145, :163-165
            feats.append(b"%d:1" % (vocab[i].get(features[14 + i - shift], 0) + offset[i]))
        return b" ".join(feats)

    n_tr = n_va = 0
    label = None
    rs = np.random.RandomState([0])
    with open(output_dir + "tr.libsvm", "wb") as out_tr, open(output_dir + "va.libsvm", "wb") as out_va:
        for features in _lines(train):                                           # :131-151
            label = features[0]
            line = label + b" " + row(features, 0) + b"\n"
            if split_decisions(1, rs)[0]:
                out_tr.write(line); n_tr += 1
            else:
                out_va.write(line); n_va += 1
    n_te = 0
    with open(output_dir + "te.libsvm", "wb") as out:                            # :153-167
        for features in _lines(test):
            out.write(label + b" " + row(features, 1) + b"\n")                    # the last train line's label
            n_te += 1
    return {"dict_sizes": dict_sizes, "feature_size": offset[N_CAT], "offsets": offset[:N_CAT],
            "min": lo, "max": hi, "lines": {"tr": n_tr, "va": n_va, "te": n_te}}


if __name__ == "__main__":
    print(preprocess(sys.argv[1], sys.argv[2], int(sys.argv[3]) if len(sys.argv) > 3 else 200))
