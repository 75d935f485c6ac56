"""wide_n_deep's host CSV decoder once a piece of a file can be decoded on its own (wide_deep_main.decode_csv_bytes, what
the device input path falls back to): the piece's errors name the file's line numbers, and decode_csv_file returns what
it returned before."""
import os

import numpy as np
import pytest

LINE1 = "1," + ",".join("%.2f" % (0.1 * i) for i in range(13)) + "," + ",".join(str(100 + i) for i in range(26))
LINE2 = "0," + ",".join("" for _ in range(13)) + "," + ",".join("" for _ in range(26))     # all defaults


def test_decode_csv_file_on_the_reader_tests_inputs(tmp_path):
    from tf_repos_b200 import wide_deep_main as wm
    p = os.path.join(tmp_path, "tr.csv")
    open(p, "w").write(LINE1 + "\n" + LINE2 + "\n")
    labels, dense, cat = wm.decode_csv_file(p)
    assert labels.dtype == np.float32 and dense.dtype == np.float32 and cat.dtype == np.int32
    assert labels.tolist() == [1.0, 0.0] and dense.shape == (2, 13) and cat.shape == (2, 26)
    assert np.array_equal(dense[0], np.asarray([float("%.2f" % (0.1 * i)) for i in range(13)], dtype=np.float32))
    assert not dense[1].any() and not cat[1].any() and cat[0].tolist() == [100 + i for i in range(26)]
    open(p, "w").write("1,2,3\n")
    with pytest.raises(ValueError) as e:
        wm.decode_csv_file(p)
    assert str(e.value) == "%s:1: Expect 40 fields but have 3 in record" % p
    open(p, "w").write("")
    labels, dense, cat = wm.decode_csv_file(p)
    assert labels.shape == (0,) and dense.shape == (0, 13) and cat.shape == (0, 26)


def test_decode_csv_bytes_is_decode_csv_file_of_the_piece_with_file_line_numbers(tmp_path):
    from tf_repos_b200 import wide_deep_main as wm
    p = os.path.join(tmp_path, "tr.csv")
    text = LINE1 + "\r\n" + "\n" + LINE2 + "\n" + LINE1          # a blank line, "\r\n", no '\n' at the end
    open(p, "wb").write(text.encode())
    want = wm.decode_csv_file(p)
    *got, n_lines = wm.decode_csv_bytes(text.encode(), p, 0)
    assert n_lines == 4 and all(np.array_equal(a, b) and a.dtype == b.dtype for a, b in zip(got, want))
    # the same error, whichever way the line is reached: as line 7 of the file, or as line 2 of a piece after 5 lines
    body = (LINE1 + "\n") * 5
    piece = LINE2 + "\n" + "1,2,3\n"
    open(p, "w").write(body + piece)
    with pytest.raises(ValueError) as whole:
        wm.decode_csv_file(p)
    with pytest.raises(ValueError) as part:
        wm.decode_csv_bytes(piece.encode(), p, 5)
    assert str(part.value) == str(whole.value) == "%s:7: Expect 40 fields but have 3 in record" % p
    # a lone '\r' ends a line for open(path, "r"), so it does for a piece
    *_, n_lines = wm.decode_csv_bytes((LINE1 + "\r" + LINE2 + "\n").encode(), p, 0)
    assert n_lines == 2
