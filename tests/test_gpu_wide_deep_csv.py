"""wide_n_deep's CSV input tokenised on the GPU (csrc/csv_device.cu, wide_deep_main.input_fn(device=)) against the host
decoder (wide_deep_main.decode_csv_file): the bits of everything the kernel accepts, the counter of everything it
declines and the host's answer or error for it, the batch sequence of a streamed multi-file multi-epoch input, and the
drop-in script with --input_parse=device against --input_parse=host."""
import os
import struct
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_FLOAT, N_INT = 14, 26


def _in_fast_path(s):
    """what decimal.cuh::parse_float converts itself: normal fp32 range, away from an fp32 rounding boundary"""
    d = abs(float(s))
    if d == 0.0:
        return True
    low = struct.unpack("<Q", struct.pack("<d", d))[0] & 0x1FFFFFFF
    return 1.1754943508222875e-38 <= d <= 3.4028234663852886e38 and not 0x0FFFFFFF <= low <= 0x10000001


def _float_field(g):
    """1-15 significant digits, the point anywhere (".5", "5."), e+-0..22, signs -- kept inside the fast path"""
    while True:
        n = int(g.integers(1, 16))
        digits = str(int(g.integers(1, 10))) + "".join(str(int(v)) for v in g.integers(0, 10, n - 1))
        pos = int(g.integers(0, n + 1))
        ex = int(g.integers(-22, 23))
        if not -22 <= ex - (n - pos) <= 22 or not -30 <= pos + ex <= 30:
            continue
        head = digits[:pos] or ("0" if g.integers(2) else "")
        tail = digits[pos:]
        body = head + ("." + tail if tail or g.integers(2) else "")
        if ex or g.integers(2):
            body += "eE"[int(g.integers(2))] + (["", "+"][int(g.integers(2))] if ex >= 0 else "-") + \
                    ("%02d" if g.integers(2) else "%d") % abs(ex)
        s = ["", "+", "-"][int(g.integers(3))] + body
        if _in_fast_path(s):
            return s


def _line(g, special=0.2):
    fl = [g.choice(["", "-0", "+7", "007", "0", "1", "0.5"]) if g.random() < special else _float_field(g)
          for _ in range(N_FLOAT)]
    it = [g.choice(["", "0", "9999", "10000", "-1", "999999999", "-0", "+7", "007", "-999999999"])
          if g.random() < 0.5 else str(int(g.integers(0, 10 ** int(g.integers(1, 10))))) for _ in range(N_INT)]
    return ",".join(list(fl) + list(it))


def _plain_line(g):
    return ",".join([str(int(g.integers(2)))] + ["%.6f" % v for v in g.random(13)] +
                    [str(int(v)) for v in g.integers(0, 12000, 26)])


def _parse(data: bytes):
    """the kernel alone on one piece -> (labels, dense, cat) host arrays of its rows, info"""
    from tf_repos_b200 import ops, text_chunks
    text = text_chunks.upload(data, "cuda")
    max_rows = data.count(b"\n") + 1
    ws = text_chunks.scratch(ops.parse_csv_device_workspace_bytes(len(data), max_rows), "cuda")
    labels, dense, cat, info = ops.parse_csv_device(text, len(data), N_FLOAT, N_INT, max_rows, ws)
    info = info.tolist()
    return tuple(t[:info[0]].cpu().numpy() for t in (labels, dense, cat)), info


def _same_bits(got, want):
    for a, b in zip(got, want):
        a, b = np.asarray(a), np.asarray(b)
        assert a.dtype == b.dtype and a.shape == b.shape
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_accepted_input_has_the_host_decoders_bits(tmp_path):
    from tf_repos_b200 import wide_deep_main as wm
    g = np.random.default_rng(11)
    lines = [_line(g) for _ in range(3000)]
    lines[5] = "," * (N_FLOAT + N_INT - 1)                                  # every field empty
    text = "".join(ln + ("\r\n" if i % 3 == 0 else "\n") for i, ln in enumerate(lines)) + _line(g)   # no '\n' at the end
    p = os.path.join(tmp_path, "tr.csv")
    open(p, "wb").write(text.encode())
    want = wm.decode_csv_file(p)
    got, info = _parse(text.encode())
    assert info == [3001, len(text), 0, 0, 0]
    _same_bits(got, want)
    assert np.signbit(want[1]).any() and (want[2] == 999999999).any() and (want[2] == -1).any()
    # and through input_fn, one batch holding everything
    (dense, cat, labels), = wm.input_fn([p], 1, 4000, device="cuda")
    assert dense.is_cuda and cat.is_cuda and labels.is_cuda
    _same_bits((labels.cpu().numpy(), dense.cpu().numpy(), cat.cpu().numpy()), want)


def _with_field(g, col, value):
    cols = _plain_line(g).split(",")
    cols[col] = value
    return ",".join(cols)


DECLINES = {   # name -> (the line, the info counter that takes it)
    "blank_line": (lambda g: "", 2),
    "fields_39": (lambda g: _plain_line(g).rsplit(",", 1)[0], 3),
    "fields_41": (lambda g: _plain_line(g) + ",1", 3),
    "quoted_field": (lambda g: _with_field(g, 3, '"5"'), 3),
    "blank_in_field": (lambda g: _with_field(g, 3, " 5"), 3),
    "tab_in_int_field": (lambda g: _with_field(g, 20, "5\t"), 3),
    "float_1e400": (lambda g: _with_field(g, 3, "1e400"), 4),
    "float_inf": (lambda g: _with_field(g, 3, "inf"), 4),
    "float_nan": (lambda g: _with_field(g, 0, "nan"), 4),
    "float_17_digits": (lambda g: _with_field(g, 3, "0.12345678901234567"), 4),
    "float_on_fp32_boundary": (lambda g: _with_field(g, 3, "16777217"), 4),      # 2^24 + 1: halfway between two fp32
    "float_subnormal": (lambda g: _with_field(g, 3, "1e-40"), 4),
    "float_underscore": (lambda g: _with_field(g, 3, "1_0"), 4),
    "float_abc": (lambda g: _with_field(g, 3, "abc"), 4),
    "id_10_digits": (lambda g: _with_field(g, 20, "1234567890"), 4),
    "id_5.0": (lambda g: _with_field(g, 20, "5.0"), 4),
    "id_abc": (lambda g: _with_field(g, 39, "abc"), 4),
    "lone_cr": (lambda g: _with_field(g, 20, "5\r6"), 4),
}


def _all_batches(files, epochs, B, device, chunk_bytes):
    """the batches as host arrays, or the ValueError the generator raised"""
    from tf_repos_b200 import wide_deep_main as wm
    out = []
    try:
        for batch in wm.input_fn(files, epochs, B, device=device, chunk_bytes=chunk_bytes):
            out.append(tuple(t.cpu().numpy() for t in batch))
    except ValueError as e:
        return str(e)
    return out


def _same_batches(got, want):
    assert type(got) is type(want)
    if isinstance(want, str):
        assert got == want
        return
    assert len(got) == len(want)
    for a, b in zip(got, want):
        _same_bits(a, b)


@pytest.mark.parametrize("name", sorted(DECLINES))
def test_declined_input_is_counted_and_decoded_by_the_host(tmp_path, name):
    make, slot = DECLINES[name]
    g = np.random.default_rng(5)
    lines = [_plain_line(g) for _ in range(60)]
    lines[45] = make(g)                                   # file line 46, in the second 4 KB piece
    data = ("\n".join(lines) + "\n").encode()
    _, info = _parse(data)
    want_info = [0, 0, 0]
    want_info[slot - 2] = 1
    assert info[0] == 60 and info[1] == len(data) and info[2:] == want_info
    p = os.path.join(tmp_path, "tr.csv")
    open(p, "wb").write(data)
    want = _all_batches([p], 1, 7, None, 4096)
    got = _all_batches([p], 1, 7, "cuda", 4096)
    _same_batches(got, want)
    if name.startswith("fields_"):
        assert want.startswith("%s:46: Expect 40 fields but have %s in record" % (p, name[-2:]))
    elif name in ("quoted_field", "float_abc", "id_5.0", "id_abc", "lone_cr"):
        assert isinstance(want, str)                      # float() / int() refuse it, or the line is cut in two
    else:
        assert sum(len(b[2]) for b in want) == (59 if name == "blank_line" else 60)


def test_streamed_batches_equal_the_host_generators(tmp_path):
    g = np.random.default_rng(9)
    files = []
    for k, n in enumerate((211, 97)):
        lines = [_line(g, special=0.5) if i % 4 else _plain_line(g) for i in range(n)]
        if k == 0:
            lines[100] = _with_field(g, 2, "0" * 5000 + "1.5")          # one line longer than a piece
            lines[150] = _with_field(g, 2, " 5")                        # one piece goes to the host decoder
        p = os.path.join(tmp_path, "tr%d.csv" % k)
        open(p, "wb").write(("\n".join(lines) + ("\n" if k == 0 else "")).encode())
        files.append(p)
    assert os.path.getsize(files[0]) > 5 * 4096
    want = _all_batches(files, 3, 37, None, 4096)
    got = _all_batches(files, 3, 37, "cuda", 4096)
    assert [len(b[2]) for b in want] == [37] * (3 * 308 // 37) + [3 * 308 % 37]
    _same_batches(got, want)
    # a batch is three contiguous row-major tensors, as WideDeep.train_step takes them
    from tf_repos_b200 import wide_deep_main as wm
    for dense, cat, labels in wm.input_fn(files, 1, 37, device="cuda", chunk_bytes=4096):
        assert dense.is_contiguous() and cat.is_contiguous() and dense.dtype == torch.float32 and cat.dtype == torch.int32
        assert dense.shape[1:] == (13,) and cat.shape[1:] == (26,) and labels.shape == dense.shape[:1]


def test_cli_device_and_host_parse_give_the_same_model(tmp_path):
    g = np.random.default_rng(3)
    runs = {}
    for mode in ("device", "host"):
        tmp = os.path.join(tmp_path, mode)
        os.makedirs(tmp + "/data")
    for name, n in (("tr0.csv", 300), ("va0.csv", 50), ("te0.csv", 77)):
        text = "".join(_plain_line(g) + "\n" for _ in range(n))
        for mode in ("device", "host"):
            open(os.path.join(tmp_path, mode, "data", name), "w").write(text)
    for mode in ("device", "host"):
        tmp = os.path.join(tmp_path, mode)
        common = [sys.executable, os.path.join(ROOT, "Model_pipeline", "wide_n_deep.py"), "--embedding_size=8",
                  "--batch_size=32", "--deep_layers=32,16", "--num_epochs=2", "--log_steps=5", "--data_dir=" + tmp + "/data",
                  "--model_dir=" + tmp + "/ckpt/m_", "--dt_dir=20261016"] + \
                 (["--input_parse=host"] if mode == "host" else [])          # device is the default
        out = []
        for task in ("train", "predict"):
            r = subprocess.run(common + ["--task_type=" + task], capture_output=True, text=True, timeout=280)
            assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
            out.append(r.stdout)
        loss = [ln for ln in out[0].splitlines() if ln.startswith("INFO:Loss for final step")]
        evals = [ln for ln in out[0].splitlines() if ln.startswith("INFO:Saving dict")]
        assert len(loss) == 1 and len(evals) == 1
        runs[mode] = (open(tmp + "/data/pred.txt", "rb").read(), loss[0], evals[0])
    assert runs["device"] == runs["host"]
    assert len(runs["device"][0].split()) == 77
