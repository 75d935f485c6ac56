"""GPU libsvm tokenizer (csrc/libsvm_device.cu, SURVEY.md 8f-1) against the host parser (strtof/strtol) and the
pure-Python oracle (oracle/libsvm.py restating decode_libsvm, DeepFM.py:65-81): bit-exact."""
import os
import random

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _host(data: bytes, F: int):
    from tf_repos_b200 import input_fn
    return input_fn._parse(data, 0, len(data), F)


def _device(data: bytes, F: int, max_rows=None, final=True):
    from tf_repos_b200 import ops
    text = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    mr = max_rows if max_rows is not None else max(1, len(data) // (2 * F + 2))
    return ops.parse_libsvm_device(text, F, mr, final)


def _same(dev_out, host_out):
    ids, vals, labels, _, needs_host = dev_out
    assert not needs_host
    assert np.array_equal(ids.cpu().numpy(), host_out[0])
    assert np.array_equal(vals.cpu().numpy().view(np.uint32), host_out[1].view(np.uint32))      # bit-exact floats
    assert np.array_equal(labels.cpu().numpy().view(np.uint32), host_out[2].view(np.uint32))


def _rand_val(rng):
    k = rng.randrange(8)
    if k == 0:
        return "1"
    if k == 1:
        return "%.6f" % rng.random()
    if k == 2:
        return repr(rng.random() * 10 ** rng.randrange(-8, 8))       # up to 17 digits -> some go to the host path
    if k == 3:
        return "%.3e" % (rng.random() * 10 ** rng.randrange(-20, 20))
    if k == 4:
        return "%d" % rng.randrange(0, 10 ** rng.randrange(1, 12))
    if k == 5:
        return "-%.4f" % rng.random()
    if k == 6:
        return "0.%s" % "".join(rng.choice("0123456789") for _ in range(rng.randrange(1, 12)))
    return "%g" % (rng.random() * 100)


def test_criteo_like_file_matches_host_and_oracle(tmp_path):
    from oracle import libsvm as olib
    from tf_repos_b200 import input_fn, synth
    ids, vals, labels = synth.criteo_batch(3000, 100_000, 39, seed=5)
    path = os.path.join(tmp_path, "tr.libsvm")
    synth.write_libsvm(path, ids, vals, labels)
    data = open(path, "rb").read()
    h = _host(data, 39)
    _same(_device(data, 39), h)
    dev = _device(data, 39)
    for r, ln in enumerate(data.decode().splitlines()[:200]):      # the oracle, line by line
        o_ids, o_vals, o_lab = olib.decode_libsvm(ln)
        assert np.array_equal(dev[0][r].cpu().numpy(), o_ids)
        assert np.array_equal(dev[1][r].cpu().numpy().view(np.uint32), o_vals.view(np.uint32))
        assert np.float32(dev[2][r].item()) == o_lab
    (d, _), = input_fn.input_fn(path, batch_size=3000, field_size=39, device="cuda")
    assert np.array_equal(d["feat_ids"][..., 0].cpu().numpy(), h[0])
    assert np.array_equal(d["feat_vals"][..., 0].cpu().numpy(), h[1])
    # unterminated last line, CRLF, runs of spaces
    data2 = data.rstrip(b"\n").replace(b"\n", b"\r\n", 5).replace(b" ", b"   ", 7)
    _same(_device(data2, 39), _host(data2, 39))
    # max_rows smaller than the file: the first rows and the byte position after them
    ids_d, vals_d, labels_d, consumed, nh = _device(data, 39, max_rows=100)
    assert ids_d.shape[0] == 100 and not nh
    assert consumed == len(b"\n".join(data.split(b"\n")[:100])) + 1
    assert np.array_equal(ids_d.cpu().numpy(), h[0][:100])
    # not the final chunk: an unterminated tail stays unparsed
    cut = data[: len(data) - 7]
    ids_c, _, _, consumed_c, _ = _device(cut, 39, final=False)
    assert consumed_c == cut.rfind(b"\n") + 1 and ids_c.shape[0] == cut.count(b"\n")


def test_number_formats_bit_exact_or_declined():
    """Every line the device accepts carries the host's bits; lines it declines are counted, never guessed."""
    rng = random.Random(7)
    F = 6
    accepted = declined = 0
    for _ in range(40):
        lines = []
        for _ in range(200):
            lines.append("%s %s" % (rng.choice(["0", "1", "0.0", "1.0"]),
                                    " ".join("%d:%s" % (rng.randrange(0, 2 ** 31 - 1), _rand_val(rng)) for _ in range(F))))
        data = ("\n".join(lines) + "\n").encode()
        ids, vals, labels, consumed, needs_host = _device(data, F)
        if needs_host:
            declined += 1
            # line by line: whatever is accepted must still be exact
            for ln in lines:
                d1 = (ln + "\n").encode()
                o = _device(d1, F)
                if not o[4]:
                    _same(o, _host(d1, F))
            continue
        accepted += 1
        _same((ids, vals, labels, consumed, needs_host), _host(data, F))
    assert accepted + declined == 40


@pytest.mark.parametrize("line", [
    "1 3:0.5 4:1",                 # too few pairs
    "1 3:0.5 4:1 5:2 6:3",         # too many
    "x 3:0.5 4:1 5:2",             # label not a number
    "1 3:0.5 4 5:2",               # token without ':'
    "1 3:0.5x 4:1 5:2",            # garbage after a value
    "1 3:inf 4:1 5:2",             # host decides
    "1 3:0.1234567890123456789 4:1 5:2",   # > 15 digits: host decides
    "1 3:1e-45 4:1 5:2",           # fp32 subnormal: host decides
    "1 12345678901:1 4:1 5:2",     # id beyond int32: host decides
    "",                            # blank line
])
def test_declined_lines_are_flagged(line):
    data = ("1 1:1 2:2 3:3\n" + line + "\n1 1:1 2:2 3:3\n").encode()
    assert _device(data, 3)[4] is True


def test_input_fn_device_batches_equal_host_batches(tmp_path):
    """repeat-before-batch semantics (DeepFM.py:83-95): same batch boundaries and values from both parsers."""
    from tf_repos_b200 import input_fn, synth
    paths = []
    for k, n in enumerate((130, 75)):
        ids, vals, labels = synth.criteo_batch(n, 5000, 15, seed=20 + k)
        p = os.path.join(tmp_path, "tr%d.libsvm" % k)
        synth.write_libsvm(p, ids, vals, labels)
        paths.append(p)
    host = list(input_fn.input_fn(paths, batch_size=64, num_epochs=2, field_size=15))
    dev = list(input_fn.input_fn(paths, batch_size=64, num_epochs=2, field_size=15, device="cuda"))
    assert len(host) == len(dev) == (2 * 205 + 63) // 64
    for (hf, hl), (df, dl) in zip(host, dev):
        assert df["feat_ids"].is_cuda and df["feat_ids"].shape == hf["feat_ids"].shape
        assert torch.equal(df["feat_ids"].cpu(), hf["feat_ids"]) and torch.equal(df["feat_vals"].cpu(), hf["feat_vals"])
        assert torch.equal(dl.cpu(), hl)


def _lines(n, F, seed):
    from tf_repos_b200 import synth
    ids, vals, labels = (t.numpy() for t in synth.criteo_batch(n, 5000, F, seed=seed))
    return ["%d " % labels[r] + " ".join("%d:%.6g" % (ids[r, f], vals[r, f]) for f in range(F)) for r in range(n)]


def _batches(files, device, **kw):
    """the batches as host tensors, or the ValueError the generator raised"""
    from tf_repos_b200 import input_fn
    out = []
    try:
        for feats, labels in input_fn.input_fn(files, device=device, **kw):
            out.append((feats["feat_ids"].cpu(), feats["feat_vals"].cpu(), labels.cpu()))
    except ValueError as e:
        return str(e)
    return out


@pytest.mark.parametrize("field_size", [0, 15])
def test_streamed_device_batches_equal_host_batches(tmp_path, field_size):
    lines = _lines(300, 15, 30)
    lines[120] = ""                                                   # declined pieces in the middle of the file
    for row, pair in ((150, "3:0.12345678901234567"), (180, "4:inf"), (200, "5:%s1.5" % ("0" * 5000))):
        lines[row] = lines[row].replace(" ", " %s " % pair, 1).rsplit(" ", 1)[0]     # 17 digits, inf, a long line
    files = [os.path.join(tmp_path, n) for n in ("tr0.libsvm", "empty.libsvm", "tr1.libsvm")]
    open(files[0], "w").write("\n".join(lines) + "\n")
    open(files[1], "w").write("")
    open(files[2], "w").write("\n".join(_lines(97, 15, 31)))           # no '\n' at the end
    assert os.path.getsize(files[0]) > 10 * 4096
    kw = dict(batch_size=37, num_epochs=3, field_size=field_size)
    host = _batches(files, None, **kw)
    dev = _batches(files, "cuda", chunk_bytes=4096, **kw)
    assert [b[2].shape[0] for b in host] == [37] * (3 * 396 // 37) + [3 * 396 % 37]
    assert len(dev) == len(host)
    for d, h in zip(dev, host):
        assert all(a.dtype == b.dtype and a.shape == b.shape for a, b in zip(d, h))
        assert torch.equal(d[0], h[0]) and torch.equal(d[1].view(torch.int32), h[1].view(torch.int32))
        assert torch.equal(d[2].view(torch.int32), h[2].view(torch.int32))
    assert torch.isinf(torch.cat([h[1] for h in host])).any()


def test_streamed_device_error_is_the_host_error(tmp_path, monkeypatch):
    from tf_repos_b200 import input_fn, text_chunks
    monkeypatch.setattr(input_fn, "CHUNK", 4096)                     # the host path cuts the device path's pieces
    lines = _lines(100, 15, 32)
    lines[30] = lines[30].rsplit(" ", 1)[0]                           # 14 pairs
    path = os.path.join(tmp_path, "tr.libsvm")
    open(path, "w").write("\n".join(lines) + "\n")
    n0, n1 = (p.count(b"\n") for p in list(text_chunks.pieces(path, 4096))[:2])
    assert n0 <= 30 < n0 + n1                                         # the ragged row is in the second piece
    host = _batches([path], None, batch_size=8)
    dev = _batches([path], "cuda", batch_size=8, chunk_bytes=4096)
    assert isinstance(host, str) and dev == host
    assert "row %d has 14 id:val pairs, field_size is 15" % (30 - n0) in host
