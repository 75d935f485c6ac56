"""CPU tests of the input_fns' shared pieces: the line cutter (text_chunks.pieces) against its definition, the "repeat
before batch" batcher (text_chunks.batches) against concatenate-then-slice, the libsvm host input_fn cut into many pieces
against the oracle, and the one --input_parse check of the drop-in scripts."""
import os
import types

import numpy as np
import pytest
import torch


def test_pieces_are_chunks_cut_at_the_last_line_end_before_each_chunk_bytes(tmp_path):
    from tf_repos_b200 import text_chunks

    def want(path, chunk_bytes):
        for data in text_chunks.chunks(path, chunk_bytes):
            pos = 0
            while pos < len(data):
                end = len(data) if len(data) - pos <= chunk_bytes else data.rfind(b"\n", pos, pos + chunk_bytes) + 1
                if end <= pos:                                   # one line longer than chunk_bytes
                    end = data.find(b"\n", pos) + 1 or len(data)
                yield data[pos:end]
                pos = end

    rng = np.random.default_rng(1)
    path = str(tmp_path / "t.txt")
    for trial in range(300):
        lines = [b"x" * int(rng.choice([0, 1, 5, 50, 300])) for _ in range(int(rng.integers(0, 40)))]
        open(path, "wb").write(b"\n".join(lines) + (b"\n" if rng.random() < 0.5 else b""))
        for chunk_bytes in (1, 2, 7, 64, 100, 1000, 10_000):
            assert list(text_chunks.pieces(path, chunk_bytes)) == list(want(path, chunk_bytes)), (trial, chunk_bytes)


def test_batches_equal_concatenate_then_slice():
    from tf_repos_b200 import text_chunks
    rng = np.random.default_rng(0)
    for trial in range(200):
        lengths = [int(n) if rng.random() < 0.7 else 0 for n in rng.integers(0, 40, int(rng.integers(0, 8)))]
        total = sum(lengths)
        rows = torch.arange(total, dtype=torch.int32)
        parts, lo = [], 0
        for n in lengths:
            parts.append((rows[lo:lo + n].reshape(n, 1).repeat(1, 3), rows[lo:lo + n].float() * 0.5))
            lo += n
        for batch_size in range(1, total + 3):
            got = list(text_chunks.batches(iter(parts), batch_size))
            want = [(rows[b:b + batch_size].reshape(-1, 1).repeat(1, 3), rows[b:b + batch_size].float() * 0.5)
                    for b in range(0, total, batch_size)]
            assert len(got) == len(want), (lengths, batch_size)
            for g, w in zip(got, want):
                assert all(a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b) for a, b in zip(g, w))


def test_libsvm_host_input_fn_in_many_pieces_matches_the_oracle(tmp_path, monkeypatch):
    from oracle import libsvm as ol
    from tf_repos_b200 import input_fn as inp
    from tf_repos_b200 import synth
    monkeypatch.setattr(inp, "CHUNK", 3000)                          # about 6 lines of 39 pairs a piece
    paths = []
    for k, n in enumerate((211, 0, 97)):
        ids, vals, labels = synth.criteo_batch(n, 10_000, 39, seed=40 + k)
        paths.append(str(tmp_path / ("tr%d.libsvm" % k)))
        synth.write_libsvm(paths[-1], ids, vals, labels)
    assert os.path.getsize(paths[0]) > 20 * 3000
    for batch_size in (1, 37, 308, 1000):
        got = list(inp.input_fn(paths, batch_size=batch_size, num_epochs=2, field_size=39))
        ref = list(ol.input_fn(paths, batch_size=batch_size, num_epochs=2))
        assert len(got) == len(ref) == -(-2 * 308 // batch_size)
        for (gf, gl), (rf, rl) in zip(got, ref):
            assert gf["feat_ids"].dtype == torch.int32 and gf["feat_vals"].dtype == torch.float32
            np.testing.assert_array_equal(gf["feat_ids"].numpy(), rf["feat_ids"])
            np.testing.assert_array_equal(gf["feat_vals"].numpy().view(np.uint32), rf["feat_vals"].view(np.uint32))
            np.testing.assert_array_equal(gl.numpy(), rl)


def test_input_parse_other_than_device_or_host_stops_the_libsvm_scripts(tmp_path, monkeypatch):
    from tf_repos_b200 import estimator, flags
    F = flags._Flags()
    monkeypatch.setattr(flags, "FLAGS", F)
    monkeypatch.setattr(estimator, "FLAGS", F)
    flags.define_common()
    dev = torch.device("cpu")
    assert flags.input_parse_device(dev) is dev
    F._parse(["--input_parse=host"])
    assert flags.input_parse_device(dev) is None
    F._parse(["--input_parse=gpu", "--data_dir=" + str(tmp_path), "--model_dir=" + str(tmp_path / "m_"),
              "--dt_dir=20261016"])
    with pytest.raises(SystemExit, match=r"input_parse must be one of \{device, host\}"):
        estimator.run(lambda: types.SimpleNamespace(device=dev), "DeepFM")
