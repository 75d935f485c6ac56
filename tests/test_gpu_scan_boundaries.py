"""The text pipelines' prefix scans (scan_sort.cuh) at their tile boundaries, through the public entry points and the
existing oracles: the one-CTA scan's carry across tiles of 1024 (line starts of 1023..2049 blocks of 4 KB, the Ali-CCP
TFRecord plan's two-array scan of lines + 1 entries, the Ali-CCP sample classify's three-array int32 scan), the CTA
scans of the Criteo per-line kernels (tiles of 256 lines) and the smart / Frappe tiled offset scan (tiles of 1024)."""
import os

import numpy as np
import pytest
import torch

from tests.test_gpu_aliccp_sample import _raw
from tests.test_gpu_aliccp_tfrecord import _file as _aliccp_file
from tests.test_gpu_criteo_feature import _dataset as _criteo_dataset, _gpu as _criteo_gpu, _oracle as _criteo_oracle
from tests.test_gpu_libsvm import _device, _host, _lines, _same
from tests.test_gpu_smart_feature import _run_both, _write_frappe, write_csv

pytestmark = pytest.mark.gpu

LS_BLOCK = 4096   # bytes per block of the line-start count (line_starts.cuh)


@pytest.fixture(scope="module")
def libsvm_text():
    text = ("\n".join(_lines(62_000, 15, 41)) + "\n").encode()
    assert len(text) > 2049 * LS_BLOCK
    return text


@pytest.mark.parametrize("blocks", [1023, 1024, 1025, 2049])
def test_line_starts_across_one_cta_tiles(libsvm_text, blocks):
    cut = libsvm_text.rfind(b"\n", 0, (blocks - 1) * LS_BLOCK + LS_BLOCK // 2) + 1
    data = libsvm_text[:cut]
    assert -(-len(data) // LS_BLOCK) == blocks
    dev, host = _device(data, 15), _host(data, 15)
    _same(dev, host)
    assert dev[0].shape[0] == host[0].shape[0] == data.count(b"\n")


def test_aliccp_tfrecord_two_array_scan(tmp_path):
    from oracle import aliccp_tfrecord as oa
    from tf_repos_b200.aliccp_tfrecord import convert
    rng = np.random.RandomState(11)
    d = tmp_path / "in"
    d.mkdir()
    for n in (1023, 1024, 1025, 2049):          # one chunk each; the plan scans n + 1 sizes and decline counts
        (d / ("part-%d" % n)).write_bytes(_aliccp_file(rng, n))
    res = convert(str(d), str(tmp_path / "gpu"))
    oa.convert(str(d), str(tmp_path / "ora"))
    names = sorted(os.listdir(tmp_path / "ora"))
    assert names == sorted(os.listdir(tmp_path / "gpu")) and len(names) == 4
    for name in names:
        assert (tmp_path / "gpu" / name).read_bytes() == (tmp_path / "ora" / name).read_bytes(), name
    assert all(o["declined"] > 0 for o in res["outputs"])


def test_aliccp_sample_three_array_scan(tmp_path):
    from oracle import aliccp_sample as oa
    from tf_repos_b200 import aliccp_sample as gs
    rng = np.random.RandomState(12)
    raw = tmp_path / "raw"
    counts = {"tr": (1023, 1024, 1025), "te": (2047, 2048, 2049)}   # one chunk per file, its lines scanned by classify
    for name, ns in counts.items():
        (raw / name).mkdir(parents=True)
        lines = _raw(rng, 300, sum(ns))
        assert len(lines) >= sum(ns)
        at = 0
        for k, n in enumerate(ns):
            (raw / name / ("f%d.csv" % k)).write_bytes(b"\n".join(lines[at:at + n]) + b"\n")
            at += n
    parts = 3
    want = oa.prepare(str(raw), str(tmp_path / "ora"), parts=parts)
    got = gs.prepare(str(raw), str(tmp_path / "gpu"), parts=parts, table_capacity=1 << 16)
    assert {k: v for k, v in got.items() if k != "device_ms"} == want
    for rel in ["feat_cnts"] + ["%s/part-%05d" % (s, p) for s in counts for p in range(parts)]:
        a, b = (open(os.path.join(tmp_path, who, rel), "rb").read() for who in ("gpu", "ora"))
        assert a == b, rel
    assert want["tr"]["samples"] and want["te"]["samples"]


@pytest.mark.parametrize("n_train,n_test", [(255, 256), (257, 513)])
def test_criteo_cta_scans_at_tile_edges(tmp_path, n_train, n_test):
    d = _criteo_dataset(tmp_path, n_train, n_test, seed=13)   # one chunk per file: tiles of 256 lines
    _, want = _criteo_oracle(d, 1)
    _, got = _criteo_gpu(d, 1)
    for name, a, b in zip(("tr.libsvm", "va.libsvm", "te.libsvm", "feature_map"), got, want):
        assert a == b, name


def test_smart_emit_tiled_scan(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    d = "in_d/"
    os.makedirs(d)
    write_csv(d + "a_part_0", 500, 14)
    for k, n in enumerate((1023, 1024, 1025, 3073)):   # one chunk per input: offsets in tiles of 1024 lines
        write_csv(d + "x%d.verify" % k, n, 15 + k)
    _run_both(d, "va")


def test_frappe_tiled_scan(tmp_path, monkeypatch):
    from oracle import smart_feature as O
    from tf_repos_b200.smart_feature import frappe_feature
    monkeypatch.chdir(tmp_path)
    for who in ("gpu", "ora"):
        os.makedirs(who + "/data")
        for k, n in enumerate((1023, 1024, 1025, 3073)):
            _write_frappe(who + "/data/f%d.libsvm" % k, n, 20 + k, edge=True)
    g = frappe_feature("gpu/data")
    r = O.frappe_feature("ora/data")
    assert len(g["outputs"]) == len(r["outputs"]) == 4
    for a, b in zip(g["outputs"], r["outputs"]):
        assert open(a, "rb").read() == open(b, "rb").read(), a
        assert g["lines"][a] == r["lines"][b]
