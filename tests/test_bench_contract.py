"""bench.py contract pieces that can be checked without a GPU: the reference arm prints exactly one JSON line with
the keys the driver reads; our arm refuses to run (no CPU fallback) when CUDA is absent."""
import json
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_one_json_line_with_the_contract_keys():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "1", "--steps", "2",
                        "--warmup", "1", "--vocab", "200000", "--batch", "512"], capture_output=True, text=True, timeout=280)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, r.stdout                      # nothing else on stdout
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "samples/s" and d["higher_is_better"] is True
    assert d["metric"].startswith("DeepFM training samples/sec") and d["n_gpus"] == 1 and d["value"] > 0
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert d["steps"] >= 1 and d["ms_per_step"] > 0 and d["scaling"] == "weak" and d["vs_baseline"] is None


def test_reference_arm_other_ranks_exit_quietly():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2"],
                       capture_output=True, text=True, timeout=120, env=env)
    assert r.returncode == 0 and r.stdout.strip() == ""


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU behaviour")
def test_b200_arm_has_no_cpu_fallback():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "1", "--warmup", "0"],
                       capture_output=True, text=True, timeout=120)
    assert r.returncode != 0 and "no CPU fallback" in (r.stderr + r.stdout)


def test_reference_arm_maps_no_product_code():
    """VERDICT r1: the reference arm must not dlopen libctr_b200.so (it used to, through `from tf_repos_b200 import synth`)."""
    code = (
        "import sys, runpy\n"
        "sys.argv = ['bench.py', '--impl', 'reference', '--vocab', '100000', '--batch', '256', '--steps', '1', '--warmup', '1']\n"
        "try:\n"
        "    runpy.run_path(%r, run_name='__main__')\n"
        "finally:\n"
        "    sys.stderr.write('LOADED_SO=%%s PKG=%%s\\n' %% ('libctr_b200' in open('/proc/self/maps').read(), 'tf_repos_b200' in sys.modules))\n"
    ) % os.path.join(ROOT, "bench.py")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=280, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "LOADED_SO=False PKG=False" in r.stderr, r.stderr[-500:]


def test_committed_bench_line_roofline_reproduces_from_its_own_numbers():
    """`frac` must follow from algorithmic bytes / avg launch duration / peak, computed from full 16-step passes only."""
    import glob
    paths = sorted(glob.glob(os.path.join(ROOT, "profiles", "bench_n1_h100*.json")))
    assert paths, "no committed bench line"
    for p in paths:
        d = json.loads([l for l in open(p) if l.startswith("{")][-1])
        r = d["roofline"]
        achieved = r["algorithmic_bytes_per_launch"] / (r["avg_launch_ms"] * 1e-3) / 1e9
        assert abs(achieved - r["achieved"]) <= 1e-6 * achieved
        assert abs(r["frac"] - achieved / r["peak"]) <= 1e-9
        assert r["launches_timed"] >= 1 and all(pp["steps"] != 16 for pp in r["partial_passes"])
        assert d["e2e"]["h2d_bytes_per_step"] > 0 and d["gpu_launches"] > 0 and "steady_state" in d and "e2e_text" in d
