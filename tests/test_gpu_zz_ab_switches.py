"""The measurement switches of DESIGN.md §5 ("A/B switches") must not change results: each alternative setting is run in
its own process (the switches are read once per process) on a small DeepFM job and compared with the default run, bit
for bit (K1 LDG vs TMA staging).  In every process the exact-deferred state must
equal the every-step state bit for bit (reference semantics: DeepFM.py:188-213, every row moves every step)."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHILD = r"""
import json, sys
import torch
sys.path.insert(0, %(root)r)
from tf_repos_b200 import synth
from tf_repos_b200.deepfm import DeepFM
B, F, N, K, P = 1024, 39, 300_000, 16, 4      # 300k rows: the sweep's grid-stride loop takes ~8 iterations
a = DeepFM(F, N, K, B, dropout="1.0,1.0,1.0", update_mode="exact", device="cuda:0", seed=0)
b = DeepFM(F, N, K, B, dropout="1.0,1.0,1.0", update_mode="exact_deferred", epoch_steps=P, device="cuda:0", seed=0)
b.fm_v.var.copy_(a.fm_v.var); b.fm_w.var.copy_(a.fm_w.var); b.dense.flat.copy_(a.dense.flat)
losses = []
for step in range(P + 2):                      # one full epoch + a 2-step flush
    ids, vals, labels = synth.criteo_batch(B, N, F, seed=100 + step, device="cuda")
    a.train_step(ids, vals, labels)
    losses.append(float(b.train_step(ids, vals, labels)[0]))
b.flush()
same = (torch.equal(a.fm_v.var, b.fm_v.var) and torch.equal(a.fm_w.var, b.fm_w.var)
        and all(torch.equal(x, y) for x, y in zip(a.fm_v.slots, b.fm_v.slots))
        and all(torch.equal(x, y) for x, y in zip(a.fm_w.slots, b.fm_w.slots)) and torch.equal(a.dense.flat, b.dense.flat))
h = lambda t: int(t.contiguous().view(torch.int32).long().sum())
print("RESULT " + json.dumps({"same": bool(same), "hash": [h(b.fm_v.var), h(b.fm_w.var), h(b.fm_v.slots[1]), h(b.dense.flat)],
                              "losses": losses}))
"""


def _run(env_extra):
    env = dict(os.environ, **env_extra)
    r = subprocess.run([sys.executable, "-c", CHILD % {"root": ROOT}], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")][-1]
    return json.loads(line[len("RESULT "):])


@pytest.fixture(scope="module")
def default_run():
    d = _run({})
    assert d["same"]
    return d


@pytest.mark.parametrize("env", [
    {"CTR_FM_EMBED_TMA": "1"},
    {"CTR_FM_EMBED_TMA": "0"},
], ids=lambda e: ",".join(f"{k}={v}" for k, v in e.items()))
def test_switch_leaves_every_bit_unchanged(default_run, env):
    d = _run(env)
    assert d["same"], "exact_deferred != exact under " + str(env)
    assert d["hash"] == default_run["hash"] and d["losses"] == default_run["losses"]

