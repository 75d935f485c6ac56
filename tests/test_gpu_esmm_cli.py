"""ESMM drop-in script end to end on TFRecord input (Model_pipeline/DeepCvrMTL.py, tf_repos_b200/esmm_main.py): train,
eval, infer, export, resume, inference against the oracle fed the same checkpoint, and a TF-named npz round trip."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import esmm_oracle as eo

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _write(path, n, seed, F=11, N=5000, maxlen=30):
    from tf_repos_b200 import tfrecord as tfr
    rng = np.random.RandomState(seed)
    recs = []
    for _ in range(n):
        y = np.float32(rng.rand() < 0.4)
        ex = {"y": y, "z": np.float32(y * (rng.rand() < 0.5)), "feat_ids": rng.randint(0, N, F).astype(np.int64),
              "a_catids": np.int64(rng.randint(0, N)), "a_shopids": np.int64(rng.randint(0, N)),
              "a_brandids": np.int64(rng.randint(0, N)), "a_intids": rng.randint(0, N, rng.randint(0, 4)).astype(np.int64)}
        for f in ("cat", "shop", "brand", "int"):
            ln = rng.randint(0, maxlen + 1)
            ex["u_%sids" % f] = rng.randint(0, N, ln).astype(np.int64)
            ex["u_%svals" % f] = (rng.rand(ln) * 3).astype(np.float32)
        recs.append(tfr.encode_example(ex))
    tfr.write_records(path, recs)


def test_esmm_cli_end_to_end(tmp_path):
    tmp = str(tmp_path)
    os.makedirs(tmp + "/data/tr"); os.makedirs(tmp + "/data/te"); os.makedirs(tmp + "/ckpt")
    _write(tmp + "/data/tr/part0.tfrecord", 120, 1); _write(tmp + "/data/tr/part1.tfrecord", 80, 2)
    _write(tmp + "/data/te/part0.tfrecord", 70, 3)
    common = [sys.executable, os.path.join(ROOT, "Model_pipeline", "DeepCvrMTL.py"), "--field_size=11",
              "--feature_size=5000", "--embedding_size=8", "--batch_size=64", "--deep_layers=16,8", "--dropout=0.9,0.9",
              "--ctr_task_wgt=0.3", "--log_steps=1", "--num_epochs=1", "--data_dir=" + tmp + "/data",
              "--model_dir=" + tmp + "/ckpt/m_", "--dt_dir=20261015"]
    mdir = tmp + "/ckpt/m_20261015"

    def run(*args):
        r = subprocess.run(common + list(args), capture_output=True, text=True, timeout=280)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        return r.stdout
    out = run("--task_type=train")
    assert "Loss for final step" in out and "CTCVR_AUC" in out
    ev = json.loads(run("--task_type=eval").strip().splitlines()[-1])
    assert set(ev) == {"loss", "CTR_AUC", "CVR_AUC", "CTCVR_AUC", "global_step"}
    assert ev["global_step"] == 4       # 200 samples / 64: three full batches + the partial one (kept)
    assert all(0.0 <= ev[k] <= 1.0 for k in ("CTR_AUC", "CVR_AUC", "CTCVR_AUC")) and ev["loss"] > 0
    run("--task_type=infer")
    lines = open(tmp + "/data/pred.txt").read().split("\n")
    assert len(lines) == 71 and lines[-1] == "" and all(len(l.split("\t")) == 2 for l in lines[:-1])
    out = run("--task_type=export", "--servable_model_dir=" + tmp + "/export")
    assert "Not Implemented, Do It Yourself!" in out and not os.path.exists(tmp + "/export")
    # the oracle with the checkpoint's variables scores the test set to the same numbers
    from tf_repos_b200 import esmm_main as em
    st = torch.load(mdir + "/ctr_b200.ckpt", map_location="cpu")
    ref = eo.ESMM(11, 5000, 8, deep_layers="16,8", dropout="0.9,0.9", ctr_task_wgt=0.3)
    for k, v in st["variables"].items():
        ref.params[k] = v.float().reshape(ref.params[k].shape).clone()
    d = em.decode([tmp + "/data/te/part0.tfrecord"], 11)
    want = []
    for idx in em.index_stream(70, 1, 64):
        batch, _, n = em.make_batch(d, idx, 64, "cpu")
        o = ref.predict({k: (v.long() if k.endswith("ids") else v) for k, v in batch.items()})
        want.append(torch.stack([o["pctr"], o["pcvr"]], 1)[:n].numpy())
    want = np.concatenate(want)
    got = np.array([[float(t) for t in l.split("\t")] for l in lines[:-1]], dtype=np.float32)
    np.testing.assert_allclose(got, want, rtol=2e-5, atol=2e-6)
    # resume from the checkpoint: a second training run continues at global_step 4
    run("--task_type=train")
    assert json.loads(run("--task_type=eval").strip().splitlines()[-1])["global_step"] == 8
    # TF-named state round trip
    from tf_repos_b200 import tf_names
    from tf_repos_b200.esmm import ESMM
    from tf_repos_b200.estimator import restore_checkpoint
    cap = json.load(open(mdir + "/esmm_shapes.json"))["occ_capacity"]
    a = ESMM(11, 5000, 8, 64, cap, deep_layers="16,8", dropout="0.9,0.9", device="cuda:0")
    restore_checkpoint(a, mdir)
    tf_names.export_npz(a, tmp + "/state.npz")
    b = ESMM(11, 5000, 8, 64, cap, deep_layers="16,8", dropout="0.9,0.9", device="cuda:0", seed=5)
    tf_names.import_npz(b, tmp + "/state.npz")
    sa, sb = tf_names.state_dict_tf(a), tf_names.state_dict_tf(b)
    assert "cvr_mlp0/weights/Adam" in sa and "ctr_out/biases/Adam_1" in sa and "embeddings/Adam" in sa
    assert sa.keys() == sb.keys() and all(np.array_equal(sa[k], sb[k]) for k in sa)
