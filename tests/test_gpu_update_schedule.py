"""The update-mode schedule (engine.SparseUpdater) through every model that drives it: exact_deferred runs as exact
where TensorFlow's update is already sparse, unknown modes raise, an overflowing sweep row list is reported once, and
ShardedDeepFM's exact_deferred state equals its exact state bit for bit."""
import pytest
import torch

pytestmark = pytest.mark.gpu

N, K, B = 4000, 8, 32
LENS = (6, 40, 6, 6, 4)        # ESMM bag lengths: u_cat, u_shop, u_brand, u_int, a_int
SMALL = dict(deep_layers="16,8", dropout="1.0,1.0", device="cuda:0")


def _criteo(seed):
    from tf_repos_b200 import synth
    return synth.criteo_batch(B, N, 39, seed=seed, device="cuda")


def _deepfm(**kw):
    from tf_repos_b200.deepfm import DeepFM
    return DeepFM(39, N, K, B, **SMALL, **kw)


def _nfm(**kw):
    from tf_repos_b200.nfm import NFM
    return NFM(39, N, K, B, **{**SMALL, "dropout": "1.0,1.0,1.0"}, **kw)


def _din(**kw):
    from tf_repos_b200.din import DIN
    return DIN(11, N, K, B, 9, max_a_int=8, attention_pooling=True, **SMALL, **kw)


def _esmm(**kw):
    from tf_repos_b200.esmm import ESMM
    return ESMM(5, N, K, B, B * sum(LENS), **SMALL, **kw)


def _sharded(**kw):
    from tf_repos_b200.sharded import ShardedDeepFM
    m = ShardedDeepFM(39, N, K, B, **SMALL, **kw)
    assert m.G == 1
    return m


def _criteo_step(m, seed):
    m.train_step(*_criteo(seed))


def _din_step(m, seed):
    from tf_repos_b200 import synth
    m.train_step(*synth.din_batch(B, N, 11, 9, 8, seed=seed, device="cuda"))


def _esmm_step(m, seed):
    from tf_repos_b200 import synth
    m.train_step(*synth.esmm_batch(B, N, 5, max_lens=LENS, min_len=0, seed=seed, device="cuda"))


MODELS = {"DeepFM": (_deepfm, _criteo_step), "NFM": (_nfm, _criteo_step), "DIN": (_din, _din_step),
          "ESMM": (_esmm, _esmm_step), "ShardedDeepFM": (_sharded, _criteo_step)}


@pytest.mark.parametrize("l2_reg", [0.0, 1e-4])
@pytest.mark.parametrize("opt", ["Adagrad", "Momentum", "ftrl", "Adam"])
@pytest.mark.parametrize("name", MODELS)
def test_exact_deferred_runs_as_exact_where_the_update_is_sparse(name, opt, l2_reg):
    make, step = MODELS[name]
    m = make(optimizer=opt, l2_reg=l2_reg, learning_rate=0.01, update_mode="exact_deferred", epoch_steps=2)
    sparse = l2_reg == 0.0 and opt != "Adam"
    assert m.update_mode == ("exact" if sparse else "exact_deferred")
    assert hasattr(m.updater, "ep") == (not sparse)
    step(m, 0)
    assert m.epoch_pos == (0 if sparse else 1)


@pytest.mark.parametrize("name", MODELS)
def test_unknown_update_mode_raises_value_error(name):
    make, _ = MODELS[name]
    with pytest.raises(ValueError, match="exact, exact_deferred, lazy"):
        make(update_mode="exact_defered")
    m = make(update_mode="lazy")
    with pytest.raises(ValueError, match="exact, exact_deferred, lazy"):
        m.set_update_mode("Exact")
    assert m.update_mode == "lazy"


@pytest.mark.parametrize("name", MODELS)
def test_check_ids_reports_a_sweep_list_overflow_once(name):
    """As test_gpu_epoch_dispatch.py::test_model_check_ids_raises_on_list_overflow, for every model class."""
    make, step = MODELS[name]
    m = make(optimizer="Adam", l2_reg=1e-4, learning_rate=5e-4, update_mode="exact_deferred", epoch_steps=2)
    e = m.updater.ep[m.tables[0].name]
    e["list"] = e["list"][:4]
    for s in range(2):
        step(m, s)
    with pytest.raises(RuntimeError, match="did not fit"):
        m.check_ids()
    m.check_ids()           # reported once


def _same_state(a, b, what):
    b.flush()
    for ta, tb in zip(a.tables, b.tables):
        assert torch.equal(ta.var, tb.var), f"{what}: {ta.name} var"
        for i, (sa, sb) in enumerate(zip(ta.slots, tb.slots)):
            assert torch.equal(sa, sb), f"{what}: {ta.name} slot {i}"
    assert torch.equal(a.dense.flat, b.dense.flat), f"{what}: dense"


def test_sharded_exact_deferred_state_equals_exact():
    """Epochs of 3 steps: a mid-epoch flush after step 1, a mid-epoch predict after step 4, epoch ends after steps 2
    and 5, and a partial epoch at the end."""
    kw = dict(optimizer="Adam", l2_reg=1e-4, learning_rate=5e-4, epoch_steps=3)
    a = _sharded(update_mode="exact", **kw)
    b = _sharded(update_mode="exact_deferred", **kw)
    for ta, tb in zip(a.tables, b.tables):
        tb.var.copy_(ta.var)
        for sa, sb in zip(ta.slots, tb.slots):
            sb.copy_(sa)
    b.dense.flat.copy_(a.dense.flat)
    for step in range(8):
        ids, vals, labels = _criteo(100 + step)
        la, lb = a.train_step(ids, vals, labels), b.train_step(ids, vals, labels)
        assert torch.equal(la[0], lb[0]), f"CE differs at step {step}"
        if step == 1:
            b.flush()
        if step == 4:
            ids_p, vals_p, _ = _criteo(500)
            assert torch.equal(a.predict(ids_p, vals_p), b.predict(ids_p, vals_p))
        if step in (1, 4, 5, 7):
            _same_state(a, b, f"after step {step}")
    a.check_ids(); b.check_ids()
