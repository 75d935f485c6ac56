"""One `last` array for an [N,K] table and the [N] table gathered with the same ids (DeepFM's fm_v and fm_w).

With Adam on the packed sweep, K in {4, ..., 256} and N % 4 == 0, the updater keeps one `last` byte per row and one row
list for both tables, and one ctr_epoch_sweep call sweeps both in one launch.  The state must stay bit for bit that of the
every-step sweep; otherwise (N % 4 != 0, non-Adam) the tables keep their own `last` arrays."""
import pytest
import torch

pytestmark = pytest.mark.gpu

F, B = 39, 128


def _pair(N, K, P, optimizer="Adam"):
    from tf_repos_b200.deepfm import DeepFM
    kw = dict(field_size=F, feature_size=N, embedding_size=K, batch_size=B, deep_layers="16", dropout="1.0",
              optimizer=optimizer, learning_rate=5e-4, l2_reg=1e-4, device="cuda:0")
    a = DeepFM(update_mode="exact", **kw)
    b = DeepFM(update_mode="exact_deferred", epoch_steps=P, **kw)
    for ta, tb in zip(a.tables, b.tables):
        tb.var.copy_(ta.var)
        for sa, sb in zip(ta.slots, tb.slots):
            sb.copy_(sa)
    b.dense.flat.copy_(a.dense.flat)
    return a, b


def _same_state(a, b, what):
    b.flush()
    for ta, tb in zip(a.tables, b.tables):
        assert torch.equal(ta.var, tb.var), f"{what}: {ta.name} var"
        for i, (sa, sb) in enumerate(zip(ta.slots, tb.slots)):
            assert torch.equal(sa, sb), f"{what}: {ta.name} slot {i}"


def _steps(a, b, seeds, N, flush_at=()):
    from tf_repos_b200 import synth
    for s in seeds:
        ids, vals, labels = synth.criteo_batch(B, N, F, seed=s, device="cuda")
        la, lb = a.train_step(ids, vals, labels), b.train_step(ids, vals, labels)
        assert torch.equal(la[0], lb[0]), f"CE differs at seed {s}"
        if s in flush_at:
            b.flush()


@pytest.mark.parametrize("K", [8, 16, 32])
def test_shared_last_with_mid_epoch_flushes_equals_every_step_sweep(K):
    N, P = 6000, 5
    a, b = _pair(N, K, P)
    u = b.updater
    assert u.shared_last
    assert u.ep["fm_w"]["last"].data_ptr() == u.ep["fm_v"]["last"].data_ptr()
    _steps(a, b, range(2 * P + 3), N, flush_at=(1, 2, 7))
    _same_state(a, b, "after two epochs with mid-epoch flushes")
    # epoch-end loss terms of both tables match the every-step sweep's l2 terms of the last step of the epoch
    a.check_ids(); b.check_ids()


def test_shared_last_switch_after_flush_resets_last():
    """A flush that reached the current step, then a mode switch: the closing sweep has nothing left to replay but
    must still return every `last` byte to 0."""
    N, P = 4000, 6
    a, b = _pair(N, 16, P)
    _steps(a, b, range(3), N)
    b.flush()
    b.set_update_mode("exact_deferred")
    assert b.epoch_pos == 0
    assert int(b.updater.ep["fm_v"]["last"].max().item()) == 0
    _same_state(a, b, "after the switch")
    _steps(a, b, range(3, 3 + P + 2), N, flush_at=(5,))
    _same_state(a, b, "one epoch later")


def test_shared_last_list_overflow_raises():
    from tf_repos_b200 import synth
    N = 4000
    _, b = _pair(N, 16, 2)
    assert b.updater.shared_last
    b.updater.ep["fm_v"]["list"] = b.updater.ep["fm_v"]["list"][:4]
    for s in range(2):
        b.train_step(*synth.criteo_batch(B, N, F, seed=s, device="cuda"))
    with pytest.raises(RuntimeError, match="did not fit"):
        b.check_ids()
    b.check_ids()


@pytest.mark.parametrize("N,optimizer", [(4001, "Adam"), (4002, "Adam"), (4000, "Adagrad")])
def test_separate_last_arrays_where_the_pair_sweep_does_not_apply(N, optimizer):
    """fm_w with N % 4 != 0 takes the generic scalar sweep (and non-Adam optimizers the scalar kernels): each table
    keeps its own `last` array, with the same results as before."""
    a, b = _pair(N, 16, 4, optimizer=optimizer)
    u = b.updater
    assert not u.shared_last
    assert u.ep["fm_w"]["last"].data_ptr() != u.ep["fm_v"]["last"].data_ptr()
    _steps(a, b, range(7), N, flush_at=(2,))
    _same_state(a, b, f"N={N} {optimizer}")


@pytest.mark.parametrize("K,shared", [(16, True), (16, False), (256, True)])
def test_rows2_with_stage_equals_rows2_without_stage(K, shared):
    """ctr_epoch_rows2 with a stage against ctr_epoch_rows2 without one (stage = NULL) on the same rows: after the
    catch-up `var` of both tables is the same, and after the apply every array, `last` and the sum(var^2) accumulators
    are."""
    from tf_repos_b200 import ops
    from tf_repos_b200.engine import OptimizerState, Table
    dev, N, n, j = torch.device("cuda:0"), 4096, 700, 5
    opt = OptimizerState("Adam", 5e-4, 1e-4, dev)
    for s in range(j + 1):
        opt.tick_epoch(s)
    g = torch.Generator(device=dev).manual_seed(3)
    uniq = torch.randperm(N, device=dev, generator=g)[:n].sort().values.int()
    n_uniq = torch.tensor([n], dtype=torch.int32, device=dev)
    gv = torch.randn(n * K, device=dev, generator=g) * 1e-3
    gw = torch.randn(n, device=dev, generator=g) * 1e-3
    runs = []
    for staged in (False, True):
        V = Table("v", N, K, opt, dev, seed=1)
        W = Table("w", N, 1, opt, dev, seed=2)
        for sl in V.slots + W.slots:
            sl.copy_(torch.rand(sl.shape, device=dev, generator=torch.Generator(device=dev).manual_seed(sl.dim())) * 1e-6)
        lv = torch.randint(0, j + 1, (N,), device=dev, generator=torch.Generator(device=dev).manual_seed(9)).to(torch.uint8)
        lw = lv if shared else lv.clone()
        ss = [torch.zeros(32, dtype=torch.float64, device=dev) for _ in range(2)]
        st = (torch.empty(3 * n * K, device=dev), torch.empty(3 * n, device=dev))
        out = {}
        for apply in (False, True):
            args = (opt.opt, apply, V, W, lv, lw, uniq, n_uniq, gv if apply else None, gw if apply else None, n,
                    opt.record(0), opt.lr_table, j, ss[0], ss[1])
            ops.epoch_rows2(*args, *(st if staged else (None, None)))
            if not apply:
                out["var_after_catch_up"] = (V.var.clone(), W.var.clone())
        torch.cuda.synchronize()
        out["final"] = [V.var, *V.slots, W.var, *W.slots, lv, lw]
        out["ss"] = ss
        runs.append(out)
    a, b = runs
    for x, y in zip(a["var_after_catch_up"], b["var_after_catch_up"]):
        assert torch.equal(x, y)
    for x, y in zip(a["final"], b["final"]):
        assert torch.equal(x, y)
    for x, y in zip(a["ss"], b["ss"]):
        assert torch.allclose(x, y, rtol=1e-6, atol=0)
