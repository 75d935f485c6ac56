"""The exact-deferred ("epoch") table kernels of csrc/epoch.cu and csrc/epoch_adam.cu, driven directly through
ops.epoch_tick / epoch_rows / epoch_rows2 / epoch_sweep / epoch_reg_loss the way engine.SparseUpdater drives them, with
no model on top, over their whole dispatch space.

Oracle: the every-row, every-step fp32 update of oracle/tf_semantics.py.  At every step each row takes the optimizer
step with G = l2*var, plus the de-duplicated gradient on the rows gathered that step (TF's sparse apply with the dense
l2_loss gradient, DeepFM.py:189-213).  The deferred kernels promise the same bits.  After every kernel call the test
checks:
  * var and every slot, bit for bit: a row whose `last` byte is L must hold the oracle state after L steps of the
    current epoch (torch.equal: the packed Adam loops may give -0 where the oracle gives +0, see adam_untouched);
  * every `last` byte: j after the catch-up of step j, j+1 after its apply, `upto` after a mid-epoch flush, 0 after
    the epoch-end sweep;
  * lr_table[j] against AdamHyper.lr_t() (or the constant lr), bit for bit;
  * the per-step l2 terms against 0.5*l2*sum(var^2) of the oracle state at the start of each step, in fp64, within
    the bound `_Tab.reg_tol` derives from the longest fp32 accumulation chain of the kernels;
  * that the packed Adam sweep's row list never overflowed (list_count <= cap, overflow counter 0).

Dispatch matrix (which branch of ctr_epoch_rows / ctr_epoch_rows2 / ctr_epoch_sweep each case reaches):

  entry point              path                          cases
  ctr_epoch_rows           epoch_rows_kernel             K in {4, 8, 16, 32, 64, 128, 256} (catch-up and apply), 4 opts
  ctr_epoch_rows           epoch_rows_generic_kernel     K in {1, 2, 3, 10, 12, 20, 100, 200}, 4 opts: whole-warp CTAs
                                                         (K=1, 2), CTAs rounded up to whole warps (K=3, 10, 12, 20,
                                                         100, 200), rows longer than a warp (K=100, 200)
  ctr_epoch_rows2          epoch_rows_kernel<WITH_W>     K in {4, 8, 32, 64, 128, 256}, 4 opts, the two tables' `last`
                                                         bytes desynchronised by flushing them at different steps
  ctr_epoch_sweep, Adam    packed (epoch_sweep_adam*)    K in {4, 12, 32, 256}; K=1 with N%4 == 0
  ctr_epoch_sweep, Adam    packed, nothing to replay     K=12, a flush directly followed by the epoch end (from == upto)
  ctr_epoch_sweep, Adam    epoch_sweep_generic_kernel    K=1 with N%4 in {1, 2, 3}; K=10; K=1 with `last` offset by 1 B
  ctr_epoch_sweep, other   epoch_sweep_kernel            K in {4, 16, 128}, Adagrad / Momentum / ftrl
  ctr_epoch_sweep, other   epoch_sweep_k1_kernel         K=1 with N%4 == 0
  ctr_epoch_sweep, other   epoch_sweep_generic_kernel    K=1 with N%4 == 3; K in {10, 12, 256}

Every rows case also runs the sweep its (K, N, optimizer) selects.  Epoch lengths P in {1, 2, 7, 32} (32 is
ctr_epoch_max_steps(): `last` bytes reach 32 and the sweeps' per-step shared arrays are full); schedules with two
mid-epoch flushes and with a flush directly followed by the epoch end; one step that gathers nothing; ids re-gathered
in later steps; ids never gathered.  The "big" cases hold >= 2e6 floats, so every sweep family runs its grid-stride
loop more than once per thread; the "extreme" cases start from zero, denormal and near-FLT_MIN states.
An Adam sweep without its row list is rejected.
"""
import math
import zlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

OPTS = ("Adam", "Adagrad", "Momentum", "ftrl")
NON_ADAM = ("Adagrad", "Momentum", "ftrl")
LR = {"Adam": 5e-3, "Adagrad": 0.05, "Momentum": 0.01, "ftrl": 0.05}
L2 = 2e-3
U32 = 2.0 ** -24          # unit roundoff of fp32
EPOCH_MAX = 32


# ---------------------------------------------------------------------------------------------------------------
# oracle + harness
# ---------------------------------------------------------------------------------------------------------------
def _oracle_step(opt_name, var, slots, G, lr, adam):
    """One every-row step (TF sparse apply over all rows, gradient G), fp32, out of place."""
    from oracle import tf_semantics as tfs
    var = var.clone(); slots = [s.clone() for s in slots]
    if opt_name == "Adam":
        tfs.adam_sparse_(var, slots[0], slots[1], G, adam.lr_t(), adam.b1, adam.b2, adam.eps)
    elif opt_name == "Adagrad":
        tfs.adagrad_(var, slots[0], G, torch.tensor(lr))
    elif opt_name == "Momentum":
        tfs.momentum_(var, slots[0], G, torch.tensor(lr), torch.tensor(0.95))
    else:
        tfs.ftrl_(var, slots[0], slots[1], G, lr)
    return var, slots


def _extreme(shape, gen, nonneg=False):
    """A mix of exact zeros, denormals, values just above FLT_MIN and (a quarter) ordinary values, on gen's device."""
    d = gen.device
    r = torch.randint(0, 4, shape, generator=gen, device=d)
    sgn = torch.where(torch.rand(shape, generator=gen, device=d) < 0.5, -1.0, 1.0)
    fmin = float(np.finfo(np.float32).tiny)
    den = torch.randint(1, 1 << 22, shape, generator=gen, device=d).double() * 2.0 ** -149
    near = fmin * (1.0 + 3.0 * torch.rand(shape, generator=gen, device=d).double())
    ordinary = torch.randn(shape, generator=gen, device=d).double() * 0.1
    x = torch.where(r == 0, torch.zeros(shape, dtype=torch.float64, device=d),
                    torch.where(r == 1, den, torch.where(r == 2, near, ordinary)))
    x = x.float()
    return x.abs() if nonneg else x * sgn.float()


class _Tab:
    """One table: device state (duck-types engine.Table for ops.epoch_rows2), its `last` bytes and scratch, and the
    oracle's states after 0..j steps of the current epoch."""

    def __init__(self, name, N, K, ost, gen, n_max, regime="normal", last_offset=0, list_cap=None):
        from tf_repos_b200 import ops
        self.name, self.N, self.K = name, N, K
        var = (torch.randn(N, K, generator=gen) * 0.1).float()
        slots = [(torch.rand(N, K, generator=gen) * 0.01 + ost.slot_init(i)).float() for i in range(ost.n_slots)]
        if regime == "extreme":
            var = _extreme((N, K), gen)
            if ost.name == "Adam":
                slots = [_extreme((N, K), gen), _extreme((N, K), gen, nonneg=True)]
            elif ost.name == "Momentum":
                slots = [_extreme((N, K), gen)]
            elif ost.name == "Adagrad":
                slots = [ost.slot_init(0) + _extreme((N, K), gen, nonneg=True)]
            else:
                slots = [ost.slot_init(0) + _extreme((N, K), gen, nonneg=True), _extreme((N, K), gen)]
        dev = "cuda"
        self.var = var.to(dev)
        self.slots = [s.to(dev) for s in slots]
        # `last` may be a view one byte into its buffer (K=1: the k1 / packed-k1 kernels need 4-byte alignment)
        self.last_buf = torch.zeros(N + last_offset, dtype=torch.uint8, device=dev)
        self.last = self.last_buf[last_offset:]
        self.ss = torch.zeros(EPOCH_MAX, dtype=torch.float64, device=dev)
        self.n_epart = ops.epoch_partials_count()
        self.partials = torch.zeros(EPOCH_MAX * self.n_epart, dtype=torch.float64, device=dev)
        self.reg = torch.zeros(EPOCH_MAX, dtype=torch.float32, device=dev)
        self.cap = list_cap if list_cap is not None else max(min(n_max * EPOCH_MAX, N), 1)   # engine.enable_epochs
        self.list = torch.empty(self.cap, dtype=torch.int32, device=dev)
        self.list_count = torch.zeros(1, dtype=torch.int32, device=dev)
        self.overflow = torch.zeros(1, dtype=torch.int32, device=dev)
        self.snaps = [(var, slots)]          # oracle state after 0, 1, ... steps of the current epoch
        self.last_exp = np.zeros(N, dtype=np.int64)
        self.reg_exp = []                    # fp64 0.5*l2*sum(var^2) at the start of each step of the epoch
        self.flush_pos = 0

    def slot(self, i):
        return self.slots[i] if i < len(self.slots) else None

    def expected(self):
        """Oracle state of every row at its own `last` step."""
        v0, s0 = self.snaps[0]
        var, slots = v0.clone(), [s.clone() for s in s0]
        for L in np.unique(self.last_exp):
            if L == 0:
                continue
            m = torch.from_numpy(self.last_exp == L)
            var[m] = self.snaps[L][0][m]
            for s, src in zip(slots, self.snaps[L][1]):
                s[m] = src[m]
        return var, slots

    def check(self, what):
        torch.cuda.synchronize()
        last = self.last.cpu().numpy().astype(np.int64)
        bad = np.nonzero(last != self.last_exp)[0]
        assert bad.size == 0, (f"{what}: {self.name} `last` of {bad.size} rows differs; row {bad[0]}: "
                               f"{last[bad[0]]} (want {self.last_exp[bad[0]]})")
        var, slots = self.expected()
        for nm, got, want in [("var", self.var, var)] + [(f"slot{i}", a, b) for i, (a, b) in
                                                          enumerate(zip(self.slots, slots))]:
            got = got.cpu()
            if not torch.equal(got, want):
                diff = (got != want).any(dim=1).nonzero().flatten()
                r = int(diff[0])
                raise AssertionError(f"{what}: {self.name} {nm} differs in {diff.numel()} rows; row {r} (last "
                                     f"{self.last_exp[r]}): {got[r, :4].tolist()} vs {want[r, :4].tolist()}")

    def oracle_step(self, opt_name, uniq, g, lr, adam):
        var, slots = self.snaps[-1]
        self.reg_exp.append(float(np.float32(0.5 * L2)) * float((var.double() ** 2).sum()))
        G = torch.tensor(L2) * var
        if uniq.numel():
            G[uniq] = g + G[uniq]
        self.snaps.append(_oracle_step(opt_name, var, slots, G, lr, adam))

    def reg_tol(self, ss_scaled):
        """Bound on |reg[s] - 0.5*l2*sum(var^2)|.  Every term var^2 >= 0 is rounded once (u), then summed in fp32 along
        chains no longer than: the elements one thread of the smallest sweep grid (2 CTAs/SM x 256 threads) folds into
        its per-step accumulator, plus float4 / unroll granularity (16), plus a 5-level warp butterfly, plus the fp32
        atomics of a CTA's 8 warps in the row kernels; everything after that is fp64.  A recursive sum of non-negative
        terms along a chain of L additions is within L*u/(1-L*u) of the exact sum; two more roundings store reg in fp32
        and add the flush's share to the epoch end's.  Products that underflow lose at most 2^-149 each."""
        from tf_repos_b200 import _lib
        n_elem = self.N * self.K
        min_threads = _lib.raw().ctr_device_sm_count() * 2 * 256
        chain = math.ceil(n_elem / min_threads) + 16 + 5 + 8 + 1
        rel = 1.01 * (chain + 3) * U32
        return rel * ss_scaled + 0.5 * L2 * n_elem * 2.0 ** -149 + 2.0 ** -149

    def check_reg(self, upto, what):
        torch.cuda.synchronize()
        got = self.reg[:upto].double().cpu().numpy()
        for s in range(upto):
            want = self.reg_exp[s]
            tol = self.reg_tol(want)
            assert abs(got[s] - want) <= tol, (f"{what}: {self.name} reg[{s}] = {got[s]!r}, fp64 oracle {want!r} "
                                               f"(|diff| {abs(got[s] - want):.3e} > bound {tol:.3e})")


class _Sched:
    """P-step epochs over one table (ops.epoch_rows) or a [N,K] + [N] pair (ops.epoch_rows2)."""

    def __init__(self, opt_name, tabs_spec, P, seed, rows2=False, regime="normal", last_offset=0, n_ids=None,
                 list_cap=None):
        from oracle import tf_semantics as tfs
        from tf_repos_b200 import engine
        self.opt_name, self.P, self.rows2 = opt_name, P, rows2
        self.lr = LR[opt_name]
        self.ost = engine.OptimizerState(opt_name, self.lr, L2, "cuda")
        self.adam = tfs.AdamHyper(self.lr)
        self.gen = torch.Generator().manual_seed(seed)
        N = tabs_spec[0][1]
        self.N = N
        self.n_ids = n_ids if n_ids is not None else min(max(N // 8, 4), 4096)
        self.pad = 37                         # uniq buffer beyond n_uniq: ids of rows nothing may touch
        self.n_max = self.n_ids + self.pad
        self.tabs = [_Tab(nm, N, K, self.ost, self.gen, self.n_max, regime, last_offset, list_cap)
                     for nm, _, K in tabs_spec]
        perm = torch.randperm(N, generator=self.gen)
        n_pool = max(int(0.6 * N), 1)
        self.pool, self.never = perm[:n_pool], perm[n_pool:]     # ids that are sometimes / never gathered
        self.t = 0                            # global step
        self.j = 0                            # step within the epoch

    def _ids(self):
        from_pool = self.pool
        if self.t == 1:
            n = 0                              # one step gathers nothing
        else:
            n = int(torch.randint(max(self.n_ids // 2, 1), self.n_ids + 1, (1,), generator=self.gen))
            n = min(n, from_pool.numel())
        pick = from_pool[torch.randperm(from_pool.numel(), generator=self.gen)[:n]]
        uniq = torch.sort(pick)[0]
        junk = self.never if self.never.numel() else self.pool
        pad = junk[torch.randint(0, junk.numel(), (self.n_max - n,), generator=self.gen)]
        buf = torch.cat([uniq, pad]).to(torch.int32).cuda()
        return uniq.long(), buf, torch.tensor([n], dtype=torch.int32, device="cuda")

    def _rows(self, apply, j, uniq_dev, n_uniq, grads):
        from tf_repos_b200 import ops
        o = self.ost
        if self.rows2:
            V, W = self.tabs
            ops.epoch_rows2(o.opt, apply, V, W, V.last, W.last, uniq_dev, n_uniq, grads[0] if apply else None,
                            grads[1] if apply else None, self.n_max, o.record(0), o.lr_table, j, V.ss, W.ss)
            return
        for t, g in zip(self.tabs, grads if apply else [None] * len(self.tabs)):
            ops.epoch_rows(o.opt, apply, t.var, t.slot(0), t.slot(1), t.last, uniq_dev, n_uniq,
                           g if apply else None, self.n_max, t.K, o.record(0), o.lr_table, j, t.ss)

    def sweep(self, t, upto, reset, what):
        from tf_repos_b200 import ops
        o = self.ost
        ops.epoch_sweep(o.opt, t.var, t.slot(0), t.slot(1), t.last, t.N, t.K, o.record(0), o.lr_table, t.flush_pos,
                        upto, reset, t.partials, t.list, t.list_count, t.ss, t.overflow)
        ops.epoch_reg_loss(t.ss, t.partials, t.n_epart, upto, 0.5 * L2, t.reg, accumulate=True)
        t.flush_pos = 0 if reset else upto
        t.last_exp[:] = 0 if reset else upto
        if reset:
            t.snaps = [t.snaps[-1]]      # the next epoch starts from the state after P steps
        t.check(what)
        assert int(t.list_count.item()) <= t.cap and int(t.overflow.item()) == 0, (
            f"{what}: {t.name} list_count {int(t.list_count.item())} > cap {t.cap}")
        t.check_reg(upto, what)
        if reset:
            t.reg_exp = []

    def step(self, flushes=()):
        """One step; flushes: [(table index, position)] flushed after this step (position j+1)."""
        from tf_repos_b200 import ops
        j, o = self.j, self.ost
        what = f"step {self.t} (epoch pos {j})"
        if j == 0:
            for t in self.tabs:
                ops.fill(t.reg, 0.0)
        o.tick_epoch(j)
        want_lr = self.adam.lr_t() if self.opt_name == "Adam" else torch.tensor(self.lr, dtype=torch.float32)
        got_lr = o.lr_table[j].cpu()
        assert torch.equal(got_lr.view(torch.int32), want_lr.view(torch.int32)), (what, got_lr, want_lr)
        uniq, uniq_dev, n_uniq = self._ids()
        # catch-up: gathered rows -> state at the start of step j
        self._rows(False, j, uniq_dev, n_uniq, None)
        for t in self.tabs:
            t.last_exp[uniq.numpy()] = j
            t.check(what + " catch-up")
        grads = []
        for t in self.tabs:
            g = (torch.randn(self.n_max, t.K, generator=self.gen) * 0.05).float()
            grads.append(g.cuda())
            t.oracle_step(self.opt_name, uniq, g[:uniq.numel()], self.lr, self.adam)
        self._rows(True, j, uniq_dev, n_uniq, grads)
        for t in self.tabs:
            t.last_exp[uniq.numpy()] = j + 1
            t.check(what + " apply")
        self.adam.finish()
        self.t += 1
        self.j += 1
        for ti, pos in flushes:
            if pos == self.j:
                self.sweep(self.tabs[ti], self.j, False, f"{what}: flush of {self.tabs[ti].name} at {pos}")
        if self.j == self.P:
            for t in self.tabs:
                self.sweep(t, self.P, True, f"{what}: epoch end of {t.name}")
            self.j = 0

    def run(self, n_steps, flushes=()):
        for _ in range(n_steps):
            self.step(flushes)
        if self.j:                       # a partial last epoch: flush it so every row is current
            for t in self.tabs:
                if self.j > t.flush_pos:
                    self.sweep(t, self.j, False, f"final flush of {t.name}")
        return self.digest()

    def digest(self):
        torch.cuda.synchronize()
        h = lambda x: int(x.contiguous().view(torch.int32).long().sum())
        return [h(x) for t in self.tabs for x in [t.var] + t.slots]


def _n_steps(P):
    return 2 * P if P <= 7 else P + 3     # two epochs; long epochs: one epoch plus the start of the next


def _run_case(case):
    """case: dict(opt, K, N, P, flush, rows2, regime, last_offset, Kw).  Returns the final state's digest."""
    opt, K, N, P = case["opt"], case["K"], case["N"], case["P"]
    rows2 = case.get("rows2", False)
    spec = [("v", N, K)] + ([("w", N, 1)] if rows2 else [])
    seed = zlib.crc32(repr((opt, K, N, P, rows2, case.get("regime", ""))).encode()) & 0xFFFF
    s = _Sched(opt, spec, P, seed, rows2=rows2, regime=case.get("regime", "normal"),
               last_offset=case.get("last_offset", 0))
    fl = []
    for ti, positions in enumerate(case.get("flush", ())):
        fl += [(ti, p) for p in positions]
    return s.run(_n_steps(P), fl)


def _rows_n(K):
    return int(min(max(100_000 // K, 250), 4001))


def _case(tag, **kw):
    kw.setdefault("flush", ())
    fl = "-".join("f" + ".".join(map(str, f)) for f in kw["flush"] if f)
    parts = [tag, kw["opt"], f"K{kw['K']}", f"N{kw['N']}", f"P{kw['P']}"] + ([fl] if fl else [])
    if kw.get("regime"):
        parts.append(kw["regime"])
    return pytest.param(kw, id="-".join(parts))


_P_ROWS = {4: 1, 8: 2, 16: 7, 32: 32, 64: 7, 128: 2, 256: 32}
_P_GEN = {1: 7, 2: 2, 3: 32, 10: 7, 12: 32, 20: 7, 100: 2, 200: 1}
_P_ROWS2 = {4: 7, 8: 2, 32: 7, 64: 32, 128: 7, 256: 2}
_FLUSH_ROWS2 = {1: ((), ()), 2: ((1,), ()), 7: ((2,), (5,)), 32: ((10,), (20,))}   # V and W at different steps

CASES = (
    # ctr_epoch_rows -> epoch_rows_kernel<OPT, LPR, VEC, APPLY>
    [_case("rows", opt=o, K=K, N=_rows_n(K), P=_P_ROWS[K], flush=(((3,),) if _P_ROWS[K] == 7 else ()))
     for K in _P_ROWS for o in OPTS]
    # ctr_epoch_rows -> epoch_rows_generic_kernel<OPT, APPLY>
    + [_case("rowsgen", opt=o, K=K, N=_rows_n(K) + (1 if K == 1 else 0), P=_P_GEN[K],
             flush=(((2, 5),) if (_P_GEN[K] == 7 and K == 10) else ()))
       for K in _P_GEN for o in OPTS]
    # ctr_epoch_rows2 -> epoch_rows_kernel<..., WITH_W>
    + [_case("rows2", opt=o, K=K, N=_rows_n(K) + 1, P=_P_ROWS2[K], rows2=True, flush=_FLUSH_ROWS2[_P_ROWS2[K]])
       for K in _P_ROWS2 for o in OPTS]
    # ctr_epoch_sweep, Adam, packed pipe (epoch_sweep_adam_kernel / epoch_sweep_adam_k1_kernel)
    + [_case("packed", opt="Adam", K=4, N=3001, P=32, flush=((11, 23),)),
       _case("packed", opt="Adam", K=12, N=1001, P=7, flush=((7,),)),
       _case("packed-big", opt="Adam", K=32, N=66_001, P=2),
       _case("packed", opt="Adam", K=256, N=300, P=7, flush=((3,),)),
       _case("packed-k1", opt="Adam", K=1, N=4000, P=32),
       _case("packed-k1-big", opt="Adam", K=1, N=2_000_000, P=2, flush=((1,),))]
    # ctr_epoch_sweep, Adam, epoch_sweep_generic_kernel<ADAM>
    + [_case("adamgen", opt="Adam", K=1, N=4001, P=7, flush=((2, 5),)),
       _case("adamgen", opt="Adam", K=1, N=4002, P=32),
       _case("adamgen", opt="Adam", K=1, N=4003, P=2, flush=((2,),)),
       _case("adamgen", opt="Adam", K=10, N=1500, P=7, flush=((7,),)),
       _case("adamgen-lastoff", opt="Adam", K=1, N=4000, P=7, last_offset=1, flush=((3,),)),
       _case("adamgen-big", opt="Adam", K=1, N=2_000_003, P=2),
       _case("adamgen", opt="Adam", K=1, N=4003, P=7, flush=((3,),), regime="extreme"),
       _case("adamgen", opt="Adam", K=10, N=1501, P=2, regime="extreme")]
    # ctr_epoch_sweep, non-Adam, epoch_sweep_kernel<OPT, UNROLL, MINB>
    + [_case("sweep", opt=o, K=4, N=3001, P=32, flush=((16,),)) for o in NON_ADAM]
    + [_case("sweep-big", opt=o, K=16, N=131_075, P=2) for o in NON_ADAM]
    + [_case("sweep", opt=o, K=128, N=500, P=7, flush=((2, 5),)) for o in NON_ADAM]
    # ctr_epoch_sweep, non-Adam, epoch_sweep_k1_kernel<OPT>
    + [_case("k1", opt=o, K=1, N=4000, P=7, flush=((3,),)) for o in NON_ADAM]
    + [_case("k1-big", opt=o, K=1, N=2_000_000, P=2) for o in NON_ADAM]
    # ctr_epoch_sweep, non-Adam, epoch_sweep_generic_kernel<OPT>
    + [_case("gen", opt=o, K=1, N=4003, P=32) for o in NON_ADAM]
    + [_case("gen", opt=o, K=10, N=1500, P=7, flush=((7,),)) for o in NON_ADAM]
    + [_case("gen", opt=o, K=12, N=800, P=2, flush=((1,),)) for o in NON_ADAM]
    + [_case("gen", opt=o, K=256, N=300, P=7, flush=((2, 5),)) for o in NON_ADAM]
    + [_case("gen-big", opt=o, K=10, N=200_003, P=2) for o in NON_ADAM]
    + [_case("gen", opt=o, K=1, N=4003, P=7, flush=((3,),), regime="extreme") for o in NON_ADAM]
    + [_case("gen", opt=o, K=12, N=801, P=7, regime="extreme") for o in NON_ADAM]
)


@pytest.mark.parametrize("case", CASES)
def test_epoch_kernels_match_every_step_oracle(case):
    _run_case(case)


# ---------------------------------------------------------------------------------------------------------------
# limits and the packed sweep's row list
# ---------------------------------------------------------------------------------------------------------------
def test_epoch_step_limits_rejected():
    from tf_repos_b200 import _lib, engine, ops
    assert ops.epoch_max_steps() == EPOCH_MAX
    ost = engine.OptimizerState("Adam", 1e-3, 1e-4, "cuda")
    ost.tick_epoch(EPOCH_MAX - 1)
    with pytest.raises(_lib.CtrError):
        ost.tick_epoch(EPOCH_MAX)
    t = _Tab("v", 64, 4, ost, torch.Generator().manual_seed(0), 8)
    uniq = torch.arange(8, dtype=torch.int32, device="cuda")
    n = torch.tensor([8], dtype=torch.int32, device="cuda")
    with pytest.raises(_lib.CtrError):
        ops.epoch_rows(ost.opt, False, t.var, t.slot(0), t.slot(1), t.last, uniq, n, None, 8, 4, ost.record(0),
                       ost.lr_table, EPOCH_MAX, t.ss)
    with pytest.raises(_lib.CtrError):
        ops.epoch_sweep(ost.opt, t.var, t.slot(0), t.slot(1), t.last, 64, 4, ost.record(0), ost.lr_table, 0,
                        EPOCH_MAX + 1, True, t.partials)
    with pytest.raises(_lib.CtrError, match="Adam needs list"):   # the Adam sweep has no path without its row list
        ops.epoch_sweep(ost.opt, t.var, t.slot(0), t.slot(1), t.last, 64, 4, ost.record(0), ost.lr_table, 0, 1, True,
                        t.partials)
    upd = engine.SparseUpdater(16, 64, 4, ost, "cuda", with_scalar_table=False)
    tab = engine.Table("v", 64, 4, ost, "cuda")
    upd.enable_epochs(EPOCH_MAX, [tab])
    for bad in (0, EPOCH_MAX + 1):
        with pytest.raises(ValueError):
            upd.enable_epochs(bad, [tab])


@pytest.mark.parametrize("K,N", [(16, 2000), (1, 4000)])
def test_packed_sweep_list_overflow_is_reported(K, N):
    """A row list smaller than the bound of include/ctr_b200.h: the packed sweep cannot catch the extra rows up, and
    must say so through the overflow counter (it adds exactly the rows it dropped)."""
    s = _Sched("Adam", [("v", N, K)], 4, seed=7, n_ids=300, list_cap=8)
    for _ in range(3):
        s.step()
    t = s.tabs[0]
    gathered = int((t.last_exp > 0).sum())
    assert gathered > 8
    from tf_repos_b200 import ops
    o = s.ost
    ops.epoch_sweep(o.opt, t.var, t.slot(0), t.slot(1), t.last, N, K, o.record(0), o.lr_table, 0, 3, False,
                    t.partials, t.list, t.list_count, t.ss, t.overflow)
    torch.cuda.synchronize()
    assert int(t.list_count.item()) == gathered
    assert int(t.overflow.item()) == gathered - 8


def test_model_check_ids_raises_on_list_overflow():
    """The same through a model: an undersized list makes check_ids() raise instead of training on stale rows."""
    from tf_repos_b200 import synth
    from tf_repos_b200.deepfm import DeepFM
    m = DeepFM(39, 5000, 8, 64, deep_layers="16", dropout="1.0", update_mode="exact_deferred", epoch_steps=2,
               device="cuda:0")
    m.updater.ep["fm_v"]["list"] = m.updater.ep["fm_v"]["list"][:4]
    for step in range(2):
        ids, vals, labels = synth.criteo_batch(64, 5000, 39, seed=step, device="cuda")
        m.train_step(ids, vals, labels)
    with pytest.raises(RuntimeError, match="did not fit"):
        m.check_ids()
    m.check_ids()           # reported once


# ---------------------------------------------------------------------------------------------------------------
# model level, at the reference's documented shapes
# ---------------------------------------------------------------------------------------------------------------
def _model_pair(cls, **kw):
    a = cls(update_mode="exact", device="cuda:0", **kw)
    b = cls(update_mode="exact_deferred", device="cuda:0", **kw)
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
    assert torch.equal(a.dense.flat, b.dense.flat), f"{what}: dense"
    for i, (sa, sb) in enumerate(zip(a.dense.slots, b.dense.slots)):
        assert torch.equal(sa, sb), f"{what}: dense slot {i}"


def _run_pair(a, b, flush_at, check_at, partial_B):
    """Two full epochs (epoch_steps each), mid-epoch flushes, then one partial batch."""
    from tf_repos_b200 import synth
    P, B, N, F = b.epoch_steps, a.B, a.N, a.F
    caps = {nm: e["list"].numel() for nm, e in b.updater.ep.items()}
    for step in range(2 * P + 1):
        bs = B if step < 2 * P else partial_B
        ids, vals, labels = synth.criteo_batch(bs, N, F, seed=1000 + step, device="cuda")
        la = a.train_step(ids, vals, labels)
        lb = b.train_step(ids, vals, labels)
        assert torch.equal(la[0], lb[0]), f"CE differs at step {step}"
        if step in flush_at:
            b.flush()
        for nm, e in b.updater.ep.items():
            assert int(e["list_count"].item()) <= caps[nm], f"{nm}: list overflow at step {step}"
        assert int(b.updater.list_overflow.item()) == 0
        if step in check_at:
            _same_state(a, b, f"after step {step}")
    _same_state(a, b, "after the partial batch")
    a.check_ids(); b.check_ids()


def test_deepfm_readme_criteo_shape_deferred_equals_exact():
    """deep_ctr/README.md's Criteo command: field_size 39, feature_size 117581 (= 1 mod 4: fm_w takes the generic
    Adam sweep), K=32 (fm_v + fm_w through ctr_epoch_rows2 at K=32, fm_v through the packed sweep), batch 256,
    deep_layers 400,400,400, dropout 0.5, Adam 5e-4, l2 1e-4, default epoch_steps."""
    from tf_repos_b200.deepfm import DeepFM
    a, b = _model_pair(DeepFM, field_size=39, feature_size=117_581, embedding_size=32, batch_size=256,
                       deep_layers="400,400,400", dropout="0.5,0.5,0.5", learning_rate=5e-4, l2_reg=1e-4,
                       optimizer="Adam")
    assert b.epoch_steps == 8 and b.update_mode == "exact_deferred"
    _run_pair(a, b, flush_at=(3, 12), check_at=(7, 10, 15), partial_B=100)


def test_nfm_adagrad_linear_table_deferred_equals_exact():
    """NFM with Adagrad at its reference K=64 and a vocabulary of 117581 rows (= 1 mod 4): the `linear` table takes
    the generic non-Adam sweep, `emb` the K=64 epoch_sweep_kernel, both gathered through ctr_epoch_rows2."""
    from tf_repos_b200.nfm import NFM
    a, b = _model_pair(NFM, field_size=39, feature_size=117_581, embedding_size=64, batch_size=256,
                       deep_layers="128,64", dropout="0.5,0.8,0.8", learning_rate=0.05, l2_reg=1e-3,
                       optimizer="Adagrad")
    assert b.update_mode == "exact_deferred"
    _run_pair(a, b, flush_at=(2, 11), check_at=(7, 15), partial_B=77)
