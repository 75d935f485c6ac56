"""Device-side building blocks shared by every model: embedding tables with TF-semantics
optimizer state, the de-duplicated sparse update, the flat buffer of dense variables and the
hyper-parameter records the kernels read.

Everything numerical happens in libctr_b200.so (tf_repos_b200/csrc); torch provides memory.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import ops

# hyper record layout (see include/ctr_b200.h): {lr_t, beta1, beta2, eps, l2_reg, aux0, aux1, aux2}
HYPER_TABLE, HYPER_DENSE, HYPER_DENSE_L2 = 0, 1, 2


class OptimizerState:
    """Host mirror of tf.train.*Optimizer construction (DeepFM.py:204-211) + device hyper records.

    record 0: embedding tables (l2_reg as given)      -- sparse rows / dense sweep
    record 1: dense variables without L2 (MLP; the fully_connected regularizer is a no-op, A.3)
    record 2: dense variables with L2 (DCN cross_w / cross_b)
    """

    def __init__(self, optimizer: str, learning_rate: float, l2_reg: float, device, adagrad_init: float = 1e-8):
        self.adagrad_init = adagrad_init   # initial_accumulator_value: 1e-8 in DeepFM.py:207, 0.1 in the canned estimators
        if optimizer not in ops.OPT_BY_NAME:
            # the reference has no branch for e.g. 'GD' although the flag help lists it (DeepFM.py:50,204-211)
            raise NameError(f"optimizer {optimizer!r} is not one of {sorted(ops.OPT_BY_NAME)}")
        self.name = optimizer
        self.opt = ops.OPT_BY_NAME[optimizer]
        self.n_slots = ops.OPT_SLOTS[self.opt]
        self.device = device
        aux = (0.0, 0.0, 0.0)
        beta1, beta2, eps = 0.9, 0.999, 1e-8
        if optimizer == "Momentum":
            aux = (0.95, 0.0, 0.0)
        elif optimizer == "ftrl":
            aux = (-0.5, 0.0, 0.0)  # learning_rate_power, l1, l2 (FtrlOptimizer defaults)
        rec = lambda l2: [learning_rate, beta1, beta2, eps, l2, *aux]
        self.hyper = torch.tensor([rec(l2_reg), rec(0.0), rec(l2_reg)], dtype=torch.float32, device=device)
        # {beta1_power, beta2_power, lr, global_step}; Adam's powers start at beta (TF _create_slots)
        self.state = torch.tensor([beta1, beta2, learning_rate, 0.0], dtype=torch.float32, device=device)

    def slot_init(self, slot: int) -> float:
        if self.name == "Adagrad":
            return self.adagrad_init
        if self.name == "ftrl" and slot == 0:
            return 0.1           # FtrlOptimizer initial_accumulator_value default
        return 0.0

    def tick(self):
        """Start of a step.  For Adam: lr_t from the current beta powers, then advance them."""
        if self.name == "Adam":
            ops.adam_tick(self.state, self.hyper)
        else:  # only the global-step counter advances (it seeds the dropout masks)
            self.tick_epoch(0)

    def tick_epoch(self, j: int):
        """exact-deferred mode: like tick(), and records this step's lr_t in lr_table[j]."""
        if self.lr_table is None:
            self.lr_table = torch.zeros(ops.epoch_max_steps(), dtype=torch.float32, device=self.device)
        ops.epoch_tick(self.state, self.hyper, self.lr_table, j, self.name == "Adam")

    lr_table = None

    def record(self, which: int) -> torch.Tensor:
        return self.hyper[which]


class Table:
    """One embedding variable [N, K] (K == 1 for the first-order weights `fm_w` [N]) + its slots."""

    def __init__(self, name: str, N: int, K: int, opt: OptimizerState, device, init_std: Optional[float] = None,
                 seed: int = 0, value: Optional[torch.Tensor] = None):
        self.name, self.N, self.K = name, N, K
        shape = (N,) if K == 1 else (N, K)
        self.var = torch.empty(shape, dtype=torch.float32, device=device)
        if value is not None:
            self.var.copy_(value.reshape(shape))
        else:
            if init_std is None:  # glorot_normal_initializer (DeepFM.py:115-116): sqrt(2/(fan_in+fan_out))
                init_std = math.sqrt(2.0 / (N + N)) if K == 1 else math.sqrt(2.0 / (N + K))
            ops.init_trunc_normal(self.var, init_std, seed)
        self.slots: List[torch.Tensor] = []
        for s in range(opt.n_slots):
            t = torch.empty(shape, dtype=torch.float32, device=device)
            ops.fill(t, opt.slot_init(s))
            self.slots.append(t)

    def slot(self, i):
        return self.slots[i] if i < len(self.slots) else None


UPDATE_MODES = ("exact", "exact_deferred", "lazy")


def _check_mode(mode: str):
    if mode not in UPDATE_MODES:
        raise ValueError(f"update_mode {mode!r} is not one of {', '.join(UPDATE_MODES)}")


class SparseUpdater:
    """K3 + K4 for a group of tables that are all gathered with the SAME ids (DeepFM: fm_v and fm_w; the first
    table is [N,K], an optional second one the [N] first-order weights), and the step schedule of its update mode.

    update_mode
      "exact": TensorFlow semantics (SURVEY.md A.4) -- every table row moves every step (dense L2 gradient +
               non-lazy sparse Adam): gathered rows are computed first into a stage buffer from the pre-step
               state, the dense sweep then advances every row with g = l2*var, and the staged rows are patched
               back (HBM-bound).
      "exact_deferred": bit-identical state to "exact"; rows nothing gathered are replayed lazily
               (csrc/epoch.cu): one pass over HBM per `epoch_steps` steps.  The l2*l2_loss terms of `loss`
               become available at the end of each epoch.  Adagrad/Momentum/Ftrl with l2_reg == 0 are truly
               sparse in TF: there is nothing to defer, and the mode becomes "exact".
      "lazy" : only gathered rows are updated (what LazyAdam would do); NOT the reference's result.

    A model's train step calls begin_step(), catch_up(ids) before the forward reads any row, and
    finish_step(ids, g_rows, g_w) with the per-occurrence gradient rows; predict() and variable reads call flush().
    `tables` are the tables it steps ([N,K] first, then the [N] table when with_scalar_table); without them only the
    buffers are built.
    """

    def __init__(self, n_ids: int, N: int, K: int, opt: OptimizerState, device, with_scalar_table: bool,
                 tables: Sequence[Table] = (), update_mode: str = "exact", epoch_steps: int = 8, l2_reg: float = 0.0):
        _check_mode(update_mode)
        self.tables = list(tables)
        self.n, self.N, self.K, self.opt = n_ids, N, K, opt
        self.uw = ops.UniqueWorkspace(n_ids, N, device)
        f32 = dict(dtype=torch.float32, device=device)
        self.g_uniq = torch.empty(max(n_ids, 1) * K, **f32)
        self.gw_uniq = torch.empty(max(n_ids, 1), **f32) if with_scalar_table else None
        self.stage_v = torch.empty(3 * max(n_ids, 1) * K, **f32)
        self.stage_w = torch.empty(3 * max(n_ids, 1), **f32) if with_scalar_table else None
        self.n_part = ops.sweep_partials_count()
        self.partials_v = torch.zeros(self.n_part, **f32)
        self.partials_w = torch.zeros(self.n_part, **f32)
        self.red_ws = torch.empty(1024, **f32)
        # [l2*l2_loss(V), l2*l2_loss(W)] of the PRE-step tables (what `loss` of this step contains)
        self.reg = torch.zeros(2, **f32)
        self.sweep_events = None  # set to [] to collect (start, end) CUDA events around the V sweep
        self.sweep_steps = []     # parallel to sweep_events: steps replayed by each pass (deferred mode)
        self.l2_reg = float(l2_reg)
        self.epoch_steps, self.epoch_pos = epoch_steps, 0
        self.update_mode = update_mode
        if update_mode == "exact_deferred":
            if self.l2_reg == 0.0 and opt.name != "Adam":
                self.update_mode = "exact"
            else:
                self.enable_epochs(epoch_steps, self.tables)

    # ---- the step schedule -----------------------------------------------------------------------------------
    def begin_step(self):
        """Start of a train step: the optimizer tick (exact_deferred: also records lr_t at the epoch position)."""
        if self.update_mode != "exact_deferred":
            self.opt.tick()
            return
        if self.epoch_pos == 0:
            for e in self.ep.values():
                ops.fill(e["reg"], 0.0)
        self.opt.tick_epoch(self.epoch_pos)

    def catch_up(self, ids_flat: torch.Tensor):
        """exact_deferred: the rows `ids_flat` gathers are brought to the start of this step (no-op otherwise)."""
        if self.update_mode == "exact_deferred":
            ops.unique_segment(ids_flat, self.uw)
            self.epoch_rows([(t, None) for t in self.tables], self.epoch_pos, apply=False)

    def finish_step(self, ids_flat: torch.Tensor, g_rows: torch.Tensor, g_w: Optional[torch.Tensor] = None):
        """The table update of this step from the per-occurrence gradient rows of `ids_flat` (g_w: those of the
        scalar table).  exact_deferred reuses the de-duplication catch_up() made of the same ids, and closes the
        epoch with the sweep of every row after its last step."""
        gw_uniq = self.gw_uniq if g_w is not None else None
        if self.update_mode == "exact_deferred":
            ops.segment_sum_rows(g_rows, g_w, self.uw, self.K, self.g_uniq, gw_uniq)
            self.epoch_rows(list(zip(self.tables, (self.g_uniq, self.gw_uniq))), self.epoch_pos, apply=True)
            self.epoch_pos += 1
            if self.epoch_pos == self.epoch_steps:
                self.epoch_sweep(self.epoch_steps, reset=True)
                self.epoch_pos = 0
        else:
            ops.unique_segment(ids_flat, self.uw)
            ops.segment_sum_rows(g_rows, g_w, self.uw, self.K, self.g_uniq, gw_uniq)
            self.apply(exact=(self.update_mode == "exact"))

    def flush(self):
        """exact_deferred: bring every row to the current step (no-op otherwise)."""
        if self.update_mode == "exact_deferred" and self.epoch_pos > self.flush_pos:
            self.epoch_sweep(self.epoch_pos, reset=False)

    def set_mode(self, mode: str):
        """Switch between exact / exact_deferred / lazy on a live model (state stays consistent).  Unlike the
        constructor, this keeps exact_deferred for every optimizer."""
        _check_mode(mode)
        if self.update_mode == "exact_deferred" and self.epoch_pos > 0:
            self.epoch_sweep(self.epoch_pos, reset=True)
            self.epoch_pos = 0
        if mode == "exact_deferred" and not hasattr(self, "ep"):
            self.enable_epochs(self.epoch_steps, self.tables)
        self.update_mode = mode

    # ---- exact-deferred ("epoch") mode: csrc/epoch.cu ------------------------------------------------
    def enable_epochs(self, P: int, tables: Sequence[Table]):
        """Allocates the per-row `last` bytes and the per-step sum(var^2) accumulators.  An [N,K] table and the [N]
        table gathered with the same ids always hold the same `last` bytes: where the packed Adam sweep can take both
        in one pass (ops.epoch_shared_last_supported) they share ONE `last` array and one row list."""
        pmax = ops.epoch_max_steps()
        if not 1 <= P <= pmax:
            raise ValueError(f"epoch_steps={P}: must be in [1, {pmax}] (the `last` bytes and lr table hold {pmax} steps)")
        dev = tables[0].var.device
        self.P = P
        self.flush_pos = 0   # steps of the current epoch every row's stored state already contains (mid-epoch flush)
        self.n_epart = ops.epoch_partials_count()
        self.ep = {}
        # rows the packed Adam sweep found but could not list (a list smaller than include/ctr_b200.h's bound)
        self.list_overflow = torch.zeros(1, dtype=torch.int32, device=dev)
        self.shared_last = (len(tables) == 2 and tables[1].K == 1 and tables[0].N == tables[1].N
                            and tables[0].K in ops.EPOCH_ROWS2_K
                            and ops.epoch_shared_last_supported(self.opt.opt, tables[0].N, tables[0].K))
        for i, t in enumerate(tables):
            # rows gathered since the last sweep, collected by the packed Adam sweep for its second pass: at most
            # n distinct ids per step, P <= pmax steps per epoch (shared: the [N,K] table's list serves both)
            cap = 1 if (self.shared_last and i == 1) else max(min(self.n * pmax, t.N), 1)
            self.ep[t.name] = dict(
                list=torch.empty(cap, dtype=torch.int32, device=dev),
                list_count=torch.zeros(1, dtype=torch.int32, device=dev),
                last=torch.zeros(t.N, dtype=torch.uint8, device=dev),
                ss=torch.zeros(pmax, dtype=torch.float64, device=dev),
                partials=torch.zeros(pmax * self.n_epart, dtype=torch.float64, device=dev),
                reg=torch.zeros(pmax, dtype=torch.float32, device=dev))
        if self.shared_last:
            ev = self.ep[tables[0].name]
            self.ep[tables[1].name].update(last=ev["last"], list=ev["list"], list_count=ev["list_count"])

    def epoch_rows(self, tables_g, j: int, apply: bool):
        """tables_g: [(Table, g_uniq or None)].  apply=False: catch the gathered rows up to the start of
        step j; apply=True: take step j with the de-duplicated gradient."""
        o, uw = self.opt, self.uw
        if (len(tables_g) == 2 and tables_g[0][0].K in ops.EPOCH_ROWS2_K and tables_g[1][0].K == 1
                and tables_g[0][0].N == tables_g[1][0].N):
            (V, gv), (W, gw) = tables_g            # fm_v + fm_w: one launch for both tables
            ev, ew = self.ep[V.name], self.ep[W.name]
            # the catch-up hands the caught-up rows to the apply of the same step through stage_v / stage_w (free in
            # this mode; see ctr_epoch_rows2)
            ops.epoch_rows2(o.opt, apply, V, W, ev["last"], ew["last"], uw.uniq, uw.n_uniq, gv if apply else None,
                            gw if apply else None, self.n, o.record(HYPER_TABLE), o.lr_table, j, ev["ss"], ew["ss"],
                            self.stage_v, self.stage_w)
            return
        for t, g in tables_g:
            e = self.ep[t.name]
            ops.epoch_rows(o.opt, apply, t.var, t.slot(0), t.slot(1), e["last"], uw.uniq, uw.n_uniq,
                           g if apply else None, self.n, t.K, o.record(HYPER_TABLE), o.lr_table, j, e["ss"])

    def epoch_sweep(self, upto: int, reset: bool):
        """All rows -> state after `upto` steps of this epoch; per-step l2*l2_loss terms -> ep[.]['reg'].  One pass per
        table, or one pass for an [N,K] + [N] pair that shares `last` (and its row list)."""
        o = self.opt
        passes = [(self.tables[0], self.tables[1])] if self.shared_last else [(t, None) for t in self.tables]
        for t, w in passes:
            e = self.ep[t.name]
            ew = self.ep[w.name] if w is not None else dict(partials=None, ss=None)
            ev = None
            if self.sweep_events is not None and t.K > 1:
                ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                ev[0].record()
            ops.epoch_sweep(o.opt, t.var, t.slot(0), t.slot(1), e["last"], t.N, t.K, o.record(HYPER_TABLE),
                            o.lr_table, self.flush_pos, upto, reset, e["partials"], e["list"], e["list_count"],
                            e["ss"], self.list_overflow, W=w, w_ss_partials=ew["partials"], w_ss_rows=ew["ss"])
            if ev is not None:
                ev[1].record()
                self.sweep_events.append(ev)
                self.sweep_steps.append(upto - self.flush_pos)   # optimizer steps this pass replayed per element
            # accumulate: a mid-epoch flush and the epoch-end sweep each contribute their share
            for x in (self.ep[u.name] for u in (t, w) if u is not None):
                ops.epoch_reg_loss(x["ss"], x["partials"], self.n_epart, upto, 0.5 * self.l2_reg, x["reg"],
                                   accumulate=True)
        self.flush_pos = 0 if reset else upto

    def check_list_overflow(self):
        """Raises if an epoch sweep dropped gathered rows (their state is then not the every-step state)."""
        ovf = getattr(self, "list_overflow", None)
        n = int(ovf.item()) if ovf is not None else 0
        if n:
            ovf.zero_()
            raise RuntimeError(f"exact-deferred epoch sweep: {n} gathered rows did not fit in the row list and were "
                               "not caught up; the table state is invalid")

    def apply(self, exact: bool):
        o, uw, hyper = self.opt, self.uw, self.opt.record(HYPER_TABLE)
        n, l2_reg = self.n, self.l2_reg
        # TF's sparse Adagrad/Momentum/Ftrl touch only gathered rows unless the dense L2 gradient
        # makes every row an index; sparse Adam decays every row regardless.
        sweep = exact and (l2_reg != 0.0 or o.name == "Adam")
        tabs = [(self.tables[0], self.g_uniq, self.stage_v, self.partials_v, 0)]
        if len(self.tables) > 1:
            tabs.append((self.tables[1], self.gw_uniq, self.stage_w, self.partials_w, 1))
        for t, g, stage, partials, ri in tabs:
            ops.opt_sparse_rows(o.opt, t.var, t.slot(0), t.slot(1), uw.uniq, uw.n_uniq, g, n, t.K, hyper,
                                stage if sweep else None)
            if sweep:
                ev = None
                if self.sweep_events is not None and ri == 0:  # bench.py: time the dominant kernel live
                    ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                    ev[0].record()
                ops.opt_dense_sweep(o.opt, t.var, t.slot(0), t.slot(1), hyper, partials)
                if ev is not None:
                    ev[1].record()
                    self.sweep_events.append(ev)
                ops.opt_patch_rows(t.var, t.slot(0), t.slot(1), uw.uniq, uw.n_uniq, stage, n, t.K, o.n_slots)
                ops.reduce_sum(partials, 0.5 * l2_reg, self.reg[ri:ri + 1], self.red_ws)


class SparseModel:
    """What every model trained through a SparseUpdater shares.  The model sets `updater`, `N` (the global
    vocabulary), `oob` (the device [count, first] of the out-of-range ids its lookups met) and `device`, and
    provides variables() (TF name -> tensor) where it has one."""

    update_mode = property(lambda self: self.updater.update_mode)
    epoch_pos = property(lambda self: self.updater.epoch_pos)
    epoch_steps = property(lambda self: self.updater.epoch_steps)

    def flush(self):
        """exact_deferred: bring every row to the current step (no-op otherwise)."""
        self.updater.flush()

    def set_update_mode(self, mode: str):
        """Switch between exact / exact_deferred / lazy on a live model (state stays consistent)."""
        self.updater.set_mode(mode)

    def check_ids(self):
        """TF raises InvalidArgumentError for ids outside [0, feature_size); we count them on device."""
        self.updater.check_list_overflow()
        cnt, first = self.oob.tolist()
        if cnt:
            self.oob.zero_()
            raise IndexError(f"{cnt} feature ids outside [0, {self.N}) (first: {first}); "
                             "TensorFlow would raise InvalidArgumentError")

    def load_variables(self, values: Dict[str, torch.Tensor]):
        vs = self.variables()
        for name, v in values.items():
            vs[name].copy_(v.to(self.device, torch.float32).reshape(vs[name].shape))


class DenseVars:
    """All dense variables of a model in ONE flat fp32 buffer (+ flat grads and slots) so that the
    optimizer apply is a single launch.  Views keep the TF variable names."""

    def __init__(self, specs: Sequence[Tuple[str, Tuple[int, ...]]], opt: OptimizerState, device,
                 l2_names: Sequence[str] = (), tail: int = 4):
        # variables with L2 first, so each group is one contiguous range
        specs = [s for s in specs if s[0] in l2_names] + [s for s in specs if s[0] not in l2_names]
        self.opt = opt
        sizes = [int(math.prod(shape)) for _, shape in specs]
        pad = lambda x: (x + 3) // 4 * 4
        offs, o = [], 0
        for sz in sizes:
            offs.append(o)
            o += pad(sz)
        self.total = o
        self.n_l2 = sum(pad(sz) for (nm, _), sz in zip(specs, sizes) if nm in l2_names)
        f32 = dict(dtype=torch.float32, device=device)
        self.flat = torch.zeros(max(self.total, 4), **f32)
        # `tail` extra floats ride along in the gradient buffer (per-rank loss terms) so that ONE
        # all-reduce covers dense gradients + loss under data parallelism
        self.grad = torch.zeros(max(self.total, 4) + tail, **f32)
        self.tail = self.grad[max(self.total, 4):]
        self.slots = []
        for s in range(opt.n_slots):
            t = torch.empty(max(self.total, 4), **f32)
            ops.fill(t, opt.slot_init(s))
            self.slots.append(t)
        self.views: Dict[str, torch.Tensor] = {}
        self.grads: Dict[str, torch.Tensor] = {}
        for (nm, shape), off, sz in zip(specs, offs, sizes):
            self.views[nm] = self.flat[off:off + sz].view(shape)
            self.grads[nm] = self.grad[off:off + sz].view(shape)

    def __getitem__(self, name):
        return self.views[name]

    def apply(self):
        o = self.opt
        s1 = lambda a, b: (self.slots[1][a:b] if o.n_slots > 1 else None)
        if self.n_l2:
            ops.opt_dense_grad(o.opt, self.flat[:self.n_l2], self.slots[0][:self.n_l2], s1(0, self.n_l2),
                               self.grad[:self.n_l2], o.record(HYPER_DENSE_L2))
        if self.total > self.n_l2:
            a, b = self.n_l2, self.total
            ops.opt_dense_grad(o.opt, self.flat[a:b], self.slots[0][a:b], s1(a, b), self.grad[a:b],
                               o.record(HYPER_DENSE))
