"""The embedding-table kernels past 2^31 elements, the size bench.py's headline trains at (feature_size 2e8 x K=16:
3.2e9 fp32 elements, 12.8 GB per tensor).  2^31 is where a signed 32-bit element index, or any 32-bit byte offset,
stops giving the same answer as a 64-bit one; every other test builds tables below it.

Shared setup.  One module-scoped set of three flat fp32 buffers (var and two slots) of E = 2^31 + 2^21 + 51 elements
(8.6 GB each: 25.8 GB for Adam).  E is 3 mod 4, so the dense sweep's scalar tail lies above 2^31.  Each test views
them as [E // K, K] for its K, without copies.  Pre-states are generated chunk by chunk (CHUNK elements) on the
device from a generator seeded by (seed, buffer, chunk), so any chunk's pre-state can be regenerated instead of
kept; the two chunks around element 2^31, the last chunk and every third chunk hold the `_extreme` mix of
test_gpu_epoch_dispatch.py (zeros, denormals, values near FLT_MIN).  CHUNK is 2^25 rather than 2^27 to keep the
peak under 30 GB while a chunk's pre-state and a step's temporaries live beside the model test's tables.

Gathered rows (per K): the rows just below and above element 2^31 (for K=12 one of them straddles it), rows in the
top 1% of the table, row N-1, and low rows, where a wrapped 32-bit offset would land.

References.
  * Gathered rows: the fp32 oracle of oracle/tf_semantics.py on the host, bit for bit (K4, epoch kernels), or
    host fp32 products and the fp64 bounds of test_gpu_fm_batch_norm.py (K1).
  * Whole tables: `_restate`, a torch-on-CUDA restatement of step_sparse (csrc/optim_steps.cuh) with one eager op
    per rounded operation, applied chunk by chunk to the regenerated pre-state.  Every test that relies on it first
    pins it bit for bit against the CPU oracle on 2^20 elements of the boundary chunks (torch's CPU sqrt is not
    correctly rounded, so the restatement itself never runs on the CPU).  torch.equal throughout: the packed Adam
    loops may give -0 where the oracle gives +0 (adam_untouched).

Each test prints its peak device memory and wall time, and skips (naming the bytes it needs) only when the device
does not have that much free.
"""
import time
import types

import numpy as np
import pytest
import torch

from tests.test_gpu_din_attention import _bits_equal, _within
from tests.test_gpu_epoch_dispatch import EPOCH_MAX, L2, _extreme, _oracle_step, _Tab
from tests.test_gpu_esmm_deepmvm_fp64 import _sweep_depth
from tests.test_gpu_fm_batch_norm import _fm_ref, gam

pytestmark = pytest.mark.gpu

B31 = 1 << 31
E = B31 + (1 << 21) + 51
CHUNK = 1 << 25
PIECE = 1 << 22                  # _extreme's fp64 temporaries are generated this many elements at a time
N_CHUNKS = -(-E // CHUNK)
EXTREME_CHUNKS = {B31 // CHUNK - 1, B31 // CHUNK, N_CHUNKS - 1} | set(range(0, N_CHUNKS, 3))
LR = {"Adam": 5e-3, "Adagrad": 0.05, "ftrl": 0.05}
GB = 1e9


# ---------------------------------------------------------------------------------------------------------------------
# memory, buffers and pre-states
# ---------------------------------------------------------------------------------------------------------------------
def _need(nbytes, what):
    """Skip (with the number of bytes) unless the device has nbytes free."""
    torch.cuda.empty_cache()                     # blocks torch caches are free for this test too
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip(f"{what} needs {nbytes} bytes ({nbytes / GB:.1f} GB) of free device memory, {free} are free")


class _Buffers:
    """The three E-element tensors, allocated on first use and freed for the model test."""

    def __init__(self):
        self.t = None

    def get(self, n):
        if self.t is None:
            _need(3 * E * 4 + (3 << 30), "three E-element fp32 tables plus chunk temporaries")
            self.t = [torch.empty(E, dtype=torch.float32, device="cuda") for _ in range(3)]
        return self.t[:n]

    def free(self):
        self.t = None
        torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def bufs():
    b = _Buffers()
    yield b
    b.free()


@pytest.fixture(autouse=True)
def _report():
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    yield
    torch.cuda.synchronize()
    print(f"\npeak device memory {torch.cuda.max_memory_allocated() / GB:.2f} GB, wall {time.time() - t0:.1f} s")


def _gen(seed, which, c):
    return torch.Generator(device="cuda").manual_seed((seed * 7919 + which) * 100_003 + c)


def _slot_init(opt, which):
    """which: 0 var, 1 slot0, 2 slot1 (engine.OptimizerState.slot_init)."""
    return {("Adagrad", 1): 1e-8, ("ftrl", 1): 0.1}.get((opt, which), 0.0)


def _chunk(seed, opt, which, c, lo=None, hi=None):
    """Pre-state of buffer `which` on elements [lo, hi) of chunk c (default: the whole chunk), as _Tab lays it out:
    ordinary chunks var ~ 0.1 N(0,1), slots init + 0.01 U(0,1); extreme chunks the _extreme mix (non-negative
    for the accumulators)."""
    c_lo, c_hi = c * CHUNK, min((c + 1) * CHUNK, E)
    g = _gen(seed, which, c)
    n = c_hi - c_lo
    if c in EXTREME_CHUNKS:
        nonneg = (opt, which) in (("Adam", 2), ("Adagrad", 1), ("ftrl", 1))
        x = torch.empty(n, dtype=torch.float32, device="cuda")
        for p in range(0, n, PIECE):
            x[p:p + PIECE] = _extreme((min(PIECE, n - p),), g, nonneg)
        if _slot_init(opt, which):
            x.add_(_slot_init(opt, which))
    elif which == 0:
        x = torch.randn(n, generator=g, device="cuda").mul_(0.1)
    else:
        x = torch.rand(n, generator=g, device="cuda").mul_(0.01).add_(_slot_init(opt, which))
    lo = c_lo if lo is None else lo
    hi = c_hi if hi is None else hi
    return x[lo - c_lo:hi - c_lo]


def _chunks(n):
    for c in range(-(-n // CHUNK)):
        yield c, c * CHUNK, min((c + 1) * CHUNK, n)


def _fill(tabs, seed, opt, n=E):
    """Write the pre-state into the first n elements of each flat table."""
    for which, t in enumerate(tabs):
        for c, lo, hi in _chunks(n):
            t[lo:hi] = _chunk(seed, opt, which, c, lo, hi)


def _row_set(K, N):
    """Rows around element 2^31, in the top 1%, N-1, and low rows; plus rows nothing may touch (`spare`)."""
    b = B31 // K
    top = N - N // 100
    rows = [0, 1, 2, 3, 17, 1000, 65_537, 1_000_003, b - 2, b - 1, b, b + 1, b + 2,
            top, top + 7, top + 1234, N - 5, N - 2, N - 1]
    spare = [4, b - 4, b + 4, top + 1, N - 3]
    assert max(rows) < N and b * K <= B31 < (b + 1) * K
    return sorted(set(rows)), spare


# ---------------------------------------------------------------------------------------------------------------------
# the restatement of step_sparse (csrc/optim_steps.cuh) and its pin against the CPU oracle
# ---------------------------------------------------------------------------------------------------------------------
def _f(x, dev):
    return torch.tensor(x, dtype=torch.float32, device=dev)


def _restate(opt, var, s0, s1, lr, g=None, l2=L2):
    """One step_sparse<OPT> in place, G = l2*var (+ g): one torch op per rounded fp32 operation, in the kernel's
    order (no contraction is possible across eager ops).  lr: 0-dim fp32 tensor on var's device."""
    d = var.device
    one = _f(1.0, d)
    G = torch.mul(_f(l2, d), var)
    if g is not None:
        G = torch.add(g, G)
    if opt == "Adam":
        b1, b2, eps = _f(0.9, d), _f(0.999, d), _f(1e-8, d)
        s0.mul_(b1).add_(torch.mul(G, torch.sub(one, b1)))
        G.mul_(G).mul_(torch.sub(one, b2))               # in place: at most two chunk-sized temporaries
        s1.mul_(b2).add_(G)
        torch.sqrt(s1, out=G).add_(eps)
        var.sub_(torch.mul(lr, s0).div_(G))
    elif opt == "Adagrad":
        s0.add_(torch.mul(G, G))
        var.sub_(torch.mul(torch.mul(lr, G), torch.div(one, torch.sqrt(s0))))
    elif opt == "ftrl":                                  # lr_power -0.5, l1 = l2(ftrl) = 0 (FtrlOptimizer defaults)
        new_acc = torch.add(s0, torch.mul(G, G))
        pn, po = torch.sqrt(new_acc), torch.sqrt(s0)
        s1.add_(torch.sub(G, torch.mul(torch.div(torch.sub(pn, po), lr), var)))
        xx = torch.sub(torch.mul(_f(0.0, d), torch.sign(s1)), s1)
        yy = torch.add(torch.div(pn, lr), torch.mul(_f(2.0, d), _f(0.0, d)))
        var.copy_(torch.where(s1.abs() > _f(0.0, d), torch.div(xx, yy), _f(0.0, d)))
        s0.copy_(new_acc)
    else:
        raise ValueError(opt)


class _Lr:
    """lr_t of every global step: AdamHyper.lr_t() (what adam_tick / epoch_tick compute) or the constant lr."""

    def __init__(self, opt, lr=None):
        from oracle import tf_semantics as tfs
        self.opt, self.lr, self.vals = opt, LR[opt] if lr is None else lr, []
        self.h = tfs.AdamHyper(self.lr)

    def __getitem__(self, t):
        while len(self.vals) <= t:
            self.vals.append(self.h.lr_t() if self.opt == "Adam" else torch.tensor(self.lr))
            self.h.finish()
        return self.vals[t]


def _pin_restatement(opt, seed, l2=L2, lr=None):
    """2^20 elements around element 2^31 (both extreme chunks), three steps -- two with G = l2*var, one with a
    gradient added -- on CUDA against oracle/tf_semantics.py on the CPU, bit for bit."""
    lo, hi = B31 - (1 << 19), B31 + (1 << 19)
    st = [torch.cat([_chunk(seed, opt, w, c, max(lo, c * CHUNK), min(hi, (c + 1) * CHUNK))
                     for c in (B31 // CHUNK - 1, B31 // CHUNK)]) for w in range(3)]
    n_sl = 1 if opt == "Adagrad" else 2
    host = [s.cpu() for s in st]
    lrs = _Lr(opt, lr)
    grad = torch.randn(hi - lo, generator=torch.Generator().manual_seed(seed)) * 0.05
    for t in range(3):
        g = grad if t == 2 else None
        _restate(opt, st[0], st[1], st[2], lrs[t].cuda(), None if g is None else g.cuda(), l2)
        G = torch.tensor(l2) * host[0]
        if g is not None:
            G = g + G
        v, sl = _oracle_step(opt, host[0], host[1:1 + n_sl], G, lrs.lr, _AdamAt(lrs[t]))
        host = [v] + sl + host[1 + n_sl:]
        for w in range(1 + n_sl):
            assert torch.equal(st[w].cpu(), host[w]), f"{opt}: the CUDA restatement differs from the oracle " \
                f"(buffer {w}, step {t}) in {int((st[w].cpu() != host[w]).sum())} elements"


class _AdamAt:
    """AdamHyper-compatible view of one step's lr_t (for _oracle_step)."""

    def __init__(self, lr_t):
        self.b1, self.b2, self.eps = torch.tensor(0.9), torch.tensor(0.999), torch.tensor(1e-8)
        self._lr = lr_t

    def lr_t(self):
        return self._lr


# ---------------------------------------------------------------------------------------------------------------------
# gathered rows on the host (every-step or lazy oracle) and the whole-table check
# ---------------------------------------------------------------------------------------------------------------------
class _Rows:
    """The oracle states of the rows a test gathers, after 0, 1, ... global steps."""

    def __init__(self, opt, seed, K, rows, tabs):
        self.opt, self.K = opt, K
        self.rows = np.asarray(rows, dtype=np.int64)
        self.n_sl = 1 if opt == "Adagrad" else 2
        idx = torch.from_numpy((self.rows[:, None] * K + np.arange(K)).reshape(-1))
        self.elem = idx                                  # flat element index of every gathered element
        self.pos = {int(r): i for i, r in enumerate(self.rows)}
        state = [t[idx.cuda()].view(-1, K).cpu() for t in tabs[:1 + self.n_sl]]
        self.snaps = [(state[0], state[1:])]
        self.lrs = _Lr(opt)

    def step(self, t, gathered, g, every_row=True):
        """Global step t.  gathered: rows (sorted), g: their gradients [n, K].  every_row: TF's every-row update
        (exact / exact-deferred); else only the gathered rows move (lazy)."""
        var, slots = self.snaps[-1]
        i = torch.tensor([self.pos[int(r)] for r in gathered], dtype=torch.long)
        G = torch.tensor(L2) * var
        if i.numel():
            G[i] = g + G[i]
        if every_row:
            nv, ns = _oracle_step(self.opt, var, slots, G, LR[self.opt], _AdamAt(self.lrs[t]))
        else:
            nv, ns = var.clone(), [s.clone() for s in slots]
            if i.numel():
                sv, ss = _oracle_step(self.opt, var[i], [s[i] for s in slots], G[i], LR[self.opt], _AdamAt(self.lrs[t]))
                nv[i] = sv
                for a, b in zip(ns, ss):
                    a[i] = b
        self.snaps.append((nv, ns))

    def at(self, steps):
        """[n_rows*K] flat values of each buffer with row r taken after steps[r] global steps."""
        out = []
        for w in range(1 + self.n_sl):
            rows = [(self.snaps[s][0] if w == 0 else self.snaps[s][1][w - 1])[r] for r, s in enumerate(steps)]
            out.append(torch.stack(rows).reshape(-1))
        return out


def _check_tables(what, opt, seed, tabs, n, t_untouched, rows=None, row_steps=None, lrs=None, sums_upto=0, l2=L2):
    """Every element of the first n elements of each table: the pre-state after t_untouched untouched-row steps
    (the restatement), except the gathered rows, which must equal rows.at(row_steps); t_untouched None checks
    nothing.  Returns the fp64 sum(var^2) of the every-step state after s steps for s < sums_upto (for the
    sweeps' l2 terms)."""
    n_tab = len(tabs)
    lrs = lrs or _Lr(opt)
    want_rows = rows.at(row_steps) if rows is not None and t_untouched is not None else None
    elem = rows.elem.numpy() if rows is not None else np.zeros(0, np.int64)
    sums = [0.0] * sums_upto
    for c, lo, hi in _chunks(n):
        st = [_chunk(seed, opt, w, c, lo, hi) for w in range(3)]
        m = (elem >= lo) & (elem < hi)
        loc = torch.from_numpy(elem[m] - lo).cuda()
        steps = max(t_untouched or 0, sums_upto)
        for s in range(steps + 1):
            if s < sums_upto:                            # the gathered rows are added from their oracle states
                for p in range(0, hi - lo, PIECE):
                    sums[s] += float(st[0][p:p + PIECE].double().square().sum())
                sums[s] -= float(st[0][loc].double().square().sum())
            if s == t_untouched:
                for w in range(n_tab):
                    exp = st[w]
                    if loc.numel():
                        exp = exp.clone()
                        exp[loc] = want_rows[w][torch.from_numpy(np.nonzero(m)[0])].cuda()
                    got = tabs[w][lo:hi]
                    if not torch.equal(got, exp):
                        bad = (got != exp).nonzero().flatten()
                        e0 = int(bad[0]) + lo
                        raise AssertionError(f"{what}: buffer {w} differs in {bad.numel()} elements of [{lo}, {hi}); "
                                             f"first at element {e0}: {float(got[e0 - lo])!r} vs "
                                             f"{float(exp[e0 - lo])!r}")
                    del exp
            if s < steps:
                _restate(opt, st[0], st[1], st[2], lrs[s].cuda(), l2=l2)
    if rows is not None:
        for s in range(sums_upto):
            sums[s] += float((rows.snaps[s][0].double() ** 2).sum())
    return sums


def _ids(rows, gen, lo_frac=0.5):
    """A random sorted subset of the rows (at least lo_frac of them)."""
    n = int(torch.randint(int(lo_frac * len(rows)), len(rows) + 1, (1,), generator=gen))
    pick = np.sort(np.asarray(rows)[torch.randperm(len(rows), generator=gen)[:n].numpy()])
    return pick


# ---------------------------------------------------------------------------------------------------------------------
# 1. K1 gathers: fm_embed_fwd (LDG K=16, TMA K=128, generic K=12), DIN's gather_scale_rows, gather_scalar
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [16, 128, 12])
def test_k1_gathers_past_2_31(bufs, K):
    from tf_repos_b200 import ops
    var, s0 = bufs.get(2)
    seed = 100 + K
    _fill([var, s0], seed, "Adam")
    N = E // K
    V = var[:N * K].view(N, K)
    W = s0[:N]
    rows, _ = _row_set(K, N)
    gen = torch.Generator().manual_seed(seed)
    B, F = 64, 39
    rows_t = torch.tensor(rows, dtype=torch.int64)
    sel = torch.randint(0, len(rows), (B, F), generator=gen)
    sel.view(-1)[:len(rows)] = torch.arange(len(rows))             # every row at least once
    ids = rows_t[sel]
    vals = (torch.rand(B, F, generator=gen) * 2 - 0.5).float()
    Vh = V[rows_t.cuda()].cpu()                                    # the gathered rows, copied by torch
    Wh = W[rows_t.cuda()].cpu()
    ref = _fm_ref(sel, vals, Vh, Wh)
    d = "cuda"
    for dt in (torch.int32, torch.int64):
        tag = f"K={K} ids {dt}"
        x = torch.full((B, F * K), float("nan"), device=d)
        yw, y2, S = (torch.full(s, float("nan"), device=d) for s in ((B,), (B,), (B, K)))
        ops.fm_embed_fwd(ids.to(dt).to(d), vals.to(d), V, W, ops.FM_DEEPFM, x=x, y_w=yw, y2=y2, S=S)
        torch.cuda.synchronize()
        _bits_equal(x, ref["x"], f"{tag}: x = V[id]*val")
        _within(S, ref["S"], ref["S_bound"], f"{tag}: S")
        _within(yw, ref["y_w"], ref["y_w_bound"], f"{tag}: y_w")
        _within(y2, ref["y2"], ref["y2_bound"], f"{tag}: y2")
    ids32 = ids.reshape(-1).to(torch.int32).to(d)
    if K in (16, 128):                                             # DIN's kernels take K in {4, ..., 256}
        wgt = vals.reshape(-1)
        out = torch.full((B * F, K), float("nan"), device=d)
        ops.gather_scale_rows(ids32, wgt.to(d), V, out, 1, K)
        _bits_equal(out, Vh[sel.reshape(-1)] * wgt[:, None], f"K={K}: gather_scale_rows")
    # the scalar gather over the whole flat buffer: int32 ids up to 2^31 - 1, i.e. byte offsets up to 2^33
    flat_ids = torch.tensor([0, 5, 1 << 30, B31 - 3, B31 - 2, B31 - 1] + [r * K for r in rows if r * K < B31],
                            dtype=torch.int64)
    out = torch.full((flat_ids.numel(),), float("nan"), device=d)
    ops.gather_scalar(flat_ids.to(torch.int32).to(d), var, out)
    _bits_equal(out, var[flat_ids.cuda()].cpu(), f"K={K}: gather_scalar")


# ---------------------------------------------------------------------------------------------------------------------
# 2. K4: exact (sparse rows to stage, dense sweep, patch) and lazy (sparse rows in place)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [16, 256, 12])
@pytest.mark.parametrize("opt", ["Adam", "ftrl", "Adagrad"])
@pytest.mark.parametrize("mode", ["exact", "lazy"])
def test_k4_sparse_rows_and_dense_sweep_past_2_31(bufs, mode, opt, K):
    from tf_repos_b200 import engine, ops
    n_sl = 1 if opt == "Adagrad" else 2
    tabs = bufs.get(1 + n_sl)
    seed = 200 + 7 * K + len(opt)
    _pin_restatement(opt, seed)
    _fill(tabs, seed, opt)
    N = E // K
    var = tabs[0][:N * K].view(N, K)
    sl = [t[:N * K].view(N, K) for t in tabs[1:]] + [None] * (2 - n_sl)
    rows, spare = _row_set(K, N)
    o = engine.OptimizerState(opt, LR[opt], L2, "cuda")
    R = _Rows(opt, seed, K, rows, tabs)
    gen = torch.Generator().manual_seed(seed)
    n_max = len(rows) + len(spare)
    stage = torch.empty(3 * n_max * K, dtype=torch.float32, device="cuda")
    partials = torch.zeros(ops.sweep_partials_count(), dtype=torch.float32, device="cuda")
    for t in range(2):
        o.tick()
        if opt == "Adam":
            assert torch.equal(o.hyper[0, 0].cpu(), R.lrs[t]), "adam_tick's lr_t"
        pick = _ids(rows, gen)
        uniq = torch.tensor(np.concatenate([pick, spare]), dtype=torch.int32, device="cuda")
        n_uniq = torch.tensor([len(pick)], dtype=torch.int32, device="cuda")
        g = (torch.randn(n_max, K, generator=gen) * 0.05).float()
        R.step(t, pick, g[:len(pick)], every_row=(mode == "exact"))
        if mode == "exact":
            ops.opt_sparse_rows(o.opt, var, sl[0], sl[1], uniq, n_uniq, g.cuda(), n_max, K, o.record(0), stage)
            partials.zero_()
            n_part = ops.opt_dense_sweep(o.opt, tabs[0], tabs[1], tabs[2] if n_sl == 2 else None, o.record(0),
                                         partials)
            ops.opt_patch_rows(var, sl[0], sl[1], uniq, n_uniq, stage, n_max, K, n_sl)
        else:
            ops.opt_sparse_rows(o.opt, var, sl[0], sl[1], uniq, n_uniq, g.cuda(), n_max, K, o.record(0))
        torch.cuda.synchronize()
        what = f"{mode} {opt} K={K} step {t}"
        got_rows = [x[torch.from_numpy(R.elem.numpy()).cuda()].cpu() for x in tabs]
        for w, want in enumerate(R.at([t + 1] * len(rows))):
            _bits_equal(got_rows[w], want, f"{what}: gathered rows, buffer {w}")
        sums = _check_tables(what, opt, seed, tabs, E, t + 1 if mode == "exact" else 0, R, [t + 1] * len(rows),
                             R.lrs, sums_upto=(t + 1 if mode == "exact" else 0))
        if mode == "exact":                      # sum(var^2) at the start of step t, fp32 partials of the sweep
            got = float(partials[:n_part].double().sum())
            _within([got], [sums[t]], [gam(_sweep_depth(E)) * sums[t]], f"{what}: the sweep's sum(var^2)")


# ---------------------------------------------------------------------------------------------------------------------
# 3. exact-deferred epoch kernels: one epoch of P = 4 with a mid-epoch flush
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("opt,K", [("Adam", 16), ("Adam", 12), ("Adagrad", 16)])
def test_epoch_kernels_past_2_31(bufs, opt, K):
    """Adam K=16: epoch_rows_kernel + the packed sweep (the headline); Adam K=12: epoch_rows_generic_kernel + the
    packed sweep; Adagrad K=16: epoch_rows_kernel + epoch_sweep_kernel<ADAGRAD>."""
    from tf_repos_b200 import engine, ops
    P, FLUSH = 4, 2
    n_sl = 1 if opt == "Adagrad" else 2
    tabs = bufs.get(1 + n_sl)
    seed = 300 + 7 * K + len(opt)
    _pin_restatement(opt, seed)
    N = E // K
    n = N * K
    _fill(tabs, seed, opt, n)
    var = tabs[0][:n].view(N, K)
    sl = [x[:n].view(N, K) for x in tabs[1:]] + [None] * (2 - n_sl)
    rows, spare = _row_set(K, N)
    o = engine.OptimizerState(opt, LR[opt], L2, "cuda")
    R = _Rows(opt, seed, K, rows, tabs)
    gen = torch.Generator().manual_seed(seed)
    n_max = len(rows) + len(spare)
    dev = "cuda"
    last = torch.zeros(N, dtype=torch.uint8, device=dev)
    ss = torch.zeros(EPOCH_MAX, dtype=torch.float64, device=dev)
    n_epart = ops.epoch_partials_count()
    partials = torch.zeros(EPOCH_MAX * n_epart, dtype=torch.float64, device=dev)
    reg = torch.zeros(EPOCH_MAX, dtype=torch.float32, device=dev)
    cap = min(n_max * EPOCH_MAX, N)
    lst = torch.empty(cap, dtype=torch.int32, device=dev)
    list_count = torch.zeros(1, dtype=torch.int32, device=dev)
    overflow = torch.zeros(1, dtype=torch.int32, device=dev)
    last_exp = {r: 0 for r in rows}
    flat_t = 0                                    # steps the rows nothing gathered hold (every row's `last`)
    tab = types.SimpleNamespace(N=n, K=1)         # _Tab.reg_tol's chain over n elements

    def check(what, t_untouched, base):
        torch.cuda.synchronize()
        want_last = torch.full((N,), t_untouched - base, dtype=torch.uint8)
        want_last[torch.tensor(rows)] = torch.tensor([last_exp[r] for r in rows], dtype=torch.uint8)
        got_last = last.cpu()
        if not torch.equal(got_last, want_last):
            bad = (got_last != want_last).nonzero().flatten()
            raise AssertionError(f"{what}: `last` differs in {bad.numel()} rows; row {int(bad[0])}: "
                                 f"{int(got_last[bad[0]])} (want {int(want_last[bad[0]])})")
        _check_tables(what, opt, seed, tabs, n, t_untouched, R, [base + last_exp[r] for r in rows], R.lrs)

    def sweep(upto, reset, base, what):
        nonlocal flat_t
        ops.epoch_sweep(o.opt, tabs[0], tabs[1], tabs[2] if n_sl == 2 else None, last, N, K, o.record(0),
                        o.lr_table, flat_t - base, upto, reset, partials, lst, list_count, ss, overflow)
        ops.epoch_reg_loss(ss, partials, n_epart, upto, 0.5 * L2, reg, accumulate=True)
        flat_t = base + upto
        for r in rows:
            last_exp[r] = 0 if reset else upto
        check(what, flat_t, base + (upto if reset else 0))
        assert int(list_count.item()) <= cap and int(overflow.item()) == 0, f"{what}: row list overflow"
        # 0.5*l2*sum(var^2) of the every-step state at the start of each step, fp64
        sums = _check_tables(what, opt, seed, tabs, n, None, R, None, R.lrs, sums_upto=upto)
        got = reg[:upto].double().cpu().numpy()
        for s in range(upto):
            want = float(np.float32(0.5 * L2)) * sums[s]
            _within([got[s]], [want], [_Tab.reg_tol(tab, want)], f"{what}: reg[{s}]")

    ops.fill(reg, 0.0)
    for j in range(P):
        what = f"{opt} K={K} step {j}"
        o.tick_epoch(j)
        want_lr = R.lrs[j]
        assert torch.equal(o.lr_table[j].cpu().view(torch.int32), want_lr.float().view(torch.int32)), what
        pick = _ids(rows, gen)
        uniq = torch.tensor(np.concatenate([pick, spare]), dtype=torch.int32, device=dev)
        n_uniq = torch.tensor([len(pick)], dtype=torch.int32, device=dev)
        ops.epoch_rows(o.opt, False, var, sl[0], sl[1], last, uniq, n_uniq, None, n_max, K, o.record(0),
                       o.lr_table, j, ss)
        for r in pick:
            last_exp[int(r)] = j
        check(what + " catch-up", flat_t, 0)
        g = (torch.randn(n_max, K, generator=gen) * 0.05).float()
        R.step(j, pick, g[:len(pick)])
        ops.epoch_rows(o.opt, True, var, sl[0], sl[1], last, uniq, n_uniq, g.cuda(), n_max, K, o.record(0),
                       o.lr_table, j, ss)
        for r in pick:
            last_exp[int(r)] = j + 1
        check(what + " apply", flat_t, 0)
        if j + 1 == FLUSH:
            sweep(FLUSH, False, 0, f"{what}: flush at {FLUSH}")
        if j + 1 == P:
            sweep(P, True, 0, f"{what}: epoch end")


# ---------------------------------------------------------------------------------------------------------------------
# 4. DeepFM at the headline's hyper-parameters, its rows shifted past element 2^31
# ---------------------------------------------------------------------------------------------------------------------
def test_deepfm_headline_config_shifted_past_2_31(bufs):
    """bench.py's configuration (K=16, Adam 5e-4, l2 1e-4, deep_layers 256,128,64, dropout 0.5, exact_deferred with
    epochs of 16 steps, batch 8192) on a table of OFF + NS rows (OFF*16 > 2^31), trained on criteo_batch ids + OFF,
    against the same model with NS rows trained on the unshifted ids.  The shift is monotone, so it keeps the unique
    order and every occurrence order, and DeepFM's L2 gradient is row-local: the CE of every step, the window
    [OFF, OFF + NS) and the dense weights must be the small model's bits; rows [0, OFF), which nothing gathers, must
    hold the untouched-row recurrence after every step; the l2 terms differ by those rows' share."""
    from tf_repos_b200 import synth
    from tf_repos_b200.deepfm import DeepFM
    bufs.free()
    OFF, NS, K, P, B = (1 << 27) + 5, 200_000, 16, 16, 8192
    NB, l2, lr, seed = OFF + NS, 1e-4, 5e-4, 400
    _need(3 * NB * (K + 1) * 4 + (2 << 30), "DeepFM with 2^31 + 3.2e6 fm_v elements")
    _pin_restatement("Adam", seed, l2, lr)
    kw = dict(deep_layers="256,128,64", dropout="0.5,0.5,0.5", l2_reg=l2, learning_rate=lr, optimizer="Adam",
              update_mode="exact_deferred", epoch_steps=P, device="cuda:0")
    big = DeepFM(39, NB, K, B, **kw)
    small = DeepFM(39, NS, K, B, **kw)
    tabs = {}
    for i, (tb, ts) in enumerate(((big.fm_v, small.fm_v), (big.fm_w, small.fm_w))):
        flat = [x.view(-1) for x in [tb.var] + tb.slots]
        n = OFF * tb.var[0].numel() if tb.var.dim() == 2 else OFF
        _fill(flat, seed + i, "Adam", n)
        for a, b in zip([tb.var] + tb.slots, [ts.var] + ts.slots):
            a[OFF:] = b
        tabs[tb.name] = (flat, n, seed + i)
    big.dense.flat.copy_(small.dense.flat)
    reg_big, reg_small = [], []
    for step in range(P + P + 7):
        ids, vals, labels = synth.criteo_batch(B, NS, 39, seed=step, device="cuda")
        ls = small.train_step(ids, vals, labels)
        lb = big.train_step(ids + OFF, vals, labels)
        assert torch.equal(ls[0], lb[0]), f"CE differs at step {step}"
        if step in (20, 34):
            big.flush(); small.flush()
        if step % P == P - 1:
            reg_big.append(big.epoch_reg_terms().double().cpu())
            reg_small.append(small.epoch_reg_terms().double().cpu())
    big.flush(); small.flush()
    big.check_ids(); small.check_ids()
    for tb, ts in ((big.fm_v, small.fm_v), (big.fm_w, small.fm_w)):
        for i, (a, b) in enumerate(zip([tb.var] + tb.slots, [ts.var] + ts.slots)):
            assert torch.equal(a[OFF:], b), f"{tb.name} buffer {i}: window differs from the small model"
    assert torch.equal(big.dense.flat, small.dense.flat), "dense variables"
    ids, vals, _ = synth.criteo_batch(B, NS, 39, seed=999, device="cuda")
    want = small.predict(ids, vals).clone()
    assert torch.equal(big.predict(ids + OFF, vals), want), "predict"
    # rows [0, OFF): the untouched-row recurrence after all 39 steps; and their share of each step's l2 term
    lrs = _Lr("Adam", lr)
    order = [big.fm_w.name, big.fm_v.name]                     # epoch_reg_terms' order
    for ti, name in enumerate(order):
        flat, n, sd = tabs[name]
        sums = _check_tables(f"{name} rows below the window", "Adam", sd, flat, n, 2 * P + 7, lrs=lrs,
                             sums_upto=2 * P, l2=l2)
        n_big, n_small = (NB, NS) if ti == 0 else (NB * K, NS * K)
        for s in range(2 * P):
            rb, rs = float(reg_big[s // P][ti, s % P]), float(reg_small[s // P][ti, s % P])
            below = float(np.float32(0.5 * l2)) * sums[s]
            tol = (_Tab.reg_tol(types.SimpleNamespace(N=n_big, K=1), below + abs(rs))
                   + _Tab.reg_tol(types.SimpleNamespace(N=n_small, K=1), abs(rs)))
            _within([rb - rs], [below], [tol], f"{name}: l2 term of step {s}, rows below the window")


# ---------------------------------------------------------------------------------------------------------------------
# 5. CRC-32C over ranges past byte 2^31 and byte 2^32
# ---------------------------------------------------------------------------------------------------------------------
def test_crc32c_past_2_31_and_2_32_bytes(bufs):
    """One 8.6 GB buffer of a repeated random 1 MiB block with distinct 1 MiB markers across byte 2^31, across byte
    2^32 and near the end; the whole range, a range 4 bytes in and a range ending mid-word, in one ctr_crc32c_ranges
    call.  Reference: tests/tf_bundle_oracle.py on the host, from the CRCs of the block's pieces and the markers
    combined by crc32c_combine / crc32c_repeat (no kernel involved)."""
    from tests import tf_bundle_oracle as tbo
    from tf_repos_b200 import ops
    (var,) = bufs.get(1)
    by = var.view(torch.uint8)
    nb = by.numel()
    BLK = 1 << 20
    gen = torch.Generator().manual_seed(5)
    block = torch.randint(0, 256, (BLK,), dtype=torch.uint8, generator=gen)
    n_full = nb // BLK
    by[:n_full * BLK].view(n_full, BLK).copy_(block.cuda().expand(n_full, BLK))
    by[n_full * BLK:] = block[:nb - n_full * BLK].cuda()
    markers = {}
    for off in (B31 - BLK // 2 - 4, (1 << 32) - 3 * 4096, nb - BLK - 8):
        m = torch.randint(0, 256, (BLK,), dtype=torch.uint8, generator=gen)
        by[off:off + BLK] = m.cuda()
        markers[off] = m.numpy().tobytes()
    blk = block.numpy().tobytes()
    memo = {}

    def crc(src, a, b):
        key = (src, a, b)
        if key not in memo:
            memo[key] = tbo.crc32c((blk if src < 0 else markers[src])[a:b])
        return memo[key]

    def host_crc(lo, hi):
        acc, p = None, lo
        while p < hi:
            inside = [o for o in markers if o <= p < o + BLK]
            if inside:
                o = inside[0]
                e = min(o + BLK, hi)
                c = crc(o, p - o, e - o)
            else:
                nxt = min([o for o in markers if o > p] + [hi])
                if p % BLK or nxt - p < BLK:
                    e = min(nxt, (p // BLK + 1) * BLK)
                    c = crc(-1, p % BLK, p % BLK + e - p)
                else:
                    e = p + (nxt - p) // BLK * BLK
                    c = tbo.crc32c_repeat(crc(-1, 0, BLK), BLK, (e - p) // BLK)
            acc = c if acc is None else tbo.crc32c_combine(acc, c, e - p)
            p = e
        return acc

    ranges = [(0, nb), (4, nb), (0, nb - 3)]
    got, got_masked = ops.crc32c([by[a:b] for a, b in ranges])
    got, got_masked = got.cpu().tolist(), got_masked.cpu().tolist()
    for (a, b), c, cm in zip(ranges, got, got_masked):
        want = host_crc(a, b)
        assert c & 0xFFFFFFFF == want, f"crc32c of bytes [{a}, {b}): {c & 0xFFFFFFFF:#010x}, want {want:#010x}"
        assert cm & 0xFFFFFFFF == tbo.mask(want), f"masked crc32c of bytes [{a}, {b})"
