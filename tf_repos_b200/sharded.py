"""Row-sharded embedding tables for DeepFM (BASELINE.json configs[4]: 1e9-row table over 8 H100s, where
fm_v + fm_w + Adam slots = 204 GB exceed one GPU's 80 GB).  Not in the reference (SURVEY.md 8e).

owner(id) = id % G, local row = id // G.  One process per GPU, data-parallel batches:

  forward   unique(my ids) -> bucket by owner -> all_to_all(ids) -> owners gather rows (after catching
            them up in exact_deferred mode) -> all_to_all(rows) -> K1 runs on the received row cache with
            ids remapped to cache positions
  backward  K2 -> segment-sum per cache row -> all_to_all(grad rows) -> owner de-duplicates what the G ranks
            sent (one contribution per rank and row, summed in rank order => deterministic) -> optimizer
            on the local shard (exact sweep / exact_deferred epochs / lazy); dense grads: all_reduce.

The result equals the single-GPU engine on the concatenated batch.  The collectives are NCCL
(torch.distributed) on the compute stream; the bucket sizes of all ranks are all-gathered first (one small host sync per step).
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.distributed as dist

from . import ops
from .base import floats, ints
from .engine import DenseVars, OptimizerState, SparseModel, SparseUpdater, Table
from .mlp import MLP


def local_rows(N: int, G: int, rank: int) -> int:
    """number of ids in [0, N) with id % G == rank"""
    return (N - rank + G - 1) // G


class ShardedDeepFM(SparseModel):
    def __init__(self, field_size, feature_size, embedding_size, batch_size, deep_layers="256,128,64",
                 dropout="0.5,0.5,0.5", l2_reg=1e-4, learning_rate=5e-4, optimizer="Adam", update_mode="exact",
                 device="cuda", seed=0, epoch_steps=8, group=None):
        self.group = group
        self.G = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.F, self.N, self.K, self.B = field_size, feature_size, embedding_size, batch_size
        self.layers, self.keep = ints(deep_layers), floats(dropout)
        self.l2_reg = float(l2_reg)
        self.device = dev = torch.device(device)
        self.seed = seed
        G, B, F, K = self.G, self.B, self.F, self.K
        self.N_local = local_rows(self.N, G, self.rank)
        self.opt = OptimizerState(optimizer, learning_rate, l2_reg, dev)
        self.V = Table("fm_v", self.N_local, K, self.opt, dev, seed=seed * 2 + 1 + 1000 * self.rank)
        self.W = Table("fm_w", self.N_local, 1, self.opt, dev, seed=seed * 2 + 2 + 1000 * self.rank)
        self.tables = [self.V, self.W]
        self.mlp = MLP(F * K, self.layers, self.keep, B, dev, seed=seed)
        self.dense = DenseVars([("fm_bias", (1,))] + self.mlp.specs(), self.opt, dev)
        self.mlp.init(self.dense, torch.Generator().manual_seed(seed))
        f32 = dict(dtype=torch.float32, device=dev)
        i32 = dict(dtype=torch.int32, device=dev)
        n = B * F
        self.n = n
        self.x = torch.empty(B, F * K, **f32); self.S = torch.empty(B, K, **f32)
        self.y_w = torch.empty(B, **f32); self.y_v = torch.empty(B, **f32)
        self.y = torch.empty(B, **f32); self.pred = torch.empty(B, **f32); self.dy = torch.empty(B, **f32)
        self.d_last = torch.empty(B, self.mlp.out_in, **f32)
        self.g_rows = torch.empty(n, K, **f32); self.g_w = torch.empty(n, **f32)
        self.loss_ce = self.dense.tail[0:1]
        self.oob = torch.zeros(2, **i32)
        # requester side
        # unique of my batch's routing keys (owner * ceil(N/G) + local row): bucket order, cache positions and the
        # gradient segments all come out of this one sort (csrc/shard.cu)
        self.n_keys = G * ((self.N + G - 1) // G)
        self.uw = ops.UniqueWorkspace(n, self.n_keys, dev)
        self.keys = torch.empty(n, **i32)
        self.counts = torch.zeros(G, **i32)
        self.count_mat = torch.zeros(G * G, **i32)
        self.local_ids = torch.empty(n, **i32)
        self.cache_v = torch.empty(n, K, **f32); self.cache_w = torch.empty(n, **f32)
        self.g_cache = torch.empty(n, K, **f32); self.gw_cache = torch.empty(n, **f32)
        # owner side (worst case: every rank asks me for n rows)
        R = G * n
        self.recv_ids = torch.zeros(R, **i32)
        self.rows_v = torch.empty(R, K, **f32); self.rows_w = torch.empty(R, **f32)
        self.recv_g = torch.empty(R, K, **f32); self.recv_gw = torch.empty(R, **f32)
        self.updater = SparseUpdater(R, self.N_local, K, self.opt, dev, True, self.tables, update_mode,
                                     epoch_steps, l2_reg)
        self.global_step = 0

    # ---- helpers ---------------------------------------------------------------------------------------
    def _a2a(self, out, inp, out_splits, in_splits):
        if self.G == 1:
            out[: inp.shape[0]].copy_(inp)
        else:
            dist.all_to_all_single(out, inp, out_splits, in_splits, group=self.group)

    def load_global_tables(self, fm_v: torch.Tensor, fm_w: torch.Tensor):
        """test helper: take my rows (id % G == rank) of full tables"""
        self.V.var.copy_(fm_v[self.rank:: self.G].to(self.device))
        self.W.var.copy_(fm_w[self.rank:: self.G].to(self.device))

    def gather_global_tables(self):
        """test helper: reassemble the full [N,K] / [N] tables on every rank"""
        self.flush()
        K = self.K
        out_v = torch.zeros(self.N, K, device=self.device); out_w = torch.zeros(self.N, device=self.device)
        for r in range(self.G):
            nl = local_rows(self.N, self.G, r)
            bv = self.V.var.clone() if r == self.rank else torch.empty(nl, K, device=self.device)
            bw = self.W.var.clone() if r == self.rank else torch.empty(nl, device=self.device)
            if self.G > 1:
                dist.broadcast(bv, r, group=self.group); dist.broadcast(bw, r, group=self.group)
            out_v[r:: self.G] = bv; out_w[r:: self.G] = bw
        return out_v, out_w

    def _lookup(self, ids: torch.Tensor, catch_up: bool = False):
        """unique -> route -> fetch rows into the cache; returns (U, send_splits, recv_splits, R)."""
        G, n = self.G, ids.numel()
        ops.shard_keys(ids.reshape(-1), self.N, G, self.keys[:n], self.oob)
        ops.unique_segment(self.keys[:n], self.uw)          # uw.inverse[i] = cache position of occurrence i
        ops.shard_split(self.uw.uniq, self.uw.n_uniq, n, self.N, G, self.counts, self.local_ids)
        self._mark("keys+sort+split")
        if G > 1:   # every rank's bucket sizes in one collective, one host sync per step
            dist.all_gather_into_tensor(self.count_mat, self.counts, group=self.group)
            cm = self.count_mat.view(G, G).tolist()
            send = cm[self.rank]
            recv = [cm[r][self.rank] for r in range(G)]
        else:
            send = self.counts.tolist()
            recv = list(send)
        U, R = sum(send), sum(recv)
        self._mark("count all-gather + host sync")
        self._a2a(self.recv_ids[:R], self.local_ids[:U], recv, send)
        self._mark("a2a ids")
        if catch_up:   # owners bring the requested rows to the start of this step
            self.updater.catch_up(self.recv_ids[:R])
        self._mark("owner: unique + catch-up rows")
        ops.gather_scale_rows(self.recv_ids[:R], None, self.V.var, self.rows_v, 1, self.K, self.oob)
        ops.gather_scalar(self.recv_ids[:R], self.W.var, self.rows_w[:R])
        self._mark("owner: gather rows")
        self._a2a(self.cache_v[:U], self.rows_v[:R], send, recv)
        self._a2a(self.cache_w[:U], self.rows_w[:R], send, recv)
        self._mark("a2a rows (v, w)")
        return U, send, recv, R

    def _forward(self, ids, vals, U, train, masks=None):
        B = ids.shape[0]
        rid = self.uw.inverse[: B * self.F].view(B, self.F)
        ops.fm_embed_fwd(rid, vals, self.cache_v[:U], self.cache_w[:U], ops.FM_DEEPFM, x=self.x[:B], y_w=self.y_w[:B],
                         y2=self.y_v[:B], S=self.S[:B], oob=self.oob)
        self._a = self.mlp.forward_hidden(self.x[:B], self.dense, train, masks, step_dev=self.opt.state[3:4])
        return self.mlp.forward_out(self._a, self.dense)

    # ---- everything between the row exchange and the gradient exchange: K1 on the row cache, MLP forward, loss head,
    # MLP backward, K2, per-cache-row gradient sums.  Static shapes and addresses (the cache is indexed through
    # uw.inverse, sizes live on the device) => replayed from ONE CUDA graph; the exchanges around it need host-side
    # split sizes and stay eager.
    def _compute_eager(self, vals, labels, masks=None):
        B, F, K, G = self.B, self.F, self.K, self.G
        rid = self.uw.inverse[: B * F].view(B, F)
        ops.fm_embed_fwd(rid, vals, self.cache_v, self.cache_w, ops.FM_DEEPFM, x=self.x, y_w=self.y_w, y2=self.y_v,
                         S=self.S, oob=self.oob)
        self._a = self.mlp.forward_hidden(self.x, self.dense, True, masks, step_dev=self.opt.state[3:4])
        y_d = self.mlp.forward_out(self._a, self.dense)
        ops.logit_loss(self.dense["fm_bias"], self.y_w, self.y_v, y_d, labels, B, y=self.y, pred=self.pred,
                       loss_ce=self.loss_ce, dy=self.dy, dbias=self.dense.grads["fm_bias"], B_total=B * G)
        self.mlp.backward_out(self._a, self.dy, self.dense, self.d_last)
        dX = self.mlp.backward_hidden(self.x, self.d_last, self.dense)
        ops.fm_embed_bwd(vals, self.x, self.S, dX, self.dy, self.dy, K, ops.FM_DEEPFM, self.g_rows, self.g_w)
        # per cache row: the lookup's sort already grouped the occurrences in cache order
        ops.segment_sum_rows(self.g_rows, self.g_w, self.uw, K, self.g_cache, self.gw_cache)

    def _compute(self, vals, labels, masks=None):
        if masks is not None or not self.use_graphs:
            return self._compute_eager(vals, labels, masks)
        if not hasattr(self, "_cg"):
            self._cg, self._cg_seen = None, 0
            self._cvals = torch.empty(self.B, self.F, dtype=torch.float32, device=self.device)
            self._clabels = torch.empty(self.B, dtype=torch.float32, device=self.device)
        self._cvals.copy_(vals, non_blocking=True); self._clabels.copy_(labels, non_blocking=True)
        if self._cg is None:
            self._cg_seen += 1
            if self._cg_seen < 3:        # warm-up visits run eagerly (lazy allocations, cudaFuncSetAttribute)
                return self._compute_eager(self._cvals, self._clabels)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, capture_error_mode="thread_local"):   # NCCL's watchdog thread keeps polling
                self._compute_eager(self._cvals, self._clabels)
            self._cg = g
        self._cg.replay()

    use_graphs = True

    # ---- optional per-phase device timing (CTR_SHARD_PHASES=1; tools/time_shard_phases.py) ---------------------
    _ph = None

    def _mark(self, name):
        if self._ph is None:
            return
        ev = torch.cuda.Event(enable_timing=True)
        ev.record()
        self._ph.append((name, ev))

    def phase_report(self):
        """{phase: mean ms} over the steps recorded since _ph was set to []"""
        torch.cuda.synchronize()
        tot, cnt = {}, {}
        for (n0, e0), (n1, e1) in zip(self._ph[:-1], self._ph[1:]):
            if n1 == "begin":
                continue
            tot[n1] = tot.get(n1, 0.0) + e0.elapsed_time(e1); cnt[n1] = cnt.get(n1, 0) + 1
        steps = max(sum(1 for n, _ in self._ph if n == "begin"), 1)
        return {k: v / steps for k, v in tot.items()}

    def predict(self, ids, vals):
        B = ids.shape[0]
        assert B == self.B
        self.flush()
        U, *_ = self._lookup(ids)
        y_d = self._forward(ids, vals, U, train=False)
        ops.logit_loss(self.dense["fm_bias"], self.y_w[:B], self.y_v[:B], y_d, None, B, y=self.y[:B], pred=self.pred[:B])
        return self.pred[:B]

    def train_step(self, ids, vals, labels, masks=None):
        B, F, K, G = ids.shape[0], self.F, self.K, self.G
        assert B == self.B
        upd = self.updater
        self._mark("begin")
        upd.begin_step()
        U, send, recv, R = self._lookup(ids, catch_up=True)
        self._compute(vals, labels, masks)
        self._mark("compute segment (K1, MLP, loss, K2, seg sums)")
        self._a2a(self.recv_g[:R], self.g_cache[:U], recv, send)
        self._a2a(self.recv_gw[:R], self.gw_cache[:U], recv, send)
        if G > 1:
            dist.all_reduce(self.dense.grad, group=self.group)
        self._mark("a2a grads (v, w) + all-reduce dense")
        upd.finish_step(self.recv_ids[:R], self.recv_g[:R], self.recv_gw[:R])
        self._mark("owner: seg sums + row apply (+ sweep at epoch end)")
        self.dense.apply()
        self.global_step += 1
        self._mark("dense apply")
        return torch.cat([self.loss_ce, upd.reg[1:2], upd.reg[0:1]])   # reg terms: this rank's shard only
