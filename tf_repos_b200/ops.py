"""Thin torch-tensor wrappers over the C ABI (include/ctr_b200.h).

PyTorch is used here only for device memory and streams: every function passes raw device
pointers and the current CUDA stream to libctr_b200.so.  No function in this module computes
anything with torch ops.
"""
from __future__ import annotations

import ctypes
from typing import Optional

import torch

from . import _lib
from ._lib import CtrError, check

FM_DEEPFM, FM_NFM, FM_PLAIN = 0, 1, 2
OPT_ADAM, OPT_ADAGRAD, OPT_MOMENTUM, OPT_FTRL = 0, 1, 2, 3
OPT_BY_NAME = {"Adam": OPT_ADAM, "Adagrad": OPT_ADAGRAD, "Momentum": OPT_MOMENTUM, "ftrl": OPT_FTRL}
OPT_SLOTS = {OPT_ADAM: 2, OPT_ADAGRAD: 1, OPT_MOMENTUM: 1, OPT_FTRL: 2}
LONG_SEG = 128

_L = _lib.raw()


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _p(t: Optional[torch.Tensor], dtype=None, name="tensor") -> Optional[int]:
    if t is None:
        return None
    if not t.is_cuda:
        raise CtrError(f"{name} must be a CUDA tensor (no CPU fallback exists)")
    if not t.is_contiguous():
        raise CtrError(f"{name} must be contiguous")
    if dtype is not None and t.dtype != dtype:
        raise CtrError(f"{name} must be {dtype}, got {t.dtype}")
    return t.data_ptr()


def fm_embed_fwd(ids, vals, V, W, mode, x=None, y_w=None, y2=None, S=None, oob=None):
    """K1.  ids [B,F] int32|int64, vals [B,F] f32, V [N,K], W [N]|None.  Outputs are caller-allocated."""
    B, F = ids.shape
    N, K = V.shape
    if ids.dtype == torch.int32:
        bits = 32
    elif ids.dtype == torch.int64:
        bits = 64
    else:
        raise CtrError(f"ids must be int32 or int64, got {ids.dtype}")
    check(
        _L.ctr_fm_embed_fwd(
            _p(ids, None, "ids"), bits, _p(vals, torch.float32, "vals"), _p(V, torch.float32, "V"),
            _p(W, torch.float32, "W"), N, B, F, K, mode, _p(x, torch.float32, "x"),
            _p(y_w, torch.float32, "y_w"), _p(y2, torch.float32, "y2"), _p(S, torch.float32, "S"),
            _p(oob, torch.int32, "oob"), _stream()),
        "ctr_fm_embed_fwd")


def fm_embed_bwd(vals, x, S, dX, dy2, dyw, K, mode, g_rows, g_w=None):
    B, F = vals.shape
    check(
        _L.ctr_fm_embed_bwd(
            _p(vals, torch.float32, "vals"), _p(x, torch.float32, "x"), _p(S, torch.float32, "S"),
            _p(dX, torch.float32, "dX"), _p(dy2, torch.float32, "dy2"), _p(dyw, torch.float32, "dyw"),
            B, F, K, mode, _p(g_rows, torch.float32, "g_rows"), _p(g_w, torch.float32, "g_w"),
            _stream()),
        "ctr_fm_embed_bwd")


def unique_segment_workspace_bytes(n: int, N: int) -> int:
    return int(_L.ctr_unique_segment_workspace_bytes(n, N))


class UniqueWorkspace:
    """Caller-owned buffers for K3 (allocated once, reused every step; graph-capture friendly)."""

    def __init__(self, n: int, N: int, device):
        self.n, self.N = n, N
        i32 = dict(dtype=torch.int32, device=device)
        self.perm = torch.empty(max(n, 1), **i32)
        self.uniq = torch.empty(max(n, 1), **i32)
        self.inverse = torch.empty(max(n, 1), **i32)
        self.seg_offsets = torch.empty(n + 1, **i32)
        self.n_uniq = torch.zeros(1, **i32)
        self.long_list = torch.zeros(n + 1, **i32)
        self.ws = torch.empty(max(unique_segment_workspace_bytes(n, N), 16), dtype=torch.uint8, device=device)


def unique_segment(ids_flat: torch.Tensor, uw: UniqueWorkspace) -> None:
    n = ids_flat.numel()
    if n > uw.n:
        raise CtrError(f"workspace was sized for n<={uw.n}, got {n}")
    uw.n_active = n   # a final partial batch (DeepFM.py:88-90 keeps it) has fewer ids than the capacity
    check(
        _L.ctr_unique_segment(
            _p(ids_flat, torch.int32, "ids"), n, uw.N, _p(uw.perm), _p(uw.uniq), _p(uw.inverse),
            _p(uw.seg_offsets), _p(uw.n_uniq), _p(uw.long_list), _p(uw.ws), uw.ws.numel(), _stream()),
        "ctr_unique_segment")


def segment_sum_rows(g_rows, g_w, uw: UniqueWorkspace, K, g_uniq, gw_uniq=None):
    check(
        _L.ctr_segment_sum_rows(
            _p(g_rows, torch.float32, "g_rows"), _p(g_w, torch.float32, "g_w"), _p(uw.perm),
            _p(uw.seg_offsets), _p(uw.n_uniq), _p(uw.long_list), getattr(uw, "n_active", uw.n), K,
            _p(g_uniq, torch.float32, "g_uniq"), _p(gw_uniq, torch.float32, "gw_uniq"), _p(uw.ws), uw.ws.numel(),
            _stream()),
        "ctr_segment_sum_rows")


def opt_sparse_rows(opt, var, slot0, slot1, uniq, n_uniq, g_uniq, n_max, K, hyper, stage=None):
    check(
        _L.ctr_opt_sparse_rows(
            opt, _p(var, torch.float32, "var"), _p(slot0, torch.float32, "slot0"),
            _p(slot1, torch.float32, "slot1"), _p(uniq, torch.int32, "uniq"),
            _p(n_uniq, torch.int32, "n_uniq"), _p(g_uniq, torch.float32, "g_uniq"), n_max, K,
            _p(hyper, torch.float32, "hyper"), _p(stage, torch.float32, "stage"), _stream()),
        "ctr_opt_sparse_rows")


def opt_dense_sweep(opt, var, slot0, slot1, hyper, sumsq_partials=None) -> int:
    n_part = ctypes.c_int(0)
    check(
        _L.ctr_opt_dense_sweep(
            opt, _p(var, torch.float32, "var"), _p(slot0, torch.float32, "slot0"),
            _p(slot1, torch.float32, "slot1"), var.numel(), _p(hyper, torch.float32, "hyper"),
            _p(sumsq_partials, torch.float32, "sumsq_partials"), ctypes.byref(n_part), _stream()),
        "ctr_opt_dense_sweep")
    return n_part.value


def sweep_partials_count() -> int:
    return int(_L.ctr_device_sm_count()) * 8


def opt_patch_rows(var, slot0, slot1, uniq, n_uniq, stage, n_max, K, n_slots):
    check(
        _L.ctr_opt_patch_rows(
            _p(var, torch.float32), _p(slot0, torch.float32), _p(slot1, torch.float32),
            _p(uniq, torch.int32), _p(n_uniq, torch.int32), _p(stage, torch.float32), n_max, K,
            n_slots, _stream()),
        "ctr_opt_patch_rows")


def opt_dense_grad(opt, var, slot0, slot1, grad, hyper):
    check(
        _L.ctr_opt_dense_grad(
            opt, _p(var, torch.float32, "var"), _p(slot0, torch.float32, "slot0"),
            _p(slot1, torch.float32, "slot1"), _p(grad, torch.float32, "grad"), var.numel(),
            _p(hyper, torch.float32, "hyper"), _stream()),
        "ctr_opt_dense_grad")


def adam_tick(state, hyper):
    """hyper: [n_hyper, 8] float32"""
    check(_L.ctr_adam_tick(_p(state, torch.float32, "state"), _p(hyper, torch.float32, "hyper"),
                           hyper.numel() // 8, _stream()), "ctr_adam_tick")


def fc_fwd(inp, Wt, b, drop_mask, keep_prob, act, out):
    M, Kd = inp.shape
    Nd = Wt.shape[1]
    check(_L.ctr_fc_fwd(_p(inp, torch.float32, "in"), _p(Wt, torch.float32, "Wt"), _p(b, torch.float32, "b"),
                        _p(drop_mask, torch.float32, "drop_mask"), float(keep_prob), M, Kd, Nd, act,
                        _p(out, torch.float32, "out"), _stream()), "ctr_fc_fwd")


def fc_bwd_workspace_bytes(M, Kd, Nd) -> int:
    return int(_L.ctr_fc_bwd_workspace_bytes(M, Kd, Nd))


def fc_fwd_grouped(inp, Wt, b, group_bias, group_P, drop_mask, keep_prob, act, out):
    M, Kd = inp.shape
    Nd = Wt.shape[1]
    check(_L.ctr_fc_fwd_grouped(_p(inp, torch.float32, "in"), _p(Wt, torch.float32, "Wt"), _p(b, torch.float32, "b"),
                                _p(group_bias, torch.float32, "group_bias"), group_P,
                                _p(drop_mask, torch.float32, "drop_mask"), float(keep_prob), M, Kd, Nd, act,
                                _p(out, torch.float32, "out"), _stream()), "ctr_fc_fwd_grouped")


def fc_bwd(inp, Wt, out, drop_mask, keep_prob, dOut, act, dIn, dW, db, ws, accumulate_din=False):
    M, Kd = inp.shape
    Nd = Wt.shape[1]
    check(_L.ctr_fc_bwd(_p(inp, torch.float32, "in"), _p(Wt, torch.float32, "Wt"), _p(out, torch.float32, "out"),
                        _p(drop_mask, torch.float32, "drop_mask"), float(keep_prob), _p(dOut, torch.float32, "dOut"),
                        M, Kd, Nd, act, _p(dIn, torch.float32, "dIn"), int(accumulate_din), _p(dW, torch.float32, "dW"),
                        _p(db, torch.float32, "db"), _p(ws), ws.numel() * ws.element_size(), _stream()), "ctr_fc_bwd")


def fc1_fwd(in_a, in_b, w, b, y):
    M, Ka = in_a.shape
    Kb = in_b.shape[1] if in_b is not None else 0
    check(_L.ctr_fc1_fwd(_p(in_a, torch.float32, "in_a"), Ka, _p(in_b, torch.float32, "in_b"), Kb,
                         _p(w, torch.float32, "w"), _p(b, torch.float32, "b"), M, _p(y, torch.float32, "y"),
                         _stream()), "ctr_fc1_fwd")


def fc1_bwd_workspace_bytes(M, Ka, Kb) -> int:
    return int(_L.ctr_fc1_bwd_workspace_bytes(M, Ka, Kb))


def fc1_bwd(in_a, in_b, w, dy, d_a, d_b, dw, db, ws):
    M, Ka = in_a.shape
    Kb = in_b.shape[1] if in_b is not None else 0
    check(_L.ctr_fc1_bwd(_p(in_a, torch.float32, "in_a"), Ka, _p(in_b, torch.float32, "in_b"), Kb,
                         _p(w, torch.float32, "w"), _p(dy, torch.float32, "dy"), M, _p(d_a, torch.float32, "d_a"),
                         _p(d_b, torch.float32, "d_b"), _p(dw, torch.float32, "dw"), _p(db, torch.float32, "db"),
                         _p(ws), ws.numel() * ws.element_size(), _stream()), "ctr_fc1_bwd")


def dropout_mask(mask, keep_prob, seed, step_dev=None):
    check(_L.ctr_dropout_mask(_p(mask, torch.float32, "mask"), mask.numel(), float(keep_prob), int(seed),
                              _p(step_dev, torch.float32, "step"), _stream()), "ctr_dropout_mask")


BN_EPS = 1e-3  # tf.contrib.layers.batch_norm default epsilon


_bn_ws = {}


def _bn_workspace(H: int, device) -> torch.Tensor:
    key = (H, str(device))
    if key not in _bn_ws:
        _bn_ws[key] = torch.empty(max(int(_L.ctr_bn_workspace_bytes(H)), 16), dtype=torch.uint8, device=device)
    return _bn_ws[key]


def bn_fwd(x, gamma, beta, moving_mean, moving_var, train: bool, decay: float, drop_mask, keep_prob, out,
           save_mean=None, save_var=None):
    n, H = x.shape
    ws = _bn_workspace(H, x.device)
    check(_L.ctr_bn_fwd(_p(x, torch.float32, "x"), n, H, _p(gamma, torch.float32, "gamma"),
                        _p(beta, torch.float32, "beta"), _p(moving_mean, torch.float32, "moving_mean"),
                        _p(moving_var, torch.float32, "moving_var"), int(train), float(decay), BN_EPS,
                        _p(drop_mask, torch.float32, "drop_mask"), float(keep_prob), _p(out, torch.float32, "out"),
                        _p(save_mean, torch.float32, "save_mean"), _p(save_var, torch.float32, "save_var"), _p(ws),
                        ws.numel(), _stream()),
          "ctr_bn_fwd")


def bn_bwd(d_out, x, save_mean, save_var, gamma, drop_mask, keep_prob, d_x, d_gamma, d_beta):
    n, H = x.shape
    ws = _bn_workspace(H, x.device)
    check(_L.ctr_bn_bwd(_p(d_out, torch.float32, "d_out"), _p(x, torch.float32, "x"), n, H,
                        _p(save_mean, torch.float32, "save_mean"), _p(save_var, torch.float32, "save_var"),
                        _p(gamma, torch.float32, "gamma"), BN_EPS, _p(drop_mask, torch.float32, "drop_mask"),
                        float(keep_prob), _p(d_x, torch.float32, "d_x"), _p(d_gamma, torch.float32, "d_gamma"),
                        _p(d_beta, torch.float32, "d_beta"), _p(ws), ws.numel(), _stream()), "ctr_bn_bwd")


def cross_fwd(x0, w, b, xL, s):
    B, D = x0.shape
    L = w.shape[0]
    check(_L.ctr_cross_fwd(_p(x0, torch.float32, "x0"), _p(w, torch.float32, "w"), _p(b, torch.float32, "b"),
                           B, D, L, _p(xL, torch.float32, "xL"), _p(s, torch.float32, "s"), _stream()),
          "ctr_cross_fwd")


def cross_bwd_workspace_bytes(B, D, L) -> int:
    return int(_L.ctr_cross_bwd_workspace_bytes(B, D, L))


def cross_bwd(x0, w, b, s, dxL, dx_in, dx0, dw, db, ws):
    B, D = x0.shape
    L = w.shape[0]
    check(_L.ctr_cross_bwd(_p(x0, torch.float32, "x0"), _p(w, torch.float32, "w"), _p(b, torch.float32, "b"),
                           _p(s, torch.float32, "s"), _p(dxL, torch.float32, "dxL"), _p(dx_in, torch.float32, "dx_in"),
                           B, D, L, _p(dx0, torch.float32, "dx0"), _p(dw, torch.float32, "dw"),
                           _p(db, torch.float32, "db"), _p(ws), ws.numel() * ws.element_size(), _stream()),
          "ctr_cross_bwd")


def mvm_fwd(x, mvm_b, x_mvm):
    """x [B, F*K] (K1 FM_PLAIN output), mvm_b [F,K] -> x_mvm [B,K] (DeepMVM.py:144-150)."""
    F, K = mvm_b.shape
    B = x.shape[0]
    check(_L.ctr_mvm_fwd(_p(x, torch.float32, "x"), _p(mvm_b, torch.float32, "mvm_b"), B, F, K,
                         _p(x_mvm, torch.float32, "x_mvm"), _stream()), "ctr_mvm_fwd")


def mvm_bwd_workspace_bytes(B, F, K) -> int:
    return int(_L.ctr_mvm_bwd_workspace_bytes(B, F, K))


def mvm_bwd(x, mvm_b, d_xmvm, dX, d_e, d_mvm_b, ws):
    """d_e [B, F*K] = d x through the product (+ dX when given); d_mvm_b [F,K] overwritten."""
    F, K = mvm_b.shape
    B = x.shape[0]
    check(_L.ctr_mvm_bwd(_p(x, torch.float32, "x"), _p(mvm_b, torch.float32, "mvm_b"),
                         _p(d_xmvm, torch.float32, "d_xmvm"), _p(dX, torch.float32, "dX"), B, F, K,
                         _p(d_e, torch.float32, "d_e"), _p(d_mvm_b, torch.float32, "d_mvm_b"), _p(ws),
                         ws.numel() * ws.element_size(), _stream()), "ctr_mvm_bwd")


def esmm_embed_fwd(feat_ids, a_ids, bag_ids, bag_wgt, bag_off, V, x, oob=None):
    """DeepCvrMTL.py:153-164.  feat_ids [B,F'], a_ids [3,B], CSR bags (bag_off [5B+1]) -> x [B,(F'+8)K]."""
    N, K = V.shape
    B, Fp = feat_ids.shape
    check(_L.ctr_esmm_embed_fwd(_p(feat_ids, torch.int32, "feat_ids"), _p(a_ids, torch.int32, "a_ids"),
                                _p(bag_ids, torch.int32, "bag_ids"), _p(bag_wgt, torch.float32, "bag_wgt"),
                                _p(bag_off, torch.int32, "bag_off"), _p(V, torch.float32, "V"), N, B, Fp, K,
                                _p(x, torch.float32, "x"), _p(oob, torch.int32, "oob"), _stream()), "ctr_esmm_embed_fwd")


def esmm_embed_bwd(dx, bag_wgt, bag_off, B, Fp, K, g_rows):
    """g_rows [n_rows, K]: per-occurrence gradient rows in the model's ids order, zero past the batch's occurrences."""
    check(_L.ctr_esmm_embed_bwd(_p(dx, torch.float32, "dx"), _p(bag_wgt, torch.float32, "bag_wgt"),
                                _p(bag_off, torch.int32, "bag_off"), B, Fp, K, g_rows.shape[0],
                                _p(g_rows, torch.float32, "g_rows"), _stream()), "ctr_esmm_embed_bwd")


def esmm_head(y_ctr, y_cvr, y, z, n, w_ctr, w_cvr, pctr, pcvr, pctcvr, losses=None, d_ctr=None, d_cvr=None):
    """DeepCvrMTL.py:205-223.  w_ctr, w_cvr: the task weights w and 1-w (each rounded to fp32 by ctypes)."""
    B = y_ctr.numel()
    check(_L.ctr_esmm_head(_p(y_ctr, torch.float32, "y_ctr"), _p(y_cvr, torch.float32, "y_cvr"),
                           _p(y, torch.float32, "y"), _p(z, torch.float32, "z"), B, int(n), float(w_ctr), float(w_cvr),
                           _p(pctr, torch.float32, "pctr"), _p(pcvr, torch.float32, "pcvr"),
                           _p(pctcvr, torch.float32, "pctcvr"), _p(losses, torch.float32, "losses"),
                           _p(d_ctr, torch.float32, "d_ctr"), _p(d_cvr, torch.float32, "d_cvr"), _stream()),
          "ctr_esmm_head")


def _dptr(t: torch.Tensor) -> int:
    """device pointer of a (possibly strided / offset) view; only the base address is used"""
    if not t.is_cuda or t.dtype != torch.float32:
        raise CtrError("expected a CUDA float32 tensor")
    return t.data_ptr()


def gather_scale_rows(ids, wgt, V, out_view, G, ld_group, oob=None):
    """out_view: tensor VIEW whose data_ptr is the first output element (e.g. x_deep[:, off:])"""
    N, K = V.shape
    check(_L.ctr_gather_scale_rows(_p(ids, torch.int32, "ids"), _p(wgt, torch.float32, "wgt"), _p(V, torch.float32, "V"),
                                   N, ids.numel(), K, G, ld_group, _dptr(out_view), _p(oob, torch.int32, "oob"),
                                   _stream()), "ctr_gather_scale_rows")


def bag_sum_fwd(ids, wgt, offsets, V, out_view, ld, oob=None):
    """oob: int32 [2] counter of ids outside [0, N) (count, first), as in gather_scale_rows"""
    N, K = V.shape
    B = offsets.numel() - 1
    check(_L.ctr_bag_sum_fwd_oob(_p(ids, torch.int32, "ids"), _p(wgt, torch.float32, "wgt"),
                                 _p(offsets, torch.int32, "offsets"), _p(V, torch.float32, "V"), N, B, K, ld,
                                 _dptr(out_view), _p(oob, torch.int32, "oob"), _stream()), "ctr_bag_sum_fwd_oob")


def bag_sum_bwd(d_out_view, ld, wgt, offsets, K, g_rows):
    B = offsets.numel() - 1
    check(_L.ctr_bag_sum_bwd(_dptr(d_out_view), ld, _p(wgt, torch.float32, "wgt"), _p(offsets, torch.int32, "offsets"),
                             B, K, _p(g_rows, torch.float32, "g_rows"), _stream()), "ctr_bag_sum_bwd")


def scale_rows(x_view, add, w, n, K, G, ld_group, out):
    """out[i] = (x_view[(i/G)*ld_group + (i%G)*K : +K] + add[i]) * w[i]   (add, w optional)"""
    check(_L.ctr_scale_rows(_dptr(x_view), _p(add, torch.float32, "add"), _p(w, torch.float32, "w"), n, K, G, ld_group,
                            _dptr(out), _stream()), "ctr_scale_rows")


def din_pool_fwd(E, z, ids, B, P, K, att, u_view, ld_u):
    check(_L.ctr_din_pool_fwd(_p(E, torch.float32, "E"), _p(z, torch.float32, "z"), _p(ids, torch.int32, "ids"),
                              B, P, K, _p(att, torch.float32, "att"), _dptr(u_view), ld_u, _stream()),
          "ctr_din_pool_fwd")


def din_pool_bwd(E, att, ids, du_view, ld_u, B, P, K, dE, dz):
    check(_L.ctr_din_pool_bwd(_p(E, torch.float32, "E"), _p(att, torch.float32, "att"), _p(ids, torch.int32, "ids"),
                              _dptr(du_view), ld_u, B, P, K, _p(dE, torch.float32, "dE"), _p(dz, torch.float32, "dz"),
                              _stream()), "ctr_din_pool_bwd")


def din_att_dz(Hh, mask, keep, dz, w2, B, P, dZ, dU, gw2_part):
    H = Hh.shape[1]
    check(_L.ctr_din_att_dz(_p(Hh, torch.float32, "Hh"), _p(mask, torch.float32, "mask"), float(keep),
                            _p(dz, torch.float32, "dz"), _p(w2, torch.float32, "w2"), B, P, H, _p(dZ, torch.float32, "dZ"),
                            _p(dU, torch.float32, "dU"), _p(gw2_part, torch.float32, "gw2_part"), _stream()),
          "ctr_din_att_dz")


def colsum_rows(part, out):
    rows, ncols = part.shape
    check(_L.ctr_colsum_rows(_p(part, torch.float32, "part"), rows, ncols, ncols, _p(out, torch.float32, "out"), _stream()),
          "ctr_colsum_rows")


def axpby(a, alpha, b, beta, out):
    check(_L.ctr_axpby(_p(a, torch.float32, "a"), float(alpha), _p(b, torch.float32, "b"), float(beta), a.numel(),
                       _p(out, torch.float32, "out"), _stream()), "ctr_axpby")


def pnn_product_check(F, K, outer):
    """Raises CtrError if pnn_product_fwd or _bwd rejects (F, K).  Called with B = 0: launches nothing."""
    check(_L.ctr_pnn_product_fwd(None, 0, F, K, int(outer), None, None), "ctr_pnn_product_fwd")
    check(_L.ctr_pnn_product_bwd(None, None, 0, F, K, int(outer), None, None), "ctr_pnn_product_bwd")


def afm_pool_check(P, K):
    """Raises CtrError if afm_pool_fwd or _bwd rejects (P, K).  Called with B = 0: launches nothing."""
    check(_L.ctr_afm_pool_fwd(None, None, None, 1.0, 0, P, K, None, None, None), "ctr_afm_pool_fwd")
    check(_L.ctr_afm_pool_bwd(None, None, None, 1.0, None, 0, P, K, None, None, None), "ctr_afm_pool_bwd")


def cross_check(D, L):
    """Raises CtrError if cross_fwd or cross_bwd rejects (D, L).  Called with B = 0: launches nothing."""
    check(_L.ctr_cross_fwd(None, None, None, 0, D, L, None, None, None), "ctr_cross_fwd")
    check(_L.ctr_cross_bwd(None, None, None, None, None, None, 0, D, L, None, None, None, None, 0, None),
          "ctr_cross_bwd")


def pnn_product_fwd(x, B, F, K, outer, z):
    check(_L.ctr_pnn_product_fwd(_p(x, torch.float32, "x"), B, F, K, int(outer), _p(z, torch.float32, "z"), _stream()),
          "ctr_pnn_product_fwd")


def pnn_product_bwd(x, dz, B, F, K, outer, dX):
    check(_L.ctr_pnn_product_bwd(_p(x, torch.float32, "x"), _p(dz, torch.float32, "dz"), B, F, K, int(outer),
                                 _p(dX, torch.float32, "dX"), _stream()), "ctr_pnn_product_bwd")


def afm_pairs_fwd(x, B, F, K, pw):
    check(_L.ctr_afm_pairs_fwd(_p(x, torch.float32, "x"), B, F, K, _p(pw, torch.float32, "pw"), _stream()),
          "ctr_afm_pairs_fwd")


def afm_pairs_bwd(x, dpw, B, F, K, dX):
    check(_L.ctr_afm_pairs_bwd(_p(x, torch.float32, "x"), _p(dpw, torch.float32, "dpw"), B, F, K,
                               _p(dX, torch.float32, "dX"), _stream()), "ctr_afm_pairs_bwd")


def afm_pool_fwd(pw, logit, mask, keep, B, P, K, att, y_emb):
    check(_L.ctr_afm_pool_fwd(_p(pw, torch.float32, "pw"), _p(logit, torch.float32, "logit"), _p(mask, torch.float32, "mask"),
                              float(keep), B, P, K, _p(att, torch.float32, "att"), _p(y_emb, torch.float32, "y_emb"),
                              _stream()), "ctr_afm_pool_fwd")


def afm_pool_bwd(pw, att, mask, keep, dy_emb, B, P, K, dpw, dlogit):
    check(_L.ctr_afm_pool_bwd(_p(pw, torch.float32, "pw"), _p(att, torch.float32, "att"), _p(mask, torch.float32, "mask"),
                              float(keep), _p(dy_emb, torch.float32, "dy_emb"), B, P, K, _p(dpw, torch.float32, "dpw"),
                              _p(dlogit, torch.float32, "dlogit"), _stream()), "ctr_afm_pool_bwd")


def dropout_apply(x, mask, keep, out):
    check(_L.ctr_dropout_apply(_p(x, torch.float32, "x"), _p(mask, torch.float32, "mask"), float(keep), x.numel(),
                               _p(out, torch.float32, "out"), _stream()), "ctr_dropout_apply")


def shard_keys(ids, N: int, G: int, keys, oob=None):
    check(_L.ctr_shard_keys(_p(ids, torch.int32, "ids"), ids.numel(), N, G, _p(keys, torch.int32, "keys"),
                            _p(oob, torch.int32, "oob"), _stream()), "ctr_shard_keys")


def shard_split(uniq_keys, n_uniq, n_max: int, N: int, G: int, counts, local_ids):
    check(_L.ctr_shard_split(_p(uniq_keys, torch.int32, "uniq"), _p(n_uniq, torch.int32, "n_uniq"), n_max, N, G,
                             _p(counts, torch.int32, "counts"), _p(local_ids, torch.int32, "local_ids"), _stream()),
          "ctr_shard_split")


def gather_scalar(ids, W, out):
    check(_L.ctr_gather_scalar(_p(ids, torch.int32, "ids"), _p(W, torch.float32, "W"), W.numel(), ids.numel(),
                               _p(out, torch.float32, "out"), _stream()), "ctr_gather_scalar")


def epoch_max_steps() -> int:
    return int(_L.ctr_epoch_max_steps())


def epoch_tick(state, hyper, lr_table, j: int, is_adam: bool):
    check(_L.ctr_epoch_tick(_p(state, torch.float32, "state"), _p(hyper, torch.float32, "hyper"),
                            hyper.numel() // 8, _p(lr_table, torch.float32, "lr_table"), j, int(is_adam),
                            _stream()), "ctr_epoch_tick")


def epoch_rows(opt, apply: bool, var, slot0, slot1, last, uniq, n_uniq, g_uniq, n_max, K, hyper, lr_table, j, ss):
    check(
        _L.ctr_epoch_rows(
            opt, int(apply), _p(var, torch.float32, "var"), _p(slot0, torch.float32, "slot0"),
            _p(slot1, torch.float32, "slot1"), _p(last, torch.uint8, "last"), _p(uniq, torch.int32, "uniq"),
            _p(n_uniq, torch.int32, "n_uniq"), _p(g_uniq, torch.float32, "g_uniq"), n_max, K,
            _p(hyper, torch.float32, "hyper"), _p(lr_table, torch.float32, "lr_table"), j,
            _p(ss, torch.float64, "ss"), _stream()),
        "ctr_epoch_rows")


def epoch_rows2(opt, apply: bool, V, W, last_v, last_w, uniq, n_uniq, g_uniq, gw_uniq, n_max, hyper, lr_table, j, ss_v, ss_w,
                stage_v=None, stage_w=None):
    """V / W: engine.Table ([N,K] and [N]) gathered with the same ids; one launch for both.  stage_v [n_max*3K] /
    stage_w [n_max*3] (both or neither): the catch-up and the apply of one step hand the rows over through them."""
    f = torch.float32
    check(
        _L.ctr_epoch_rows2(
            opt, int(apply), _p(V.var, f, "var"), _p(V.slot(0), f), _p(V.slot(1), f), _p(last_v, torch.uint8, "last"),
            _p(W.var, f, "w_var"), _p(W.slot(0), f), _p(W.slot(1), f), _p(last_w, torch.uint8, "w_last"),
            _p(uniq, torch.int32, "uniq"), _p(n_uniq, torch.int32, "n_uniq"), _p(g_uniq, f, "g_uniq"),
            _p(gw_uniq, f, "gw_uniq"), n_max, V.K, _p(hyper, f, "hyper"), _p(lr_table, f, "lr_table"), j,
            _p(ss_v, torch.float64, "ss"), _p(ss_w, torch.float64, "ss_w"), _p(stage_v, f, "stage"),
            _p(stage_w, f, "w_stage"), _stream()),
        "ctr_epoch_rows2")


EPOCH_ROWS2_K = (4, 8, 16, 32, 64, 128, 256)


def epoch_partials_count() -> int:
    return int(_L.ctr_device_sm_count()) * 6


def epoch_sweep(opt, var, slot0, slot1, last, n_rows, K, hyper, lr_table, from_: int, upto: int, reset: bool,
                ss_partials, list_buf=None, list_count=None, ss_rows=None, list_overflow=None, W=None,
                w_ss_partials=None, w_ss_rows=None):
    """list_buf / list_count / ss_rows: scratch of the Adam sweep (required for Adam).
    list_overflow: int32 [1] counter; gathered rows that did not fit in list_buf are added to it (see check_ids).
    W: the scalar table [n_rows] (engine.Table) that shares `last` (epoch_shared_last_supported), swept in the same
    pass with its own w_ss_partials / w_ss_rows."""
    f = torch.float32
    w_var, w_slot0, w_slot1 = (W.var, W.slot(0), W.slot(1)) if W is not None else (None, None, None)
    n_part = ctypes.c_int(0)
    check(
        _L.ctr_epoch_sweep(
            opt, _p(var, f, "var"), _p(slot0, f, "slot0"), _p(slot1, f, "slot1"), _p(w_var, f, "w_var"),
            _p(w_slot0, f, "w_slot0"), _p(w_slot1, f, "w_slot1"), _p(last, torch.uint8, "last"), n_rows, K,
            _p(hyper, f, "hyper"), _p(lr_table, f, "lr_table"), from_, upto, int(reset),
            _p(ss_partials, torch.float64, "ss_partials"), _p(w_ss_partials, torch.float64, "w_ss_partials"),
            ctypes.byref(n_part), _p(list_buf, torch.int32, "list"), (list_buf.numel() if list_buf is not None else 0),
            _p(list_count, torch.int32, "list_count"), _p(ss_rows, torch.float64, "ss_rows"),
            _p(w_ss_rows, torch.float64, "w_ss_rows"), _p(list_overflow, torch.int32, "list_overflow"), _stream()),
        "ctr_epoch_sweep")
    return n_part.value


def epoch_shared_last_supported(opt, n_rows: int, K: int) -> bool:
    """Whether an [n_rows, K] table and a scalar [n_rows] table can share one `last` array (ctr_epoch_sweep)."""
    return bool(_L.ctr_epoch_shared_last_supported(opt, n_rows, K))


def epoch_reg_loss(ss_rows, ss_partials, n_partials, upto, scale, reg, accumulate=False):
    check(
        _L.ctr_epoch_reg_loss(_p(ss_rows, torch.float64, "ss_rows"), _p(ss_partials, torch.float64, "ss_partials"),
                              n_partials, upto, float(scale), _p(reg, torch.float32, "reg"), int(accumulate),
                              _stream()),
        "ctr_epoch_reg_loss")


def selftest_adam_packed(regime: int, seed: int, n: int, steps: int, lr: float, l2: float, device) -> tuple:
    """(elements with differing bits, rejected trajectories, total) of the packed Adam loops vs the scalar step"""
    out = torch.zeros(3, dtype=torch.int64, device=device)
    check(_L.ctr_selftest_adam_packed(int(regime), int(seed), int(n), int(steps), float(lr), float(l2),
                                      _p(out, torch.int64, "out3"), _stream()), "ctr_selftest_adam_packed")
    return tuple(out.tolist())


def selftest_divsqrt(seed: int, n: int, device) -> tuple:
    """(sqrt mismatches, div mismatches) of the sweeps' in-range IEEE fast paths vs sqrt.rn / div.rn on n operands"""
    mism = torch.zeros(2, dtype=torch.int64, device=device)
    check(_L.ctr_selftest_divsqrt(int(seed), int(n), _p(mism, torch.int64, "mismatches"), _stream()),
          "ctr_selftest_divsqrt")
    return tuple(int(x) for x in mism.tolist())


def reduce_sum(inp, scale, out, ws):
    check(
        _L.ctr_reduce_sum(_p(inp, torch.float32, "in"), inp.numel(), float(scale), _p(out, torch.float32, "out"),
                          _p(ws, torch.float32, "ws"), ws.numel() * 4, _stream()),
        "ctr_reduce_sum")


def l2_loss(t, out, ws, scale: float = 1.0):
    """out[0] = scale * 0.5 * sum(t^2)"""
    check(
        _L.ctr_l2_loss(_p(t, torch.float32, "t"), t.numel(), float(scale), _p(out, torch.float32, "out"), _p(ws),
                       ws.numel() * ws.element_size(), _stream()),
        "ctr_l2_loss")


def logit_loss(bias, y_a, y_b, y_c, labels, B, y=None, pred=None, loss_ce=None, dy=None, dbias=None, B_total=None):
    check(
        _L.ctr_logit_loss(
            _p(bias, torch.float32, "bias"), _p(y_a, torch.float32, "y_a"), _p(y_b, torch.float32, "y_b"),
            _p(y_c, torch.float32, "y_c"), _p(labels, torch.float32, "labels"), B, B_total or B,
            _p(y, torch.float32, "y"), _p(pred, torch.float32, "pred"), _p(loss_ce, torch.float32, "loss_ce"),
            _p(dy, torch.float32, "dy"), _p(dbias, torch.float32, "dbias"), _stream()),
        "ctr_logit_loss")


def wd_input_fwd(ids, dense, emb, wide_cat, wide_num, wide_bias, num_perm, NB, K, flat_ids, x, lin):
    B, Fc = ids.shape
    Fd = dense.shape[1]
    check(_L.ctr_wd_input_fwd(_p(ids, torch.int32, "ids"), _p(dense, torch.float32, "dense"), _p(emb, torch.float32, "emb"),
                              _p(wide_cat, torch.float32, "wide_cat"), _p(wide_num, torch.float32, "wide_num"),
                              _p(wide_bias, torch.float32, "wide_bias"), _p(num_perm, torch.int32, "num_perm"), B, Fc, Fd,
                              NB, K, _p(flat_ids, torch.int32, "flat_ids"), _p(x, torch.float32, "x"),
                              _p(lin, torch.float32, "lin"), _stream()), "ctr_wd_input_fwd")


def wd_input_bwd(dX, dy, dense, B, Fc, Fd, K, g_rows, g_cat, g_num, g_bias):
    check(_L.ctr_wd_input_bwd(_p(dX, torch.float32, "dX"), _p(dy, torch.float32, "dy"), _p(dense, torch.float32, "dense"),
                              B, Fc, Fd, K, _p(g_rows, torch.float32, "g_rows"), _p(g_cat, torch.float32, "g_cat"),
                              _p(g_num, torch.float32, "g_num"), _p(g_bias, torch.float32, "g_bias"), _stream()),
          "ctr_wd_input_bwd")


def wd_serve_input(data, offsets, example_base: int, emb, wide_cat, wide_num, wide_bias, num_perm, NB, K, x, lin, err):
    """Serialized tf.Examples data[offsets[b], offsets[b+1]) (uint8, offsets int64 [n+1]) -> x [n, 26K+13] and lin [n]
    as wd_input_fwd writes them; err int64 [1] (uint64 bits, ~0 = none) is min-folded."""
    n = offsets.numel() - 1
    check(_L.ctr_wd_serve_input(_p(data, torch.uint8, "data"), _p(offsets, torch.int64, "offsets"), n, example_base,
                                _p(emb, torch.float32, "emb"), _p(wide_cat, torch.float32, "wide_cat"),
                                _p(wide_num, torch.float32, "wide_num"), _p(wide_bias, torch.float32, "wide_bias"),
                                _p(num_perm, torch.int32, "num_perm"), NB, K, _p(x, torch.float32, "x"),
                                _p(lin, torch.float32, "lin"), _p(err, torch.int64, "err"), _stream()),
          "ctr_wd_serve_input")


def parse_libsvm_device_workspace_bytes(n_bytes: int, max_rows: int) -> int:
    return int(_L.ctr_parse_libsvm_device_workspace_bytes(n_bytes, max_rows))


def parse_libsvm_device_core(text: torch.Tensor, n_bytes: int, F: int, max_rows: int, ws: torch.Tensor,
                             final_chunk: bool = True):
    """decode_libsvm (DeepFM.py:65-81) of text[:n_bytes], a uint8 CUDA tensor; ws holds at least
    parse_libsvm_device_workspace_bytes(n_bytes, max_rows) device bytes.  Returns (ids int32 [max_rows,F], vals f32
    [max_rows,F], labels f32 [max_rows], info int64 [5] on the device) without waiting for the device: info = (rows,
    bytes consumed, blank lines, malformed lines, lines with a number for the host), and when any of the last three is
    non-zero the piece holds something only the host parser may decide and the outputs must be discarded."""
    assert text.is_cuda and text.dtype == torch.uint8 and text.is_contiguous() and 0 <= n_bytes <= text.numel()
    dev = text.device
    ids = torch.empty(max_rows, F, dtype=torch.int32, device=dev)
    vals = torch.empty(max_rows, F, dtype=torch.float32, device=dev)
    labels = torch.empty(max_rows, dtype=torch.float32, device=dev)
    info = torch.empty(5, dtype=torch.int64, device=dev)
    check(_L.ctr_parse_libsvm_device(text.data_ptr(), n_bytes, F, max_rows, int(final_chunk), ids.data_ptr(),
                                     vals.data_ptr(), labels.data_ptr(), info.data_ptr(), _p(ws, torch.uint8, "ws"),
                                     ws.numel(), _stream()), "ctr_parse_libsvm_device")
    return ids, vals, labels, info


def parse_libsvm_device(text: torch.Tensor, F: int, max_rows: int, final_chunk: bool = True):
    """parse_libsvm_device_core of the whole of text with its own workspace, waiting for the result.  Returns (ids
    int32 [rows,F], vals f32 [rows,F], labels f32 [rows], consumed bytes, needs_host) -- when needs_host is True the
    chunk holds something only the host parser may decide (blank/malformed line, exotic number) and the outputs must
    be discarded."""
    n = text.numel()
    ws = torch.empty(parse_libsvm_device_workspace_bytes(n, max_rows), dtype=torch.uint8, device=text.device)
    ids, vals, labels, info = parse_libsvm_device_core(text, n, F, max_rows, ws, final_chunk)
    rows, consumed, blank, bad, host = (int(x) for x in info.tolist())
    return ids[:rows], vals[:rows], labels[:rows], consumed, bool(blank or bad or host)


def parse_csv_device_workspace_bytes(n_bytes: int, max_rows: int) -> int:
    return int(_L.ctr_parse_csv_device_workspace_bytes(n_bytes, max_rows))


def parse_csv_device(text: torch.Tensor, n_bytes: int, n_float: int, n_int: int, max_rows: int, ws: torch.Tensor,
                     final_chunk: bool = True):
    """tf.decode_csv (wide_n_deep.py:55-73) of text[:n_bytes], a uint8 CUDA tensor; ws holds at least
    parse_csv_device_workspace_bytes(n_bytes, max_rows) device bytes.  Returns (labels f32 [max_rows], dense f32
    [max_rows, n_float-1], cat int32 [max_rows, n_int], info int64 [5] on the device) without waiting for the device:
    info = (rows, bytes consumed, blank lines, malformed lines, lines with a number for the host), and when any of the
    last three is non-zero the piece holds something only the host decoder may decide and the outputs must be
    discarded."""
    assert text.is_cuda and text.dtype == torch.uint8 and text.is_contiguous() and 0 <= n_bytes <= text.numel()
    dev = text.device
    labels = torch.empty(max_rows, dtype=torch.float32, device=dev)
    dense = torch.empty(max_rows, n_float - 1, dtype=torch.float32, device=dev)
    cat = torch.empty(max_rows, n_int, dtype=torch.int32, device=dev)
    info = torch.empty(5, dtype=torch.int64, device=dev)
    check(_L.ctr_parse_csv_device(text.data_ptr(), n_bytes, n_float, n_int, max_rows, int(final_chunk),
                                  labels.data_ptr(), dense.data_ptr(), cat.data_ptr(), info.data_ptr(),
                                  _p(ws, torch.uint8, "ws"), ws.numel(), _stream()), "ctr_parse_csv_device")
    return labels, dense, cat, info


def tfrecord_frame(buf, final_chunk: bool, max_records: int):
    """Frames the TFRecords of a host uint8 numpy buffer (ctr_tfrecord_frame).  Returns (rec_off int64 [records],
    consumed, error class, error offset, bytes the next record needs)."""
    import numpy as np
    rec_off = np.empty(max(max_records, 1), dtype=np.int64)
    info = np.zeros(5, dtype=np.int64)
    check(_L.ctr_tfrecord_frame(buf.ctypes.data, buf.nbytes, int(final_chunk), rec_off.ctypes.data, max_records,
                                info.ctypes.data), "ctr_tfrecord_frame")
    n, consumed, cls, at, need = (int(x) for x in info)
    return rec_off[:n], consumed, cls, at, need


def tfrecord_scan(chunk, rec_off, record_base: int, F: int, labels_mask: int, lens, err):
    """Pass 1 over the framed records of a uint8 CUDA chunk: lens int32 [n,5], err uint64-as-int64 [1] (min-folded)."""
    n = rec_off.numel()
    check(_L.ctr_tfrecord_scan(_p(chunk, torch.uint8, "chunk"), chunk.numel(), _p(rec_off, torch.int64, "rec_off"), n,
                               record_base, F, labels_mask, _p(lens, torch.int32, "lens"), _p(err, torch.int64, "err"),
                               _stream()), "ctr_tfrecord_scan")


def tfrecord_emit_din(stage, slot_off, slot_len, B, F, P, a_int_off, feat_ids, a_ids, a_int_ids, u_ids, u_wgt, y):
    check(_L.ctr_tfrecord_emit_din(_p(stage, torch.uint8, "stage"), _p(slot_off, torch.int64, "slot_off"),
                                   _p(slot_len, torch.int32, "slot_len"), B, F, P, _p(a_int_off, torch.int32, "a_int_off"),
                                   _p(feat_ids, torch.int32, "feat_ids"), _p(a_ids, torch.int32, "a_ids"),
                                   _p(a_int_ids, torch.int32, "a_int_ids"), _p(u_ids, torch.int32, "u_ids"),
                                   _p(u_wgt, torch.float32, "u_wgt"), _p(y, torch.float32, "y"), _stream()),
          "ctr_tfrecord_emit_din")


def din_serve_scan(data, offsets, example_base: int, F: int, B: int, max_a_int: int, slot_off, slot_len, a_int_off,
                   maxima, err):
    """One serving slice of serialized tf.Examples data[offsets[b], offsets[b+1]) (uint8, offsets int64 [n+1], n <= B)
    -> slot_off int64 [B], slot_len int32 [B] and a_int_off int32 [B+1] for tfrecord_emit_din; maxima int32 [2]
    (longest behaviour list, longest a_int bag; zeroed by the caller) and err int64 [1] (uint64 bits, ~0 = none) are
    folded into."""
    n = offsets.numel() - 1
    check(_L.ctr_din_serve_scan(_p(data, torch.uint8, "data"), _p(offsets, torch.int64, "offsets"), n, example_base, F, B,
                                max_a_int, _p(slot_off, torch.int64, "slot_off"), _p(slot_len, torch.int32, "slot_len"),
                                _p(a_int_off, torch.int32, "a_int_off"), _p(maxima, torch.int32, "maxima"),
                                _p(err, torch.int64, "err"), _stream()), "ctr_din_serve_scan")


def esmm_serve_scan(data, offsets, example_base: int, F: int, B: int, occ_capacity: int, slot_off, slot_len, bag_off,
                    total, err):
    """One serving slice of serialized tf.Examples data[offsets[b], offsets[b+1]) (uint8, offsets int64 [n+1], n <= B)
    -> slot_off int64 [B], slot_len int32 [B] and bag_off int32 [5B+1] for tfrecord_emit_esmm; total int64 [1] = the
    slice's occurrences (bag_off is all zeros when it exceeds occ_capacity); err int64 [1] (uint64 bits, ~0 = none) is
    folded into."""
    n = offsets.numel() - 1
    check(_L.ctr_esmm_serve_scan(_p(data, torch.uint8, "data"), _p(offsets, torch.int64, "offsets"), n, example_base, F,
                                 B, occ_capacity, _p(slot_off, torch.int64, "slot_off"),
                                 _p(slot_len, torch.int32, "slot_len"), _p(bag_off, torch.int32, "bag_off"),
                                 _p(total, torch.int64, "total"), _p(err, torch.int64, "err"), _stream()),
          "ctr_esmm_serve_scan")


def tfrecord_emit_esmm(stage, slot_off, slot_len, B, F, bag_off, feat_ids, a_ids, bag_ids, bag_wgt, y, z):
    check(_L.ctr_tfrecord_emit_esmm(_p(stage, torch.uint8, "stage"), _p(slot_off, torch.int64, "slot_off"),
                                    _p(slot_len, torch.int32, "slot_len"), B, F, _p(bag_off, torch.int32, "bag_off"),
                                    _p(feat_ids, torch.int32, "feat_ids"), _p(a_ids, torch.int32, "a_ids"),
                                    _p(bag_ids, torch.int32, "bag_ids"), _p(bag_wgt, torch.float32, "bag_wgt"),
                                    _p(y, torch.float32, "y"), _p(z, torch.float32, "z"), _stream()),
          "ctr_tfrecord_emit_esmm")


def init_trunc_normal(t, stddev: float, seed: int):
    check(_L.ctr_init_trunc_normal(_p(t, torch.float32, "t"), t.numel(), float(stddev), int(seed), _stream()),
          "ctr_init_trunc_normal")


def fill(t, value: float):
    check(_L.ctr_fill(_p(t, torch.float32, "t"), t.numel(), float(value), _stream()), "ctr_fill")


def crc32c_workspace_bytes(n: int, total_bytes: int) -> int:
    return int(_L.ctr_crc32c_workspace_bytes(n, total_bytes))


def crc32c(tensors, crc=None, masked=None, ws=None):
    """CRC-32C of the bytes of each contiguous CUDA tensor (any dtype; a uint8 view gives any 4-byte aligned byte
    range) in one ctr_crc32c_ranges call on the current stream.  Returns device int32 tensors (crc, masked): the
    standard CRC-32C and TensorFlow's masked form, as the low 32 bits of each element (`& 0xFFFFFFFF` on the host)."""
    tensors = list(tensors)
    n = len(tensors)
    if n == 0:
        raise CtrError("crc32c: no tensors")
    dev = tensors[0].device
    rng = torch.empty(n, 2, dtype=torch.int64)
    for i, t in enumerate(tensors):
        if t.device != dev:
            raise CtrError(f"crc32c: tensor {i} is on {t.device}, not {dev}")
        rng[i, 0], rng[i, 1] = _p(t, None, f"tensors[{i}]"), t.numel() * t.element_size()
    total = int(rng[:, 1].sum())
    rng = rng.to(dev)
    i32 = dict(dtype=torch.int32, device=dev)
    crc = torch.empty(n, **i32) if crc is None else crc
    masked = torch.empty(n, **i32) if masked is None else masked
    need = crc32c_workspace_bytes(n, total)
    if ws is None or ws.numel() < need:
        ws = torch.empty(need, dtype=torch.uint8, device=dev)
    check(_L.ctr_crc32c_ranges(_p(rng, torch.int64, "ranges"), n, total, _p(crc, torch.int32, "crc"),
                               _p(masked, torch.int32, "masked"), _p(ws, torch.uint8, "ws"), ws.numel(), _stream()),
          "ctr_crc32c_ranges")
    return crc, masked


def auc_counts(pred, label, thresholds, counts):
    """counts int64 [2, 201] += tf.metrics.auc's per-class histogram of #{t in thresholds : t < pred} (row 0: label 0,
    row 1: label != 0 or NaN); a NaN pred counts above every threshold.  pred, label f32 [n]; thresholds f32 [200]."""
    n = pred.numel()
    if label.numel() != n:
        raise CtrError(f"auc_counts: {n} predictions, {label.numel()} labels")
    if thresholds.numel() != 200 or counts.numel() != 2 * 201:
        raise CtrError("auc_counts: thresholds must be f32 [200] and counts int64 [2, 201]")
    check(_L.ctr_auc_counts(_p(pred, torch.float32, "pred"), _p(label, torch.float32, "label"), n,
                            _p(thresholds, torch.float32, "thresholds"), _p(counts, torch.int64, "counts"), _stream()),
          "ctr_auc_counts")


def format_preds_workspace_bytes(n: int) -> int:
    return int(_L.ctr_format_preds_workspace_bytes(n))


def format_preds(a, b, out, offset, ws):
    """Appends "%f\\n" % a[r] (b None) or "%f\\t%f\\n" % (a[r], b[r]) for every row to the uint8 device buffer out at
    the device int64 offset[0], and advances offset[0]; Python's "%f" bytes for every float32.  Bytes past the end of
    out are not written, offset still advances: offset[0] > out.numel() means out was too small."""
    n = a.numel()
    if b is not None and b.numel() != n:
        raise CtrError(f"format_preds: columns of {n} and {b.numel()} rows")
    check(_L.ctr_format_preds(_p(a, torch.float32, "a"), _p(b, torch.float32, "b"), n, _p(out, torch.uint8, "out"),
                              out.numel(), _p(offset, torch.int64, "offset"), _p(ws, torch.uint8, "ws"), ws.numel(),
                              _stream()),
          "ctr_format_preds")
