"""ctypes binding of libctr_b200.so (the C ABI declared in include/ctr_b200.h).

There is deliberately NO fallback: if the shared library is missing, or a call returns an error
status, this raises.  The product path never routes through oracle/ or through PyTorch eager ops
for the hot path (sparse gather, interaction, scatter-add, optimizer).
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_int32, c_int64, c_size_t, c_uint64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libctr_b200.so")


class CtrError(RuntimeError):
    pass


def _load() -> ctypes.CDLL:
    if not os.path.exists(LIB_PATH):
        raise CtrError(
            f"{LIB_PATH} not found: build it with `make` (or `python -c 'import __graft_entry__ as g; "
            "g.build()'`). There is no CPU/eager fallback for the hot path."
        )
    return ctypes.CDLL(LIB_PATH)


_lib = _load()

P = c_void_p
# name -> (restype, argtypes).  Keep in the same order as include/ctr_b200.h.
SIGNATURES = {
    "ctr_abi_version": (c_int, []),
    "ctr_last_error": (c_char_p, []),
    "ctr_launch_count": (c_int64, []),
    "ctr_device_sm_count": (c_int, []),
    "ctr_fm_embed_fwd": (c_int, [P, c_int, P, P, P, c_int64, c_int, c_int, c_int, c_int, P, P, P, P, P, P]),
    "ctr_fm_embed_bwd": (c_int, [P, P, P, P, P, P, c_int, c_int, c_int, c_int, P, P, P]),
    "ctr_unique_segment_workspace_bytes": (c_size_t, [c_int64, c_int64]),
    "ctr_unique_segment": (c_int, [P, c_int64, c_int64, P, P, P, P, P, P, P, c_size_t, P]),
    "ctr_segment_sum_rows": (c_int, [P, P, P, P, P, P, c_int64, c_int, P, P, P, c_size_t, P]),
    "ctr_opt_sparse_rows": (c_int, [c_int, P, P, P, P, P, P, c_int64, c_int, P, P, P]),
    "ctr_opt_dense_sweep": (c_int, [c_int, P, P, P, c_int64, P, P, ctypes.POINTER(c_int), P]),
    "ctr_opt_patch_rows": (c_int, [P, P, P, P, P, P, c_int64, c_int, c_int, P]),
    "ctr_opt_dense_grad": (c_int, [c_int, P, P, P, P, c_int64, P, P]),
    "ctr_adam_tick": (c_int, [P, P, c_int, P]),
    "ctr_epoch_max_steps": (c_int, []),
    "ctr_epoch_tick": (c_int, [P, P, c_int, P, c_int, c_int, P]),
    "ctr_epoch_rows": (c_int, [c_int, c_int, P, P, P, P, P, P, P, c_int64, c_int, P, P, c_int, P, P]),
    "ctr_epoch_rows2": (c_int, [c_int, c_int, P, P, P, P, P, P, P, P, P, P, P, P, c_int64, c_int, P, P, c_int, P, P, P,
                                P, P]),
    "ctr_epoch_shared_last_supported": (c_int, [c_int, c_int64, c_int]),
    "ctr_epoch_sweep": (c_int, [c_int, P, P, P, P, P, P, P, c_int64, c_int, P, P, c_int, c_int, c_int, P, P,
                                ctypes.POINTER(c_int), P, c_int64, P, P, P, P, P]),
    "ctr_epoch_reg_loss": (c_int, [P, P, c_int, c_int, c_float, P, c_int, P]),
    "ctr_selftest_divsqrt": (c_int, [c_uint64, c_int64, P, P]),
    "ctr_selftest_adam_packed": (c_int, [c_int, c_uint64, c_int64, c_int, c_float, c_float, P, P]),
    "ctr_reduce_sum": (c_int, [P, c_int64, c_float, P, P, c_size_t, P]),
    "ctr_l2_loss_workspace_bytes": (c_size_t, [c_int64]),
    "ctr_l2_loss": (c_int, [P, c_int64, c_float, P, P, c_size_t, P]),
    "ctr_logit_loss": (c_int, [P, P, P, P, P, c_int, c_int, P, P, P, P, P, P]),
    "ctr_fc_fwd": (c_int, [P, P, P, P, c_float, c_int, c_int, c_int, c_int, P, P]),
    "ctr_fc_bwd_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "ctr_fc_fwd_grouped": (c_int, [P, P, P, P, c_int, P, c_float, c_int, c_int, c_int, c_int, P, P]),
    "ctr_fc_bwd": (c_int, [P, P, P, P, c_float, P, c_int, c_int, c_int, c_int, P, c_int, P, P, P, c_size_t, P]),
    "ctr_fc1_fwd": (c_int, [P, c_int, P, c_int, P, P, c_int, P, P]),
    "ctr_fc1_bwd_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "ctr_fc1_bwd": (c_int, [P, c_int, P, c_int, P, P, c_int, P, P, P, P, P, c_size_t, P]),
    "ctr_dropout_mask": (c_int, [P, c_int64, c_float, c_uint64, P, P]),
    "ctr_bn_workspace_bytes": (c_size_t, [c_int]),
    "ctr_bn_fwd": (c_int, [P, c_int, c_int, P, P, P, P, c_int, c_float, c_float, P, c_float, P, P, P, P, c_size_t, P]),
    "ctr_bn_bwd": (c_int, [P, P, c_int, c_int, P, P, P, c_float, P, c_float, P, P, P, P, c_size_t, P]),
    "ctr_cross_fwd": (c_int, [P, P, P, c_int, c_int, c_int, P, P, P]),
    "ctr_cross_bwd_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "ctr_cross_bwd": (c_int, [P, P, P, P, P, P, c_int, c_int, c_int, P, P, P, P, c_size_t, P]),
    "ctr_mvm_fwd": (c_int, [P, P, c_int, c_int, c_int, P, P]),
    "ctr_mvm_bwd_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "ctr_mvm_bwd": (c_int, [P, P, P, P, c_int, c_int, c_int, P, P, P, c_size_t, P]),
    "ctr_esmm_embed_fwd": (c_int, [P, P, P, P, P, P, c_int64, c_int, c_int, c_int, P, P, P]),
    "ctr_esmm_embed_bwd": (c_int, [P, P, P, c_int, c_int, c_int, c_int64, P, P]),
    "ctr_esmm_head": (c_int, [P, P, P, P, c_int, c_int, c_float, c_float, P, P, P, P, P, P, P]),
    "ctr_gather_scale_rows": (c_int, [P, P, P, c_int64, c_int64, c_int, c_int, c_int64, P, P, P]),
    "ctr_bag_sum_fwd_oob": (c_int, [P, P, P, P, c_int64, c_int, c_int, c_int64, P, P, P]),
    "ctr_bag_sum_bwd": (c_int, [P, c_int64, P, P, c_int, c_int, P, P]),
    "ctr_scale_rows": (c_int, [P, P, P, c_int64, c_int, c_int, c_int64, P, P]),
    "ctr_din_pool_fwd": (c_int, [P, P, P, c_int, c_int, c_int, P, P, c_int64, P]),
    "ctr_din_pool_bwd": (c_int, [P, P, P, P, c_int64, c_int, c_int, c_int, P, P, P]),
    "ctr_din_att_dz": (c_int, [P, P, c_float, P, P, c_int, c_int, c_int, P, P, P, P]),
    "ctr_colsum_rows": (c_int, [P, c_int, c_int, c_int, P, P]),
    "ctr_axpby": (c_int, [P, c_float, P, c_float, c_int64, P, P]),
    "ctr_pnn_product_fwd": (c_int, [P, c_int, c_int, c_int, c_int, P, P]),
    "ctr_pnn_product_bwd": (c_int, [P, P, c_int, c_int, c_int, c_int, P, P]),
    "ctr_afm_pairs_fwd": (c_int, [P, c_int, c_int, c_int, P, P]),
    "ctr_afm_pairs_bwd": (c_int, [P, P, c_int, c_int, c_int, P, P]),
    "ctr_afm_pool_fwd": (c_int, [P, P, P, c_float, c_int, c_int, c_int, P, P, P]),
    "ctr_afm_pool_bwd": (c_int, [P, P, P, c_float, P, c_int, c_int, c_int, P, P, P]),
    "ctr_dropout_apply": (c_int, [P, P, c_float, c_int64, P, P]),
    "ctr_shard_keys": (c_int, [P, c_int64, c_int64, c_int, P, P, P]),
    "ctr_shard_split": (c_int, [P, P, c_int64, c_int64, c_int, P, P, P]),
    "ctr_gather_scalar": (c_int, [P, P, c_int64, c_int64, P, P]),
    "ctr_wd_input_fwd": (c_int, [P, P, P, P, P, P, P, c_int, c_int, c_int, c_int, c_int, P, P, P, P]),
    "ctr_wd_input_bwd": (c_int, [P, P, P, c_int, c_int, c_int, c_int, P, P, P, P, P]),
    "ctr_wd_serve_input": (c_int, [P, P, c_int64, c_int64, P, P, P, P, P, c_int, c_int, P, P, P, P]),
    "ctr_parse_libsvm": (c_int64, [c_char_p, c_size_t, c_int, c_int64, c_int, P, P, P, ctypes.POINTER(c_size_t)]),
    "ctr_libsvm_count_fields": (c_int, [c_char_p, c_size_t]),
    "ctr_parse_libsvm_device_workspace_bytes": (c_size_t, [c_size_t, c_int64]),
    "ctr_parse_libsvm_device": (c_int, [P, c_size_t, c_int, c_int64, c_int, P, P, P, P, P, c_size_t, P]),
    "ctr_parse_csv_device_workspace_bytes": (c_size_t, [c_size_t, c_int64]),
    "ctr_parse_csv_device": (c_int, [P, c_size_t, c_int, c_int, c_int64, c_int, P, P, P, P, P, c_size_t, P]),
    "ctr_criteo_table_bytes": (c_size_t, [c_int64]),
    "ctr_criteo_stats_workspace_bytes": (c_size_t, [c_size_t]),
    "ctr_criteo_stats": (c_int, [P, c_size_t, c_int64, P, c_int64, P, P, P, c_size_t, P]),
    "ctr_criteo_vocab_workspace_bytes": (c_size_t, [c_int64]),
    "ctr_criteo_vocab": (c_int, [P, c_int64, c_int64, P, P, P, c_size_t, P]),
    "ctr_criteo_emit_workspace_bytes": (c_size_t, [c_size_t]),
    "ctr_criteo_emit_plan": (c_int, [P, c_size_t, c_int, c_int64, P, P, c_int64, P, P, P, P, c_int, P, P, c_size_t, P]),
    "ctr_criteo_emit_write": (c_int, [P, c_size_t, c_int, P, P, c_int64, P, P, P, P, c_int, P, P, P, c_size_t, P]),
    "ctr_tfrecord_frame": (c_int, [P, c_size_t, c_int, P, c_int64, P]),
    "ctr_tfrecord_scan": (c_int, [P, c_size_t, P, c_int64, c_int64, c_int, c_int, P, P, P]),
    "ctr_tfrecord_emit_din": (c_int, [P, P, P, c_int, c_int, c_int, P, P, P, P, P, P, P, P]),
    "ctr_tfrecord_emit_esmm": (c_int, [P, P, P, c_int, c_int, P, P, P, P, P, P, P, P]),
    "ctr_din_serve_scan": (c_int, [P, P, c_int64, c_int64, c_int, c_int, c_int, P, P, P, P, P, P]),
    "ctr_aliccp_workspace_bytes": (c_size_t, [c_size_t]),
    "ctr_aliccp_plan": (c_int, [P, c_size_t, c_int64, P, P, c_size_t, P]),
    "ctr_aliccp_declines": (c_int, [P, c_size_t, P, c_size_t, P, P]),
    "ctr_aliccp_write": (c_int, [P, c_size_t, P, P, P, c_size_t, P]),
    "ctr_aliccp_sample_count_table_bytes": (c_size_t, [c_int64]),
    "ctr_aliccp_sample_md5_table_bytes": (c_size_t, [c_int64]),
    "ctr_aliccp_sample_chunk_workspace_bytes": (c_size_t, [c_size_t, c_int64]),
    "ctr_aliccp_sample_classify": (c_int, [P, c_size_t, c_int64, c_int, P, c_int64, P, c_int64, P, P, c_size_t, P]),
    "ctr_aliccp_sample_place": (c_int, [P, c_size_t, c_int64, c_int64, c_uint64, c_int64, P, c_int64, P, c_int64, P, P,
                                        P, c_int64, P, P, c_int64, P, c_size_t, P]),
    "ctr_aliccp_sample_resolve": (c_int, [P, c_int64, P, c_int64, P, c_int64, P, P, P]),
    "ctr_aliccp_sample_count_commons": (c_int, [P, P, P, P, c_int64, P, c_int64, P, P]),
    "ctr_aliccp_sample_vocab_workspace_bytes": (c_size_t, [c_int64]),
    "ctr_aliccp_sample_vocab": (c_int, [P, c_int64, c_int64, P, P, P, c_size_t, P]),
    "ctr_aliccp_sample_feat_cnts": (c_int, [P, P, c_size_t, c_int64, P]),
    "ctr_aliccp_sample_render": (c_int, [P, P, P, P, c_int64, P, c_int64, P, P, P]),
    "ctr_aliccp_sample_emit": (c_int, [P, c_size_t, c_int64, c_int64, c_uint64, P, c_int64, P, P, P, c_int64, P, c_int64,
                                       c_int64, P, P, P, c_size_t, P]),
    "ctr_aliccp_sample_order_workspace_bytes": (c_size_t, [c_int64]),
    "ctr_aliccp_sample_order": (c_int, [P, P, c_int64, c_int64, P, P, c_size_t, P]),
    "ctr_smart_map_table_bytes": (c_size_t, [c_int64]),
    "ctr_smart_map_workspace_bytes": (c_size_t, [c_size_t]),
    "ctr_smart_map_build": (c_int, [P, c_size_t, P, c_int64, P, P, P, c_size_t, P]),
    "ctr_smart_emit_workspace_bytes": (c_size_t, [c_size_t]),
    "ctr_smart_emit_plan": (c_int, [P, c_size_t, P, P, c_int64, P, P, P, c_size_t, P]),
    "ctr_smart_emit_write": (c_int, [P, c_size_t, P, P, c_int64, P, P, P, c_size_t, P]),
    "ctr_smart_build_table_bytes": (c_size_t, [c_int64]),
    "ctr_smart_build_insert_workspace_bytes": (c_size_t, [c_size_t]),
    "ctr_smart_build_insert": (c_int, [P, c_size_t, c_int64, P, c_int64, P, c_int64, P, P, P, c_size_t, P]),
    "ctr_smart_build_workspace_bytes": (c_size_t, [c_int64]),
    "ctr_smart_build_finish": (c_int, [P, c_int64, P, P, P, P, c_size_t, P]),
    "ctr_smart_build_render": (c_int, [P, c_int64, P, P, P, c_size_t, P]),
    "ctr_frappe_workspace_bytes": (c_size_t, [c_size_t]),
    "ctr_frappe_plan": (c_int, [P, c_size_t, P, P, c_size_t, P]),
    "ctr_frappe_write": (c_int, [P, c_size_t, P, P, c_size_t, P]),
    "ctr_crc32c_workspace_bytes": (c_size_t, [c_int, c_int64]),
    "ctr_crc32c_ranges": (c_int, [P, c_int, c_int64, P, P, P, c_size_t, P]),
    "ctr_auc_counts": (c_int, [P, P, c_int64, P, P, P]),
    "ctr_format_preds_workspace_bytes": (c_size_t, [c_int64]),
    "ctr_format_preds": (c_int, [P, P, c_int64, P, c_int64, P, P, c_size_t, P]),
    "ctr_init_trunc_normal": (c_int, [P, c_int64, c_float, c_uint64, P]),
    "ctr_fill": (c_int, [P, c_int64, c_float, P]),
}

for _name, (_res, _args) in SIGNATURES.items():
    _fn = getattr(_lib, _name)  # AttributeError here == header/library mismatch: fail loudly
    _fn.restype = _res
    _fn.argtypes = _args


def last_error() -> str:
    return (_lib.ctr_last_error() or b"").decode("utf-8", "replace")


def check(status: int, what: str) -> None:
    if status != 0:
        raise CtrError(f"{what} failed with status {status}: {last_error()}")


def raw():
    """The ctypes CDLL (for tests that check symbol export)."""
    return _lib


def launch_count() -> int:
    return int(_lib.ctr_launch_count())


def abi_version() -> int:
    return int(_lib.ctr_abi_version())
