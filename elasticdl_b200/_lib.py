"""ctypes binding of libb200ps.so (include/b200ps.h).

There is deliberately NO fallback: if the CUDA library is missing or a call
fails, an exception is raised.  The product path never routes through a CPU
implementation.
"""
import ctypes
import os

from elasticdl_b200 import build as _build

ABI_VERSION = 2  # B200PS_ABI_VERSION of include/b200ps.h
MAX_SHARDS = 16
MAX_SEGS = 96

OK, EINVAL, ECUDA, ENOTFOUND, EWIDTH, ERANGE, ESTATE = 0, -1, -2, -3, -4, -5, -6


class Seg(ctypes.Structure):
    _fields_ = [
        ("table", ctypes.c_int32),
        ("n", ctypes.c_int32),
        ("ids_dev", ctypes.c_void_p),
        ("n_dev", ctypes.c_void_p),
        ("rows_dev", ctypes.c_void_p),
    ]


DEEPFM_TILE_MAXG = 38  # B200_DEEPFM_TILE_MAXG: id groups the tile towers hold
# floats of `scratch` the tile towers need: W1 in tile column order and the tile counter (DeepFM), W1 and the cross
# weights and the counters (B200_DEEPFM_DCN_SCRATCH)
DEEPFM_TILE_SCRATCH = 320 * 16 + 16
DEEPFM_DCN_SCRATCH = 320 * 20 + 16


class DeepFMRows(ctypes.Structure):  # b200_deepfm_rows_t (include/b200_deepfm.h)
    _fields_ = [
        ("uniq", ctypes.c_void_p),
        ("deep_base", ctypes.c_void_p * DEEPFM_TILE_MAXG), ("wide_base", ctypes.c_void_p * DEEPFM_TILE_MAXG),
        ("deep_stride", ctypes.c_int64), ("wide_stride", ctypes.c_int64),
        ("deep_param_off", ctypes.c_int64), ("wide_param_off", ctypes.c_int64),
    ]


class DeepFMArgs(ctypes.Structure):  # b200_deepfm_args_t (include/b200_deepfm.h)
    _fields_ = [
        ("G", ctypes.c_int32), ("B", ctypes.c_int32),
        ("inv", ctypes.c_void_p), ("n_unique", ctypes.c_void_p),
        ("bet_wide", ctypes.c_void_p), ("bet_deep", ctypes.c_void_p),
        ("dense", ctypes.c_void_p), ("labels", ctypes.c_void_p),
        ("params", ctypes.c_void_p), ("grads", ctypes.c_void_p),
        ("gsum_wide", ctypes.c_void_p), ("gsum_deep", ctypes.c_void_p),
        ("loss", ctypes.c_void_p), ("logits", ctypes.c_void_p), ("scratch", ctypes.c_void_p),
        ("rows", ctypes.POINTER(DeepFMRows)),
    ]


class CensusArgs(ctypes.Structure):  # b200_census_args_t (include/b200_census.h)
    _fields_ = [
        ("B", ctypes.c_int32), ("reference_reshape", ctypes.c_int32),
        ("ids", ctypes.c_void_p), ("labels", ctypes.c_void_p), ("params", ctypes.c_void_p),
        ("loss", ctypes.c_void_p), ("logits", ctypes.c_void_p), ("grads", ctypes.c_void_p),
        ("uniq", ctypes.c_void_p), ("n_unique", ctypes.c_void_p), ("gsum", ctypes.c_void_p),
        ("error", ctypes.c_void_p), ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_size_t),
    ]


class CsqlArgs(ctypes.Structure):  # b200_csql_args_t (include/b200_census_sqlflow.h)
    _fields_ = CensusArgs._fields_


class FrappeArgs(ctypes.Structure):  # b200_frappe_args_t (include/b200_frappe.h)
    _fields_ = [
        ("B", ctypes.c_int32), ("pad_", ctypes.c_int32),
        ("ids", ctypes.c_void_p), ("inv", ctypes.c_void_p), ("n_unique", ctypes.c_void_p),
        ("bet_deep", ctypes.c_void_p), ("bet_wide", ctypes.c_void_p), ("labels", ctypes.c_void_p),
        ("params", ctypes.c_void_p), ("loss", ctypes.c_void_p), ("logits", ctypes.c_void_p),
        ("grads", ctypes.c_void_p), ("gsum_deep", ctypes.c_void_p), ("gsum_wide", ctypes.c_void_p),
        ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_size_t),
    ]


FC_MAX_TABLES, FC_MAX_BLOCKS = 8, 16  # B200_FC_DNN_MAX_TABLES, B200_FC_DNN_MAX_BLOCKS


class FcBlock(ctypes.Structure):  # b200_fc_block_t (include/b200_fc_dnn.h)
    _fields_ = [("kind", ctypes.c_int32), ("src", ctypes.c_int32), ("width", ctypes.c_int32),
                ("offset", ctypes.c_int32)]


class FcLayout(ctypes.Structure):  # b200_fc_layout_t
    _fields_ = [
        ("F", ctypes.c_int32), ("n_blocks", ctypes.c_int32), ("n_tables", ctypes.c_int32),
        ("loss_mean", ctypes.c_int32), ("table_rows", ctypes.c_int32 * FC_MAX_TABLES),
        ("table_dim", ctypes.c_int32 * FC_MAX_TABLES), ("table_string", ctypes.c_int32 * FC_MAX_TABLES),
        ("blocks", FcBlock * FC_MAX_BLOCKS),
    ]


class FcDnnArgs(ctypes.Structure):  # b200_fc_dnn_args_t
    _fields_ = [
        ("B", ctypes.c_int64), ("n_numeric", ctypes.c_int32), ("n_ids", ctypes.c_int32),
        ("n_strings", ctypes.c_int32), ("W", ctypes.c_int32),
        ("numeric", ctypes.c_void_p), ("ids", ctypes.c_void_p), ("strings", ctypes.c_void_p),
        ("inv", ctypes.c_void_p), ("n_unique", ctypes.c_void_p), ("rows", ctypes.c_void_p),
        ("labels", ctypes.c_void_p), ("params", ctypes.c_void_p), ("loss", ctypes.c_void_p),
        ("logits", ctypes.c_void_p), ("grads", ctypes.c_void_p), ("gsum", ctypes.c_void_p),
        ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_size_t),
    ]


class DeepctrWdlArgs(ctypes.Structure):  # b200_deepctr_wdl_args_t (include/b200_deepctr_wdl.h)
    _fields_ = [
        ("B", ctypes.c_int64), ("ids", ctypes.c_void_p), ("dense", ctypes.c_void_p), ("labels", ctypes.c_void_p),
        ("params", ctypes.c_void_p), ("loss", ctypes.c_void_p), ("logits", ctypes.c_void_p),
        ("grads", ctypes.c_void_p), ("error", ctypes.c_void_p), ("workspace", ctypes.c_void_p),
        ("workspace_bytes", ctypes.c_size_t),
    ]


DeepctrDeepfmArgs = DeepctrWdlArgs  # b200_deepctr_deepfm_args_t (include/b200_deepctr_deepfm.h) has the same fields


LR_MAX_BOUNDARIES = 32  # B200PS_LR_MAX_BOUNDARIES
LR_PIECEWISE, LR_EXPONENTIAL, LR_INVERSE_TIME, LR_POLYNOMIAL = 1, 2, 3, 4


class LrSchedule(ctypes.Structure):  # b200ps_lr_schedule_t (include/b200ps.h)
    _fields_ = [
        ("kind", ctypes.c_int32), ("n_boundaries", ctypes.c_int32), ("staircase", ctypes.c_int32),
        ("cycle", ctypes.c_int32),
        ("initial_learning_rate", ctypes.c_double), ("decay_steps", ctypes.c_double), ("decay_rate", ctypes.c_double),
        ("end_learning_rate", ctypes.c_double), ("power", ctypes.c_double),
        ("boundaries", ctypes.c_double * LR_MAX_BOUNDARIES), ("values", ctypes.c_float * (LR_MAX_BOUNDARIES + 1)),
    ]


class PSError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("b200ps error %d: %s" % (code, msg))
        self.code = code


class PSNotFound(PSError, KeyError):
    pass


class PSRangeError(PSError, ValueError):
    pass


# every symbol include/b200ps.h declares: name -> (restype, argtypes)
_vp, _i, _i64, _f, _sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float, ctypes.c_size_t
_segp = ctypes.POINTER(Seg)
SYMBOLS = {
    "b200ps_last_error": (ctypes.c_char_p, []),
    "b200ps_abi_version": (_i, []),
    "b200ps_create": (_i, [_i, _i, ctypes.c_char_p, ctypes.c_char_p, _i, ctypes.c_uint, ctypes.POINTER(_vp)]),
    "b200ps_destroy": (_i, [_vp]),
    "b200ps_clone_view": (_i, [_vp, _i, ctypes.POINTER(_vp)]),
    "b200ps_shard_create_local": (_i, [_vp, _i, _i]),
    "b200ps_shard_export": (_i, [_vp, _i, _vp, _sz, ctypes.POINTER(_sz)]),
    "b200ps_shard_import": (_i, [_vp, _i, _vp, _sz]),
    "b200ps_table_register": (_i, [_vp, ctypes.c_char_p, _i, ctypes.c_char_p, _i64, ctypes.c_uint64]),
    "b200ps_table_register_pair": (_i, [_vp, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p, _i64, ctypes.c_uint64]),
    "b200ps_table_register_hashed": (_i, [_vp, ctypes.c_char_p, _i, ctypes.c_char_p, _i64, ctypes.c_uint64]),
    "b200ps_dense_register": (_i, [_vp, ctypes.c_char_p, _i, _i64, _i]),
    "b200ps_lookup": (_i, [_vp, ctypes.c_char_p]),
    "b200ps_commit": (_i, [_vp]),
    "b200ps_pull_rows": (_i, [_vp, _segp, _i, _vp]),
    "b200ps_set_rows": (_i, [_vp, _segp, _i, _vp]),
    "b200ps_pull_rows_pair": (_i, [_vp, _segp, ctypes.POINTER(_vp), _i, _vp]),
    "b200ps_push_rows_pair": (_i, [_vp, _segp, ctypes.POINTER(_vp), _i, _vp]),
    "b200ps_xchg_create": (_i, [_vp, _i, _i, ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int32)]),
    "b200ps_xchg_pull": (_i, [_vp, _vp, _vp, _vp, _vp, _vp]),
    "b200ps_xchg_profile": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, ctypes.POINTER(ctypes.c_float), _vp]),
    "b200ps_xchg_push": (_i, [_vp, _vp, _vp, _vp]),
    "b200ps_pull_dense": (_i, [_vp, _segp, _i, _vp]),
    "b200ps_set_dense": (_i, [_vp, _segp, _i, _vp]),
    "b200ps_slot_rows": (_i, [_vp, _i, _i, _segp, _i, _vp]),
    "b200ps_slot_dense": (_i, [_vp, _i, _i, _segp, _i, _vp]),
    "b200ps_push_begin": (_i, [_vp, _f, ctypes.POINTER(ctypes.c_int32), _vp]),
    "b200ps_set_lr_schedule": (_i, [_vp, ctypes.POINTER(LrSchedule)]),
    "b200ps_push_rows": (_i, [_vp, _segp, _i, _vp]),
    "b200ps_push_dense": (_i, [_vp, _segp, _i, _vp]),
    "b200ps_push_dense_reduce": (_i, [_vp, _i, ctypes.POINTER(_vp), _i, _f, _i, _vp]),
    "b200ps_push_dense_allreduce": (_i, [_vp, _i, _vp, ctypes.POINTER(_vp), _i, _f, _f, _f, _f, _f, _vp]),
    "b200ps_push_end": (_i, [_vp, _vp, _vp]),
    "b200ps_bump_step": (_i, [_vp, _vp]),
    "b200ps_push_begin_shard": (_i, [_vp, _i, _f, ctypes.POINTER(ctypes.c_int32), _vp]),
    "b200ps_push_end_shard": (_i, [_vp, _i, _vp]),
    "b200ps_raw_register": (_i, [_vp, ctypes.c_char_p, _sz]),
    "b200ps_raw_ptr": (_i, [_vp, _i, _i, ctypes.POINTER(_vp), ctypes.POINTER(_sz)]),
    "b200ps_table_rows_ptr": (_i, [_vp, _i, _i, ctypes.POINTER(ctypes.POINTER(_f)), ctypes.POINTER(_i64),
                                   ctypes.POINTER(_i64), ctypes.POINTER(_i64)]),
    "b200ps_barrier": (_i, [_vp, _vp]),
    "b200ps_kernel_sgd": (_i, [_vp, _vp, _f, ctypes.c_longlong, _vp]),
    "b200ps_kernel_momentum": (_i, [_vp, _vp, _vp, _f, _i, _f, ctypes.c_longlong, _vp]),
    "b200ps_kernel_adam": (_i, [_vp, _vp, _vp, _vp, _f, ctypes.c_longlong, ctypes.c_longlong, _f, _f, _f, _vp, _vp]),
    "b200ps_kernel_adagrad": (_i, [_vp, _vp, _vp, _f, ctypes.c_longlong, _f, _vp]),
    "b200ps_unique_workspace": (_sz, [_i, _i64]),
    "b200ps_unique": (_i, [_vp, _vp, _i, _i64, _vp, _vp, _vp, _vp, _sz, _vp]),
    "b200ps_unique_bounded_workspace": (_sz, [_i, _i64, ctypes.POINTER(_i64)]),
    "b200ps_unique_bounded": (_i, [_vp, _vp, _i, _i64, ctypes.POINTER(_i64), _vp, _vp, _vp, _vp, _sz, _vp]),
    "b200ps_unique_bounded_i32": (_i, [_vp, _vp, _i, _i64, ctypes.POINTER(_i64), _vp, _vp, _vp, _vp, _sz, _vp]),
    "b200ps_unique_bounded_ex": (_i, [_vp, _vp, _i, _i, _i64, ctypes.POINTER(_i64), _vp, _vp, _vp, _vp, _sz, _i, _vp]),
    "b200ps_debug_buffer": (_i, [_vp, _sz]),
    "b200ps_unique_packed": (_i, [_vp, _vp, ctypes.POINTER(ctypes.c_int32), _i, _i64, ctypes.POINTER(_i64), _vp, _vp, _vp, _vp,
                                  _sz, _i, _vp]),
    "b200ps_packed_ids_bytes": (_sz, [ctypes.POINTER(ctypes.c_int32), _i, _i64]),
    "b200ps_segment_sum": (_i, [_vp, _vp, _vp, _i, _i64, _i, _vp, _vp]),
    "b200ps_gather_rows": (_i, [_vp, _vp, _vp, _i, _i64, _i, _vp, _vp]),
    "b200ps_sparse_workspace": (_sz, [_i64, _i64, _i]),
    "b200ps_sparse_prep": (_i, [_vp, _vp, _vp, _i, _i64, _i64, _i, _vp, _vp, _sz, _vp]),
    "b200ps_bag_prep": (_i, [_vp, _vp, _i, _vp, _i64, _i, _i64, _i64, _i64, _i, _vp, _vp, _sz, _vp]),
    "b200ps_sparse_combine": (_i, [_vp, _vp, _vp, _vp, _sz, _i64, _i64, _i, _i, _vp, _vp]),
    "b200ps_sparse_combine_grad": (_i, [_vp, _vp, _vp, _vp, _sz, _i64, _i64, _i, _i, _i64, _vp, _vp]),
    "b200ps_sparse_combine_weighted": (_i, [_vp, _vp, _vp, _vp, _vp, _sz, _i64, _i64, _i, _i, _vp, _vp]),
    "b200ps_sparse_combine_weighted_grad": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _sz, _i64, _i64, _i, _i, _i64, _vp, _vp,
                                                 _vp]),
    "b200ps_shard_state": (_i, [_vp, _i, ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(_i64), ctypes.POINTER(ctypes.c_int32)]),
    "b200ps_set_shard_state": (_i, [_vp, _i, ctypes.c_int32, _i64, ctypes.c_int32]),
    "b200ps_snapshot_state": (_i, [_vp, _vp, _vp]),
    "b200ps_try_init": (_i, [_vp, _i, ctypes.POINTER(_i)]),
    "b200ps_finish_init": (_i, [_vp, _i, ctypes.c_int32, _vp]),
    "b200ps_table_size": (_i, [_vp, _i, _i, ctypes.POINTER(_i64)]),
    "b200ps_table_ids": (_i, [_vp, _i, _i, _vp, _i64, ctypes.POINTER(_i64)]),
    "b200ps_check": (_i, [_vp]),
    "b200ps_launch_count": (_i64, [_vp]),
    # include/b200_deepfm.h
    "b200_deepfm_param_count": (_sz, [_i]),
    "b200_deepfm_fwd_bwd": (_i, [ctypes.POINTER(DeepFMArgs), _vp]),
    "b200_deepfm_forward": (_i, [ctypes.POINTER(DeepFMArgs), _vp]),
    "b200_deepfm_fwd_bwd_mma": (_i, [ctypes.POINTER(DeepFMArgs), _vp]),
    "b200_deepfm_mma_launch_count": (_i64, []),
    "b200_deepfm_launch_count": (_i64, []),
    "b200_deepfm_fwd_bwd_tile": (_i, [ctypes.POINTER(DeepFMArgs), _vp]),
    "b200_deepfm_forward_tile": (_i, [ctypes.POINTER(DeepFMArgs), _vp]),
    "b200_deepfm_publish_loss": (_i, [_vp, _vp, _i, _vp, _vp]),
    "b200_deepfm_tile_prologue": (_i, [ctypes.POINTER(DeepFMArgs), _vp]),
    "b200_deepfm_tile_main": (_i, [ctypes.POINTER(DeepFMArgs), _vp]),
    "b200_deepfm_tile_launch_count": (_i64, []),
    "b200_deepfm_last_error": (ctypes.c_char_p, []),
    "b200_deepfm_dcn_param_count": (_sz, [_i]),
    "b200_deepfm_dcn_fwd_bwd_tile": (_i, [ctypes.POINTER(DeepFMArgs), _vp]),
    "b200_deepfm_dcn_tile_prologue": (_i, [ctypes.POINTER(DeepFMArgs), _vp]),
    "b200_deepfm_dcn_tile_main": (_i, [ctypes.POINTER(DeepFMArgs), _vp]),
    "b200_deepfm_dcn_forward_tile": (_i, [ctypes.POINTER(DeepFMArgs), _vp]),
    "b200_deepfm_dcn_launch_count": (_i64, []),
    "b200_deepfm_wide_deep_fwd_bwd_tile": (_i, [ctypes.POINTER(DeepFMArgs), _vp]),
    "b200_deepfm_wide_deep_tile_prologue": (_i, [ctypes.POINTER(DeepFMArgs), _vp]),
    "b200_deepfm_wide_deep_tile_main": (_i, [ctypes.POINTER(DeepFMArgs), _vp]),
    "b200_deepfm_wide_deep_forward_tile": (_i, [ctypes.POINTER(DeepFMArgs), _vp]),
    "b200_deepfm_xdeepfm_param_count": (_sz, [_i]),
    "b200_deepfm_xdeepfm_scratch_floats": (_sz, [_i, _i]),
    "b200_deepfm_xdeepfm_fwd_bwd_tile": (_i, [ctypes.POINTER(DeepFMArgs), _vp]),
    "b200_deepfm_xdeepfm_tile_prologue": (_i, [ctypes.POINTER(DeepFMArgs), _vp]),
    "b200_deepfm_xdeepfm_tile_main": (_i, [ctypes.POINTER(DeepFMArgs), _vp]),
    "b200_deepfm_xdeepfm_forward_tile": (_i, [ctypes.POINTER(DeepFMArgs), _vp]),
    "b200_deepfm_xdeepfm_launch_count": (_i64, []),
    # include/b200_features.h
    "b200feat_last_error": (ctypes.c_char_p, []),
    "b200feat_transform": (_i, [_vp, _i, _vp, _i, _vp, _i, _vp, _i, _i, _vp, _i, _i, _i64, _vp, _i, _vp, _vp]),
    "b200feat_hash_strings": (_i, [_vp, _i, _i64, _i64, _vp, _vp]),
    "b200feat_hash_ints": (_i, [_vp, _i64, _i64, _vp, _vp]),
    "b200feat_bucketize": (_i, [_vp, _i64, _vp, _i, _vp, _vp]),
    "b200feat_transform_ext": (_i, [_vp, _vp, _i, _vp, _i, _vp, _i, _vp, _i, _i, _vp, _i, _i, _i64, _vp, _i, _vp, _vp]),
    "b200feat_vocab_slots": (_i64, [_i64]),
    "b200feat_vocab_build": (_i, [_vp, _i64, _i, _i64, _vp, ctypes.POINTER(_i64)]),
    "b200feat_index_lookup": (_i, [_vp, _i, _i64, _vp, _vp, _i64, ctypes.c_int32, ctypes.c_int32, _i64, _vp, _vp]),
    "b200feat_log_round": (_i, [_vp, _i, _i64, _i64, _i64, _i, ctypes.c_double, _vp, _vp]),
    "b200feat_round_identity": (_i, [_vp, _i, _i64, _i64, _i64, _vp, _vp]),
    "b200feat_fingerprint64": (_i, [_vp, _i, _i64, _vp, _vp]),
    "b200feat_launch_count": (_i64, []),
}
# include/b200_census.h
CENSUS_SYMBOLS = {
    "b200_census_workspace_bytes": (_sz, [_i64]),
    "b200_census_tower": (_i, [ctypes.POINTER(CensusArgs), _vp]),
    "b200_census_last_error": (ctypes.c_char_p, []),
    "b200_census_launch_count": (_i64, []),
}
# include/b200_census_sqlflow.h
CSQL_SYMBOLS = {
    "b200_csql_workspace_bytes": (_sz, [_i64]),
    "b200_csql_tower": (_i, [ctypes.POINTER(CsqlArgs), _vp]),
    "b200_csql_forward": (_i, [ctypes.POINTER(CsqlArgs), _vp]),
    "b200_csql_last_error": (ctypes.c_char_p, []),
    "b200_csql_launch_count": (_i64, []),
}
# include/b200_frappe.h
FRAPPE_SYMBOLS = {
    "b200_frappe_workspace_bytes": (_sz, [_i64]),
    "b200_frappe_tower": (_i, [ctypes.POINTER(FrappeArgs), _vp]),
    "b200_frappe_forward": (_i, [ctypes.POINTER(FrappeArgs), _vp]),
    "b200_frappe_last_error": (ctypes.c_char_p, []),
    "b200_frappe_launch_count": (_i64, []),
}
# include/b200_fc_dnn.h
FC_DNN_SYMBOLS = {
    "b200_fc_dnn_params": (_i64, [ctypes.POINTER(FcLayout)]),
    "b200_fc_dnn_workspace_bytes": (_sz, [ctypes.POINTER(FcLayout), _i64]),
    "b200_fc_dnn_fill_empty": (_i, [ctypes.POINTER(FcLayout), _vp, _vp, _i64, _i, _vp]),
    "b200_fc_dnn_tower": (_i, [ctypes.POINTER(FcLayout), ctypes.POINTER(FcDnnArgs), _vp]),
    "b200_fc_dnn_forward": (_i, [ctypes.POINTER(FcLayout), ctypes.POINTER(FcDnnArgs), _vp]),
    "b200_fc_dnn_last_error": (ctypes.c_char_p, []),
    "b200_fc_dnn_launch_count": (_i64, []),
}
# include/b200_deepctr_wdl.h
DEEPCTR_WDL_SYMBOLS = {
    "b200_deepctr_wdl_workspace_bytes": (_sz, [_i64]),
    "b200_deepctr_wdl_tower": (_i, [ctypes.POINTER(DeepctrWdlArgs), _vp]),
    "b200_deepctr_wdl_forward": (_i, [ctypes.POINTER(DeepctrWdlArgs), _vp]),
    "b200_deepctr_wdl_last_error": (ctypes.c_char_p, []),
    "b200_deepctr_wdl_launch_count": (_i64, []),
}
# include/b200_deepctr_deepfm.h
DEEPCTR_DEEPFM_SYMBOLS = {
    "b200_deepctr_deepfm_workspace_bytes": (_sz, [_i64]),
    "b200_deepctr_deepfm_tower": (_i, [ctypes.POINTER(DeepctrDeepfmArgs), _vp]),
    "b200_deepctr_deepfm_forward": (_i, [ctypes.POINTER(DeepctrDeepfmArgs), _vp]),
    "b200_deepctr_deepfm_last_error": (ctypes.c_char_p, []),
    "b200_deepctr_deepfm_launch_count": (_i64, []),
}
# include/b200_metrics.h
METRICS_MAX_THRESHOLDS = 16384  # B200_METRICS_MAX_THRESHOLDS
METRICS_SYMBOLS = {
    "b200_metrics_auc_update": (_i, [_vp, _vp, _i64, _vp, ctypes.c_int32, _vp, _vp, _vp]),
    "b200_metrics_last_error": (ctypes.c_char_p, []),
    "b200_metrics_launch_count": (_i64, []),
}

_lib = None


def lib():
    """Load (building in-tree first if the sources are newer) the CUDA library."""
    global _lib
    if _lib is None:
        path = _build.LIB
        if not os.path.exists(path) or _build._stale():
            path = _build.build()
        handle = ctypes.CDLL(path)
        for name, (res, args) in list(SYMBOLS.items()) + list(CENSUS_SYMBOLS.items()) + list(FRAPPE_SYMBOLS.items())\
                + list(METRICS_SYMBOLS.items()) + list(FC_DNN_SYMBOLS.items()) + list(CSQL_SYMBOLS.items())\
                + list(DEEPCTR_WDL_SYMBOLS.items()) + list(DEEPCTR_DEEPFM_SYMBOLS.items()):
            fn = getattr(handle, name)  # AttributeError if the ABI drifted: fail loudly
            fn.restype = res
            fn.argtypes = args
        if handle.b200ps_abi_version() != ABI_VERSION:
            raise ImportError("libb200ps.so ABI version %d, this package needs %d: rebuild it"
                              % (handle.b200ps_abi_version(), ABI_VERSION))
        _lib = handle
    return _lib


def check(rc):
    """Turn a negative return code into the matching Python exception."""
    if rc >= 0:
        return rc
    msg = lib().b200ps_last_error().decode("utf-8", "replace")
    if rc == ENOTFOUND:
        raise PSNotFound(rc, msg)
    if rc == ERANGE:
        raise PSRangeError(rc, msg)
    if rc in (EINVAL, EWIDTH):
        raise ValueError("b200ps error %d: %s" % (rc, msg))
    raise PSError(rc, msg)


def check_call(rc, name, last_error):
    """Raise for a non-zero return code of the tower or metrics entry point `name`: ValueError for EINVAL (an
    argument it refused), RuntimeError otherwise, with the message of its own last_error()."""
    if rc:
        msg = last_error().decode("utf-8", "replace")
        raise (ValueError if rc == EINVAL else RuntimeError)("%s failed (%d): %s" % (name, rc, msg))
