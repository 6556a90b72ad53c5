"""ctypes binding of libmm_b200.so — the C-ABI declared in include/mm_b200.h.

This is the only place the product touches native code.  There is NO fallback: if the
library is missing or a symbol cannot be resolved, importing/using the ops raises.
"""
from __future__ import annotations

import ctypes as C
import os
import re
from pathlib import Path

_PKG = Path(__file__).resolve().parent
LIB_PATH = _PKG / "_lib" / "libmm_b200.so"
HEADER_PATH = _PKG.parent / "include" / "mm_b200.h"

MM_MAX_TABLES = 64
MM_I32, MM_I64, MM_F32, MM_F64 = 0, 1, 2, 3
ACTIVATIONS = {
    None: 0, "linear": 0, "relu": 1, "sigmoid": 2, "tanh": 3, "selu": 4, "elu": 5, "gelu": 6,
}
COMBINERS = {"mean": 0, "sum": 1, "sqrtn": 2, "max": 3}


class GatherTable(C.Structure):
    """mm_gather_table (include/mm_b200.h)."""

    _fields_ = [
        ("weights", C.c_void_p),
        ("indices", C.c_void_p),
        ("rows", C.c_int64),
        ("dim", C.c_int32),
        ("out_col", C.c_int32),
    ]


class LookupTable(C.Structure):
    """mm_lookup_table (include/mm_b200.h)."""

    _fields_ = [
        ("weights", C.c_void_p),
        ("indices", C.c_void_p),
        ("rows", C.c_int64),
        ("slot", C.c_int32),
        ("idx_bytes", C.c_int32),
        ("peer_weights_host", C.POINTER(C.c_void_p)),
    ]


class SparseTable(C.Structure):
    """mm_sparse_table (include/mm_b200.h)."""

    _fields_ = [
        ("weights", C.c_void_p),
        ("rows", C.c_int64),
        ("indices", C.c_void_p),
        ("idx_bytes", C.c_int32),
        ("reserved", C.c_int32),
        ("grad_rows", C.c_void_p),
        ("rep_map", C.c_void_p),
        ("state1", C.c_void_p),
        ("state2", C.c_void_p),
        ("mirror", C.c_void_p),
        ("dense_grad", C.c_void_p),
    ]


class WideBlock(C.Structure):
    """mm_wide_block (include/mm_b200.h)."""

    _fields_ = [
        ("indices", C.c_void_p),
        ("rows", C.c_int64),
        ("offset", C.c_int64),
        ("idx_bytes", C.c_int32),
        ("reserved", C.c_int32),
    ]


class WideBag(C.Structure):
    """mm_wide_bag (include/mm_b200.h)."""

    _fields_ = [
        ("values", C.c_void_p),
        ("offsets", C.c_void_p),
        ("rows", C.c_int64),
        ("offset", C.c_int64),
        ("nnz", C.c_int64),
        ("idx_bytes", C.c_int32),
        ("off_dtype", C.c_int32),
        ("length", C.c_int32),
        ("mode", C.c_int32),
    ]


WIDE_MODES = {"multi_hot": 0, "count": 1}  # MM_WIDE_MULTI_HOT / MM_WIDE_COUNT
OPTIMIZERS = {"sgd": 0, "adagrad": 1, "adam": 2}
LOSS_KINDS = {"binary_crossentropy": 0, "mse": 1}  # MM_LOSS_BCE / MM_LOSS_MSE
# mm_inbatch_pairwise_fwd / _bwd loss kinds (MM_PAIRWISE_*), by the reference's registry names
PAIRWISE_KINDS = {"bpr": 0, "bpr-max": 1, "top1": 2, "top1_v2": 3, "top1-max": 4, "logistic": 5, "hinge": 6}
HYPER_LR, HYPER_BETA1, HYPER_BETA2, HYPER_EPS, HYPER_STEP, HYPER_LR_T, HYPER_COUNT = 0, 1, 2, 3, 4, 5, 8
# K25 learning-rate schedules (MM_SCHED_*): kinds, the parameter layout of the device array, its size and boundary limit
SCHED_KINDS = {"ExponentialDecay": 1, "PiecewiseConstantDecay": 2, "PolynomialDecay": 3, "InverseTimeDecay": 4,
               "CosineDecay": 5}
SCHED_KIND, SCHED_INIT, SCHED_DECAY_STEPS, SCHED_RATE, SCHED_POWER, SCHED_FLAG, SCHED_NB = 0, 1, 2, 3, 4, 5, 6
SCHED_MAX_BOUNDARIES, SCHED_BOUNDARIES = 32, 8
SCHED_VALUES = SCHED_BOUNDARIES + SCHED_MAX_BOUNDARIES
SCHED_COUNT = SCHED_VALUES + SCHED_MAX_BOUNDARIES + 1
CONCAT_L2_CTAS = 512  # MM_CONCAT_L2_CTAS: mm_concat_backward_l2's partials per slice
# K24 limits and launch shape (MM_PRETRAINED_*)
PRETRAINED_MAX_DIM, PRETRAINED_MAX_OUT, PRETRAINED_CTAS_PER_SM = 1024, 256, 8


class ConcatPiece(C.Structure):
    """mm_concat_piece (include/mm_b200.h)."""

    _fields_ = [
        ("src", C.c_void_p),
        ("src_stride", C.c_int64),
        ("width", C.c_int32),
        ("dtype", C.c_int32),
        ("out_col", C.c_int32),
        ("reserved", C.c_int32),
    ]


class ColumnSlice(C.Structure):
    """mm_column_slice (include/mm_b200.h)."""

    _fields_ = [
        ("dst", C.c_void_p),
        ("dst_stride", C.c_int64),
        ("col", C.c_int32),
        ("width", C.c_int32),
    ]


class MetricsHead(C.Structure):
    """mm_metrics_head (include/mm_b200.h)."""

    _fields_ = [
        ("targets", C.c_void_p),
        ("sample_weight", C.c_void_p),
        ("metric_weights", C.c_void_p * 2),
        ("target_dtype", C.c_int32),
        ("loss_kind", C.c_int32),
        ("pred_form", C.c_int32),
        ("n_thresholds", C.c_int32),
        ("thresholds", C.c_float * 4),
    ]


# mm_metrics_update state layout (include/mm_b200.h, K17)
METRICS_MAX_HEADS, METRICS_MAX_THRESHOLDS, METRICS_MAX_BUCKETS = 8, 4, 1024
METRICS_LOSS, METRICS_COUNT, METRICS_INVALID, METRICS_SET0, METRICS_SET_STRIDE = 0, 1, 2, 3, 12
METRICS_POS, METRICS_NEG, METRICS_SQ_ERR, METRICS_W_SUM, METRICS_TP, METRICS_FP = 0, 1, 2, 3, 4, 8
METRICS_SCALARS = 27
PRED_ACT, PRED_HEAD = 0, 1

_vp, _i, _i64, _f, _u64 = C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_uint64
_tables = C.POINTER(GatherTable)

# name -> (restype, argtypes); must list every function declared in include/mm_b200.h
SIGNATURES = {
    "mm_version": (_i, []),
    "mm_last_error": (C.c_char_p, []),
    "mm_launch_count": (_i64, []),
    "mm_init_uniform_hash": (_i, [_vp, _i64, _u64, _f, _f, _vp]),
    "mm_gather_multi": (_i, [_tables, _i, _i, _i64, _vp, _i64, _vp, _vp]),
    "mm_gather_bag": (_i, [_vp, _i64, _i, _vp, _i, _vp, _i, _i64, _i, _vp, _i64, _i, _vp, _vp]),
    "mm_gather_seq": (_i, [_vp, _i64, _i, _vp, _i, _i64, _i, _i, _vp, _i64, _i, _vp, _vp]),
    "mm_concat_columns": (_i, [C.POINTER(ConcatPiece), _i, _i64, _vp, _i64, _vp]),
    "mm_concat_split": (_i, [C.POINTER(ConcatPiece), _i, _i64, _vp, _i, _vp]),
    "mm_l2_normalize": (_i, [_vp, _i64, _i, _i64, _vp, _i64, _vp]),
    "mm_scale_shift": (_i, [_vp, _i64, _i, _i64, _vp, _vp, _vp, _i64, _vp]),
    "mm_cross_combine": (_i, [_vp, _vp, _vp, _i64, _i, _i64, _i64, _i64, _vp, _i64, _vp]),
    "mm_dot_interaction": (_i, [_vp, _i64, _i, _i, _i64, _vp, _i, _i64, _i, _vp, _i64, _vp, _i, _vp]),
    "mm_dlrm_lookup_interact": (_i, [C.POINTER(LookupTable), _i, _i64, _i, _i, _i, _vp, _i64, _i, _vp, _i64, _vp, _i, _vp, _i, _vp]),
    "mm_dense_fp32": (_i, [_vp, _i64, _i, _i64, _vp, _vp, _i, _i, _vp, _i64, _vp, _i64, _vp]),
    "mm_tc_padded_k": (_i, [_i]),
    "mm_tc_padded_n": (_i, [_i]),
    "mm_split_rows": (_i, [_vp, _i64, _i, _i64, _vp, _i, _vp]),
    "mm_split_weights": (_i, [_vp, _i, _i, _vp, _i, _i, _vp]),
    "mm_dense_tc": (_i, [_vp, _i64, _i, _i, _vp, _i, _i, _vp, _i, _i, _vp, _vp, _i64, _vp, _i64,
                         _vp, _i, _vp]),
    "mm_dense_tc_dropout": (_i, [_vp, _i64, _i, _i, _vp, _i, _i, _vp, _i, _i, _vp, _i64, _vp, _i, _f, _u64, _vp, _i, _vp]),
    "mm_dense_tc_head": (_i, [_vp, _i64, _i, _i, _vp, _i, _i, _vp, _i, _i, _vp, _f, _i, _vp, _vp]),
    "mm_mlp_tc_supported": (_i, [_i, _i, C.POINTER(C.c_int), _i]),
    "mm_mlp_tc": (_i, [_vp, _i64, _i, _i, C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.POINTER(C.c_void_p), C.POINTER(C.c_int),
                       _vp, _i64, _vp, _f, _i, _vp, _vp]),
    "mm_mlp_tc_heads": (_i, [_vp, _i64, _i, _i, C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.POINTER(C.c_void_p), C.POINTER(C.c_int),
                             _i, _vp, _vp, C.POINTER(C.c_int), _vp, _vp]),
    "mm_mlp_tc_pairs": (_i, [_vp, _vp, _i64, _i, _i, C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.POINTER(C.c_void_p),
                             C.POINTER(C.c_int), _vp, _i64, _vp, _f, _i, _vp, _i, _vp, C.POINTER(C.c_int), _vp]),
    "mm_mlp_tc_operand_out": (_i, [_vp, _i64, _i, _i, C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.POINTER(C.c_void_p),
                                   C.POINTER(C.c_int), _vp, _i64, _vp, _vp]),
    "mm_tower2_small_supported": (_i, [_i, _i, _i]),
    "mm_tower2_small": (_i, [C.POINTER(ConcatPiece), _i, _i64, _vp, _i, _vp, _i, _vp, _i, _vp, _i, _vp, _i64, _vp, _vp]),
    "mm_rowwise_dot": (_i, [_vp, _vp, _i64, _i, _i64, _i64, _vp, _vp]),
    "mm_catalog_workspace_bytes": (_i64, [_i64, _i64, _i]),
    "mm_catalog_score": (_i, [_vp, _i64, _i, _vp, _i64, _vp, _vp, _i, _vp, _i, _vp, _vp, _vp, _i64, _vp]),
    "mm_inbatch_softmax_ce": (_i, [_vp, _vp, _i64, _i64, _i, _vp, _vp, _i, _i, _f, _vp, _vp, _f, _vp, _vp, _i64, _vp]),
    "mm_shard_gather_push": (_i, [_tables, _i, _i, _i64, _i64, _i, _i, _i, C.POINTER(C.c_void_p), _i64, _vp, _vp]),
    "mm_init_uniform_hash_rows": (_i, [_vp, _i64, _i, _u64, _f, _f, _i64, _i64, _vp]),
    "mm_positive_scores": (_i, [_vp, _vp, _i64, _i, _vp, _f, _vp, _i64, _vp]),
    "mm_inbatch_scores_tc": (_i, [_vp, _vp, _i64, _i64, _i, _vp, _vp, _i, _i, _f, _vp, _f, _vp, _i64, _vp]),
    "mm_inbatch_scores": (_i, [_vp, _vp, _vp, _i64, _i64, _i, _vp, _vp, _i, _i, _f, _vp, _vp, _f,
                               _vp, _i64, _vp]),
    "mm_fm_pairwise": (_i, [_vp, _i64, _i, _i, _vp, _vp]),
    "mm_deepfm_head": (_i, [C.POINTER(LookupTable), C.POINTER(C.c_int64), _i, _i64, _i, C.POINTER(ConcatPiece), C.POINTER(C.c_int64), _i,
                            _vp, _vp, _vp, _i64, _vp, _vp, _i, _vp, _vp, _vp]),
    "mm_heads_fwd_bwd": (_i, [_vp, _i64, _i, _i64, _i, _vp, _vp, C.POINTER(C.c_int), C.POINTER(C.c_float), C.POINTER(C.c_void_p),
                              C.POINTER(C.c_int), C.POINTER(C.c_void_p), _vp, _vp, _vp, _i64, _i, _vp, _vp, _vp]),
    "mm_dense_wgrad": (_i, [_vp, _i64, _i, _i64, _vp, _i, _i64, _vp, _vp, _vp]),
    "mm_dense_wgrad_split": (_i, [_vp, _i64, _i, _i, _vp, _i, _i64, _vp, _vp, _vp]),
    "mm_dense_dgrad": (_i, [_vp, _i64, _i, _i64, _vp, _i, _vp, _i64, _vp, _i64, _vp]),
    "mm_relu_mask": (_i, [_vp, _i64, _i, _i64, _vp, _i64, _vp]),
    "mm_dlrm_interact_backward": (_i, [C.POINTER(LookupTable), _i, _i64, _i, _vp, _i64, _i, _i, _vp, _i64,
                                       C.POINTER(C.c_void_p), _i64, _vp, _i64, _i, _i, _vp]),
    "mm_sparse_rows_apply": (_i, [C.POINTER(SparseTable), _i, _i64, _i, _i, _vp, _vp]),
    "mm_bag_grad_rows": (_i, [_vp, _i64, _i, _i64, _vp, _i, _vp, _i, _i, _i64, _i64, _i, _vp, _vp, _vp]),
    "mm_dense_apply": (_i, [_i, _vp, _vp, _vp, _vp, _i64, _vp, _f, _vp]),
    "mm_opt_tick": (_i, [_vp, _vp]),
    "mm_opt_tick_schedule": (_i, [_vp, _vp, _vp]),
    "mm_fill_i32": (_i, [_vp, _i64, C.c_int32, _vp]),
    "mm_cross_backward": (_i, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _i, _i64, _i, _vp, _i64, _vp, _i, _vp]),
    "mm_concat_backward": (_i, [C.POINTER(C.c_void_p), C.POINTER(C.c_int64), _i, _i64, _i, C.POINTER(ColumnSlice), _i, _vp]),
    "mm_concat_backward_l2": (_i, [C.POINTER(C.c_void_p), C.POINTER(C.c_int64), _i, _i64, _i, C.POINTER(ColumnSlice), _i, _vp, _i64,
                                   C.POINTER(C.c_float), _vp, _i64, _vp, _vp]),
    "mm_inbatch_softmax_ce_backward": (_i, [_vp, _vp, _i64, _i64, _i, _vp, _vp, _i, _i, _f, _vp, _f, _vp, _vp, _vp, _vp, _i,
                                            _vp, _vp, _vp, _vp, _vp]),
    "mm_catalog_softmax_ce_workspace_bytes": (_i64, [_i64, _i64, _i]),
    "mm_catalog_softmax_ce_backward": (_i, [_vp, _vp, _i64, _i64, _i, _vp, _vp, _i, _f, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp,
                                            _i64, _vp]),
    "mm_catalog_smoothed_ce_workspace_bytes": (_i64, [_i64, _i64, _i]),
    "mm_catalog_smoothed_ce_backward": (_i, [_vp, _vp, _i64, _i64, _i, _vp, _vp, _i, _f, _f, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp,
                                             _vp, _i64, _vp]),
    "mm_catalog_mean_logit_workspace_bytes": (_i64, [_i64]),
    "mm_catalog_mean_logit": (_i, [_vp, _vp, _i64, _i64, _i, _vp, _vp, _vp, _i64, _vp]),
    "mm_slices_add_dense_workspace_bytes": (_i64, [_i64]),
    "mm_slices_add_dense": (_i, [_vp, _i, _vp, _i64, _i, _vp, _i64, _vp, _i64, _vp]),
    "mm_l2_normalize_backward": (_i, [_vp, _vp, _i64, _i, _i64, _i64, _vp, _i64, _vp]),
    "mm_deepfm_head_fwd_bwd": (_i, [_vp, _i64, C.POINTER(C.c_int64), _i, C.POINTER(WideBlock), _i, C.POINTER(ConcatPiece),
                                    C.POINTER(C.c_int64), _i, _vp, _vp, _vp, _i64, _i, _i, _vp, _vp, _i, _vp, _vp, _i, _vp, _i, _vp,
                                    _i64, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "mm_fm_concat_backward": (_i, [C.POINTER(C.c_void_p), C.POINTER(C.c_int64), _i, _i64, _i, _vp, _i64, _vp, C.POINTER(ColumnSlice),
                                   _i, _vp]),
    "mm_wide_rows_apply": (_i, [_vp, _vp, _vp, _i64, C.POINTER(WideBlock), _i, _i64, _vp, _vp, _vp, C.POINTER(C.c_int64), _i, _vp,
                                _vp, _vp, _vp, _i, _vp, _vp]),
    "mm_metrics_workspace_bytes": (_i64, [_i64, _i]),
    "mm_wide_deep_head_fwd_bwd": (_i, [C.POINTER(WideBlock), _i, C.POINTER(WideBag), _i, _vp, _vp, _vp, _i64, _i, _i, _vp, _vp, _i, _vp,
                                       _vp, _i, _i, _vp, _i, _vp, _i64, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "mm_wide_bag_grad": (_i, [C.POINTER(WideBag), _i64, _vp, _vp, _vp, _vp]),
    "mm_metrics_update": (_i, [_vp, _i64, _i, C.POINTER(MetricsHead), _i, _i, _vp, _vp, _i64, _vp]),
    "mm_mmoe_heads_fwd_bwd": (_i, [_vp, _i64, _i, _i, _i64, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), _i, _f, _vp, _vp,
                                   C.POINTER(C.c_int), C.POINTER(C.c_float), C.POINTER(C.c_void_p), C.POINTER(C.c_int),
                                   C.POINTER(C.c_void_p), _vp, _vp, _vp, _i64, _i, C.POINTER(C.c_void_p), C.POINTER(C.c_int64),
                                   _vp, _vp, _vp]),
    "mm_mmoe_mix_fwd": (_i, [_vp, _i64, _i, _i, _i64, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), _i, _f, _vp, _vp, _vp, _i, _vp]),
    "mm_mmoe_mix_bwd": (_i, [_vp, _i64, _i, _i, _i64, _vp, _i, _f, _vp, _vp, _i64, _i, C.POINTER(C.c_void_p), C.POINTER(C.c_int64),
                             _vp]),
    "mm_mmoe_task_heads_fwd_bwd": (_i, [C.POINTER(C.c_void_p), C.POINTER(C.c_int64), _i64, _i, _i, _vp, _vp, C.POINTER(C.c_int),
                                        C.POINTER(C.c_float), C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.POINTER(C.c_void_p),
                                        _vp, _vp, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), _i, _vp, _vp, _vp]),
    "mm_inbatch_pairwise_fwd": (_i, [_vp, _vp, _i64, _i64, _i, _vp, _vp, _i, _i, _f, _f, _i, _f, _vp, _vp, _vp, _vp]),
    "mm_inbatch_pairwise_bwd": (_i, [_vp, _vp, _i64, _i64, _i, _vp, _vp, _i, _i, _f, _f, _i, _f, _vp, _vp, _vp, _vp, _vp, _vp,
                                     _vp, _vp]),
    "mm_ncf_head_fwd_bwd": (_i, [_vp, _i64, _vp, _i, _vp, _i64, _vp, _i, _i, _vp, _i64, _i, _i, _i64, _i, _vp, _vp, C.POINTER(C.c_int),
                                 C.POINTER(C.c_float), C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.POINTER(C.c_void_p), _f, _vp,
                                 _i64, _i, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp]),
    "mm_pretrained_gather": (_i, [_vp, _i64, _i, _i64, _vp, _i, _i64, _vp, _i64, _vp, _vp]),
    "mm_pretrained_project": (_i, [_vp, _i64, _i, _i64, _vp, _i, _i64, _vp, _vp, _i, _vp, _i64, _vp, _vp]),
    "mm_pretrained_backward_workspace_bytes": (_i64, [_i64, _i, _i]),
    "mm_pretrained_project_backward": (_i, [_vp, _i64, _i, _i64, _vp, _i, _i64, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), _i,
                                            _vp, _i64, _i, _vp, _vp, _vp, _i64, _vp]),
}


def declared_symbols() -> list[str]:
    """Function names declared in include/mm_b200.h (parsed from the header text)."""
    text = HEADER_PATH.read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(mm_[a-z0-9_]+)\s*\(", text)))


_lib = None


def load() -> C.CDLL:
    """Load the shared library and bind every entry point; raise loudly if anything is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -m models_b200.csrc.build` "
            "(or __graft_entry__.build()). There is no CPU/PyTorch fallback for this path."
        )
    lib = C.CDLL(os.fspath(LIB_PATH))
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:  # pragma: no cover - only on a broken build
            raise RuntimeError(f"libmm_b200.so does not export {name}") from e
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error() -> str:
    return load().mm_last_error().decode("utf-8", "replace")


def check(rc: int, what: str) -> None:
    if rc == 0:
        return
    msg = last_error()
    if rc < 0:
        raise ValueError(f"{what}: {msg} (code {rc})")
    raise RuntimeError(f"{what}: {msg} (cudaError {rc})")
