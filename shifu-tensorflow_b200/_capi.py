"""ctypes binding of include/shifu_b200.h (the C-ABI a JNI shim binds the same way, INTEGRATION.md).

No compute lives here: every call forwards to libshifu_b200.so.  If the library has not been built the
import fails loudly - there is no Python / CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import logging
import os
from typing import Optional, Sequence

import numpy as np

# A step runs on up to five streams (main, side, two exchange streams, descriptor prefetch); with the default of 8 hardware
# queues CUDA maps several of them onto one queue and their kernels falsely serialise (an exchange kernel that waits for
# its peers then holds back an unrelated GEMM).  Read by the driver when the context is created, i.e. at the first CUDA call.
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libshifu_b200.so")

SB_MAX_HIDDEN = 32
SB_NCCL_ID_BYTES = 128
ACT_SIGMOID, ACT_TANH, ACT_RELU, ACT_LEAKYRELU, ACT_NONE = 0, 1, 2, 3, -1
LOSS_MSE, LOSS_SIGMOID_CE = 0, 1
OPT_ADADELTA, OPT_ADAM, OPT_SGD, OPT_MOMENTUM, OPT_ADAGRAD, OPT_RMSPROP, OPT_FTRL = 0, 1, 2, 3, 4, 5, 6
OPT_RPROP = 8                   # iRPROP-: learning_rate is the start step size (7 is not an optimizer)
# TF 1.x defaults of the hyperparameters make_desc fills in when the caller passes none: RMSPropOptimizer's (decay,
# epsilon, momentum) differ from the values every other optimizer gets
_RMSPROP_DEFAULTS = dict(rho=0.9, epsilon=1e-10, momentum=0.0)
_OTHER_DEFAULTS = dict(rho=0.95, epsilon=1e-8, momentum=0.9)
INITIAL_ACCUMULATOR, L1, L2 = 0.1, 0.0, 0.0     # Adagrad / FTRL (Trainer(initial_accumulator=, l1=, l2=))
PREC_FP32, PREC_BF16, PREC_FP32_TC, PREC_BF16X2 = 0, 1, 2, 3
SB_REASON_RAISE, SB_REASON_LOWER, SB_REASON_MAGNITUDE = 0, 1, 2
REASON_ORDERS = {"raise": SB_REASON_RAISE, "lower": SB_REASON_LOWER, "magnitude": SB_REASON_MAGNITUDE}
SB_OK, SB_ERR_INVALID, SB_ERR_CUDA, SB_ERR_NCCL, SB_ERR_IO, SB_ERR_STATE, SB_ERR_FORMAT = 0, -1, -2, -3, -4, -5, -6


class NetDesc(C.Structure):
    _fields_ = [
        ("n_features", C.c_int32), ("n_hidden", C.c_int32),
        ("hidden", C.c_int32 * SB_MAX_HIDDEN), ("acts", C.c_int32 * SB_MAX_HIDDEN),
        ("loss", C.c_int32), ("optimizer", C.c_int32),
        ("learning_rate", C.c_float), ("rho", C.c_float), ("epsilon", C.c_float),
        ("beta1", C.c_float), ("beta2", C.c_float), ("momentum", C.c_float),
        ("max_batch", C.c_int32), ("precision", C.c_int32),
    ]


def make_desc(n_features: int, hidden: Sequence[int], acts: Sequence[int], loss: int = LOSS_MSE,
              optimizer: int = OPT_ADADELTA, learning_rate: float = 0.001, rho: Optional[float] = None,
              epsilon: Optional[float] = None, beta1: float = 0.9, beta2: float = 0.999, momentum: Optional[float] = None,
              max_batch: int = 128, precision: int = PREC_FP32) -> NetDesc:
    """rho / epsilon / momentum left at None take the TF 1.x default of `optimizer`: RMSProp decay 0.9, epsilon 1e-10,
    momentum 0.0; every other optimizer rho 0.95, epsilon 1e-8, momentum 0.9."""
    dflt = _RMSPROP_DEFAULTS if optimizer == OPT_RMSPROP else _OTHER_DEFAULTS
    rho = dflt["rho"] if rho is None else rho
    epsilon = dflt["epsilon"] if epsilon is None else epsilon
    momentum = dflt["momentum"] if momentum is None else momentum
    if len(hidden) != len(acts):
        raise ValueError("hidden and acts must have the same length")
    if len(hidden) > SB_MAX_HIDDEN:
        raise ValueError("at most %d hidden layers" % SB_MAX_HIDDEN)
    d = NetDesc()
    d.n_features, d.n_hidden = int(n_features), len(hidden)
    for i, (h, a) in enumerate(zip(hidden, acts)):
        d.hidden[i], d.acts[i] = int(h), int(a)
    d.loss, d.optimizer = int(loss), int(optimizer)
    d.learning_rate, d.rho, d.epsilon = learning_rate, rho, epsilon
    d.beta1, d.beta2, d.momentum = beta1, beta2, momentum
    d.max_batch, d.precision = int(max_batch), int(precision)
    return d


class CellFlag(C.Structure):
    _fields_ = [("row", C.c_int64), ("slot", C.c_int32), ("len", C.c_int32), ("offset", C.c_int64)]


COL_SKIP, COL_TARGET, COL_WEIGHT = -1, -2, -3


class PerfSummary(C.Structure):
    _fields_ = [("rows", C.c_int64), ("pos", C.c_int64), ("neg", C.c_int64), ("n_distinct", C.c_int64),
                ("w_pos", C.c_double), ("w_neg", C.c_double), ("auc", C.c_double), ("w_auc", C.c_double),
                ("ap", C.c_double), ("w_ap", C.c_double), ("ks", C.c_double), ("w_ks", C.c_double),
                ("ks_score", C.c_float), ("w_ks_score", C.c_float)]


class PerfPoint(C.Structure):
    _fields_ = [("threshold", C.c_float), ("tp", C.c_int64), ("fp", C.c_int64), ("w_tp", C.c_double), ("w_fp", C.c_double)]


class ShifuB200Error(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__("[%d] %s" % (code, msg))
        self.code = code


_lib = None

# name -> (restype, argtypes); the single source of truth for tests/test_capi_symbols.py
_P = C.POINTER
_f32p, _f64p, _vp, _cp = _P(C.c_float), _P(C.c_double), C.c_void_p, C.c_char_p
PROTOTYPES = {
    "sb_version": (C.c_char_p, []),
    "sb_last_error": (C.c_char_p, []),
    "sb_device_count": (C.c_int, []),
    "sb_device_mem_info": (C.c_int, [C.c_int, _P(C.c_uint64), _P(C.c_uint64)]),
    "sb_host_alloc": (C.c_int, [_P(_vp), C.c_uint64]),
    "sb_host_free": (C.c_int, [_vp]),
    "sb_nccl_unique_id": (C.c_int, [_vp]),
    "sb_trainer_create": (C.c_int, [_P(NetDesc), C.c_int, _vp, C.c_int, C.c_int, _P(_vp)]),
    "sb_trainer_destroy": (C.c_int, [_vp]),
    "sb_trainer_ipc_handle": (C.c_int, [_vp, _vp]),
    "sb_trainer_set_peer_handles": (C.c_int, [_vp, _vp, C.c_int32]),
    "sb_trainer_clear_peer_handles": (C.c_int, [_vp]),
    "sb_trainer_exchange_base": (C.c_void_p, [_vp]),
    "sb_trainer_set_peer_pointers": (C.c_int, [_vp, _P(_vp), C.c_int32]),
    "sb_trainer_param_count": (C.c_int64, [_vp]),
    "sb_trainer_set_params": (C.c_int, [_vp, _f32p, C.c_int64]),
    "sb_trainer_get_params": (C.c_int, [_vp, _f32p, C.c_int64]),
    "sb_trainer_init_xavier": (C.c_int, [_vp, C.c_uint64]),
    "sb_trainer_get_grads": (C.c_int, [_vp, _f32p, C.c_int64]),
    "sb_trainer_step": (C.c_int, [_vp, _f32p, _f32p, _f32p, C.c_int32, _f32p]),
    "sb_trainer_set_sparse": (C.c_int, [_vp, C.c_int32, C.c_int32, C.c_int32]),
    "sb_trainer_set_deterministic": (C.c_int, [_vp, C.c_int32]),
    "sb_trainer_set_optimizer_params": (C.c_int, [_vp, C.c_float, C.c_float, C.c_float]),
    "sb_trainer_set_fixed_layers": (C.c_int, [_vp, _P(C.c_int32), C.c_int32, C.c_int32]),
    "sb_trainer_step_sparse": (C.c_int, [_vp, _f32p, _P(C.c_int32), _f32p, _f32p, C.c_int32, _f32p]),
    "sb_trainer_predict_sparse": (C.c_int, [_vp, _f32p, _P(C.c_int32), C.c_int64, _f32p]),
    "sb_trainer_eval_loss_sparse": (C.c_int, [_vp, _f32p, _P(C.c_int32), _f32p, _f32p, C.c_int64, _f32p]),
    "sb_trainer_step_async": (C.c_int, [_vp, _f32p, _f32p, _f32p, C.c_int32]),
    "sb_trainer_accumulate": (C.c_int, [_vp, _f32p, _f32p, _f32p, C.c_int32, _f32p]),
    "sb_trainer_apply_accumulated": (C.c_int, [_vp]),
    "sb_trainer_apply_accumulated_mean": (C.c_int, [_vp, C.c_int64]),
    "sb_trainer_loss_resident": (C.c_int, [_vp, C.c_int64, C.c_int32, _f32p]),
    "sb_trainer_broadcast_state": (C.c_int, [_vp, C.c_int32]),
    "sb_trainer_load_dataset": (C.c_int, [_vp, _f32p, _f32p, _f32p, C.c_int64]),
    "sb_trainer_dataset_on_host": (C.c_int, [_vp]),
    "sb_trainer_step_resident": (C.c_int, [_vp, C.c_int64, C.c_int32, _f32p]),
    "sb_trainer_step_resident_async": (C.c_int, [_vp, C.c_int64, C.c_int32]),
    "sb_trainer_run_resident": (C.c_int, [_vp, C.POINTER(C.c_int64), C.c_int32, C.c_int32]),
    "sb_trainer_accumulate_resident": (C.c_int, [_vp, C.c_int64, C.c_int32, _f32p]),
    "sb_trainer_set_row_order": (C.c_int, [_vp, C.POINTER(C.c_int64), C.c_int64]),
    "sb_trainer_last_loss": (C.c_int, [_vp, _f32p]),
    "sb_trainer_loss_history": (C.c_int, [_vp, C.c_int64, C.c_int32, _f32p]),
    "sb_trainer_sync": (C.c_int, [_vp]),
    "sb_trainer_stream": (C.c_void_p, [_vp]),
    "sb_trainer_kernels_per_step": (C.c_int, [_vp, C.c_int32]),
    "sb_trainer_eval_loss": (C.c_int, [_vp, _f32p, _f32p, _f32p, C.c_int64, _f32p]),
    "sb_trainer_predict": (C.c_int, [_vp, _f32p, C.c_int64, _f32p]),
    "sb_trainer_save_checkpoint": (C.c_int, [_vp, _cp]),
    "sb_trainer_load_checkpoint": (C.c_int, [_vp, _cp]),
    "sb_trainer_global_step": (C.c_int64, [_vp]),
    "sb_trainer_export_savedmodel": (C.c_int, [_vp, _cp]),
    "sb_model_load": (C.c_int, [_cp, _cp, _cp, _cp, C.c_int, C.c_int, _P(_vp)]),
    "sb_model_create": (C.c_int, [_P(NetDesc), _f32p, C.c_int64, C.c_int, _P(_vp)]),
    "sb_model_destroy": (C.c_int, [_vp]),
    "sb_model_n_features": (C.c_int32, [_vp]),
    "sb_model_n_layers": (C.c_int32, [_vp]),
    "sb_model_score": (C.c_int, [_vp, _f32p, C.c_int64, _f32p]),
    "sb_model_score_row_f64": (C.c_int, [_vp, _f64p, C.c_int32, _f64p]),
    "sb_model_score_device": (C.c_int, [_vp, _vp, C.c_int64, _vp]),
    "sb_model_sensitivity": (C.c_int, [_vp, _vp, _vp, C.c_int64, _P(C.c_int32), C.c_int32, _f32p, _f64p, _f64p, _f64p, _vp]),
    "sb_model_reason_codes": (C.c_int, [_vp, _vp, C.c_int64, _P(C.c_int32), C.c_int32, _f32p, C.c_int32, C.c_int32, _vp, _vp,
                                        _vp]),
    "sb_model_sync": (C.c_int, [_vp]),
    "sb_model_stream": (C.c_void_p, [_vp]),
    "sb_debug_model_batch_stats": (C.c_int, [_vp, _P(C.c_int64), C.c_int32]),
    "sb_debug_model_hold": (C.c_int, [_vp, C.c_int32, C.c_int32]),
    "sb_debug_model_routes": (C.c_int, [_vp, C.c_char_p, C.c_int32]),
    "sb_debug_model_bytes": (C.c_int, [_vp, _P(C.c_int64)]),
    "sb_ensemble_load": (C.c_int, [_P(_cp), C.c_int32, _cp, _cp, _cp, C.c_int, C.c_int, _P(_vp)]),
    "sb_ensemble_create": (C.c_int, [_P(NetDesc), _P(_f32p), _P(C.c_int64), C.c_int32, C.c_int, _P(_vp)]),
    "sb_ensemble_destroy": (C.c_int, [_vp]),
    "sb_ensemble_size": (C.c_int32, [_vp]),
    "sb_ensemble_score": (C.c_int, [_vp, _vp, C.c_int64, _vp, _vp]),
    "sb_ensemble_score_device": (C.c_int, [_vp, _vp, C.c_int64, _vp, _vp]),
    "sb_ensemble_score_row_f64": (C.c_int, [_vp, _f64p, C.c_int32, _f64p]),
    "sb_ensemble_sync": (C.c_int, [_vp]),
    "sb_ensemble_stream": (C.c_void_p, [_vp]),
    "sb_debug_ensemble_routes": (C.c_int, [_vp, C.c_char_p, C.c_int32]),
    "sb_debug_ensemble_bytes": (C.c_int, [_vp, _P(C.c_int64)]),
    "sb_ensemble_sensitivity": (C.c_int, [_vp, C.c_int32, _vp, _vp, C.c_int64, _P(C.c_int32), C.c_int32, _f32p, _f64p, _f64p, _f64p,
                                          _vp]),
    "sb_ensemble_reason_codes": (C.c_int, [_vp, C.c_int32, _vp, C.c_int64, _P(C.c_int32), C.c_int32, _f32p, C.c_int32, C.c_int32,
                                           _vp, _vp, _vp]),
    "sb_perf_create": (C.c_int, [C.c_int, C.c_int64, _P(_vp)]),
    "sb_perf_destroy": (C.c_int, [_vp]),
    "sb_perf_reset": (C.c_int, [_vp]),
    "sb_perf_add": (C.c_int, [_vp, _vp, C.c_int32, _vp, _vp, C.c_int64, _vp]),
    "sb_perf_summary_get": (C.c_int, [_vp, _P(PerfSummary)]),
    "sb_perf_points": (C.c_int, [_vp, C.c_int32, C.c_int32, _f64p, C.c_int32, _P(PerfPoint)]),
    "sb_perf_sync": (C.c_int, [_vp]),
    "sb_perf_stream": (C.c_void_p, [_vp]),
    "sb_debug_perf_runs": (C.c_int, [_vp, _f32p, _P(C.c_int64), _P(C.c_int64), _f64p, _f64p, C.c_int64, _P(C.c_int64)]),
    "sb_debug_perf_bytes": (C.c_int, [_vp, _P(C.c_int64)]),
    "sb_text_parse": (C.c_int, [_cp, C.c_int64, C.c_char, _P(C.c_int32), C.c_int32, C.c_int32, _f32p, _f32p, _f32p, C.c_int64,
                                _P(C.c_int64), _P(CellFlag), C.c_int64, _P(C.c_int64), C.c_int]),
    "sb_text_parse_device": (C.c_int, [_cp, C.c_int64, C.c_char, _P(C.c_int32), C.c_int32, C.c_int32, _P(_f32p), _P(_f32p), _P(_f32p),
                                       _P(C.c_int64), _P(CellFlag), C.c_int64, _P(C.c_int64), C.c_int, _f32p]),
    "sb_device_alloc_f32": (C.c_int, [_P(_f32p), C.c_int64, C.c_int]),
    "sb_device_free": (C.c_int, [_vp]),
    "sb_device_patch_f32": (C.c_int, [_f32p, C.c_int64, C.c_float]),
    "sb_device_read_f32": (C.c_int, [_f32p, C.c_int64, _f32p]),
    "sb_device_gather_rows": (C.c_int, [_f32p, C.c_int32, _P(C.c_int64), C.c_int64, _f32p, C.c_int]),
    "sb_debug_text_parse_host": (C.c_int, [_cp, C.c_int64, C.c_char, _P(C.c_int32), C.c_int32, C.c_int32, _f32p, _f32p, _f32p,
                                           C.c_int64, _P(C.c_int64), _P(CellFlag), C.c_int64, _P(C.c_int64)]),
    "sb_savedmodel_write": (C.c_int, [_cp, _P(NetDesc), _f32p, C.c_int64]),
    "sb_savedmodel_read": (C.c_int, [_cp, _cp, _cp, _cp, _P(NetDesc), _P(C.c_int32), _f32p, C.c_int64, _P(C.c_int64)]),
    "sb_debug_gemm_layer": (C.c_int, [C.c_int32, C.c_int32, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _P(C.c_int32),
                                      C.c_char_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_int32, C.c_int32, C.c_int32, C.c_int64, C.c_int]),
    "sb_debug_step_trace": (C.c_int, [_vp, C.POINTER(C.c_uint64), C.c_int32, C.c_char_p, C.c_int32, C.POINTER(C.c_int32)]),
    "sb_debug_gemm_bench": (C.c_int, [_f32p, _f32p, _f32p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_int32, C.c_int32, C.c_int, C.c_int32, _f32p]),
    "sb_debug_gemm_bf16_cfg": (C.c_int, [_f32p, _f32p, _f32p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                         C.c_int32, C.c_int32, C.c_int]),
    "sb_debug_gemm_epilogue": (C.c_int, [_f32p, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                         C.c_int32, C.c_int32, C.c_int, C.c_int32, _f32p]),
    "sb_debug_gemm_fwd_out": (C.c_int, [_f32p, _f32p, _f32p, _f32p, C.c_float, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p,
                                        _P(C.c_int32), C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                        C.c_int32, C.c_int32, C.c_int32, C.c_int]),
    "sb_debug_out_layer": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, _f32p, _f32p, C.c_float, _f32p, _f32p, _f32p,
                                     _f32p, _f32p, _f32p, _f32p, _f32p, _P(C.c_int32), _P(C.c_int32), C.c_char_p, C.c_int32,
                                     C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int]),
    "sb_debug_embed": (C.c_int, [C.c_int32, C.c_int32, _f32p, _P(C.c_int32), _f32p, _f32p, _P(C.c_int32), C.c_int32, C.c_int32,
                                 C.c_int32, C.c_int32, C.c_int]),
    "sb_debug_trainer_buffer": (C.c_int, [_vp, C.c_int32, _vp, C.c_int64, C.c_int32]),
    "sb_debug_first_kernel": (C.c_int, [_vp, _f32p, _f32p, _f32p, _P(C.c_int32), C.c_int64, C.c_int32, C.c_int32, C.c_char_p,
                                        C.c_int32]),
    "sb_debug_force_host_set": (C.c_int, [_vp, C.c_int32]),
    "sb_debug_exchange": (C.c_int, [_vp, C.c_int32, C.c_float, C.c_int32, C.c_int32, _f32p, _P(C.c_int32), C.c_char_p,
                                    C.c_int32]),
    "sb_debug_exchange_layout": (C.c_int, [_vp, _P(C.c_int32), C.c_int32, _P(C.c_int64), C.c_int64, _P(C.c_int32)]),
    "sb_debug_optimizer": (C.c_int, [_vp, C.c_float, C.c_int32, _f32p, C.c_char_p, C.c_int32]),
}

DEBUG_BUF_THETA, DEBUG_BUF_S1, DEBUG_BUF_S2, DEBUG_BUF_GRAD, DEBUG_BUF_SHADOW = 0, 1, 2, 3, 4
# the step's input stage (sb_debug_first_kernel): batch operand, its y / w, slot (0, 0)'s scalars; the resident set (read-only)
DEBUG_BUF_BATCH_X = DEBUG_BUF_SHADOW + SB_MAX_HIDDEN
DEBUG_BUF_BATCH_Y, DEBUG_BUF_BATCH_W, DEBUG_BUF_SCAL = DEBUG_BUF_BATCH_X + 1, DEBUG_BUF_BATCH_X + 2, DEBUG_BUF_BATCH_X + 3
DEBUG_BUF_DS_X, DEBUG_BUF_DS_Y, DEBUG_BUF_DS_W, DEBUG_BUF_DS_P = (DEBUG_BUF_BATCH_X + 4, DEBUG_BUF_BATCH_X + 5, DEBUG_BUF_BATCH_X + 6,
                                                                  DEBUG_BUF_BATCH_X + 7)
SCAL_LOSS_SUM, SCAL_NNZ, SCAL_COUNT = 0, 1, 4
DEBUG_XINFO_WORDS, DEBUG_XWORK_WORDS = 24, 8
DEBUG_MSTAT_WORDS = 6
ENSEMBLE_MAX = 32       # SB_ENSEMBLE_MAX: members of one ensemble
ENSEMBLE_STATS = ("mean", "max", "min", "median")     # sb_ensemble_score's stats columns
PERF_ACTION_RATE, PERF_RECALL, PERF_FPR, PERF_SCORE = 0, 1, 2, 3
PERF_AXES = {"action_rate": PERF_ACTION_RATE, "recall": PERF_RECALL, "fpr": PERF_FPR, "score": PERF_SCORE}
PERF_MAX_ROWS = 2**31 - 1     # rows one performance handle holds
SMALL_ROWS = 128        # score_rows.cuh: an fp32 model scores batches of up to this many rows in one launch
# score.cu model_chunk_rows: a model runs every scoring call in forwards of at most this many rows (its max_batch)
MODEL_CHUNK_ROWS = {PREC_FP32: 16384, PREC_BF16: 65536, PREC_FP32_TC: 32768, PREC_BF16X2: 32768}


def lib():
    """Load libshifu_b200.so (once).  Raises ImportError when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "libshifu_b200.so is missing (%s). Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "or `python shifu-tensorflow_b200/build.py`. There is no CPU fallback." % LIB_PATH)
    L = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    _lib = L
    return L


def check(status: int) -> None:
    if status != SB_OK:
        raise ShifuB200Error(status, lib().sb_last_error().decode("utf-8", "replace"))


def _f32(a, shape=None) -> np.ndarray:
    a = np.ascontiguousarray(a, dtype=np.float32)
    if shape is not None and a.shape != shape:
        a = a.reshape(shape)
    return a


def _ptr(a):
    if a is None:
        return None
    if hasattr(a, "ptr") and not isinstance(a, np.ndarray):      # DeviceArray
        return a.ptr
    return a.ctypes.data_as(_f32p)


def _in_ptr(a, dtype=np.float32):
    """-> (void pointer, shape) of a numpy array (host), a DeviceArray or a CUDA tensor (device); numpy arrays must be
    C-contiguous `dtype` (fp32 by default), anything else is converted to one"""
    name = np.dtype(dtype).name
    if isinstance(a, DeviceArray):
        return C.c_void_p(C.cast(a.ptr, _vp).value), a.shape
    if hasattr(a, "data_ptr") and getattr(a, "is_cuda", False):
        if not a.is_contiguous() or str(a.dtype) != "torch." + name:
            raise ValueError("a device tensor must be contiguous " + name)
        return C.c_void_p(a.data_ptr()), tuple(a.shape)
    if hasattr(a, "numpy") and not isinstance(a, np.ndarray):
        a = a.numpy()
    if not (isinstance(a, np.ndarray) and a.dtype == dtype and a.flags.c_contiguous):
        raise ValueError("a host array must be C-contiguous %s (it is read in place)" % name)
    return a.ctypes.data_as(_vp), a.shape


class DeviceArray:
    """fp32 array that lives in GPU memory (library-owned; what sb_text_parse_device returns).  Accepted by
    Trainer.load_dataset / eval_loss / predict in place of a numpy array."""

    def __init__(self, ptr, shape, device: int = 0, owner: bool = True):
        self.ptr, self.shape, self.device, self._own = ptr, tuple(shape), device, owner

    @classmethod
    def empty(cls, shape, device: int = 0) -> "DeviceArray":
        p = _f32p()
        n = int(np.prod(shape))
        check(lib().sb_device_alloc_f32(C.byref(p), max(n, 1), device))
        return cls(p, shape, device)

    def __len__(self):
        return self.shape[0]

    @property
    def size(self) -> int:
        return int(np.prod(self.shape))

    def numpy(self) -> np.ndarray:
        out = np.empty(self.shape, np.float32)
        if self.size:
            check(lib().sb_device_read_f32(self.ptr, self.size, _ptr(out)))
        return out

    def patch(self, flat_index: int, value: float):
        check(lib().sb_device_patch_f32(self.ptr, int(flat_index), float(value)))

    def take_rows(self, rows) -> "DeviceArray":
        """rows (host int64 indices) gathered on the device into a new DeviceArray"""
        rows = np.ascontiguousarray(rows, dtype=np.int64)
        n_cols = int(np.prod(self.shape[1:])) if len(self.shape) > 1 else 1
        out = DeviceArray.empty((len(rows),) + self.shape[1:], self.device)
        check(lib().sb_device_gather_rows(self.ptr, n_cols, rows.ctypes.data_as(_P(C.c_int64)), len(rows), out.ptr, self.device))
        return out

    def free(self):
        if self._own and self.ptr:
            lib().sb_device_free(C.cast(self.ptr, _vp))
        self.ptr = None

    __del__ = free


class Trainer:
    """Owns one sb_trainer_t.  X is [rows, n_features] float32, y / w are [rows] (or [rows,1])."""

    def __init__(self, desc: NetDesc, device: int = 0, nccl_id: Optional[bytes] = None, rank: int = 0, world: int = 1,
                 deterministic: bool = False, initial_accumulator: Optional[float] = None, l1: Optional[float] = None,
                 l2: Optional[float] = None, fixed_layers: Sequence[int] = (), fixed_bias: bool = True):
        """initial_accumulator / l1 / l2 (Adagrad, FTRL; None = TF's default): see set_optimizer_params;
        fixed_layers / fixed_bias: see set_fixed_layers"""
        self._h = C.c_void_p()
        self.desc = desc
        idbuf = None
        if nccl_id is not None:
            if len(nccl_id) != SB_NCCL_ID_BYTES:
                raise ValueError("nccl_id must be %d bytes" % SB_NCCL_ID_BYTES)
            idbuf = C.create_string_buffer(bytes(nccl_id), SB_NCCL_ID_BYTES)
        check(lib().sb_trainer_create(C.byref(desc), device, C.cast(idbuf, _vp) if idbuf is not None else None,
                                      rank, world, C.byref(self._h)))
        self.n_params = int(lib().sb_trainer_param_count(self._h))
        self.n_features = int(desc.n_features)
        if deterministic:
            self.set_deterministic(True)
        if (initial_accumulator, l1, l2) != (None, None, None):
            self.set_optimizer_params(INITIAL_ACCUMULATOR if initial_accumulator is None else initial_accumulator,
                                      L1 if l1 is None else l1, L2 if l2 is None else l2)
        if len(fixed_layers) > 0:
            self.set_fixed_layers(fixed_layers, fixed_bias)

    def set_fixed_layers(self, layers: Sequence[int], fix_bias: bool = True):
        """Fine-tuning: never change the weights of these layers, nor their biases when fix_bias (Shifu's FixedLayers /
        FixedBias; sb_trainer_set_fixed_layers).  Layers are numbered from 1: hidden layers 1..n_hidden, the output layer
        n_hidden + 1.  Their values, optimizer state and bf16 shadows keep their bits, get_grads reports 0 for them, and a
        step skips the GEMMs only they need.  Before the first step and before the peer exchange is set up, on every rank."""
        arr = np.ascontiguousarray([int(x) for x in layers], dtype=np.int32)
        ptr = arr.ctypes.data_as(_P(C.c_int32)) if arr.size else None
        check(lib().sb_trainer_set_fixed_layers(self._h, ptr, int(arr.size), 1 if fix_bias else 0))

    def set_deterministic(self, on: bool = True):
        """fixed-order reductions in every training kernel (sb_trainer_set_deterministic); before the first step"""
        check(lib().sb_trainer_set_deterministic(self._h, 1 if on else 0))

    def set_optimizer_params(self, initial_accumulator: float = INITIAL_ACCUMULATOR, l1: float = L1, l2: float = L2):
        """Adagrad / FTRL: accum's start value (> 0) and FTRL's l1 / l2 strengths (>= 0) (sb_trainer_set_optimizer_params);
        before the first step"""
        check(lib().sb_trainer_set_optimizer_params(self._h, float(initial_accumulator), float(l1), float(l2)))

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            lib().sb_trainer_destroy(self._h)
            self._h = None

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    # ---- peer-memory gradient exchange (CUDA IPC) ----
    def ipc_handle(self) -> bytes:
        buf = C.create_string_buffer(64)
        check(lib().sb_trainer_ipc_handle(self._h, C.cast(buf, _vp)))
        return buf.raw

    def set_peer_handles(self, handles: Sequence[bytes]):
        blob = b"".join(handles)
        buf = C.create_string_buffer(blob, len(blob))
        check(lib().sb_trainer_set_peer_handles(self._h, C.cast(buf, _vp), len(handles)))

    def clear_peer_handles(self):
        check(lib().sb_trainer_clear_peer_handles(self._h))

    @property
    def exchange_base(self) -> int:
        return int(lib().sb_trainer_exchange_base(self._h) or 0)

    def set_peer_pointers(self, bases: Sequence[int]):
        """in-process peers: every rank's exchange_base in rank order"""
        arr = (C.c_void_p * len(bases))(*[C.c_void_p(int(b)) for b in bases])
        check(lib().sb_trainer_set_peer_pointers(self._h, arr, len(bases)))

    # ---- parameters ----
    def set_params(self, flat):
        flat = _f32(flat).reshape(-1)
        check(lib().sb_trainer_set_params(self._h, _ptr(flat), flat.size))

    def get_params(self) -> np.ndarray:
        out = np.empty(self.n_params, np.float32)
        check(lib().sb_trainer_get_params(self._h, _ptr(out), out.size))
        return out

    def get_grads(self) -> np.ndarray:
        out = np.empty(self.n_params, np.float32)
        check(lib().sb_trainer_get_grads(self._h, _ptr(out), out.size))
        return out

    def init_xavier(self, seed: int):
        check(lib().sb_trainer_init_xavier(self._h, seed))

    # ---- steps ----
    def _xyw(self, X, y, w):
        if isinstance(X, DeviceArray):          # device-resident set: pointers pass through
            rows = X.shape[0]
            if len(X.shape) != 2 or X.shape[1] != self.n_features or y.size != rows or (w is not None and w.size != rows):
                raise ValueError("device arrays must be X [rows, %d], y [rows], w [rows]" % self.n_features)
            return X, y, w, rows
        X = _f32(X)
        rows = X.shape[0]
        if X.ndim != 2 or X.shape[1] != self.n_features:
            raise ValueError("X must be [rows, %d]" % self.n_features)
        y = _f32(y).reshape(-1)
        w = None if w is None else _f32(w).reshape(-1)
        if y.size != rows or (w is not None and w.size != rows):
            raise ValueError("y / w length must equal rows")
        return X, y, w, rows

    def step(self, X, y, w=None) -> float:
        X, y, w, rows = self._xyw(X, y, w)
        loss = C.c_float()
        check(lib().sb_trainer_step(self._h, _ptr(X), _ptr(y), _ptr(w), rows, C.byref(loss)))
        return float(loss.value)

    # ---- wide+deep: dense block + index matrix (oracle/wide_deep.py) ----
    def set_sparse(self, n_dense: int, n_onehot: int, n_cat: int):
        check(lib().sb_trainer_set_sparse(self._h, n_dense, n_onehot, n_cat))
        self._sparse = (n_dense, n_cat)

    def _xd_idx(self, Xd, idx):
        n_dense, n_cat = self._sparse
        Xd = _f32(Xd)
        idx = np.ascontiguousarray(idx, dtype=np.int32)
        if Xd.ndim != 2 or Xd.shape[1] != n_dense or idx.shape != (Xd.shape[0], n_cat):
            raise ValueError("Xd must be [rows, %d], idx [rows, %d]" % (n_dense, n_cat))
        return Xd, idx

    def step_sparse(self, Xd, idx, y, w=None) -> float:
        Xd, idx = self._xd_idx(Xd, idx)
        y = _f32(y).reshape(-1)
        w = None if w is None else _f32(w).reshape(-1)
        loss = C.c_float()
        check(lib().sb_trainer_step_sparse(self._h, _ptr(Xd), idx.ctypes.data_as(_P(C.c_int32)), _ptr(y), _ptr(w), Xd.shape[0],
                                           C.byref(loss)))
        return float(loss.value)

    def predict_sparse(self, Xd, idx) -> np.ndarray:
        Xd, idx = self._xd_idx(Xd, idx)
        out = np.empty(Xd.shape[0], np.float32)
        check(lib().sb_trainer_predict_sparse(self._h, _ptr(Xd), idx.ctypes.data_as(_P(C.c_int32)), Xd.shape[0], _ptr(out)))
        return out

    def eval_loss_sparse(self, Xd, idx, y, w=None) -> float:
        Xd, idx = self._xd_idx(Xd, idx)
        y = _f32(y).reshape(-1)
        w = None if w is None else _f32(w).reshape(-1)
        loss = C.c_float()
        check(lib().sb_trainer_eval_loss_sparse(self._h, _ptr(Xd), idx.ctypes.data_as(_P(C.c_int32)), _ptr(y), _ptr(w), Xd.shape[0],
                                                C.byref(loss)))
        return float(loss.value)

    def step_async(self, X, y, w=None) -> None:
        """queue one step on HOST buffers without waiting (X/y/w should be pinned and not reused for two more steps)"""
        X, y, w, rows = self._xyw(X, y, w)
        check(lib().sb_trainer_step_async(self._h, _ptr(X), _ptr(y), _ptr(w), rows))

    def accumulate(self, X, y, w=None) -> float:
        X, y, w, rows = self._xyw(X, y, w)
        loss = C.c_float()
        check(lib().sb_trainer_accumulate(self._h, _ptr(X), _ptr(y), _ptr(w), rows, C.byref(loss)))
        return float(loss.value)

    def apply_accumulated(self, total_pushes: Optional[int] = None):
        """one update from the accumulated gradients; total_pushes = divisor over ALL ranks (default world * n_acc)"""
        if total_pushes is None:
            check(lib().sb_trainer_apply_accumulated(self._h))
        else:
            check(lib().sb_trainer_apply_accumulated_mean(self._h, int(total_pushes)))

    def loss_resident(self, row_offset: int, rows: int) -> float:
        loss = C.c_float()
        check(lib().sb_trainer_loss_resident(self._h, row_offset, rows, C.byref(loss)))
        return float(loss.value)

    def broadcast_state(self, root: int = 0):
        check(lib().sb_trainer_broadcast_state(self._h, root))

    def load_dataset(self, X, y, w=None):
        X, y, w, rows = self._xyw(X, y, w)
        check(lib().sb_trainer_load_dataset(self._h, _ptr(X), _ptr(y), _ptr(w), rows))
        self.dataset_rows = rows
        logging.info("resident set: %d rows placed in %s" % (rows, "pinned host memory (each step reads its rows over PCIe)"
                                                              if self.dataset_on_host else "HBM"))

    @property
    def dataset_on_host(self) -> bool:
        """True when the loaded set did not fit in device memory and lives in pinned host memory (load_dataset)"""
        return lib().sb_trainer_dataset_on_host(self._h) == 1

    def debug_force_host_set(self, on: bool = True):
        """test hook: the next load_dataset places the set in pinned host memory whatever its size"""
        check(lib().sb_debug_force_host_set(self._h, int(bool(on))))

    def step_resident(self, row_offset: int, rows: int) -> float:
        loss = C.c_float()
        check(lib().sb_trainer_step_resident(self._h, row_offset, rows, C.byref(loss)))
        return float(loss.value)

    def step_resident_async(self, row_offset: int, rows: int):
        check(lib().sb_trainer_step_resident_async(self._h, row_offset, rows))

    def run_resident(self, row_offsets, rows: int):
        """n update steps over the resident set in one call (asynchronous; the reference's per-epoch batch loop)"""
        offs = np.ascontiguousarray(row_offsets, dtype=np.int64).reshape(-1)
        check(lib().sb_trainer_run_resident(self._h, offs.ctypes.data_as(C.POINTER(C.c_int64)), offs.size, rows))

    def accumulate_resident(self, row_offset: int, rows: int) -> float:
        loss = C.c_float()
        check(lib().sb_trainer_accumulate_resident(self._h, row_offset, rows, C.byref(loss)))
        return float(loss.value)

    def set_row_order(self, rows=None):
        """the resident steps read logical row r as row rows[r] of the loaded set (sb_trainer_set_row_order); None: the
        physical order"""
        if rows is None:
            check(lib().sb_trainer_set_row_order(self._h, None, 0))
            return
        order = np.ascontiguousarray(rows, dtype=np.int64).reshape(-1)
        check(lib().sb_trainer_set_row_order(self._h, order.ctypes.data_as(C.POINTER(C.c_int64)), order.size))

    def last_loss(self) -> float:
        loss = C.c_float()
        check(lib().sb_trainer_last_loss(self._h, C.byref(loss)))
        return float(loss.value)

    def loss_history(self, first_step: int, n: int) -> np.ndarray:
        """mini-batch losses of update steps first_step .. first_step+n-1 (1-based global_step); waits for the GPU"""
        out = np.empty(n, np.float32)
        check(lib().sb_trainer_loss_history(self._h, first_step, n, _ptr(out)))
        return out

    def sync(self):
        check(lib().sb_trainer_sync(self._h))

    @property
    def stream(self) -> int:
        return int(lib().sb_trainer_stream(self._h) or 0)

    def kernels_per_step(self, rows: int) -> int:
        n = lib().sb_trainer_kernels_per_step(self._h, rows)
        if n < 0:
            check(n)
        return n

    def eval_loss(self, X, y, w=None) -> float:
        X, y, w, rows = self._xyw(X, y, w)
        loss = C.c_float()
        check(lib().sb_trainer_eval_loss(self._h, _ptr(X), _ptr(y), _ptr(w), rows, C.byref(loss)))
        return float(loss.value)

    def predict(self, X) -> np.ndarray:
        X = _f32(X)
        out = np.empty(X.shape[0], np.float32)
        check(lib().sb_trainer_predict(self._h, _ptr(X), X.shape[0], _ptr(out)))
        return out

    def debug_step_trace(self):
        """-> (names, stamps[k,16] uint64 ns) of the last step's GEMM launches (needs SB_STEP_TRACE=1 at creation)"""
        buf = np.zeros((32, 16), np.uint64)
        names = C.create_string_buffer(4096)
        k = C.c_int32()
        check(lib().sb_debug_step_trace(self._h, buf.ctypes.data_as(C.POINTER(C.c_uint64)), 32, names, 4096, C.byref(k)))
        return names.value.decode().split(","), buf[:k.value].copy()

    # ---- exchange test hooks (sb_debug_trainer_buffer / sb_debug_exchange / sb_debug_exchange_layout) ----
    def debug_buffer_dtype(self, which: int):
        """element type of buffer `which` of debug_buffer"""
        if which in (DEBUG_BUF_BATCH_X, DEBUG_BUF_DS_X):
            return np.float32 if self.desc.precision == PREC_FP32 else np.uint16
        if which == DEBUG_BUF_DS_P:
            return np.int32
        return np.float32 if which < DEBUG_BUF_SHADOW or which >= DEBUG_BUF_BATCH_X else np.uint16

    def debug_buffer(self, which: int, value: Optional[np.ndarray] = None, n: Optional[int] = None,
                     refresh_shadows: bool = False) -> Optional[np.ndarray]:
        """value None: -> a copy of one raw arena buffer (which < DEBUG_BUF_SHADOW: float32 [n_params]; DEBUG_BUF_SHADOW + l:
        the uint16 bits of hidden layer l's shadow, n values = np * in * ld_out) or input-stage buffer (DEBUG_BUF_BATCH_X ..
        DEBUG_BUF_DS_P, n values of debug_buffer_dtype; include/shifu_b200.h gives the shapes).  Otherwise write `value`
        (of the type read), refreshing the shadows from theta if asked."""
        dtype = self.debug_buffer_dtype(which)
        if value is None:
            out = np.empty(self.n_params if n is None else n, dtype)
            check(lib().sb_debug_trainer_buffer(self._h, which, out.ctypes.data_as(_vp), out.size, 0))
            return out
        value = np.ascontiguousarray(value, dtype=dtype).reshape(-1)
        check(lib().sb_debug_trainer_buffer(self._h, which, value.ctypes.data_as(_vp), value.size, 2 if refresh_shadows else 1))
        return None

    def debug_first_kernel(self, X=None, y=None, w=None, idx=None, row_offset: int = 0, rows: Optional[int] = None,
                           clear: bool = False) -> str:
        """what a step queues before layer 0, waited for (sb_debug_first_kernel): host rows X / y / w (idx: the dense block and
        index matrix of a sparse trainer), or with X None rows [row_offset, row_offset + rows) of the resident set -> the
        kernel launched ("none" for a bf16-resident batch)"""
        route = C.create_string_buffer(64)
        if X is None:
            check(lib().sb_debug_first_kernel(self._h, None, None, None, None, int(row_offset), int(rows), int(clear), route, 64))
            return route.value.decode()
        X, y = _f32(X), _f32(y).reshape(-1)
        w = None if w is None else _f32(w).reshape(-1)
        idx_p = None
        if idx is not None:
            idx = np.ascontiguousarray(idx, dtype=np.int32)
            idx_p = idx.ctypes.data_as(_P(C.c_int32))
        n = X.shape[0] if rows is None else int(rows)
        if y.size < n or (w is not None and w.size < n) or X.shape[0] < n:
            raise ValueError("X, y, w hold fewer than rows = %d rows" % n)
        check(lib().sb_debug_first_kernel(self._h, _ptr(X), _ptr(y), _ptr(w), idx_p, int(row_offset), n, int(clear), route, 64))
        return route.value.decode()

    def debug_exchange(self, slot_mask: int, gscale: float = 0.0, grid: int = 0, alone: bool = False):
        """queue one exchange of the slots in slot_mask as a step does, without waiting -> (lr_t, grid, kernel name)"""
        lr_t, g = C.c_float(), C.c_int32()
        route = C.create_string_buffer(64)
        check(lib().sb_debug_exchange(self._h, int(slot_mask), float(gscale), int(grid), int(alone), C.byref(lr_t), C.byref(g),
                                      route, 64))
        return float(lr_t.value), int(g.value), route.value.decode()

    def debug_optimizer(self, gscale: float = 0.0, tail: int = 0):
        """queue one single-GPU optimizer pass over the raw gradient buffer without waiting (tail = 1: the step's split
        tail; sb_debug_optimizer) -> (lr_t, route)"""
        lr_t = C.c_float()
        route = C.create_string_buffer(256)
        check(lib().sb_debug_optimizer(self._h, float(gscale), int(tail), C.byref(lr_t), route, 256))
        return float(lr_t.value), route.value.decode()

    def debug_exchange_layout(self) -> dict:
        info = (C.c_int32 * DEBUG_XINFO_WORDS)()
        n = C.c_int32()
        check(lib().sb_debug_exchange_layout(self._h, info, DEBUG_XINFO_WORDS, None, 0, C.byref(n)))
        work = np.zeros((n.value, DEBUG_XWORK_WORDS), np.int64)
        check(lib().sb_debug_exchange_layout(self._h, info, DEBUG_XINFO_WORDS, work.ctypes.data_as(_P(C.c_int64)), work.size,
                                             C.byref(n)))
        s = info[0]
        return dict(slots=s, sms=info[1], ll=bool(info[2]), share_device=bool(info[3]), rank=info[4], world=info[5], np=info[6],
                    begin=list(info[8:8 + s]), end=list(info[16:16 + s]),
                    work=[dict(zip(("off", "count", "out_dim", "mat_off", "ld_out", "np", "layer", "part_stride"),
                                   (int(v) for v in row))) for row in work])

    @property
    def global_step(self) -> int:
        return int(lib().sb_trainer_global_step(self._h))

    def save_checkpoint(self, path: str):
        check(lib().sb_trainer_save_checkpoint(self._h, path.encode()))

    def load_checkpoint(self, path: str):
        check(lib().sb_trainer_load_checkpoint(self._h, path.encode()))

    def export_savedmodel(self, export_dir: str):
        check(lib().sb_trainer_export_savedmodel(self._h, export_dir.encode()))


def _sensitivity(n_features, call, X, w, cols, values, deltas) -> dict:
    """Model.sensitivity / Ensemble.sensitivity: the arguments checked and converted, then call(X, w, rows, cols, n_cols,
    values, sum_sq, sum, w_sum, deltas) of the C entry point"""
    xp, shape = _in_ptr(X)
    if len(shape) != 2 or shape[1] != n_features:
        raise ValueError("X must be [rows, %d]" % n_features)
    rows = int(shape[0])
    wp, wshape = _in_ptr(w) if w is not None else (None, (rows,))
    if int(np.prod(wshape)) != rows:
        raise ValueError("w must hold one weight per row")
    cl = None if cols is None else np.ascontiguousarray(cols, dtype=np.int32).reshape(-1)
    n_cols = n_features if cl is None else cl.size
    vl = None if values is None else _f32(values).reshape(-1)
    if vl is not None and vl.size != n_cols:
        raise ValueError("values must hold one value per list position (%d)" % n_cols)
    sum_sq, total, w_sum = np.zeros(n_cols), np.zeros(n_cols), C.c_double()
    if deltas is True:
        d_out = np.empty((rows, n_cols), np.float32)
        dp = d_out.ctypes.data_as(_vp)
    elif deltas is False or deltas is None:
        d_out, dp = None, None
    else:
        d_out = deltas
        dp = _in_ptr(deltas)[0]
    check(call(xp, wp, rows, None if cl is None else cl.ctypes.data_as(_P(C.c_int32)), 0 if cl is None else cl.size,
               None if vl is None else _ptr(vl), sum_sq.ctypes.data_as(_f64p), total.ctypes.data_as(_f64p), C.byref(w_sum), dp))
    return {"sum_sq": sum_sq, "sum": total, "w_sum": float(w_sum.value), "deltas": d_out}


def _reason_codes(n_features, call, X, k, cols, values, order, scores, pos, d) -> dict:
    """Model.reason_codes / Ensemble.reason_codes: the arguments checked and converted, then call(X, rows, cols, n_cols,
    values, k, order, pos, d, scores) of the C entry point"""
    xp, shape = _in_ptr(X)
    if len(shape) != 2 or shape[1] != n_features:
        raise ValueError("X must be [rows, %d]" % n_features)
    rows = int(shape[0])
    cl = None if cols is None else np.ascontiguousarray(cols, dtype=np.int32).reshape(-1)
    n_cols = n_features if cl is None else cl.size
    vl = None if values is None else _f32(values).reshape(-1)
    if vl is not None and vl.size != n_cols:
        raise ValueError("values must hold one value per list position (%d)" % n_cols)
    if order not in REASON_ORDERS:
        raise ValueError("order must be one of %s" % sorted(REASON_ORDERS))

    def out(buf, dtype, shape):
        if buf is None or buf is True:
            a = np.empty(shape, dtype)
            return a, a.ctypes.data_as(_vp)
        return buf, _in_ptr(buf, dtype)[0]

    p_out, pp = out(pos, np.int32, (rows, k))
    d_out, dp = out(d, np.float32, (rows, k))
    s_out, sp = out(scores, np.float32, (rows,)) if scores is not False and scores is not None else (None, None)
    check(call(xp, rows, None if cl is None else cl.ctypes.data_as(_P(C.c_int32)), 0 if cl is None else cl.size,
               None if vl is None else _ptr(vl), int(k), REASON_ORDERS[order], pp, dp, sp))
    return {"pos": p_out, "d": d_out, "scores": s_out}


class Model:
    """Owns one sb_model_t (batched scorer)."""

    def __init__(self, handle):
        self._h = handle
        self.n_features = int(lib().sb_model_n_features(self._h))

    @classmethod
    def load(cls, saved_model_dir: str, input_name: str, output_name: str, tag: str = "serve", device: int = 0,
             precision: int = PREC_FP32) -> "Model":
        h = C.c_void_p()
        enc = lambda s: None if s is None else s.encode()
        check(lib().sb_model_load(enc(saved_model_dir), enc(input_name), enc(output_name), enc(tag), device, precision,
                                  C.byref(h)))
        return cls(h)

    @classmethod
    def create(cls, desc: NetDesc, flat_params, device: int = 0) -> "Model":
        h = C.c_void_p()
        flat = _f32(flat_params).reshape(-1)
        check(lib().sb_model_create(C.byref(desc), _ptr(flat), flat.size, device, C.byref(h)))
        return cls(h)

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            lib().sb_model_destroy(self._h)
            self._h = None

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def score(self, X) -> np.ndarray:
        X = _f32(X)
        if X.ndim != 2 or X.shape[1] != self.n_features:
            raise ValueError("X must be [rows, %d]" % self.n_features)
        out = np.empty(X.shape[0], np.float32)
        check(lib().sb_model_score(self._h, _ptr(X), X.shape[0], _ptr(out)))
        return out

    def score_row_f64(self, row) -> float:
        row = np.ascontiguousarray(row, dtype=np.float64).reshape(-1)
        out = C.c_double()
        check(lib().sb_model_score_row_f64(self._h, row.ctypes.data_as(_f64p), row.size, C.byref(out)))
        return float(out.value)

    def score_device(self, dX_ptr: int, rows: int, dOut_ptr: int):
        check(lib().sb_model_score_device(self._h, C.c_void_p(dX_ptr), rows, C.c_void_p(dOut_ptr)))

    def sensitivity(self, X, w=None, cols=None, values=None, deltas=False) -> dict:
        """Column sensitivity (sb_model_sensitivity): for each list position k, d[r, k] = s(X[r]) - s(X[r] with column
        cols[k] set to values[k]).  -> {"sum_sq": sum_r w d^2, "sum": sum_r w d (float64 [n_cols]), "w_sum": sum_r w,
        "deltas": d [rows, n_cols] or None}.
        X / w: numpy arrays (host) or CUDA tensors / DeviceArrays on the model's device.  cols: None for every column in
        order.  values: None for 0 at every position.  deltas: False (not computed), True (returned as a host array) or a
        device buffer of rows * n_cols floats to write them into."""
        return _sensitivity(self.n_features, lambda *a: lib().sb_model_sensitivity(self._h, *a), X, w, cols, values, deltas)

    def reason_codes(self, X, k, cols=None, values=None, order="raise", scores=False, pos=None, d=None) -> dict:
        """Per-row reason codes (sb_model_reason_codes): for each row, the k list positions whose deltas
        d = s(X[r]) - s(X[r] with column cols[j] set to values[j]) rank first in `order` ("raise": largest d first,
        "lower": smallest d first, "magnitude": largest |d| first; NaN last, ties to the smaller position).
        -> {"pos": int32 [rows, k], "d": their deltas float32 [rows, k], "scores": the base scores [rows] or None}.
        X: a numpy array (host) or a CUDA tensor / DeviceArray on the model's device.  cols / values as in sensitivity.
        pos / d: None (returned as host arrays) or a buffer of rows * k int32 / float32 to write into; scores: False (not
        computed), True (a host array) or a buffer of rows floats."""
        return _reason_codes(self.n_features, lambda *a: lib().sb_model_reason_codes(self._h, *a), X, k, cols, values, order,
                             scores, pos, d)

    def sync(self):
        check(lib().sb_model_sync(self._h))

    @property
    def stream(self) -> int:
        return int(lib().sb_model_stream(self._h) or 0)

    def batch_stats(self) -> dict:
        """counters since creation (sb_debug_model_batch_stats): compute() batches, their rows, the largest batch, batches
        run by the one-launch fp32 kernel / by the captured tensor-core graph, and one-launch fp32 forwards of any entry point"""
        st = np.zeros(DEBUG_MSTAT_WORDS, np.int64)
        check(lib().sb_debug_model_batch_stats(self._h, st.ctypes.data_as(_P(C.c_int64)), st.size))
        return dict(zip(("batches", "rows", "max_fill", "small", "graph", "small_launches"), (int(v) for v in st)))

    def hold(self, k: int, timeout_ms: int):
        """the next compute() batch waits until k rows are queued or timeout_ms have passed (sb_debug_model_hold)"""
        check(lib().sb_debug_model_hold(self._h, int(k), int(timeout_ms)))

    def routes(self) -> str:
        """the kernels of the last forward, "+"-joined (sb_debug_model_routes)"""
        buf = C.create_string_buffer(256)
        check(lib().sb_debug_model_routes(self._h, buf, len(buf)))
        return buf.value.decode()

    def device_bytes(self) -> int:
        """the device bytes the model allocated (sb_debug_model_bytes)"""
        out = C.c_int64()
        check(lib().sb_debug_model_bytes(self._h, C.byref(out)))
        return int(out.value)


class Ensemble:
    """Owns one sb_ensemble_t: K bagged member models scored from one staged copy of the rows, with each row's mean,
    max, min and median of the member scores formed on the GPU."""

    def __init__(self, handle, n_features: int):
        self._h = handle
        self.n_features = int(n_features)
        self.k = int(lib().sb_ensemble_size(self._h))

    @classmethod
    def load(cls, saved_model_dirs: Sequence[str], input_name: str, output_name: str, tag: str = "serve", device: int = 0,
             precision: int = PREC_FP32) -> "Ensemble":
        enc = lambda s: None if s is None else s.encode()
        dirs = (_cp * max(len(saved_model_dirs), 1))(*[enc(d) for d in saved_model_dirs])
        h = C.c_void_p()
        check(lib().sb_ensemble_load(dirs, len(saved_model_dirs), enc(input_name), enc(output_name), enc(tag), device,
                                     precision, C.byref(h)))
        e = cls(h, 0)
        e.n_features = savedmodel_read(saved_model_dirs[0], input_name, output_name, tag)[0]
        return e

    @classmethod
    def create(cls, descs: Sequence[NetDesc], flats, device: int = 0) -> "Ensemble":
        k = len(descs)
        flats = [_f32(f).reshape(-1) for f in flats]
        if len(flats) != k:
            raise ValueError("one flat parameter vector per descriptor")
        d_arr = (NetDesc * max(k, 1))(*descs)
        f_arr = (_f32p * max(k, 1))(*[_ptr(f) for f in flats])
        n_arr = (C.c_int64 * max(k, 1))(*[f.size for f in flats])
        h = C.c_void_p()
        check(lib().sb_ensemble_create(d_arr, f_arr, n_arr, k, device, C.byref(h)))
        return cls(h, descs[0].n_features)

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            lib().sb_ensemble_destroy(self._h)
            self._h = None

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def score(self, X, scores: bool = True, stats: bool = True):
        """-> (scores [rows, k] in member order or None, stats [rows, 4] = mean, max, min, median or None).  X: a numpy
        array (host) or a CUDA tensor / DeviceArray on the ensemble's device."""
        if isinstance(X, np.ndarray) or not (hasattr(X, "data_ptr") or isinstance(X, DeviceArray)):
            X = _f32(X)
        xp, shape = _in_ptr(X)
        if len(shape) != 2 or shape[1] != self.n_features:
            raise ValueError("X must be [rows, %d]" % self.n_features)
        rows = int(shape[0])
        s = np.empty((rows, self.k), np.float32) if scores else None
        t = np.empty((rows, 4), np.float32) if stats else None
        check(lib().sb_ensemble_score(self._h, xp, rows, None if s is None else s.ctypes.data_as(_vp),
                                      None if t is None else t.ctypes.data_as(_vp)))
        return s, t

    def score_device(self, dX_ptr: int, rows: int, dScores_ptr: Optional[int], dStats_ptr: Optional[int]):
        """device pointers, asynchronous on the ensemble's stream (sync() waits); either output pointer may be None"""
        check(lib().sb_ensemble_score_device(self._h, C.c_void_p(dX_ptr), rows, C.c_void_p(dScores_ptr) if dScores_ptr else None,
                                             C.c_void_p(dStats_ptr) if dStats_ptr else None))

    def score_row_f64(self, row) -> np.ndarray:
        """compute() of every member: -> float64 [k + 4] (the k member scores, then mean, max, min, median)"""
        row = np.ascontiguousarray(row, dtype=np.float64).reshape(-1)
        out = np.empty(self.k + 4, np.float64)
        check(lib().sb_ensemble_score_row_f64(self._h, row.ctypes.data_as(_f64p), row.size, out.ctypes.data_as(_f64p)))
        return out

    def _stat(self, stat: str) -> int:
        if stat not in ENSEMBLE_STATS:
            raise ValueError("stat must be one of %s" % (ENSEMBLE_STATS,))
        return ENSEMBLE_STATS.index(stat)

    def sensitivity(self, X, w=None, cols=None, values=None, deltas=False, stat="mean") -> dict:
        """Column sensitivity of one statistic S of the member scores (sb_ensemble_sensitivity): for each list position
        k, d[r, k] = S(X[r]) - S(X[r] with column cols[k] set to values[k]), stat one of ENSEMBLE_STATS.  Arguments and
        result as Model.sensitivity."""
        st = self._stat(stat)
        return _sensitivity(self.n_features, lambda *a: lib().sb_ensemble_sensitivity(self._h, st, *a), X, w, cols, values,
                            deltas)

    def reason_codes(self, X, k, cols=None, values=None, order="raise", stat="mean", scores=False, pos=None, d=None) -> dict:
        """Per-row reason codes of one statistic S of the member scores (sb_ensemble_reason_codes): the k list positions
        whose deltas d = S(X[r]) - S(X[r] with column cols[j] set to values[j]) rank first in `order`, stat one of
        ENSEMBLE_STATS; scores: S(X[r]).  Arguments and result as Model.reason_codes."""
        st = self._stat(stat)
        return _reason_codes(self.n_features, lambda *a: lib().sb_ensemble_reason_codes(self._h, st, *a), X, k, cols, values,
                             order, scores, pos, d)

    def sync(self):
        check(lib().sb_ensemble_sync(self._h))

    @property
    def stream(self) -> int:
        return int(lib().sb_ensemble_stream(self._h) or 0)

    def routes(self) -> str:
        """the kernels of the last chunk, "+"-joined (sb_debug_ensemble_routes)"""
        buf = C.create_string_buffer(16384)
        check(lib().sb_debug_ensemble_routes(self._h, buf, len(buf)))
        return buf.value.decode()

    def device_bytes(self) -> int:
        """the device bytes the ensemble allocated (sb_debug_ensemble_bytes)"""
        out = C.c_int64()
        check(lib().sb_debug_ensemble_bytes(self._h, C.byref(out)))
        return int(out.value)


class Performance:
    """Owns one sb_perf_t: exact ROC AUC, PR AUC (average precision), KS and operating points of scored rows, each
    weighted and unweighted, computed on the GPU from one radix sort of the scores (include/shifu_b200.h defines them)."""

    def __init__(self, device: int = 0, reserve_rows: int = 0):
        h = C.c_void_p()
        check(lib().sb_perf_create(device, int(reserve_rows), C.byref(h)))
        self._h = h

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            lib().sb_perf_destroy(self._h)
            self._h = None

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def add(self, scores, y, w=None, stride: int = 1):
        """numpy rows: scores[r * stride] (float32), y[r] (0 / 1), w[r] (None: 1); returns once the rows have been read"""
        y = _f32(y).reshape(-1)
        s = _f32(scores).reshape(-1)
        rows = y.size
        if rows and s.size < (rows - 1) * stride + 1:
            raise ValueError("scores must hold (rows - 1) * stride + 1 values")
        if w is not None:
            w = _f32(w).reshape(-1)
            if w.size != rows:
                raise ValueError("w must hold one weight per row")
        check(lib().sb_perf_add(self._h, s.ctypes.data_as(_vp), int(stride), y.ctypes.data_as(_vp),
                                None if w is None else w.ctypes.data_as(_vp), rows, None))

    def add_device(self, ptr: int, y_ptr: int, w_ptr: Optional[int], rows: int, stride: int = 1,
                   after_stream: Optional[int] = None):
        """device pointers (ints): queued on the handle's stream behind the work queued on after_stream so far"""
        check(lib().sb_perf_add(self._h, C.c_void_p(ptr), int(stride), C.c_void_p(y_ptr), C.c_void_p(w_ptr) if w_ptr else None,
                                int(rows), C.c_void_p(after_stream) if after_stream else None))

    def summary(self) -> dict:
        s = PerfSummary()
        check(lib().sb_perf_summary_get(self._h, C.byref(s)))
        return {name: getattr(s, name) for name, _ in PerfSummary._fields_}

    def points(self, axis, levels, weighted: bool = False) -> dict:
        """-> {"threshold" float32, "tp", "fp" int64, "w_tp", "w_fp" float64}, one entry per level.  axis: "action_rate",
        "recall", "fpr", "score" or its PERF_* number"""
        ax = PERF_AXES[axis] if isinstance(axis, str) else int(axis)
        lv = np.ascontiguousarray(levels, dtype=np.float64).reshape(-1)
        out = (PerfPoint * max(lv.size, 1))()
        check(lib().sb_perf_points(self._h, ax, 1 if weighted else 0, lv.ctypes.data_as(_f64p), lv.size, out))
        a = np.frombuffer(out, dtype=np.dtype([("threshold", "<f4"), ("tp", "<i8"), ("fp", "<i8"), ("w_tp", "<f8"),
                                               ("w_fp", "<f8")], align=True), count=lv.size)
        return {name: a[name].copy() for name in a.dtype.names}

    def reset(self):
        check(lib().sb_perf_reset(self._h))

    def sync(self):
        check(lib().sb_perf_sync(self._h))

    @property
    def stream(self) -> int:
        return int(lib().sb_perf_stream(self._h) or 0)

    def runs(self) -> dict:
        """the whole run table (sb_debug_perf_runs): t, tp, fp, w_tp, w_fp per distinct score, highest first"""
        n = C.c_int64()
        check(lib().sb_debug_perf_runs(self._h, None, None, None, None, None, 0, C.byref(n)))
        m = int(n.value)
        t, tp, fp = np.empty(m, np.float32), np.empty(m, np.int64), np.empty(m, np.int64)
        wtp, wfp = np.empty(m, np.float64), np.empty(m, np.float64)
        check(lib().sb_debug_perf_runs(self._h, _ptr(t), tp.ctypes.data_as(_P(C.c_int64)), fp.ctypes.data_as(_P(C.c_int64)),
                                       wtp.ctypes.data_as(_f64p), wfp.ctypes.data_as(_f64p), m, C.byref(n)))
        return {"t": t, "tp": tp, "fp": fp, "w_tp": wtp, "w_fp": wfp}

    def device_bytes(self) -> int:
        """the device bytes the handle holds (sb_debug_perf_bytes)"""
        out = C.c_int64()
        check(lib().sb_debug_perf_bytes(self._h, C.byref(out)))
        return int(out.value)


def nccl_unique_id() -> bytes:
    buf = C.create_string_buffer(SB_NCCL_ID_BYTES)
    check(lib().sb_nccl_unique_id(C.cast(buf, _vp)))
    return buf.raw


def device_count() -> int:
    return int(lib().sb_device_count())


def device_mem_info(device: int = 0):
    """-> (free, total) bytes of device memory (cudaMemGetInfo)"""
    f, t = C.c_uint64(), C.c_uint64()
    check(lib().sb_device_mem_info(int(device), C.byref(f), C.byref(t)))
    return int(f.value), int(t.value)


def savedmodel_write(export_dir: str, desc: NetDesc, flat_params) -> None:
    flat = _f32(flat_params).reshape(-1)
    check(lib().sb_savedmodel_write(export_dir.encode(), C.byref(desc), _ptr(flat), flat.size))


def savedmodel_read(saved_model_dir: str, input_name: str, output_name: str, tag: str = "serve"):
    """-> (n_features, hidden list, acts list, out_act, flat params)"""
    d = NetDesc()
    out_act = C.c_int32(0)
    n = C.c_int64(0)
    args = (saved_model_dir.encode(), input_name.encode(), output_name.encode(), tag.encode())
    check(lib().sb_savedmodel_read(*args, C.byref(d), C.byref(out_act), None, 0, C.byref(n)))
    flat = np.empty(n.value, np.float32)
    check(lib().sb_savedmodel_read(*args, C.byref(d), C.byref(out_act), _ptr(flat), flat.size, C.byref(n)))
    return int(d.n_features), [int(d.hidden[i]) for i in range(d.n_hidden)], [int(d.acts[i]) for i in range(d.n_hidden)], \
        int(out_act.value), flat


def debug_gemm_bf16(A: np.ndarray, B: np.ndarray, split_k: int = 1, device: int = 0, a_mn: bool = False,
                    b_mn: bool = False, cg: int = 0, bn: int = 0) -> np.ndarray:
    """D[M,N] = sum_k A(m,k) B(n,k) through the wgmma kernel (operands rounded to bf16 on the device).
    A is [M,K] (K-major) or, with a_mn, [K,M] (MN-major); B is [N,K] or, with b_mn, [K,N]."""
    A, B = _f32(A), _f32(B)
    (K, M) = A.shape if a_mn else A.shape[::-1]
    (K2, N) = B.shape if b_mn else B.shape[::-1]
    assert K == K2
    D = np.zeros((M, N), np.float32)
    check(lib().sb_debug_gemm_bf16_cfg(_ptr(A), _ptr(B), _ptr(D), M, N, K, split_k, int(a_mn), int(b_mn), cg, bn, device))
    return D


GEMM_FWD, GEMM_DA, GEMM_DW = 0, 1, 2
PARTS = {PREC_FP32: 1, PREC_BF16: 1, PREC_FP32_TC: 3, PREC_BF16X2: 2}


def debug_gemm_layer(kind: int, precision: int, A: np.ndarray, W: np.ndarray, act: int = ACT_NONE,
                     bias: Optional[np.ndarray] = None, aux: Optional[np.ndarray] = None, addend: Optional[np.ndarray] = None,
                     colsum: Optional[np.ndarray] = None, grad: Optional[np.ndarray] = None, M: Optional[int] = None,
                     row0: int = 0, r0: int = 0, r1: Optional[int] = None, sms: int = 0, clear_n4: int = 0, device: int = 0):
    """One forward / dA / dW GEMM of a training step through the step's own launch code (sb_debug_gemm_layer):
      GEMM_FWD: A [a_rows, K] (batch = rows row0 .. row0 + M - 1, M defaults to the rest), W [K, N], bias [N], addend [M, N]
      GEMM_DA : A = dZ_l [M, K], W = W_l [N, K], aux = A_{l-1} [M, N], colsum [N] (in/out, zeros by default)
      GEMM_DW : A [a_rows, M] (batch = rows row0 .. row0 + K - 1), W = dZ [K, N], grad [M, N] (in/out, zeros by default),
                rows r0 .. r1 - 1 (r1 defaults to M)
    -> (out [np, M, N] or None, colsum or None, grad or None, guard count, route name)"""
    A, W = _f32(A), _f32(W)
    nparts = PARTS[precision]
    out = cs = g = None
    if kind == GEMM_DW:
        a_rows, Mx = A.shape
        K, N = W.shape
        if row0 + K > a_rows:
            raise ValueError("the batch of K = %d rows at row0 = %d runs past A" % (K, row0))
        g = np.zeros((Mx, N), np.float32) if grad is None else _f32(grad).copy()
        a_rows_arg, M = a_rows, Mx
    elif kind == GEMM_DA:
        M, K = A.shape
        N = W.shape[0]
        assert W.shape == (N, K) and np.shape(aux) == (M, N)
        cs = np.zeros(N, np.float32) if colsum is None else _f32(colsum).copy()
        a_rows_arg = M
    else:
        a_rows_arg, K = A.shape
        N = W.shape[1]
        M = a_rows_arg - row0 if M is None else M
    if kind != GEMM_DW:
        out = np.zeros((nparts, M, N), np.float32)
    bias = None if bias is None else _f32(bias)
    aux = None if aux is None else _f32(aux)
    addend = None if addend is None else _f32(addend)
    guard = C.c_int32(-1)
    route = C.create_string_buffer(64)
    check(lib().sb_debug_gemm_layer(kind, precision, _ptr(A), _ptr(W), _ptr(bias), _ptr(aux), _ptr(addend), _ptr(out), _ptr(cs),
                                    _ptr(g), C.byref(guard), route, 64, M, N, K, a_rows_arg, row0, act, r0,
                                    M if r1 is None else r1, sms, clear_n4, device))
    return out, cs, g, int(guard.value), route.value.decode()


def debug_gemm_split(A: np.ndarray, B: np.ndarray, np_parts: int, device: int = 0) -> np.ndarray:
    """D[M,N] = A[M,K] B[N,K]^T with every fp32 value split into np_parts bf16 parts (1 = plain bf16): the forward GEMM of
    a step in that precision (debug_gemm_layer, act none, zero bias), its stored parts summed in float64"""
    prec = {1: PREC_BF16, 2: PREC_BF16X2, 3: PREC_FP32_TC}.get(np_parts)
    if prec is None:
        raise ShifuB200Error(SB_ERR_INVALID, "np_parts=%r outside 1..3" % (np_parts,))
    A, B = _f32(A), _f32(B)
    assert A.shape[1] == B.shape[1]
    out, _, _, guard, _ = debug_gemm_layer(GEMM_FWD, prec, A, B.T.copy(), ACT_NONE, bias=np.zeros(B.shape[0], np.float32),
                                           device=device)
    if guard != 0:
        raise ShifuB200Error(SB_ERR_STATE, "%d sentinel elements around the output changed" % guard)
    return out.astype(np.float64).sum(axis=0)


def debug_gemm_bench(M: int, N: int, K: int, split_k: int = 1, a_mn: bool = False, b_mn: bool = False, cg: int = 0,
                     bn: int = 0, iters: int = 50, device: int = 0) -> float:
    """average device ms per launch of one tile configuration (random operands)"""
    rng = np.random.default_rng(0)
    A = rng.standard_normal((K, M) if a_mn else (M, K), dtype=np.float32)
    B = rng.standard_normal((K, N) if b_mn else (N, K), dtype=np.float32)
    D = np.zeros((M, N), np.float32)
    ms = C.c_float()
    check(lib().sb_debug_gemm_bench(_ptr(A), _ptr(B), _ptr(D), M, N, K, split_k, int(a_mn), int(b_mn), cg, bn, device,
                                    iters, C.byref(ms)))
    return float(ms.value)


def debug_gemm_epilogue(A: np.ndarray, W: np.ndarray, act: int, bias: Optional[np.ndarray] = None,
                        aux: Optional[np.ndarray] = None, bm_wg: int = 0, iters: int = 0, device: int = 0):
    """One plain-bf16 forward (aux None: act(A W + bias), W [K,N]) or dA (aux given: (A W^T) * act'(aux), W [N,K]) GEMM
    with its fused epilogue -> (out [M,N] fp32 of the bf16 results, column sums [N] or None, ms per launch or None).
    bm_wg: 0 = the planner's tile, 64 / 128 = the ping-pong kernel's warpgroup tile rows, 256 = the forward GEMM's
    128 x 256 tile"""
    A, W = _f32(A), _f32(W)
    M, K = A.shape
    da = aux is not None
    N = W.shape[0] if da else W.shape[1]
    assert W.shape == ((N, K) if da else (K, N))
    bias = _f32(bias) if bias is not None else None
    aux = _f32(aux) if da else None
    out = np.zeros((M, N), np.float32)
    cs = np.zeros(N, np.float32) if da else None
    ms = C.c_float()
    check(lib().sb_debug_gemm_epilogue(_ptr(A), _ptr(W), _ptr(bias) if bias is not None else None,
                                       _ptr(aux) if da else None, _ptr(out), _ptr(cs) if da else None, M, N, K, int(da),
                                       act, bm_wg, device, iters, C.byref(ms)))
    return out, cs, (float(ms.value) if iters > 0 else None)


def debug_gemm_fwd_out(A: np.ndarray, W: np.ndarray, bias: np.ndarray, wo: np.ndarray, bo: float, y: np.ndarray,
                       w: np.ndarray, act: int, loss: int, np_parts: int = 1, row0: int = 0, M: Optional[int] = None,
                       grid: int = 0, g_bL: Optional[np.ndarray] = None, g_wo: Optional[np.ndarray] = None, g_bo: float = 0.0,
                       loss_sum: float = 0.0, device: int = 0):
    """The fused output-layer GEMM of a training step (last hidden layer N <= 256) on rows row0 .. row0 + M - 1 of
    A [a_rows, K] (M defaults to the rest of A), W [K, N], y / w [M].  g_bL, g_wo [N], g_bo and loss_sum are the initial
    values the kernel adds into (zeros by default).  -> (dZ [np_parts, M, N] fp32 of the bf16 parts, g_bL, g_wo, g_bo,
    loss_sum, number of changed sentinel elements around dZ)"""
    A, W, bias, wo = _f32(A), _f32(W), _f32(bias), _f32(wo)
    a_rows, K = A.shape
    K2, N = W.shape
    assert K == K2
    M = a_rows - row0 if M is None else M
    y, w = _f32(y).reshape(-1), _f32(w).reshape(-1)
    assert y.size == M and w.size == M
    g_bL = _f32(g_bL).copy() if g_bL is not None else np.zeros(N, np.float32)
    g_wo = _f32(g_wo).copy() if g_wo is not None else np.zeros(N, np.float32)
    gbo, ls, guard = C.c_float(g_bo), C.c_float(loss_sum), C.c_int32(-1)
    dZ = np.zeros((max(np_parts, 1), max(M, 0), N), np.float32)
    check(lib().sb_debug_gemm_fwd_out(_ptr(A), _ptr(W), _ptr(bias), _ptr(wo), float(bo), _ptr(y), _ptr(w), _ptr(dZ),
                                      _ptr(g_bL), _ptr(g_wo), C.byref(gbo), C.byref(ls), C.byref(guard), M, N, K, a_rows, row0,
                                      act, loss, np_parts, grid, device))
    return dZ, g_bL, g_wo, float(gbo.value), float(ls.value), int(guard.value)


def debug_out_layer(precision: int, A: np.ndarray, wo: np.ndarray, bo: float, act: int, loss: int,
                    y: Optional[np.ndarray] = None, w: Optional[np.ndarray] = None, do_loss: bool = True, do_bwd: bool = True,
                    det: bool = False, g_bL: Optional[np.ndarray] = None, g_wo: Optional[np.ndarray] = None, g_bo: float = 0.0,
                    loss_sum: float = 0.0, sms: int = 0, M: Optional[int] = None, H: Optional[int] = None, device: int = 0):
    """The output layer of a step on its own (sb_debug_out_layer) through the step's launch code, on A_L = A [M, H]
    (M, H default to A's shape), wo [H], y / w [M] (do_loss).  g_bL, g_wo [H], g_bo and loss_sum are the initial values the
    kernel adds into (zeros by default).  -> dict with yhat [M], dZ [np, M, H] (fp32 of the stored parts), g_bL, g_wo,
    g_bo, loss_sum, guard (changed sentinel elements), repeat_same (det: 1 if a second launch gave the same bits, else
    -1) and route (the kernel instantiation)"""
    A, wo = _f32(A), _f32(wo)
    M = A.shape[0] if M is None else M
    H = A.shape[1] if H is None else H
    nparts = PARTS.get(precision, 1)
    y = None if y is None else _f32(y).reshape(-1)
    w = None if w is None else _f32(w).reshape(-1)
    yhat = np.zeros(max(M, 0), np.float32)
    dZ = np.zeros((nparts, max(M, 0), max(H, 0)), np.float32)
    g_bL = _f32(g_bL).copy() if g_bL is not None else np.zeros(max(H, 0), np.float32)
    g_wo = _f32(g_wo).copy() if g_wo is not None else np.zeros(max(H, 0), np.float32)
    gbo, ls, guard, same = C.c_float(g_bo), C.c_float(loss_sum), C.c_int32(-1), C.c_int32(-1)
    route = C.create_string_buffer(64)
    check(lib().sb_debug_out_layer(precision, int(det), int(do_loss), int(do_bwd), _ptr(A), _ptr(wo), float(bo), _ptr(y), _ptr(w),
                                   _ptr(yhat), _ptr(dZ), _ptr(g_bL), _ptr(g_wo), C.byref(gbo), C.byref(ls), C.byref(guard),
                                   C.byref(same), route, 64, M, H, act, loss, sms, device))
    return dict(yhat=yhat, dZ=dZ, g_bL=g_bL, g_wo=g_wo, g_bo=float(gbo.value), loss_sum=float(ls.value),
                guard=int(guard.value), repeat_same=int(same.value), route=route.value.decode())


def debug_embed(precision: int, idx: np.ndarray, n_onehot: int, H: int, We: Optional[np.ndarray] = None,
                dZ: Optional[np.ndarray] = None, grad: Optional[np.ndarray] = None, device: int = 0):
    """The wide+deep embedding kernels of a sparse step (sb_debug_embed) through the step's launch code, idx [rows, n_cat]:
    dZ None: the gather of W_e [n_onehot, H] -> E [rows, H]; dZ [rows, H] given: the scatter-add into W_e's gradient
    rows, grad [n_onehot, H] their initial value (zeros by default) -> the rows after it.  -> (result, guard count)"""
    idx = np.ascontiguousarray(idx, dtype=np.int32)
    rows, n_cat = idx.shape if idx.ndim == 2 else (0, 0)
    scatter = dZ is not None
    We = None if We is None else _f32(We)
    dZ = None if dZ is None else _f32(dZ)
    out = (np.zeros((n_onehot, H), np.float32) if grad is None else _f32(grad).copy()) if scatter else np.zeros((rows, H), np.float32)
    guard = C.c_int32(-1)
    check(lib().sb_debug_embed(precision, int(scatter), _ptr(We), idx.ctypes.data_as(_P(C.c_int32)), _ptr(dZ), _ptr(out),
                               C.byref(guard), rows, H, n_onehot, n_cat, device))
    return out, int(guard.value)


def text_parse_device(text: bytes, col_map: Sequence[int], n_feat: int, delim: str = "|", device: int = 0, flag_cap: int = 65536):
    """sb_text_parse_device: -> (X DeviceArray [rows, n_feat], y DeviceArray [rows], w DeviceArray [rows], flags, text, kernel_ms)"""
    if not text.endswith(b"\n"):
        text = text + b"\n"
    cm = (C.c_int32 * len(col_map))(*[int(c) for c in col_map])
    dX, dy, dw = _f32p(), _f32p(), _f32p()
    flags = (CellFlag * flag_cap)()
    n_rows, n_flags, kms = C.c_int64(0), C.c_int64(0), C.c_float(0)
    check(lib().sb_text_parse_device(text, len(text), delim.encode()[:1], cm, len(col_map), n_feat, C.byref(dX), C.byref(dy), C.byref(dw),
                                     C.byref(n_rows), flags, flag_cap, C.byref(n_flags), device, C.byref(kms)))
    if n_flags.value > flag_cap:
        raise ShifuB200Error(SB_ERR_FORMAT, "%d cells need the slow path, more than flag_cap=%d" % (n_flags.value, flag_cap))
    fl = [(int(flags[i].row), int(flags[i].slot), int(flags[i].offset), int(flags[i].len)) for i in range(n_flags.value)]
    n = n_rows.value
    return DeviceArray(dX, (n, n_feat), device), DeviceArray(dy, (n,), device), DeviceArray(dw, (n,), device), fl, text, float(kms.value)


def text_parse(text: bytes, col_map: Sequence[int], n_feat: int, delim: str = "|", device: int = 0, host_debug: bool = False,
               flag_cap: int = 65536):
    """GPU ingest of delimiter-separated numeric text -> (X [rows, n_feat] f32, y [rows] f32, w [rows] f32, flags).
    flags = [(row, slot, offset, length)] for cells the exact fast path declined; the caller resolves them with float().
    host_debug=True runs the identical state machine on the host (unit tests only)."""
    if not text.endswith(b"\n"):
        text = text + b"\n"
    max_rows = text.count(b"\n")
    cm = (C.c_int32 * len(col_map))(*[int(c) for c in col_map])
    X = np.zeros((max_rows, n_feat), np.float32)
    y = np.zeros(max_rows, np.float32)
    w = np.ones(max_rows, np.float32)
    flags = (CellFlag * flag_cap)()
    n_rows, n_flags = C.c_int64(0), C.c_int64(0)
    args = [text, len(text), delim.encode()[:1], cm, len(col_map), n_feat, _ptr(X), _ptr(y), _ptr(w), max_rows, C.byref(n_rows),
            flags, flag_cap, C.byref(n_flags)]
    if host_debug:
        check(lib().sb_debug_text_parse_host(*args))
    else:
        check(lib().sb_text_parse(*args, device))
    if n_flags.value > flag_cap:
        raise ShifuB200Error(SB_ERR_FORMAT, "%d cells need the slow path, more than flag_cap=%d" % (n_flags.value, flag_cap))
    fl = [(int(flags[i].row), int(flags[i].slot), int(flags[i].offset), int(flags[i].len)) for i in range(n_flags.value)]
    n = n_rows.value
    return X[:n], y[:n], w[:n], fl, text
