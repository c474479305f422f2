"""shifu-tensorflow_b200: H100-native tabular-DNN train / score hot path behind shifu-tensorflow's plug-in seams.

Only what the path needs lives here:
  csrc/        CUDA kernels (sm_90a: wgmma / TMA / mbarrier) + the C-ABI (include/shifu_b200.h)
  _capi.py     ctypes binding of that C-ABI
  trainer.py   host mirror of the reference worker script (ssgd_monitor.py): env-var contract, ModelConfig.json,
               load_data, batch schedule, metrics socket line, SavedModel export
  scorer.py    host mirror of the reference Java scorer (TensorflowModel: init / compute / releaseResource), and its
               bagged form (TensorflowEnsemble: every member of a run's models/ per row, with their statistics), and
               computePerformance on both (AUC, average precision, KS and the gains / ROC / PR tables of a scored set)
"""
from . import _capi as capi  # noqa: F401
from ._capi import (Trainer, Model, Ensemble, Performance, NetDesc, make_desc, ShifuB200Error,  # noqa: F401
                    ACT_SIGMOID, ACT_TANH, ACT_RELU, ACT_LEAKYRELU, ACT_NONE,
                    LOSS_MSE, LOSS_SIGMOID_CE, OPT_ADADELTA, OPT_ADAM, OPT_SGD, OPT_MOMENTUM,
                    OPT_ADAGRAD, OPT_RMSPROP, OPT_FTRL, OPT_RPROP,
                    PREC_FP32, PREC_BF16, PREC_FP32_TC, PREC_BF16X2)

__all__ = ["capi", "Trainer", "Model", "Ensemble", "Performance", "NetDesc", "make_desc", "ShifuB200Error"]
