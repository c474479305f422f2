"""TEST INFRASTRUCTURE ONLY - the TF 1.x optimizers past the reference's four: Adagrad, RMSProp and FTRL, restated from
TF 1.x core/kernels/training_ops.cc (library code, not in the reference tree) like shifu_oracle.Optimizer's forms.

    Adagrad  (ApplyAdagrad)                    accum += g^2;  theta -= lr g / sqrt(accum)
    RMSProp  (ApplyRMSProp, not centered)      ms += (g^2 - ms)(1 - decay);  mom = momentum mom + lr g / sqrt(ms + eps);
                                               theta -= mom
    FTRL     (ApplyFtrl, lr_power = -0.5,      a' = accum + g^2;  linear += g - (sqrt(a') - sqrt(accum)) / lr theta;
              no l2 shrinkage)                 q = sqrt(a') / lr + 2 l2;
                                               theta = |linear| > l1 ? (sign(linear) l1 - linear) / q : 0;  accum = a'

State in the two streams of shifu_oracle.Optimizer: s1 = accum | ms | accum, s2 = - | mom | linear.  FTRL's theta does not
depend on the previous theta except through `linear`: a parameter whose |linear| <= l1 is exactly 0 (with l1 = 0 and a
zero gradient from the start, linear stays 0 and so does the parameter) - TF's arithmetic, kept.

Nothing under shifu-tensorflow_b200/ imports this file.  oracle/tf_golden_optimizers.py writes TF's own three steps of
each rule, so that a machine with TF pins them."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from . import shifu_oracle as so

OPT_ADAGRAD, OPT_RMSPROP, OPT_FTRL = 4, 5, 6

# TF 1.x constructor defaults of the hyperparameters that differ from shifu_oracle.OptConfig's
RMSPROP_DEFAULTS = dict(rho=0.9, eps=1e-10, momentum=0.0)       # tf.train.RMSPropOptimizer(decay, epsilon, momentum)


@dataclass
class OptConfig(so.OptConfig):
    initial_accumulator: float = 0.1   # Adagrad / FTRL initial_accumulator_value (TF default)
    l1: float = 0.0                    # FTRL l1_regularization_strength
    l2: float = 0.0                    # FTRL l2_regularization_strength
    # TF 1.x RMSPropOptimizer._create_slots builds its `rms` slot with a ones initializer (every other slot of every TF
    # optimizer starts at 0 or at initial_accumulator_value).  Unpinned by the reference, which never uses RMSProp;
    # default True, the C-ABI implements exactly this default.
    rmsprop_ms_starts_at_one: bool = True


def tf_config(kind: int, lr: float, **kw) -> OptConfig:
    """OptConfig with TF's defaults of `kind` (RMSProp: decay 0.9, epsilon 1e-10, momentum 0) under the caller's values"""
    base = dict(RMSPROP_DEFAULTS) if kind == OPT_RMSPROP else {}
    base.update(kw)
    return OptConfig(kind=kind, lr=lr, **base)


def initial_slots(cfg: so.OptConfig, n: int, dtype=np.float32):
    """(s1, s2) before the first update"""
    s1, s2 = np.zeros(n, dtype), np.zeros(n, dtype)
    if cfg.kind in (OPT_ADAGRAD, OPT_FTRL):
        s1[:] = cfg.initial_accumulator
    elif cfg.kind == OPT_RMSPROP and cfg.rmsprop_ms_starts_at_one:
        s1[:] = 1
    return s1, s2


class Optimizer(so.Optimizer):
    """shifu_oracle.Optimizer plus the three rules above; the reference's four are shifu_oracle's, unchanged"""

    def __init__(self, cfg: so.OptConfig, n: int, dtype=np.float32):
        super().__init__(cfg, n, dtype)
        self.s1, self.s2 = initial_slots(cfg, n, dtype)

    def apply(self, theta: np.ndarray, g: np.ndarray) -> np.ndarray:
        c, dt = self.cfg, theta.dtype.type
        if c.kind == OPT_ADAGRAD:
            self.t += 1
            self.s1 = self.s1 + g * g
            return theta - dt(c.lr) * g / np.sqrt(self.s1)
        if c.kind == OPT_RMSPROP:
            self.t += 1
            self.s1 = self.s1 + (g * g - self.s1) * (dt(1) - dt(c.rho))
            self.s2 = dt(c.momentum) * self.s2 + dt(c.lr) * g / np.sqrt(self.s1 + dt(c.eps))
            return theta - self.s2
        if c.kind == OPT_FTRL:
            self.t += 1
            lr = dt(c.lr)
            a = self.s1 + g * g
            sa = np.sqrt(a)
            self.s2 = self.s2 + (g - (sa - np.sqrt(self.s1)) / lr * theta)
            self.s1 = a
            q = sa / lr + dt(2) * dt(c.l2)
            l1 = dt(c.l1)
            return np.where(np.abs(self.s2) > l1, (np.sign(self.s2) * l1 - self.s2) / q, dt(0)).astype(theta.dtype)
        return super().apply(theta, g)


class CleanTrainer(so.CleanTrainer):
    def __init__(self, net, params, opt: so.OptConfig, loss=so.LOSS_MSE, dtype=np.float32):
        super().__init__(net, params, opt, loss, dtype)
        self.opt = Optimizer(opt, self.theta.size, dtype)


class Bf16Trainer(so.Bf16Trainer):
    def __init__(self, net, params, opt: so.OptConfig, loss=so.LOSS_MSE, fused_out=True):
        super().__init__(net, params, opt, loss, fused_out)
        self.opt = Optimizer(opt, self.theta.size, np.float32)


class SyncReplicasTrainer(so.SyncReplicasTrainer):
    def __init__(self, net, params, opt: so.OptConfig, R: int, loss=so.LOSS_MSE, dtype=np.float32):
        super().__init__(net, params, opt, R, loss, dtype)
        self.opt = Optimizer(opt, self.theta.size, dtype)
