"""numpy float32 restatement of RPROP (SB_OPT_RPROP, the iRPROP- form of Igel and Huesken), and the oracle's trainers with it.

The rule is what opt_update computes (csrc/kernels.cuh) and what torch.optim.Rprop(lr, etas=(0.5, 1.2),
step_sizes=(1e-6, 50)) computes, in torch's order, every operation one float32 rounding:

    p    = g * prev
    step = min(max(step * (p > 0 ? 1.2 : p < 0 ? 0.5 : 1), 1e-6), 50)     (clamped on every update)
    g    = p < 0 ? 0 : g                                                 (a sign flip: no move now, no flip next time)
    theta = g > 0 ? theta - step : g < 0 ? theta + step : theta          (g = +-0: theta keeps its bits)
    prev = g

prev starts at 0 and step at the learning rate, so a product that underflows to 0 counts as "no change", as in torch.
The Optimizer / trainers below are oracle/tf_optimizers.py's with this rule as optimizer 8; every other optimizer is
theirs, unchanged."""
import numpy as np

from oracle import shifu_oracle as so
from oracle import tf_optimizers as tfo

RPROP = 8
ETA_PLUS, ETA_MINUS = np.float32(1.2), np.float32(0.5)
STEP_MIN, STEP_MAX = np.float32(1e-6), np.float32(50.0)


def rprop_update(theta, g, prev, step):
    """one update on float32 arrays -> (theta', prev', step'); the inputs are not modified"""
    theta, g, prev, step = (np.asarray(v, np.float32) for v in (theta, g, prev, step))
    p = g * prev
    f = np.where(p > 0, ETA_PLUS, np.where(p < 0, ETA_MINUS, np.float32(1.0)))
    step = np.minimum(np.maximum(step * f, STEP_MIN), STEP_MAX)
    g = np.where(p < 0, np.float32(0.0), g)
    theta = np.where(g > 0, theta - step, np.where(g < 0, theta + step, theta))
    return theta, g, step


def start_state(lr, n):
    """(prev, step) before the first update"""
    return np.zeros(n, np.float32), np.full(n, np.float32(lr), np.float32)


class Optimizer(tfo.Optimizer):
    """tf_optimizers.Optimizer plus RPROP (float32 only): s1 = prev, s2 = step"""

    def __init__(self, cfg: so.OptConfig, n: int, dtype=np.float32):
        super().__init__(cfg, n, dtype)
        if cfg.kind == RPROP:
            assert dtype == np.float32, "RPROP is restated in float32"
            self.s1, self.s2 = start_state(cfg.lr, n)

    def apply(self, theta: np.ndarray, g: np.ndarray) -> np.ndarray:
        if self.cfg.kind != RPROP:
            return super().apply(theta, g)
        self.t += 1
        theta, self.s1, self.s2 = rprop_update(theta, g, self.s1, self.s2)
        return theta


class CleanTrainer(so.CleanTrainer):
    def __init__(self, net, params, opt: so.OptConfig, loss=so.LOSS_MSE, dtype=np.float32):
        super().__init__(net, params, opt, loss, dtype)
        self.opt = Optimizer(opt, self.theta.size, dtype)


class SyncReplicasTrainer(so.SyncReplicasTrainer):
    def __init__(self, net, params, opt: so.OptConfig, R: int, loss=so.LOSS_MSE, dtype=np.float32):
        super().__init__(net, params, opt, R, loss, dtype)
        self.opt = Optimizer(opt, self.theta.size, dtype)
