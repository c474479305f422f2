"""float64 reference of the optimizer update (opt_update in csrc/kernels.cuh) with error bounds, and the bf16 shadow bits a
refreshed run must hold; shared by the kernel tests of the single-GPU optimizer pass (test_optimizer_pass.py) and of the
peer exchange (test_exchange_kernels.py).

Bounds for the master and state.  u = 2^-24; every float32 operation rounds once (an FMA once for two), so an
expression of k operations is within about k u of its terms' magnitudes, and an input error e of a later operand
propagates with its coefficient.  With S the sum of the magnitudes of an expression's terms the check is
|got - ref| <= C u S, C = 16 (at least twice the operation count of the longest chain below):
  SGD        theta' = theta - lr g                               S_t = |theta| + lr |g|
  Momentum   s1' = s1 m + g                                      S_1 = |s1| m + |g|
             theta' = theta - lr s1'                             S_t = |theta| + lr S_1
  Adam       s1' = s1 + (g - s1)(1 - b1)                         S_1 = |s1| + (1 - b1)(|g| + |s1|)
             s2' = s2 + (g g - s2)(1 - b2)                       S_2 = s2 + (1 - b2)(g g + s2)  (<= 3 s2' / b2: no
                                                                 cancellation, the terms are >= 0)
             theta' = theta - lr s1' / (sqrt(s2') + eps)         S_t = |theta| + lr S_1 / D + |step| (1 + S_2 / (2 s2'))
                                                                 (D = sqrt(s2') + eps; sqrt halves s2's relative error)
  Adadelta   s1' = s1 rho + g g (1 - rho)                        S_1 = s1 rho + g g (1 - rho)
             upd = sqrt(s2 + eps) / sqrt(s1' + eps) g            S_u = |upd| (1 + S_1 / (2 (s1' + eps)))
             s2' = s2 rho + upd upd (1 - rho)                    S_2 = s2 rho + 3 upd upd (1 - rho)
             theta' = theta - upd lr                             S_t = |theta| + lr S_u
The TF 1.x forms of the later three (s1 >= 0 throughout; Adagrad's and FTRL's accum > 0):
  Adagrad    s1' = s1 + g g                                      S_1 = s1 + g g
             theta' = theta - lr g / sqrt(s1')                   S_t = |theta| + |step| (1 + S_1 / (2 s1'))
  RMSProp    s1' = s1 + (g g - s1)(1 - rho)                      S_1 = s1 + (1 - rho)(g g + s1)
             q = lr g / sqrt(s1' + eps)                          S_q = |q| (1 + (S_1 + eps) / (2 (s1' + eps)))
             s2' = m s2 + q                                      S_2 = m |s2| + S_q
             theta' = theta - s2'                                S_t = |theta| + S_2
  FTRL       a = s1 + g g, sa = sqrt(a), r = sqrt(s1)            S_a = s1 + g g
             d = sa - r  (cancels: both terms carry their own    S_d = sa (1 + S_a / (2 a)) + r
             error, not one relative to d)
             s2' = s2 + g - d / lr theta                         S_2 = |s2| + |g| + S_d |theta| / lr
             Q = sa / lr + 2 l2                                  S_Q = sa (1 + S_a / (2 a)) / lr + 2 l2
             theta' = |s2'| > l1 ? (sgn(s2') l1 - s2') / Q : 0   S_t = (l1 + |s2'| + S_2) / Q + |theta'| S_Q / Q
             (s1' = a, S_1 = S_a).  The branch itself is checked apart from the bound: where |s2'| < l1 - C u S_2 the
             kernel's theta' is +0.0, where |s2'| > l1 + C u S_2 it is non-zero.
1 - beta and 1 - rho are exact in float32 for beta, rho in [1/2, 1] (Sterbenz), so the reference uses the same constants.
An exact case (SGD, lr = 2^-4, gscale = 1/4, dyadic theta and gradients with few bits) has no rounding anywhere and must
match the float64 result bit for bit."""
import math

import numpy as np

from conftest import bf16_round

FP32, BF16, FP32_TC, BF16X2 = 0, 1, 2, 3
PNAME = {FP32: "fp32", BF16: "bf16", FP32_TC: "fp32_tc", BF16X2: "bf16x2"}
NPARTS = {FP32: 1, BF16: 1, FP32_TC: 3, BF16X2: 2}
ADADELTA, ADAM, SGD, MOMENTUM, ADAGRAD, RMSPROP, FTRL = 0, 1, 2, 3, 4, 5, 6
ONAME = {ADADELTA: "adadelta", ADAM: "adam", SGD: "sgd", MOMENTUM: "momentum", ADAGRAD: "adagrad", RMSPROP: "rmsprop",
         FTRL: "ftrl"}
EXT = (ADAGRAD, RMSPROP, FTRL)          # opt_group: the rules of the OPT_EXT instantiations
U = 2.0 ** -24
C_BOUND = 16.0
RHO, EPS, BETA1, BETA2, MOM = 0.95, 1e-8, 0.9, 0.999, 0.9


def uses_s1(kind):
    """the optimizer reads and writes s1 (opt_uses_s1)"""
    return kind != SGD


def uses_s2(kind):
    """the optimizer reads and writes s2 (opt_uses_s2)"""
    return kind not in (SGD, MOMENTUM, ADAGRAD)


def s1_start(kind, v):
    """raw s1 from a draw v: a squared-gradient accumulator (Adadelta, RMSProp) >= 0, Adagrad's and FTRL's accum > 0"""
    if kind in (ADAGRAD, FTRL):
        return (np.abs(v) + 0.01).astype(np.float32)
    return (np.abs(v) if kind in (ADADELTA, RMSPROP) else v).astype(np.float32)


def shadow_bits(theta, part):
    """bf16 bits of bf16_residual(theta, part), round to nearest even"""
    x = np.asarray(theta, np.float32).copy()
    for _ in range(part):
        x = (x - bf16_round(x)).astype(np.float32)
    return (bf16_round(x).view(np.uint32) >> 16).astype(np.uint16)


def reference(kind, lr, th, a, b, g, l1=0.0, l2=0.0):
    """float64 opt_update on float32 inputs -> (theta', s1', s2', S_t, S_1, S_2); l1 / l2: FTRL's strengths"""
    th, a, b, g = (np.asarray(v, np.float64) for v in (th, a, b, g))
    lr = float(lr)
    f = lambda v: float(np.float32(v))
    rho, eps, b1, b2, m = f(RHO), f(EPS), f(BETA1), f(BETA2), f(MOM)
    zero = np.zeros_like(th)
    if kind == SGD:
        return th - lr * g, a, b, np.abs(th) + lr * np.abs(g), zero, zero
    if kind == MOMENTUM:
        a2 = a * m + g
        S1 = np.abs(a) * m + np.abs(g)
        return th - lr * a2, a2, b, np.abs(th) + lr * S1, S1, zero
    if kind == ADAM:
        a2 = a + (g - a) * (1 - b1)
        b2_ = b + (g * g - b) * (1 - b2)
        S1 = np.abs(a) + (1 - b1) * (np.abs(g) + np.abs(a))
        S2 = b + (1 - b2) * (g * g + b)
        D = np.sqrt(b2_) + eps
        step = lr * a2 / D
        rel2 = np.divide(S2, 2 * b2_, out=np.zeros_like(S2), where=b2_ > 0)
        return th - step, a2, b2_, np.abs(th) + lr * S1 / D + np.abs(step) * (1 + rel2), S1, S2
    if kind == ADADELTA:
        a2 = a * rho + g * g * (1 - rho)
        S1 = a * rho + g * g * (1 - rho)
        upd = np.sqrt(b + eps) / np.sqrt(a2 + eps) * g
        Su = np.abs(upd) * (1 + S1 / (2 * (a2 + eps)))
        b2_ = b * rho + upd * upd * (1 - rho)
        S2 = b * rho + 3 * upd * upd * (1 - rho)
        return th - upd * lr, a2, b2_, np.abs(th) + lr * Su, S1, S2
    if kind == ADAGRAD:
        a2 = a + g * g
        S1 = a + g * g
        step = lr * g / np.sqrt(a2)
        return th - step, a2, b, np.abs(th) + np.abs(step) * (1 + S1 / (2 * a2)), S1, zero
    if kind == RMSPROP:
        a2 = a + (g * g - a) * (1 - rho)
        S1 = a + (1 - rho) * (g * g + a)
        q = lr * g / np.sqrt(a2 + eps)
        Sq = np.abs(q) * (1 + (S1 + eps) / (2 * (a2 + eps)))
        b2_ = m * b + q
        S2 = m * np.abs(b) + Sq
        return th - b2_, a2, b2_, np.abs(th) + S2, S1, S2
    if kind == FTRL:
        l1, l2 = f(l1), f(l2)
        acc = a + g * g
        Sa = a + g * g
        sa, r = np.sqrt(acc), np.sqrt(a)
        Ssa = sa * (1 + Sa / (2 * acc))
        d = sa - r
        Sd = Ssa + r
        b2_ = b + g - d / lr * th
        S2 = np.abs(b) + np.abs(g) + Sd * np.abs(th) / lr
        Q = sa / lr + 2 * l2
        SQ = Ssa / lr + 2 * l2
        t2 = np.where(np.abs(b2_) > l1, (np.sign(b2_) * l1 - b2_) / Q, 0.0)
        return t2, acc, b2_, (l1 + np.abs(b2_) + S2) / Q + np.abs(t2) * SQ / Q, Sa, S2
    raise ValueError(kind)


def lr_t_of(kind, lr, step):
    if kind != ADAM:
        return float(np.float32(lr))
    b1, b2 = float(np.float32(BETA1)), float(np.float32(BETA2))
    return float(np.float32(lr)) * math.sqrt(1 - b2 ** step) / (1 - b1 ** step)


def check_l1_branch(kind, got_theta, ref_s2, S2, l1, what):
    """FTRL: theta' is +0.0 (bit for bit) where the reference's |s2'| is clearly at most l1, non-zero where it is clearly
    above; elements within C u S_2 of l1 only meet the continuous bound"""
    if kind != FTRL:
        return
    l1 = float(np.float32(l1))
    band = C_BOUND * U * S2
    inside = np.abs(ref_s2) < l1 - band
    outside = np.abs(ref_s2) > l1 + band
    bits = np.asarray(got_theta, np.float32).view(np.uint32)
    bad = np.flatnonzero(inside & (bits != 0))
    assert bad.size == 0, "%s: %d elements with |s2'| < l1 are not +0.0, first at %s: %r" % (
        what, bad.size, bad[:8], np.asarray(got_theta)[bad[:8]])
    bad = np.flatnonzero(outside & (np.asarray(got_theta) == 0))
    assert bad.size == 0, "%s: %d elements with |s2'| > l1 are 0, first at %s" % (what, bad.size, bad[:8])


def _bits_equal(got, want, what):
    g, w = np.asarray(got), np.asarray(want)
    gv = g.view(np.uint32 if g.dtype == np.float32 else np.uint16)
    wv = w.view(np.uint32 if w.dtype == np.float32 else np.uint16)
    bad = np.flatnonzero(gv.reshape(-1) != wv.reshape(-1))
    assert bad.size == 0, "%s: %d elements differ, first at %s: got %r want %r" % (
        what, bad.size, bad[:8], g.reshape(-1)[bad[:8]], w.reshape(-1)[bad[:8]])
