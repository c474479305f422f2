"""float64 reference of an ensemble's column sensitivity and reason codes (sb_ensemble_sensitivity /
sb_ensemble_reason_codes), with a bound per (row, column) pair, built on sensitivity_ref.pair_scores.

Each member's pair score is held by sensitivity_ref as an interval [s - e, s + e].  The statistic S of the K member
scores is then bounded as an interval too:
  mean    the mean of the members' centres, half-width sum(e) / K plus the fp32 rounding of K - 1 adds and the divide,
          taken as (K + 1) u sum(|s| + e) / K
  max / min / median
          order statistics are monotone in every member score, so S lies between the statistic of the lower ends and
          that of the upper ends; the even-K median (a + b) * 0.5f adds one rounding, u max|end|
A delta d = S(base) - S(pair) is within the two intervals' half-widths plus u |d| for its fp32 subtraction."""
import numpy as np

from out_layer_ref import U
from sensitivity_ref import pair_scores

STATS = ("mean", "max", "min", "median")


def stat_interval(s, e, stat):
    """member scores s and their bounds e [K, ...] -> (centre, half-width) [...] of the statistic `stat`"""
    s, e = np.asarray(s, np.float64), np.asarray(e, np.float64)
    K = s.shape[0]
    if stat == "mean":
        mag = (np.abs(s) + e).sum(0)
        return s.mean(0), e.sum(0) / K + (K + 1) * U * mag / K
    lo, hi = s - e, s + e
    if stat == "max":
        a, b = lo.max(0), hi.max(0)
        return 0.5 * (a + b), 0.5 * (b - a)
    if stat == "min":
        a, b = lo.min(0), hi.min(0)
        return 0.5 * (a + b), 0.5 * (b - a)
    i, j = (K - 1) // 2, K // 2
    ls, hs = np.sort(lo, axis=0), np.sort(hi, axis=0)
    a, b = 0.5 * (ls[i] + ls[j]), 0.5 * (hs[i] + hs[j])
    r = 0.0 if i == j else U * np.maximum(np.abs(a), np.abs(b))
    return 0.5 * (a + b), 0.5 * (b - a) + r


def member_pair_scores(X, members, prec, cols, values):
    """members: [(layers, acts)] -> (s0, e0) [K, M] of the base rows and (s, e) [K, C, M] of the pairs, each member's
    float64 scores and bounds from sensitivity_ref.pair_scores"""
    base, pairs = [], []
    for layers, acts in members:
        b, p = pair_scores(X, layers, acts, prec, cols, values)
        base.append(b)
        pairs.append(p)
    s0 = np.stack([b[0] for b in base]), np.stack([b[1] for b in base])
    s = np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])
    return s0, s


def deltas(member_scores, stat):
    """member_pair_scores' result -> (d, bound) [M, C] of d = S(base) - S(pair), and (S(base), its bound) [M]"""
    (s0, e0), (s, e) = member_scores
    c0, h0 = stat_interval(s0, e0, stat)
    c, h = stat_interval(s, e, stat)
    d = c0[None, :] - c
    return (d.T, (h0[None, :] + h + U * np.abs(d)).T), (c0, h0)
