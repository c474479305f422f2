"""The definitions of include/shifu_b200.h's sb_perf_* restated in float64 and exact integers (numpy int64 never
overflows here: every count product is below 2^62 for at most 2^31 - 1 rows).

runs()      the run table: t_j (the distinct scores, highest first, -0 folded into +0), TP_j, FP_j (int64) and WTP_j, WFP_j
            (float64 cumulative sums in row order within a run and run order across runs).
summary()   the metrics from a run table; auc and ks from exact integers and one fp64 division, as the header defines them.
points()    the operating points by their definitions: the first run whose axis value reaches the level, or the last run
            whose threshold reaches it.

Bounds.  The device sums the same non-negative fp64 terms as runs() in another fixed association.  Any association of k
non-negative terms is within (k - 1) u of their exact sum S (u = 2^-53), so a cumulative weight of the device and of runs()
differ by at most g S with g = 2 n u (weight_bound).  The metrics follow by Abel summation (a sum of increments of one
monotone sequence weighted by a bounded monotone or bounded-variation one moves by at most the sequences' error times the
other's total variation), plus m u for the m-term sums and a few u for the divisions:
    w_auc:  3 g + (m + 8) u                      (g for WFP against TV(WTP) + WTP_m = 2 Wp, g Wp Wn for WTP)
    ap:     (m + 8) u                            (exact counts: one rounded division per term)
    w_ap:   2 g (TV(r) + 1) + (m + 8) u           r_j = WTP_j / (WTP_j + WFP_j), the precision along the table
    w_ks:   4 g + 8 u                            (both products and both totals perturbed by g)
each doubled, since runs() itself has the same error (metric_bounds)."""
import numpy as np

U = 2.0 ** -53
AXES = ("action_rate", "recall", "fpr", "score")


def keys_order(s):
    """row indices sorted by descending score, ties in row order (the device's stable sort)"""
    s = np.asarray(s, np.float32) + np.float32(0.0)          # -0 -> +0
    return np.argsort(-s.astype(np.float64), kind="stable"), s


def runs(s, y, w=None):
    order, s = keys_order(s)
    ss = s[order]
    yy = np.asarray(y, np.float32)[order] == 1.0
    ww = np.ones(len(ss)) if w is None else np.asarray(w, np.float32)[order].astype(np.float64)
    if len(ss) == 0:
        z = np.zeros(0, np.int64)
        return {"t": np.zeros(0, np.float32), "tp": z, "fp": z, "w_tp": np.zeros(0), "w_fp": np.zeros(0)}
    tail = np.append(ss[1:] != ss[:-1], True)
    tp = np.cumsum(yy.astype(np.int64))[tail]
    fp = np.cumsum((~yy).astype(np.int64))[tail]
    w_tp = np.cumsum(np.where(yy, ww, 0.0))[tail]
    w_fp = np.cumsum(np.where(yy, 0.0, ww))[tail]
    return {"t": ss[tail], "tp": tp, "fp": fp, "w_tp": w_tp, "w_fp": w_fp}


def runs_from_counts(t, p, n, wp, wn):
    """a run table from per-run counts and weight sums, runs in descending t (e.g. a bincount of quantised scores)"""
    return {"t": np.asarray(t, np.float32), "tp": np.cumsum(p).astype(np.int64), "fp": np.cumsum(n).astype(np.int64),
            "w_tp": np.cumsum(np.asarray(wp, np.float64)), "w_fp": np.cumsum(np.asarray(wn, np.float64))}


def _prev(a):
    return np.concatenate([np.zeros(1, a.dtype), a[:-1]])


def summary(r):
    tp, fp, wtp, wfp, t = r["tp"], r["fp"], r["w_tp"], r["w_fp"], r["t"]
    m = len(t)
    nan = float("nan")
    out = {"n_distinct": m, "pos": int(tp[-1]) if m else 0, "neg": int(fp[-1]) if m else 0,
           "w_pos": float(wtp[-1]) if m else 0.0, "w_neg": float(wfp[-1]) if m else 0.0,
           "auc": nan, "w_auc": nan, "ap": nan, "w_ap": nan, "ks": nan, "w_ks": nan, "ks_score": nan, "w_ks_score": nan}
    if m == 0:
        return out
    P, N, Wp, Wn = out["pos"], out["neg"], out["w_pos"], out["w_neg"]
    tp0, fp0, wtp0, wfp0 = _prev(tp), _prev(fp), _prev(wtp), _prev(wfp)
    p, n = tp - tp0, fp - fp0
    if P * N > 0:
        a2 = int(np.sum(n * (2 * tp0 + p)))                  # int64, exact
        out["auc"] = float(a2) / float(2 * P * N)
        d = np.abs(tp * N - fp * P)
        j = int(np.argmax(d))                                # the first maximum
        out["ks"], out["ks_score"] = float(int(d[j])) / float(P * N), float(t[j])
    if P > 0:
        out["ap"] = float(np.sum(p / P * (tp / (tp + fp))))
    if Wp * Wn > 0:
        out["w_auc"] = float(np.sum((wfp - wfp0) * (wtp0 + (wtp - wtp0) / 2))) / (Wp * Wn)
        wd = np.abs(wtp * Wn - wfp * Wp)
        j = int(np.argmax(wd))
        out["w_ks"], out["w_ks_score"] = float(wd[j]) / (Wp * Wn), float(t[j])
    if Wp > 0:
        wp = wtp - wtp0
        with np.errstate(invalid="ignore", divide="ignore"):
            out["w_ap"] = float(np.sum(np.where(wp > 0, wp / Wp * (wtp / (wtp + wfp)), 0.0)))
    return out


def axis_values(r, axis, weighted):
    if weighted:
        tp, fp = r["w_tp"], r["w_fp"]
        P, N = (tp[-1], fp[-1]) if len(tp) else (0.0, 0.0)
    else:
        tp, fp = r["tp"], r["fp"]
        P, N = (int(tp[-1]), int(fp[-1])) if len(tp) else (0, 0)
    num, den = {"action_rate": (tp + fp, P + N), "recall": (tp, P), "fpr": (fp, N)}[axis]
    return np.asarray(num, np.float64), float(den)


def points(r, axis, levels, weighted=False):
    """-> list of (threshold, tp, fp, w_tp, w_fp) by a plain sweep over the table"""
    out = []
    m = len(r["t"])
    for lv in levels:
        if axis == "score":
            js = [j for j in range(m) if float(r["t"][j]) >= lv]
            j = js[-1] if js else None
        else:
            num, den = axis_values(r, axis, weighted)
            if den == 0:
                raise ValueError("axis undefined")
            j = next(j for j in range(m) if num[j] / den >= lv)
        if j is None:
            out.append((float("inf"), 0, 0, 0.0, 0.0))
        else:
            out.append((float(r["t"][j]), int(r["tp"][j]), int(r["fp"][j]), float(r["w_tp"][j]), float(r["w_fp"][j])))
    return out


def weight_bound(n):
    """|device - runs()| of a cumulative weight sum, relative to it"""
    return 2 * max(n, 1) * U


def metric_bounds(r, n):
    """absolute bounds on |device - summary()| of the weighted metrics and of ap (module docstring)"""
    g = 2 * weight_bound(n)                 # the device's and the reference's errors together
    m = len(r["t"])
    wtp, wfp = r["w_tp"], r["w_fp"]
    with np.errstate(invalid="ignore", divide="ignore"):
        prec = np.where(wtp + wfp > 0, wtp / (wtp + wfp), 0.0)
    tv = float(np.sum(np.abs(np.diff(prec)))) if m > 1 else 0.0
    mu = 2 * (m + 8) * U
    return {"w_auc": 3 * g + mu, "ap": mu, "w_ap": 2 * g * (tv + 1) + mu, "w_ks": 4 * g + 16 * U}
