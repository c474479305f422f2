"""float64 reference of column sensitivity (sb_model_sensitivity) with a bound per (row, column) pair, built on
score_ref.py.

The library computes layer 0's pre-activation once per row and each pair (row r, list position k: column c set to v) as
the rank-1 update z0' = z0 + (v - x_c) W0[c, :], then runs layers 1..L and the output unit on the pair rows.  The
reference does the same in float64 on the model's view of the inputs (bf16(X), bf16(v) and the bf16 W0 shadow in BF16;
the fp32 values otherwise), which is the exact pre-activation of the modified row: rank1_scores equals brute-force
re-scoring of modified rows to float64 rounding (tests/test_sensitivity.py).

Bound of z0' (u = 2^-24, c = score_ref.contraction_c, S = |x| |W0| the original row's contraction magnitude):
  c S + 4u (|z0| + |b|)       z0 as score_ref bounds it: the GEMM's contraction and its fp32 result (the GEMM stores its
                              fp32 accumulator, or in FP32 the fp32 sum with the bias)
  (c + 4u) (|x_c| + |v|) |W0[c]|   the update: the delta is formed from the bf16 parts of x_c and v times W0's parts, so
                              it leaves out the same part products the GEMM leaves out for the row (c relative to the
                              term's magnitude, taken for the removed term x_c W0[c] and the added term v W0[c]), and
                              its products round in fp32
  4u (|z0'| + |b|)            two fp32 roundings of z0': the update's add and the bias add (FP32: one fused add)
The base slot (delta 0) gets the same bound with the update term 0.  From z0' on, every layer is bounded as score_ref
does it (BF16: the stored value as an interval of bf16 values; otherwise the exact model with contraction, activation
and part-storage terms, the inputs' errors carried in quadrature), and the output unit is out_layer_ref.output_layer.
A delta d = s(base) - s(pair) is within the sum of the two scores' bounds, plus u |d| for its fp32 subtraction."""
import numpy as np

from conftest import bf16_round
from out_layer_ref import U, activation
from score_ref import BF16, FP32, NPARTS, _carried, _e_act, contraction_c, out_unit


def model_view(X, prec):
    """the inputs as layer 0's GEMM sees them, float64"""
    X = np.asarray(X, np.float32)
    return (bf16_round(X) if prec == BF16 else X).astype(np.float64)


def _layers_from(z, e_z, layers, acts, prec):
    """(z0, its bound) [M, N0] -> (y_hat, bound) [M]: layer 0's activation and store, layers 1..L and the output unit,
    bounded as score_ref.hidden_forward / score bound them"""
    bf = prec == BF16
    a = e = None
    for li, ((W, b), act) in enumerate(zip(layers[:-1], acts)):
        if li > 0:
            Wm = (bf16_round(W) if bf else W).astype(np.float64)
            b64 = b.astype(np.float64)
            z = a @ Wm + b64
            e_z = contraction_c(prec, W.shape[0]) * (np.abs(a) @ np.abs(Wm)) + 4 * U * (np.abs(z) + np.abs(b64)) + _carried(e, Wm)
        v = activation(z, act)
        if bf:
            with np.errstate(over="ignore"):
                lo = bf16_round((activation(z - e_z, act) - _e_act(v, act)).astype(np.float32)).astype(np.float64)
                hi = bf16_round((activation(z + e_z, act) + _e_act(v, act)).astype(np.float32)).astype(np.float64)
            a, e = 0.5 * (lo + hi), 0.5 * (hi - lo)
        else:
            a = v
            e = e_z + _e_act(v, act)
            if prec != FP32:
                e = e + 2.0 ** (1 - 8 * NPARTS[prec]) * np.abs(v)
    if NPARTS[prec] > 1:
        e = e + 2 * U * np.abs(a)
    M = a.shape[0]
    wo, bo = layers[-1]
    r = out_unit(a, e, wo, bo, np.zeros(M, np.float32), np.ones(M, np.float32), acts[-1], 0, 1)["yhat"]
    return r


def pair_scores(X, layers, acts, prec, cols, values, block=32):
    """-> (s0, e0) [M] of the base rows and (s, e) [K, M] of the pairs (list position k, row r): float64 scores in
    precision mode prec and their bounds (module docstring)"""
    W0, b0 = layers[0]
    xm = model_view(X, prec)
    Wm = (bf16_round(W0) if prec == BF16 else W0).astype(np.float64)
    vm = model_view(np.asarray(values, np.float32), prec)
    b64 = b0.astype(np.float64)
    c = contraction_c(prec, W0.shape[0])
    z0 = xm @ Wm
    S = np.abs(xm) @ np.abs(Wm)
    z = z0 + b64

    def bound(zp, upd):
        return c * S + 4 * U * (np.abs(z) + np.abs(b64)) + upd + 4 * U * (np.abs(zp) + np.abs(b64))

    s0, e0 = _layers_from(z, bound(z, 0.0), layers, acts, prec)
    K, M = len(cols), xm.shape[0]
    s, e = np.empty((K, M)), np.empty((K, M))
    for k0 in range(0, K, block):
        ks = range(k0, min(K, k0 + block))
        zs, es = [], []
        for k in ks:
            col = int(cols[k])
            xc = xm[:, col:col + 1]
            zp = z + (vm[k] - xc) * Wm[col]
            zs.append(zp)
            es.append(bound(zp, (c + 4 * U) * (np.abs(xc) + abs(vm[k])) * np.abs(Wm[col])))
        yh, eb = _layers_from(np.concatenate(zs), np.concatenate(es), layers, acts, prec)
        s[k0:k0 + len(ks)] = yh.reshape(len(ks), M)
        e[k0:k0 + len(ks)] = eb.reshape(len(ks), M)
    return (s0, e0), (s, e)


def _plain_forward(a, layers, acts, bf):
    for (W, b), act in zip(layers[:-1], acts):
        Wm = (bf16_round(W) if bf else W).astype(np.float64)
        a = activation(a @ Wm + b.astype(np.float64), act)
    wo, bo = layers[-1]
    return activation(a @ np.asarray(wo, np.float64) + np.float64(bo), 0)


def rank1_scores(X, layers, acts, prec, cols, values):
    """[K, M] float64 scores of the pairs through the rank-1 update of layer 0 (no bounds)"""
    W0, b0 = layers[0]
    bf = prec == BF16
    xm, vm = model_view(X, prec), model_view(np.asarray(values, np.float32), prec)
    Wm = (bf16_round(W0) if bf else W0).astype(np.float64)
    z = xm @ Wm + b0.astype(np.float64)
    out = []
    for k, col in enumerate(cols):
        zp = z + (vm[k] - xm[:, col:col + 1]) * Wm[col]
        a = activation(zp, acts[0])
        out.append(_plain_forward(a, layers[1:], acts[1:], bf))
    return np.array(out)


def brute_scores(X, layers, acts, prec, cols, values):
    """[K, M] float64 scores of the modified rows, each re-scored in full"""
    out = []
    for k, col in enumerate(cols):
        Xk = np.array(X, np.float32)
        Xk[:, col] = np.float32(values[k])
        out.append(_plain_forward(model_view(Xk, prec), layers, acts, prec == BF16))
    return np.array(out)
