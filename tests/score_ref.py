"""float64 reference of a model's score with a bound per row, shared by the scoring-path tests (test_score_paths.py).

Each row is carried through the hidden layers as a value a and a bound e_a, with u = 2^-24 and c the contraction constant
of the step's GEMMs (contraction_c: (K + 2) u for FP32, 3e-6 for np = 1 and 3 bf16 parts, 2e-5 for np = 2):
  FP32, FP32_TC, BF16X2   the exact model on the fp32 inputs and weights.  Per layer, with S = |a_{l-1}| |W|:
                            e_z = P(e_{l-1}, W) + c S + 4u (|pre| + |b|)      (the bias add and the fp32 pre-activation)
                            e_a = e_z + e_act                                 (every activation is 1-Lipschitz)
                          e_act = 4u (|a| + 1) for sigmoid / tanh (a few ulp of expf / tanhf), 4u |a| for relu, leakyrelu
                          and none (exact but for leakyrelu's one multiply).  Storing a as np bf16 parts adds
                          2^(1 - 8 np) |a|; FP32 stores a itself.
  BF16                    rounding-aware: the kernels round X and the W shadow to bf16, multiply exactly, accumulate in
                          fp32 and store each activation as bf16.  The reference does the same in float64 on bf16(X) and
                          bf16(W), with e_z as above.  Every activation is monotone, so the stored value lies in
                          [bf16(act(z - e_z) - e_act), bf16(act(z + e_z) + e_act)]: where both ends are the same bf16 value
                          the element is exact (bound 0), otherwise it is carried as the middle of the span, bound half of it.
P is the error a layer's inputs carry into its outputs.  The worst case e_{l-1} |W| grows by sum_k |W_kj| (~ 30 at the
eval net's widths) per layer and bounds nothing after three layers; the inputs' errors are separate roundings of separate
elements, so P adds them in quadrature: P = KAPPA sqrt(e_{l-1}^2 W^2), KAPPA = 4.  Every other term is a worst case.
The output unit is out_layer_ref.output_layer (y_hat and its bound) on A_L, with P(e_a, w_o) as the bound its inputs
carry; e_a includes 2u |a| where the kernel rebuilds A_L from its bf16 parts in fp32."""
import numpy as np

from conftest import bf16_round
from out_layer_ref import ACTS, MSE, U, activation, output_layer

FP32, BF16, FP32_TC, BF16X2 = 0, 1, 2, 3
NPARTS = {FP32: 1, BF16: 1, FP32_TC: 3, BF16X2: 2}
SMOOTH = (ACTS["sigmoid"], ACTS["tanh"])
KAPPA = 4.0


def contraction_c(prec, K):
    """the bound of a K-term contraction relative to the sum of its terms' magnitudes (test_gemm_layer.py's module
    docstring): the fp32 FMA chain, or the tensor-core contraction of 1, 2 or 3 bf16 parts"""
    return (K + 2) * U if prec == FP32 else {1: 3e-6, 2: 2e-5, 3: 3e-6}[NPARTS[prec]]


def unflatten(flat, F, hidden):
    """the flat parameter vector -> [(W [in, out], b [out]) per hidden layer] + [(w_o [H], b_o)] (fp32)"""
    flat = np.asarray(flat, np.float32).ravel()
    out, o, prev = [], 0, F
    for h in list(hidden) + [1]:
        W = flat[o:o + prev * h].reshape(prev, h)
        o += prev * h
        out.append((W, flat[o:o + h]))
        o += h
        prev = h
    assert o == flat.size, (o, flat.size)
    W, b = out[-1]
    return out[:-1] + [(W[:, 0], np.float32(b[0]))]


def _e_act(a, act):
    return 4 * U * (np.abs(a) + 1) if act in SMOOTH else 4 * U * np.abs(a)


def _carried(e, W):
    """P: the bound the inputs' errors e [M, K] carry through W [K, N] (module docstring)"""
    return KAPPA * np.sqrt((e * e) @ (W * W))


def stored_inputs(X, prec):
    """the rows as layer 0 reads them: bf16 in BF16, else fp32 (float64)"""
    return (bf16_round(X) if prec == BF16 else np.asarray(X, np.float32)).astype(np.float64)


def pre_activation(a, e, W, b, prec):
    """-> (z, e_z) float64: a W + b of inputs a within e (None: exact) and its bound (module docstring)"""
    Wm = (bf16_round(W) if prec == BF16 else W).astype(np.float64)
    b64 = b.astype(np.float64)
    z = a @ Wm + b64
    e_z = contraction_c(prec, W.shape[0]) * (np.abs(a) @ np.abs(Wm)) + 4 * U * (np.abs(z) + np.abs(b64))
    if e is not None:
        e_z += _carried(e, Wm)
    return z, e_z


def hidden_forward(X, layers, acts, prec, exact=None, z0=None):
    """-> (A_L, e_a) float64 [M, H_L]: the last hidden layer as the kernels store it, and its bound (module docstring).
    exact (a list): receives each BF16 layer's fraction of elements known exactly.  z0: (z, e_z) of layer 0's
    pre-activation, where the caller evaluates it itself (wide_deep_ref.py); X is then not read"""
    bf = prec == BF16
    a = None if z0 is not None else stored_inputs(X, prec)
    e = None                                         # the inputs are exact
    for l, ((W, b), act) in enumerate(zip(layers[:-1], acts)):
        z, e_z = z0 if (l == 0 and z0 is not None) else pre_activation(a, e, W, b, prec)
        v = activation(z, act)
        if bf:
            with np.errstate(over="ignore"):         # exp of a saturated sigmoid's argument
                lo = bf16_round((activation(z - e_z, act) - _e_act(v, act)).astype(np.float32)).astype(np.float64)
                hi = bf16_round((activation(z + e_z, act) + _e_act(v, act)).astype(np.float32)).astype(np.float64)
            a, e = 0.5 * (lo + hi), 0.5 * (hi - lo)
            if exact is not None:
                exact.append(float(np.mean(lo == hi)))
        else:
            a = v
            e = e_z + _e_act(v, act)
            if prec != FP32:
                e += 2.0 ** (1 - 8 * NPARTS[prec]) * np.abs(v)
    if NPARTS[prec] > 1:
        e = e + 2 * U * np.abs(a)
    return a, e


def out_unit(a, e_a, wo, bo, y, w, act, loss, d):
    """output_layer on A_L = a within e_a, its inputs' errors carried by P (y_hat and the loss; not the gradients)"""
    with np.errstate(over="ignore"):                 # exp(-z) of a saturated score: inf, and y_hat 0
        return output_layer(a, np.zeros_like(a), wo, bo, y, w, act, loss, d,
                            e_z_add=_carried(e_a, np.asarray(wo, np.float64)[:, None])[:, 0])


def validation_loss(a, e_a, wo, bo, y, w, act, B, depth):
    """-> (loss, bound) of a validation pass (Trainer.eval_loss, eval_loss_sparse) over A_L = a within e_a: the MSE sums of
    output_layer over pieces of at most B rows, added up and divided by n_nz.  depth(m): the reduction depth of the
    output-layer launch over a piece of m rows.  A set without a non-zero weight: (0, 0)"""
    n, nnz = len(y), np.count_nonzero(w)
    if nnz == 0:
        return 0.0, 0.0
    total, bound = 0.0, 0.0
    for r0 in range(0, n, B):
        s = slice(r0, min(n, r0 + B))
        ref = out_unit(a[s], e_a[s], wo, bo, y[s], w[s], act, MSE, depth(s.stop - s.start))
        total += ref["loss"][0]
        bound += ref["loss"][1] + ref["d"] * U * abs(ref["loss"][0])
    return total / nnz, bound / nnz + 2 * U * abs(total / nnz)


def scores(a, e, layers, acts):
    """-> (y_hat, e_yhat) float64 [M] of the output unit on A_L = a within e"""
    M = a.shape[0]
    wo, bo = layers[-1]
    return out_unit(a, e, wo, bo, np.zeros(M, np.float32), np.ones(M, np.float32), acts[-1], 0, 1)["yhat"]


def score(X, layers, acts, prec, exact=None):
    """-> (y_hat, e_yhat) float64 [M] of the rows X [M, F] (fp32) in precision mode prec"""
    return scores(*hidden_forward(X, layers, acts, prec, exact), layers, acts)
