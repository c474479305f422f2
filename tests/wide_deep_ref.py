"""float64 reference of the wide+deep forward with a bound per row, shared by the wide+deep path tests
(test_wide_deep_paths.py).  It is score_ref.py's model with layer 0's pre-activation evaluated sparsely, as the step's
embedding gather and layer-0 GEMM evaluate it (oracle/wide_deep.py):

    z0 = Xd W_d + E + b0,     E[r] = sum over c of W_e[idx[r, c]]   (idx = -1 adds nothing)

with u = 2^-24, a = Xd as layer 0 reads it (score_ref.stored_inputs) and E as the gather reads W_e: the fp32 rows (FP32),
the bf16 shadow (BF16), or the sum of the np bf16 parts (FP32_TC, BF16X2), whose truncation against the fp32 rows of the
exact model is added to the bound:
    e_z0 = contraction_c(prec, n_dense) |a| |W_d|                  the dense GEMM (score_ref.py)
         + n_cat np u sum |terms|  +  sum |parts - W_e|             the gather (test_embed.py) and the parts' truncation
         + 4u (|pre| + |E| + |b0|)                                 the epilogue's two fp32 adds (test_gemm_layer.py)
Layers 1..L, the BF16 rounding of every activation and the output unit are score_ref.hidden_forward / out_unit."""
import numpy as np

from conftest import bf16_round
from out_layer_ref import U
from score_ref import BF16, FP32, NPARTS, contraction_c, hidden_forward, scores, stored_inputs


def stored_parts(x, prec):
    """[np, ...] float64: x as the step stores it - its bf16 parts (bf16_residual), or the fp32 values"""
    if prec == FP32:
        return x.astype(np.float64)[None]
    r, parts = x.astype(np.float32), []
    for _ in range(NPARTS[prec]):
        p = bf16_round(r)
        parts.append(p.astype(np.float64))
        r = (r - p).astype(np.float32)
    return np.stack(parts)


def gather(T, idx):
    """[rows, H] float64: sum over c of T[idx[:, c]], -1 adding nothing"""
    out = np.zeros((idx.shape[0], T.shape[1]))
    for c in range(idx.shape[1]):
        j = idx[:, c]
        hit = j >= 0
        out[hit] += T[j[hit]]
    return out


def layer0_sparse(Xd, idx, W0, b0, prec):
    """-> (z0, e_z0) float64 [rows, h_0] of layer 0 on the dense block Xd [rows, n_dense] and the one-hot indices idx
    [rows, n_cat] (module docstring)"""
    n_dense = Xd.shape[1]
    Wd, We = W0[:n_dense], W0[n_dense:]
    a = stored_inputs(Xd, prec)
    Wdm = (bf16_round(Wd) if prec == BF16 else Wd).astype(np.float64)
    pre = a @ Wdm
    parts = stored_parts(We, prec)
    read = parts.sum(axis=0)                                  # the row the gather adds
    model = read if prec in (FP32, BF16) else We.astype(np.float64)
    E = gather(model, idx)
    e_E = idx.shape[1] * NPARTS[prec] * U * gather(np.abs(parts).sum(axis=0), idx) + gather(np.abs(read - model), idx)
    b64 = b0.astype(np.float64)
    z = pre + E + b64
    e_z = contraction_c(prec, n_dense) * (np.abs(a) @ np.abs(Wdm)) + e_E + 4 * U * (np.abs(pre) + np.abs(E) + np.abs(b64))
    return z, e_z


def hidden_forward_sparse(Xd, idx, layers, acts, prec, exact=None):
    """-> (A_L, e_a) as score_ref.hidden_forward, layer 0 evaluated sparsely"""
    W0, b0 = layers[0]
    return hidden_forward(None, layers, acts, prec, exact, z0=layer0_sparse(Xd, idx, W0, b0, prec))


def score_sparse(Xd, idx, layers, acts, prec, exact=None):
    """-> (y_hat, e_yhat) float64 [rows] of the wide+deep rows (Xd, idx) in precision mode prec"""
    return scores(*hidden_forward_sparse(Xd, idx, layers, acts, prec, exact), layers, acts)
