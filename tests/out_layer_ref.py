"""float64 reference of the output layer with error bounds, shared by the output-layer kernel tests (test_gemm_fwd_out.py:
A_L from the fused GEMM; test_out_layer.py: A_L as an input).

Given a = A_L [M, H] known within e_a, with u = 2^-24:
  z               e_z = sum_c |w_o| e_a + (H + 4) u (sum_c |a w_o| + |b_o|)
  y_hat           e_yh = y_hat (1 - y_hat) e_z exp(e_z) + 8u y_hat + 2^-147   (sigmoid' varies by at most exp(e_z) over
                  the interval; expf / division a few ulp; expf of a very negative z is subnormal)
  dz              e_dz = |w| / n_nz (0.625 e_z + 16u) + 8u |dz|      (|d dz / dz| <= 0.625 |w| / n_nz for MSE)
  loss term       e_l = |w| (e_z + 8u (|z| + 1))                       (|d loss / dz| <= |w|)
  g = dZ_L        e_g = 2 |dz w_o| e_a + |w_o| e_dz + 4u |g|          (|act''| <= 2 in terms of the output)
  sums            the sum of the terms' bounds + d u sum |terms|, d = the depth of the kernel's reduction
e_a carries a few ulp of the act' evaluation besides the error of a itself.  relu / leakyrelu: where a may sit on the
wrong side of the kink (`kink`), act' may flip; such an element is left out of the element-wise dZ check and its flip
|dz w_o| (1 - alpha) is added to the bound of its db_L column."""
import numpy as np

ACTS = {"sigmoid": 0, "tanh": 1, "relu": 2, "leakyrelu": 3, "none": -1}
MSE, CE = 0, 1
LOSSES = {"mse": MSE, "ce": CE}
U = 2.0 ** -24
ALPHA = 0.2


def activation(z, act):
    if act == ACTS["sigmoid"]:
        return 1.0 / (1.0 + np.exp(-z))
    if act == ACTS["tanh"]:
        return np.tanh(z)
    if act == ACTS["relu"]:
        return np.maximum(z, 0.0)
    if act == ACTS["leakyrelu"]:
        return np.where(z > 0, z, ALPHA * z)
    return z


def act_grad(a, act):
    if act == ACTS["sigmoid"]:
        return a * (1.0 - a)
    if act == ACTS["tanh"]:
        return 1.0 - a * a
    if act == ACTS["relu"]:
        return (a > 0).astype(np.float64)
    if act == ACTS["leakyrelu"]:
        return np.where(a > 0, 1.0, ALPHA)
    return np.ones_like(a)


def output_layer(a, e_a, wo, bo, y, w, act, loss, d, kink=None, e_z_add=0.0):
    """float64 values and bounds (module docstring) of every output of the layer on a [M, H] (float64) within e_a:
    y_hat, g = dZ_L and e_g, and (value, bound) of db_L, dw_o, db_o and the loss sum for a reduction depth d.
    e_z_add [M]: a bound on z the caller derived itself, added to e_z"""
    f64 = np.float64
    wo64 = wo.astype(f64)
    H = a.shape[1]
    aw = a * wo64
    z = aw.sum(axis=1) + f64(bo)
    e_z = e_a @ np.abs(wo64) + (H + 4) * U * (np.abs(aw).sum(axis=1) + abs(f64(bo))) + e_z_add
    yh = 1.0 / (1.0 + np.exp(-z))
    y64, w64 = y.astype(f64), w.astype(f64)
    nnz = np.count_nonzero(w)
    inv = 1.0 / nnz if nnz else 0.0
    if loss == MSE:
        per = w64 * (yh - y64) ** 2
        dz = 2 * w64 * (yh - y64) * yh * (1 - yh) * inv
    else:
        per = w64 * (np.maximum(z, 0) - z * y64 + np.log1p(np.exp(-np.abs(z))))
        dz = w64 * (yh - y64) * inv
    e_per = np.abs(w64) * (e_z + 8 * U * (np.abs(z) + 1))
    e_dz = np.abs(w64) * inv * (0.625 * e_z + 16 * U) + 8 * U * np.abs(dz)
    dzw = np.abs(dz)[:, None] * np.abs(wo64)[None, :]
    g = dz[:, None] * wo64[None, :] * act_grad(a, act)
    e_g = 2 * dzw * e_a + np.abs(wo64)[None, :] * e_dz[:, None] + 4 * U * np.abs(g)
    if kink is not None:
        flip = np.where(kink, dzw * (1.0 - (ALPHA if act == ACTS["leakyrelu"] else 0.0)), 0.0)
    else:
        kink = np.zeros(a.shape, bool)
        flip = 0.0
    dza = dz[:, None] * a
    return {"yhat": (yh, yh * (1 - yh) * e_z * np.exp(e_z) + 8 * U * yh + 2.0 ** -147),
            "g": g, "e_g": e_g, "kink": kink,
            "db_L": (g.sum(axis=0), (e_g + flip).sum(axis=0) + d * U * np.abs(g).sum(axis=0)),
            "dw_o": (dza.sum(axis=0), (np.abs(dz)[:, None] * e_a + np.abs(a) * e_dz[:, None]).sum(axis=0)
                     + d * U * np.abs(dza).sum(axis=0)),
            "db_o": (dz.sum(), e_dz.sum() + d * U * np.abs(dz).sum()),
            "loss": (per.sum(), e_per.sum() + d * U * np.abs(per).sum()),
            "d": d}
