"""Kernel-level checks of the wide+deep first layer's embedding kernels (kernels.cuh: embed_gather_kernel,
embed_scatter_kernel) through the sb_debug_embed hook, which launches them with the step's own Net::enqueue_embed on a
Net whose W_0 holds W_e below three dense rows.

Oracle: float64 of the same operation on the values the kernels read, with u = 2^-24:
  gather       E[r] = sum over c with idx[r, c] >= 0 of W_e[idx[r, c]] as stored (every bf16 shadow part, or the fp32
               row), within (n_cat np) u sum |terms|
  scatter-add  W_e's gradient row j gains the sum over every (r, c) with idx[r, c] = j of dZ_0[r] as stored (the sum of
               its parts, or fp32), in any order (red.global), within (count_j + np) u (sum |terms| + |init|); a row
               nobody selected keeps its initial value bit for bit
W_e's dense neighbours, b_0 and dZ_0's pad columns and rows past the batch hold NaN; the hook counts every write
outside E's batch columns or W_e's gradient rows."""
import numpy as np
import pytest

from oracle import wide_deep as wd
from wide_deep_ref import stored_parts

FP32, BF16, FP32_TC, BF16X2 = 0, 1, 2, 3
PRECS = {"fp32": FP32, "bf16": BF16, "fp32tc": FP32_TC, "bf16x2": BF16X2}
NP = {FP32: 1, BF16: 1, FP32_TC: 3, BF16X2: 2}
U = 2.0 ** -24
WIDTHS = [1, 3, 4, 5, 8, 12, 36, 127, 128, 129, 256, 257, 300, 1024]
ROWS = [1, 7, 8, 9, 130, 2048]
VOCAB = {1: [37], 4: [5, 9, 3, 17], 50: [7] * 50}
OUTS = ("gather", "scatter")

_worst = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if _worst:
        print("\nworst error / bound: " + ", ".join("%s %.3g" % (k, _worst[k]) for k in OUTS if k in _worst))


def _index(rows, n_cat, seed, hot=None):
    vocab = VOCAB[n_cat]
    _, idx, _, _ = wd.synth_wide_deep_batch(rows, 2, vocab, seed)
    if rows > 1:
        idx[1] = -1                         # a row with every value missing
    if hot is not None:
        idx[:, 0] = hot                     # every row selects the same embedding row
    return idx.astype(np.int32), int(sum(vocab))


def _note(name, err, tol):
    pos = tol > 0
    r = float(np.max(err[pos] / tol[pos])) if pos.any() else 0.0
    _worst[name] = max(_worst.get(name, 0.0), r)
    return r


def _gather(sb, prec, idx, n_onehot, H, seed):
    rng = np.random.RandomState(seed)
    We = (rng.standard_normal((n_onehot, H)) * 0.5).astype(np.float32)
    E, guard = sb.capi.debug_embed(prec, idx, n_onehot, H, We=We)
    assert guard == 0, "%d guard elements around E changed" % guard
    O = wd.onehot_matrix(idx, n_onehot, np.float64)
    parts = stored_parts(We, prec)
    want = O @ parts.sum(axis=0)
    tol = idx.shape[1] * NP[prec] * U * (O @ np.abs(parts).sum(axis=0))
    err = np.abs(E - want)
    r = _note("gather", err, tol)
    assert (err <= tol).all(), "gather off by %.3g x its bound at %s" % (r, np.unravel_index(np.argmax(err - tol), err.shape))


def _scatter(sb, prec, idx, n_onehot, H, seed):
    rng = np.random.RandomState(seed + 1)
    rows = idx.shape[0]
    dZ = rng.standard_normal((rows, H)).astype(np.float32)
    init = (rng.standard_normal((n_onehot, H)) * 0.1).astype(np.float32)
    got, guard = sb.capi.debug_embed(prec, idx, n_onehot, H, dZ=dZ, grad=init)
    assert guard == 0, "%d guard elements around W_e's gradient rows changed" % guard
    O = wd.onehot_matrix(idx, n_onehot, np.float64)
    parts = stored_parts(dZ, prec)
    count = O.sum(axis=0)[:, None]
    gain = O.T @ parts.sum(axis=0)
    tol = (count + NP[prec]) * U * (O.T @ np.abs(parts).sum(axis=0) + np.abs(init))
    err = np.abs(got.astype(np.float64) - init - gain)
    r = _note("scatter", err, tol)
    assert (err <= tol).all(), "scatter off by %.3g x its bound at %s" % (r, np.unravel_index(np.argmax(err - tol), err.shape))
    unused = count[:, 0] == 0
    assert got[unused].tobytes() == init[unused].tobytes(), "an embedding row nobody selected changed"


@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("H", WIDTHS)
@pytest.mark.parametrize("prec", sorted(PRECS))
def test_gather_and_scatter(sb, prec, H, rows):
    # H % 8 != 0: the gather's scalar tail; H % 4 != 0: the scatter's scalar red.global; H > 256: several passes per lane
    n_cat = sorted(VOCAB)[(WIDTHS.index(H) + ROWS.index(rows)) % len(VOCAB)]
    idx, n_onehot = _index(rows, n_cat, H + rows)
    _gather(sb, PRECS[prec], idx, n_onehot, H, H * 7 + rows)
    _scatter(sb, PRECS[prec], idx, n_onehot, H, H * 7 + rows)


@pytest.mark.gpu
@pytest.mark.parametrize("H", [5, 128, 257])
@pytest.mark.parametrize("n_cat", sorted(VOCAB))
@pytest.mark.parametrize("prec", sorted(PRECS))
def test_categorical_columns(sb, prec, n_cat, H):
    idx, n_onehot = _index(2048, n_cat, n_cat)
    _gather(sb, PRECS[prec], idx, n_onehot, H, n_cat)
    _scatter(sb, PRECS[prec], idx, n_onehot, H, n_cat)


@pytest.mark.gpu
@pytest.mark.parametrize("H", [3, 4, 129, 1024])
@pytest.mark.parametrize("prec", sorted(PRECS))
def test_hot_embedding_row(sb, prec, H):
    # 2048 rows add into one embedding row: 2048 atomics per element of that row
    idx, n_onehot = _index(2048, 4, 5, hot=11)
    _gather(sb, PRECS[prec], idx, n_onehot, H, 3)
    _scatter(sb, PRECS[prec], idx, n_onehot, H, 3)


# ------------------------------------------------------------------------------------------------------------ no GPU
def _call(sb, prec=FP32_TC, scatter=0, rows=8, H=16, n_onehot=10, n_cat=2, drop=(), bad_idx=None):
    import ctypes as C
    buf = {k: np.ones(4096, np.float32) for k in ("We", "dZ", "out")}
    for k in drop:
        buf[k] = None
    idx = np.zeros(4096, np.int32)
    if bad_idx is not None:
        idx[max(rows * n_cat - 1, 0)] = bad_idx
    guard = C.c_int32(-1)
    ptr = sb.capi._ptr
    return sb.capi.lib().sb_debug_embed(prec, scatter, ptr(buf["We"]), None if "idx" in drop else idx.ctypes.data_as(C.POINTER(C.c_int32)),
                                        ptr(buf["dZ"]), ptr(buf["out"]), None if "guard" in drop else C.byref(guard), rows, H,
                                        n_onehot, n_cat, 0)


INVALID = {
    "precision=4": dict(prec=4), "precision=-1": dict(prec=-1), "scatter=2": dict(scatter=2), "rows=0": dict(rows=0),
    "H=0": dict(H=0), "n_onehot=0": dict(n_onehot=0), "n_cat=0": dict(n_cat=0), "rows=-1": dict(rows=-1),
    "no_idx": dict(drop=("idx",)), "no_out": dict(drop=("out",)), "no_guard": dict(drop=("guard",)),
    "gather_no_We": dict(drop=("We",)), "scatter_no_dZ": dict(scatter=1, drop=("dZ",)),
    "idx=n_onehot": dict(bad_idx=10), "idx=-2": dict(bad_idx=-2), "idx=INT_MIN": dict(bad_idx=-2 ** 31),
    "scatter_idx=-2": dict(scatter=1, bad_idx=-2),
}


@pytest.mark.parametrize("case", sorted(INVALID))
def test_invalid_arguments_rejected_before_any_device_call(sb, case):
    # refused on a machine without a GPU, so no device work happens before the check
    assert _call(sb, **INVALID[case]) == sb.capi.SB_ERR_INVALID, sb.capi.lib().sb_last_error()
