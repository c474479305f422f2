"""Kernel-level checks of the fused output-layer GEMM (gemm_fwd_out.cuh) through the sb_debug_gemm_fwd_out hook, which
launches it the way a training step does (last hidden layer N <= 256).

Oracle: float64 of the same operation, z = act(A W + b) . w_o + b_o, y_hat = sigmoid(z), the loss term and dz
(SUM_BY_NONZERO_WEIGHTS), g = dZ_L = dz w_o act'(a), and the sums db_L = sum_r g, dw_o = sum_r dz a, db_o = sum_r dz,
loss = sum_r loss term.  np = 1 takes A and W rounded to bf16 (the kernel then multiplies exactly and accumulates in
fp32); np = 2 / 3 takes the fp32 inputs (the kernel splits them into bf16 parts).

Tolerances follow the arithmetic, with u = 2^-24 (the output-layer half is out_layer_ref.output_layer):
  pre-activation  e_pre = c_np * (|A| |W| + |b|): the fp32-class bound of the tensor-core contraction that
                  test_gemm_split.py holds the split GEMM to (c = 3e-6 for np = 1 and 3, 2e-5 for np = 2)
  a = act(pre)    e_a = e_pre + 4u (|a| + 1)                         (|act'| <= 1, a few ulp of tanhf / expf)
  z               e_z = sum_c |w_o| e_a + (N + 4) u (sum_c |a w_o| + |b_o|)
  dz              e_dz = |w| / n_nz (0.625 e_z + 16u) + 8u |dz|      (|d dz / dz| <= 0.625 |w| / n_nz for MSE)
  loss term       e_l = |w| (e_z + 8u (|z| + 1))                       (|d loss / dz| <= |w|)
  g               e_g = 2 |dz w_o| e_a + |w_o| e_dz + 4u |g|          (|act''| <= 2 in terms of the output)
  dZ_L (np = 1)   e_g + one bf16 ulp (2^-7 |g|); np = 2 / 3: the sum of the parts within e_g + 2^(1 - 8 np) |g|
  sums            the sum of the terms' bounds + d u sum |terms|, d = tiles + 20 (the depth of the kernel's reduction:
                  two rows per thread, 3 shuffle rounds, one add per tile, 4 warp slots, one atomic per CTA)
So a sum is held relative to the sum of the absolute values of its terms: a dropped row or a shifted column misses by
far more than its bound.  relu / leakyrelu: where |pre| lies within e_pre of the kink, act' may flip; such an element is
left out of the element-wise dZ check and its flip |dz w_o| (1 - alpha) is added to the bound of its db_L column.  z,
dz and dw_o = sum dz a are continuous at the kink and need no extra term.

The in/out sums are pre-filled with non-zero values: the kernel must add into them, never store."""
import numpy as np
import pytest

from conftest import bf16_round
from out_layer_ref import ACTS, CE, LOSSES, MSE, U, output_layer
from out_layer_ref import activation as _act

ACC = {1: 3e-6, 2: 2e-5, 3: 3e-6}
OUTS = ("dZ", "db_L", "dw_o", "db_o", "loss")

_worst = {}
_cache = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if _worst:
        print("\nworst error / bound: " + ", ".join("%s %.3g" % (k, _worst[k]) for k in OUTS if k in _worst))


def _operands(M, N, K, seed, a_rows=None, row0=0):
    """A [a_rows, K] with the batch at rows row0 .. row0 + M - 1 (the other rows 100x larger), W [K, N], bias, w_o, b_o, y, w"""
    key = (M, N, K, seed, a_rows, row0)
    if key not in _cache:
        rng = np.random.RandomState(seed * 7919 + M * 31 + N * 7 + K)
        a_rows = M if a_rows is None else a_rows
        A = (np.clip(rng.standard_normal((a_rows, K)), -4, 4) * 0.5).astype(np.float32)
        A[:row0] *= 100
        A[row0 + M:] *= 100
        lim = np.sqrt(6.0 / (K + N))
        W = rng.uniform(-lim, lim, (K, N)).astype(np.float32)
        bias = rng.uniform(-0.3, 0.3, N).astype(np.float32)
        wo = rng.uniform(-1, 1, N).astype(np.float32) * np.float32(np.sqrt(6.0 / (N + 1)))
        bo = np.float32(0.3)
        y = (rng.uniform(size=M) < 0.2).astype(np.float32)
        w = rng.choice(np.array([0.0, 1.0, 2.5], np.float32), size=M).astype(np.float32)
        init = [rng.standard_normal(N).astype(np.float32) * 0.1, rng.standard_normal(N).astype(np.float32) * 0.1,
                np.float32(0.37), np.float32(1.25)]
        _cache.clear()
        _cache[key] = (A, W, bias, wo, bo, y, w, init)
    return _cache[key]


def _reference(A, W, bias, wo, bo, y, w, act, loss, np_parts, row0, M):
    """float64 values and bounds (module docstring) of every output"""
    f64 = np.float64
    Ab, Wb = A[row0:row0 + M], W
    if np_parts == 1:
        Ab, Wb = bf16_round(Ab), bf16_round(Wb)
    A64, W64, b64 = Ab.astype(f64), Wb.astype(f64), bias.astype(f64)
    pre = A64 @ W64 + b64
    e_pre = ACC[np_parts] * (np.abs(A64) @ np.abs(W64) + np.abs(b64))
    a = _act(pre, act)
    e_a = e_pre + 4 * U * (np.abs(a) + 1)
    kink = np.abs(pre) <= e_pre if act in (ACTS["relu"], ACTS["leakyrelu"]) else None
    return output_layer(a, e_a, wo, bo, y, w, act, loss, (M + 63) // 64 + 20, kink)


def _note(name, err, tol):
    err, tol = np.broadcast_arrays(np.asarray(err, np.float64), np.asarray(tol, np.float64))
    pos = tol > 0                        # a zero bound (a row of weight 0) admits no error; the assertion checks it
    r = float(np.max(err[pos] / tol[pos])) if pos.any() else 0.0
    _worst[name] = max(_worst.get(name, 0.0), r)
    return r


def _check_outputs(got, ref, init, np_parts, what=""):
    dZ, g_bL, g_wo, g_bo, loss_sum, guard = got
    assert guard == 0, "%s: %d sentinel elements around dZ_L changed" % (what, guard)
    g, e_g, ok = ref["g"], ref["e_g"], ~ref["kink"]
    if np_parts == 1:
        err, tol = np.abs(dZ[0] - g), 2.0 ** -7 * np.abs(g) + e_g
    else:
        err, tol = np.abs(dZ.astype(np.float64).sum(axis=0) - g), e_g + 2.0 ** (1 - 8 * np_parts) * np.abs(g)
        for k in range(1, np_parts):     # part k is the bf16 of what parts 0 .. k-1 leave: at most 2^-8 of part k-1
            assert (np.abs(dZ[k]) <= 2.0 ** -8 * np.abs(dZ[k - 1])).all(), "%s: part %d not below part %d" % (what, k, k - 1)
    bad = (err > tol) & ok
    _note("dZ", err[ok], tol[ok])
    assert not bad.any(), "%s: %d dZ_L elements off, first at %s: %r vs %r (bound %r)" % (
        what, bad.sum(), np.argwhere(bad)[0], dZ[0][bad][0], g[bad][0], tol[bad][0])
    # in/out: the result minus the value passed in is the contribution (fp32 atomics onto the initial value add d u |init|)
    for name, val, i0 in (("db_L", g_bL, init[0]), ("dw_o", g_wo, init[1]), ("db_o", g_bo, init[2]), ("loss", loss_sum, init[3])):
        want, tol = ref[name]
        val, i0 = np.asarray(val, np.float64), np.asarray(i0, np.float64)
        tol = tol + ref["d"] * U * (np.abs(i0) + np.abs(want))
        err = np.abs(val - i0 - want)
        r = _note(name, err, tol)
        assert (err <= tol).all(), "%s: %s off by %.3g x its bound (worst at %s)" % (what, name, r, np.argmax(err / tol))


def _run(sb, M, N, K, act="relu", loss=MSE, np_parts=1, grid=0, seed=0, a_rows=None, row0=0, scale_wo=None):
    A, W, bias, wo, bo, y, w, init = _operands(M, N, K, seed, a_rows, row0)
    if scale_wo is not None:
        wo = (wo * np.float32(scale_wo)).astype(np.float32)
    ref = _reference(A, W, bias, wo, bo, y, w, ACTS[act], loss, np_parts, row0, M)
    got = sb.capi.debug_gemm_fwd_out(A, W, bias, wo, bo, y, w, ACTS[act], loss, np_parts=np_parts, row0=row0, M=M, grid=grid,
                                     g_bL=init[0], g_wo=init[1], g_bo=init[2], loss_sum=init[3])
    _check_outputs(got, ref, init, np_parts, "M=%d N=%d K=%d %s loss=%d np=%d grid=%d" % (M, N, K, act, loss, np_parts, grid))
    return got, ref


SHAPES = [
    # (M, N, K)
    (8192, 256, 512),        # cfg2's last hidden layer
    (4096, 128, 256),        # cfg1's
    (100, 50, 200),          # cfg0's
    (130, 24, 40),           # the bf16 small step test's
] + [(333, n, 136) for n in (1, 8, 63, 64, 65, 127, 128, 129, 200, 255, 256)] + [
    (m, 200, 72) for m in (1, 8, 9, 63, 65)       # the second row half of a fragment (rows r0 + 8) absent, the first present
] + [(200, 96, k) for k in (8, 72, 2000)]


@pytest.mark.gpu
@pytest.mark.parametrize("loss", sorted(LOSSES))
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_shapes_match_fp64(sb, M, N, K, loss):
    _run(sb, M, N, K, "relu", LOSSES[loss])


@pytest.mark.gpu
@pytest.mark.parametrize("loss", sorted(LOSSES))
@pytest.mark.parametrize("grid", [1, 3])
def test_several_tiles_per_cta(sb, grid, loss):
    # 16 tiles on 1 or 3 CTAs: the z-partial double buffer, the wait on the dZ_L staging tiles between tiles, and the loss
    # / column sums carried over the tiles of a CTA
    _run(sb, 1000, 160, 100, "relu", LOSSES[loss], grid=grid)


@pytest.mark.gpu
def test_natural_grid_runs_a_second_wave(sb):
    # 141 tiles: more than one per SM on any H100
    _run(sb, 9000, 100, 136, "tanh", CE)


@pytest.mark.gpu
@pytest.mark.parametrize("loss", sorted(LOSSES))
@pytest.mark.parametrize("N", [40, 100, 250])          # BN = 64, 128, 256
@pytest.mark.parametrize("act", sorted(ACTS))
def test_activations(sb, act, N, loss):
    _run(sb, 300, N, 72, act, LOSSES[loss])


@pytest.mark.gpu
@pytest.mark.parametrize("loss", sorted(LOSSES))
@pytest.mark.parametrize("act", ["relu", "tanh"])
@pytest.mark.parametrize("N", [50, 200])
@pytest.mark.parametrize("np_parts", [2, 3])
def test_split_parts(sb, np_parts, N, act, loss):
    # the fp32-class modes: A and W as np bf16 parts, dZ_L as np bf16 parts that add up to g at the fp32-class bound
    _run(sb, 500, N, 300, act, LOSSES[loss], np_parts=np_parts)


@pytest.mark.gpu
@pytest.mark.parametrize("np_parts", [1, 3])
def test_resident_row_offset(sb, np_parts):
    # the batch read at a row offset inside a larger A, as a step on the HBM-resident set reads it: the rows past the batch
    # end are real (100x larger) data, not TMA zero fill, and must not leak into the last tile
    M, N, K, row0 = 300, 120, 72, 77
    got, _ = _run(sb, M, N, K, "relu", CE, np_parts=np_parts, a_rows=row0 + M + 50, row0=row0)
    A, W, bias, wo, bo, y, w, init = _operands(M, N, K, 0, row0 + M + 50, row0)
    alone = sb.capi.debug_gemm_fwd_out(A[row0:row0 + M], W, bias, wo, bo, y, w, ACTS["relu"], CE, np_parts=np_parts,
                                       g_bL=init[0], g_wo=init[1], g_bo=init[2], loss_sum=init[3])
    np.testing.assert_array_equal(got[0], alone[0])


@pytest.mark.gpu
def test_no_nonzero_weight(sb):
    # n_nz = 0: dz = 0 everywhere, so dZ_L is zero and the sums come back exactly as they went in
    M, N, K = 200, 90, 64
    A, W, bias, wo, bo, y, w, init = _operands(M, N, K, 3)
    for loss in (MSE, CE):
        dZ, g_bL, g_wo, g_bo, loss_sum, guard = sb.capi.debug_gemm_fwd_out(
            A, W, bias, wo, bo, y, np.zeros(M, np.float32), ACTS["relu"], loss, g_bL=init[0], g_wo=init[1], g_bo=init[2],
            loss_sum=init[3])
        assert guard == 0
        np.testing.assert_array_equal(dZ, 0.0)
        np.testing.assert_array_equal(g_bL, init[0])
        np.testing.assert_array_equal(g_wo, init[1])
        assert g_bo == init[2] and loss_sum == init[3]


@pytest.mark.gpu
@pytest.mark.parametrize("loss", sorted(LOSSES))
@pytest.mark.parametrize("act", ["relu", "sigmoid"])
def test_extreme_logits(sb, act, loss):
    # |z| up to ~100: the CE loss needs the softplus form max(z, 0) - z y + log1p(exp(-|z|)), MSE's dz vanishes in fp32
    M, N, K = 256, 128, 64
    A, W, bias, wo, bo, y, w, init = _operands(M, N, K, 0)
    a = _act(bf16_round(A).astype(np.float64) @ bf16_round(W).astype(np.float64) + bias, ACTS[act])
    z = a @ wo.astype(np.float64) + bo
    got, _ = _run(sb, M, N, K, act, LOSSES[loss], scale_wo=100.0 / np.abs(z - bo).max())
    assert all(np.isfinite(np.asarray(v)).all() for v in got[:5])


@pytest.mark.gpu
def test_two_launches_are_bit_identical(sb):
    M, N, K = 2000, 200, 300
    A, W, bias, wo, bo, y, w, _ = _operands(M, N, K, 5)
    first = sb.capi.debug_gemm_fwd_out(A, W, bias, wo, bo, y, w, ACTS["leakyrelu"], CE)
    second = sb.capi.debug_gemm_fwd_out(A, W, bias, wo, bo, y, w, ACTS["leakyrelu"], CE)
    np.testing.assert_array_equal(first[0], second[0])


INVALID = {
    "N=0": dict(N=0), "N=257": dict(N=257), "np=0": dict(np_parts=0), "np=4": dict(np_parts=4), "loss=2": dict(loss=2),
    "act=4": dict(act=4), "act=-2": dict(act=-2), "grid=-1": dict(grid=-1), "M=0": dict(M=0), "K=0": dict(K=0),
    "row0=-1": dict(row0=-1), "past_a_rows": dict(row0=5),
}


@pytest.mark.parametrize("case", sorted(INVALID))
def test_invalid_arguments_rejected_before_any_device_call(sb, case):
    # refused on a machine without a GPU
    kw = dict(M=64, N=64, K=64, np_parts=1, loss=MSE, act=ACTS["relu"], grid=0, row0=0)
    kw.update(INVALID[case])
    M, N, K = kw.pop("M"), kw.pop("N"), kw.pop("K")
    A = np.ones((64, K), np.float32)        # 64 rows of A: row0 = 5 runs past them
    W = np.ones((K, N), np.float32)
    v, m = np.ones(N, np.float32), np.ones(M, np.float32)
    act, loss = kw.pop("act"), kw.pop("loss")
    with pytest.raises(sb.capi.ShifuB200Error) as e:
        sb.capi.debug_gemm_fwd_out(A, W, v, v, 0.0, m, m, act, loss, M=M, **kw)
    assert e.value.code == sb.capi.SB_ERR_INVALID
