"""Kernel-level checks of the ping-pong forward / dA GEMM (gemm_pp.cuh) with its fused epilogues, through the
sb_debug_gemm_epilogue hook.

Oracle: float64 on the bf16-rounded operands.  The kernel accumulates exact bf16 products in fp32 and rounds its result to
bf16 once, so an element may differ by one bf16 ulp where fp32 summation order flips a rounding."""
import numpy as np
import pytest

from conftest import bf16_round

ACTS = {"sigmoid": 0, "tanh": 1, "relu": 2, "leakyrelu": 3, "none": -1}

SHAPES = [
    # (M, N, K)
    (100, 50, 200),          # ragged M / N / K: TMA zero fill, clipped stores
    (130, 129, 72),
    (1024, 64, 256),         # N = 64 tiles
    (4096, 512, 1000),       # cfg1 forward 0 (K tail)
    (4096, 256, 128),        # cfg1 dA 2
    (4096, 512, 256),        # cfg1 dA 1
    (8192, 1024, 2000),      # cfg2 forward 0
    (8192, 512, 256),        # cfg2 dA 2
    (8192, 1024, 512),       # cfg2 dA 1
    (128 * 132, 384, 128),   # 396 tiles of 128 rows on 132 SMs: three per CTA, so warpgroup 0 gets one tile more
]

_cache = {}


def _operands(M, N, K, da):
    key = (M, N, K, da)
    if key not in _cache:
        rng = np.random.RandomState(M * 7 + N * 3 + K + da)
        A = bf16_round((rng.standard_normal((M, K)) * 0.5).astype(np.float32))
        W = bf16_round((rng.standard_normal((N, K) if da else (K, N)) * 0.5).astype(np.float32))
        prod = A.astype(np.float64) @ (W.astype(np.float64).T if da else W.astype(np.float64))
        _cache.clear()
        _cache[key] = (A, W, prod)
    return _cache[key]


def _act(z, act):
    if act == ACTS["sigmoid"]:
        return 1.0 / (1.0 + np.exp(-z))
    if act == ACTS["tanh"]:
        return np.tanh(z)
    if act == ACTS["relu"]:
        return np.maximum(z, 0.0)
    if act == ACTS["leakyrelu"]:
        return np.where(z > 0, z, 0.2 * z)
    return z


def _act_grad(a, act):
    if act == ACTS["sigmoid"]:
        return a * (1.0 - a)
    if act == ACTS["tanh"]:
        return 1.0 - a * a
    if act == ACTS["relu"]:
        return (a > 0).astype(np.float64)
    if act == ACTS["leakyrelu"]:
        return np.where(a > 0, 1.0, 0.2)
    return np.ones_like(a)


def _check_bf16(out, ref, K):
    # one bf16 ulp of the reference (2^-7 relative at most) plus the fp32 accumulation error of the product
    tol = np.abs(ref) * 2.0 ** -7 + 1e-5 * np.sqrt(K)
    bad = np.abs(out - ref) > tol
    assert not bad.any(), "%d elements off, first at %s: %r vs %r" % (bad.sum(), np.argwhere(bad)[0], out[bad][0], ref[bad][0])


def _forward(sb, M, N, K, act, bm_wg):
    A, W, prod = _operands(M, N, K, 0)
    bias = (np.random.RandomState(N).standard_normal(N) * 0.1).astype(np.float32)
    out, _, _ = sb.capi.debug_gemm_epilogue(A, W, act, bias=bias, bm_wg=bm_wg)
    _check_bf16(out, _act(prod + bias.astype(np.float64), act), K)


def _dA(sb, M, N, K, act, bm_wg):
    A, W, prod = _operands(M, N, K, 1)
    rng = np.random.RandomState(M + N)
    if act == ACTS["sigmoid"]:
        aux = rng.uniform(0.0, 1.0, (M, N))
    elif act == ACTS["tanh"]:
        aux = rng.uniform(-1.0, 1.0, (M, N))
    else:
        aux = rng.standard_normal((M, N))
    aux = bf16_round(aux.astype(np.float32))
    out, cs, _ = sb.capi.debug_gemm_epilogue(A, W, act, aux=aux, bm_wg=bm_wg)
    dz = prod * _act_grad(aux.astype(np.float64), act)
    _check_bf16(out, dz, K)
    ref_cs = dz.sum(axis=0)
    err = np.abs(cs - ref_cs)
    tol = 1e-5 * np.sqrt(M) * max(1.0, np.abs(ref_cs).max()) + 1e-6 * np.abs(dz).sum(axis=0)
    assert (err <= tol).all(), (err.max(), np.argmax(err - tol))


@pytest.mark.gpu
@pytest.mark.parametrize("bm_wg", [64, 128])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_forward_matches_fp64(sb, M, N, K, bm_wg):
    _forward(sb, M, N, K, ACTS["relu"], bm_wg)


@pytest.mark.gpu
@pytest.mark.parametrize("bm_wg", [64, 128])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_dA_matches_fp64(sb, M, N, K, bm_wg):
    _dA(sb, M, N, K, ACTS["relu"], bm_wg)


@pytest.mark.gpu
@pytest.mark.parametrize("bm_wg", [64, 128])
@pytest.mark.parametrize("act", sorted(ACTS))
@pytest.mark.parametrize("M,N,K", [(130, 129, 72), (1024, 320, 256)])
def test_activations(sb, M, N, K, act, bm_wg):
    _forward(sb, M, N, K, ACTS[act], bm_wg)
    _dA(sb, M, N, K, ACTS[act], bm_wg)


@pytest.mark.gpu
@pytest.mark.parametrize("bm_wg", [64, 128])
@pytest.mark.parametrize("da", [0, 1])
def test_identity_is_exact(sb, da, bm_wg):
    # A = I: the output is W (forward) or W^T (dA) itself, bit for bit - a swizzle or descriptor mistake moves elements
    M, N = 320, 192
    A = np.eye(M, dtype=np.float32)
    W = bf16_round(np.random.RandomState(5).standard_normal((N, M) if da else (M, N)).astype(np.float32))
    if da:
        out, cs, _ = sb.capi.debug_gemm_epilogue(A, W, ACTS["none"], aux=np.zeros((M, N), np.float32), bm_wg=bm_wg)
        np.testing.assert_array_equal(out, W.T)
        np.testing.assert_allclose(cs, W.astype(np.float64).sum(axis=1), rtol=1e-5, atol=1e-5)
    else:
        out, _, _ = sb.capi.debug_gemm_epilogue(A, W, ACTS["none"], bias=np.zeros(N, np.float32), bm_wg=bm_wg)
        np.testing.assert_array_equal(out, W)
