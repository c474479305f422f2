"""Kernel-level parity of the wgmma GEMM (gemm_tc.cuh) through the C-ABI test hook.

Oracle: float64 matmul of the bf16-rounded operands (the kernel multiplies exact bf16 products and accumulates
in fp32 registers, so the only difference is fp32 summation order/rounding)."""
import numpy as np
import pytest

from conftest import bf16_round

SHAPES = [
    # (M, N, K, split_k)
    (128, 128, 64, 1),        # one tile, one k-block
    (128, 64, 128, 1),        # BN = 64 path
    (256, 256, 256, 1),       # several tiles
    (100, 50, 200, 1),        # ragged M/N/K (cfg0 layer shapes): TMA zero fill + guarded stores
    (4096, 512, 1000, 1),     # cfg1 layer-0 forward, K tail (1000 % 64 != 0)
    (1000, 512, 4096, 4),     # cfg1 layer-0 dW as split-K over the batch
    (512, 256, 4096, 16),     # deeper split
    (130, 129, 72, 2),        # everything ragged + split
    (8192, 1024, 2000, 1),    # cfg2 layer-0 forward (persistent: > 132 tiles, several per CTA)
]


LAYOUTS = {"KK": (False, False),   # dA GEMM:      dZ_l [rows,out]  x  W_l [in,out] as B[N=in, K=out]
           "KM": (False, True),    # forward GEMM: A_{l-1} [rows,in] x W_l [in,out] as B stored [K=in, N=out]
           "MM": (True, True)}     # dW GEMM:      A_{l-1} [rows,in] and dZ_l [rows,out], both stored [K=rows, *]


@pytest.mark.gpu
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("M,N,K,split_k", SHAPES)
def test_gemm_bf16_matches_fp64(sb, M, N, K, split_k, layout):
    a_mn, b_mn = LAYOUTS[layout]
    rng = np.random.RandomState(M * 7 + N * 3 + K)
    A = bf16_round(rng.standard_normal((M, K)).astype(np.float32))
    B = bf16_round(rng.standard_normal((N, K)).astype(np.float32))
    D = sb.capi.debug_gemm_bf16(A.T.copy() if a_mn else A, B.T.copy() if b_mn else B, split_k=split_k, a_mn=a_mn, b_mn=b_mn)
    ref = A.astype(np.float64) @ B.astype(np.float64).T
    # fp32 accumulation over K terms of magnitude ~1: error ~ sqrt(K) * 2^-24 * |sum|-ish; 1e-3 absolute is generous
    err = np.abs(D - ref).max()
    scale = np.sqrt(K)
    assert err <= 2e-5 * scale * 4, "max abs err %g (K=%d)" % (err, K)


TILES = [(1, 64), (1, 128)]   # (cfg_cg = 1: the tile is forced, BN)


@pytest.mark.gpu
@pytest.mark.parametrize("cg,bn", TILES)
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("M,N,K,split_k", [(300, 200, 136, 1), (1000, 512, 1024, 2), (2048, 1024, 512, 1)])
def test_gemm_every_tile_configuration(sb, M, N, K, split_k, layout, cg, bn):
    """each instantiated tile shape (128xBN) on ragged and multi-wave problems, forced through the debug hook (the planner
    would not pick every one of them here)"""
    if bn == 64 and N > 64:
        N = 64
    a_mn, b_mn = LAYOUTS[layout]
    rng = np.random.RandomState(M + N + K + cg * 7 + bn)
    A = bf16_round(rng.standard_normal((M, K)).astype(np.float32))
    B = bf16_round(rng.standard_normal((N, K)).astype(np.float32))
    D = sb.capi.debug_gemm_bf16(A.T.copy() if a_mn else A, B.T.copy() if b_mn else B, split_k=split_k, a_mn=a_mn, b_mn=b_mn,
                                cg=cg, bn=bn)
    ref = A.astype(np.float64) @ B.astype(np.float64).T
    assert np.abs(D - ref).max() <= 8e-5 * np.sqrt(K)


@pytest.mark.gpu
@pytest.mark.parametrize("cg,bn", TILES)
def test_gemm_identity_exact_pair_tiles(sb, cg, bn):
    """A = [I; I] (256 x 128), B arbitrary: D must be exactly [B^T; B^T] for every tile configuration"""
    rng = np.random.RandomState(2)
    n = 64 if bn == 64 else 256
    A = np.vstack([np.eye(128, dtype=np.float32)] * 2)
    B = bf16_round(rng.standard_normal((n, 128)).astype(np.float32))
    D = sb.capi.debug_gemm_bf16(A, B, cg=cg, bn=bn)
    np.testing.assert_array_equal(D, np.vstack([B.T, B.T]))


@pytest.mark.gpu
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_gemm_identity_exact(sb, layout):
    """A = I, B arbitrary bf16: the result must be exactly B^T - any swizzle / descriptor / layout mistake shows up
    as a permutation."""
    a_mn, b_mn = LAYOUTS[layout]
    rng = np.random.RandomState(1)
    K = 128
    A = np.eye(128, K, dtype=np.float32)
    B = bf16_round(rng.standard_normal((128, K)).astype(np.float32))
    D = sb.capi.debug_gemm_bf16(A.T.copy() if a_mn else A, B.T.copy() if b_mn else B, a_mn=a_mn, b_mn=b_mn)
    np.testing.assert_array_equal(D, B.T)
