"""The forward GEMM on 128 x 256 tiles (gemm_wide.cuh), forced through the sb_debug_gemm_epilogue hook (bm_wg = 256),
against float64 on the bf16-rounded operands: the cfg2 shapes the planner gives it, ragged M / N / K, every activation
and the identity.  Plus the hook's argument checks, which need no GPU."""
import numpy as np
import pytest

from conftest import bf16_round
from test_gemm_pp import ACTS, _forward

WIDE = 256

SHAPES = [
    # (M, N, K)
    (8192, 1024, 2000),   # cfg2 forward 0
    (8192, 512, 1024),    # cfg2 forward 1
    (1000, 300, 2000),    # M % 128 != 0, the second 256-wide tile 44 columns wide, K tail
    (1000, 1000, 2000),   # the fourth tile 232 columns wide
    (130, 129, 72),       # one partial tile in every direction
    (128 * 140, 512, 128),  # 280 tiles on 132 SMs: a CTA runs up to three, the buffer and ring are reused
]


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_wide_forward_matches_fp64(sb, M, N, K):
    _forward(sb, M, N, K, ACTS["relu"], WIDE)


@pytest.mark.gpu
@pytest.mark.parametrize("act", sorted(ACTS))
@pytest.mark.parametrize("M,N,K", [(130, 300, 72), (1024, 320, 1024)])
def test_wide_activations(sb, M, N, K, act):
    _forward(sb, M, N, K, ACTS[act], WIDE)


@pytest.mark.gpu
def test_wide_identity_is_exact(sb):
    # A = I: the output is W itself, bit for bit - a swizzle or descriptor mistake moves elements
    M, N = 320, 384
    A = np.eye(M, dtype=np.float32)
    W = bf16_round(np.random.RandomState(5).standard_normal((M, N)).astype(np.float32))
    out, _, _ = sb.capi.debug_gemm_epilogue(A, W, ACTS["none"], bias=np.zeros(N, np.float32), bm_wg=WIDE)
    np.testing.assert_array_equal(out, W)


@pytest.mark.parametrize("bm_wg,da", [(96, False), (-1, False), (512, False), (WIDE, True)])
def test_tile_selector_rejected_before_any_device_call(sb, bm_wg, da):
    # no tile of that height, or the wide tile for the dA GEMM (it has no dA epilogue): refused on a machine without a GPU
    A = np.ones((64, 64), np.float32)
    kw = dict(aux=np.zeros((64, 64), np.float32)) if da else dict(bias=np.zeros(64, np.float32))
    with pytest.raises(sb.capi.ShifuB200Error) as e:
        sb.capi.debug_gemm_epilogue(A, A, ACTS["relu"], bm_wg=bm_wg, **kw)
    assert e.value.code == sb.capi.SB_ERR_INVALID
