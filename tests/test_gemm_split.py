"""The tensor-core parity GEMM (SB_PREC_FP32_TC / SB_PREC_BF16X2): fp32 operands held as 3 / 2 bf16 parts, the part
products with i + j < np accumulated in fp32 by the SAME wgmma kernel over an extended K axis.  Checked against a
float64 contraction of the fp32 inputs; the bound is relative to sum_k |a_k b_k| (what an fp32 dot product is held to)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _case(sb, M, N, K, parts, seed=0):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((M, K), dtype=np.float32) * np.exp(rng.standard_normal((M, K), dtype=np.float32))
    B = rng.standard_normal((N, K), dtype=np.float32)
    D = sb.capi.debug_gemm_split(A, B, parts)
    ref = A.astype(np.float64) @ B.astype(np.float64).T
    scale = np.abs(A).astype(np.float64) @ np.abs(B).astype(np.float64).T
    return np.abs(D - ref).max(), (np.abs(D - ref) / scale).max()


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (300, 200, 1000), (4096, 512, 1000), (8192, 1024, 2000), (100, 50, 200), (33, 7, 19)])
def test_three_parts_are_fp32_class(sb, M, N, K):
    _, rel = _case(sb, M, N, K, 3)
    # fp32-class: an fp32 FMA chain of length K is allowed K * 6e-8 (1.2e-4 at K = 2000) and typically lands at
    # sqrt(K) * 6e-8 ~ 3e-6; the tensor core's fp32 accumulation (alignment truncation inside a k-block) measures 0.7 - 1.4e-6
    assert rel <= 3e-6, rel


@pytest.mark.parametrize("M,N,K", [(300, 200, 1000), (8192, 1024, 2000)])
def test_two_parts_and_one_part_error_levels(sb, M, N, K):
    _, rel2 = _case(sb, M, N, K, 2)
    _, rel1 = _case(sb, M, N, K, 1)
    assert rel2 <= 2e-5, rel2                # ~2^-16
    assert 1e-4 <= rel1 <= 1e-2, rel1        # plain bf16: ~2^-9 per operand (sanity: the split really adds precision)
