"""The dW GEMM on 128 x 256 tiles (gemm_dw.cuh), and the optimizer pass on the run layouts it has to handle.

dW: forced through the debug hook (cfg_cg = 1, bn = 256, MM layout = the dW layout) against float64 on the bf16-rounded
operands, on the cfg1 / cfg2 dW shapes, ragged M / N and split-K 1, 2, 8; the split-precision parts (np = 2, 3) through
whole training steps whose layer-0 dW the planner puts on 256-wide tiles.  Optimizer: fp32 master against the oracle over
three steps for all four optimizers on shapes with unaligned runs and a matrix whose out_dim is not a multiple of 4, and
the bf16 shadow the pass writes against the one refreshed from the master."""
import numpy as np
import pytest

from conftest import bf16_round
from oracle import shifu_oracle as so
from util import make_pair

pytestmark = pytest.mark.gpu

DW_SHAPES = [
    # (M = in, N = out, K = rows, split_k)
    (2000, 1024, 8192, 2),    # cfg2 dW_0 as planned
    (1024, 512, 8192, 8),     # cfg2 dW_1
    (1000, 512, 4096, 1),     # cfg1 dW_0
    (1000, 512, 4096, 8),
    (2000, 1000, 1024, 2),    # ragged M (2000 % 128 != 0), N not a multiple of 256
    (488, 300, 640, 8),       # the second exchange chunk of cfg1's W_0, N ragged inside the second tile
    (130, 258, 200, 1),       # everything ragged, N % 4 != 0: the scalar red path
]


@pytest.mark.parametrize("M,N,K,split_k", DW_SHAPES)
def test_dw_256_wide_tiles_match_fp64(sb, M, N, K, split_k):
    rng = np.random.RandomState(M + 3 * N + K + split_k)
    A = bf16_round(rng.standard_normal((M, K)).astype(np.float32))
    B = bf16_round(rng.standard_normal((N, K)).astype(np.float32))
    D = sb.capi.debug_gemm_bf16(A.T.copy(), B.T.copy(), split_k=split_k, a_mn=True, b_mn=True, cg=1, bn=256)
    ref = A.astype(np.float64) @ B.astype(np.float64).T
    assert np.abs(D - ref).max() <= 8e-5 * np.sqrt(K)


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True)])
def test_256_wide_tiles_only_for_the_dw_layout(sb, a_mn, b_mn):
    A = np.ones((64, 64), np.float32)
    with pytest.raises(sb.capi.ShifuB200Error):
        sb.capi.debug_gemm_bf16(A, A, a_mn=a_mn, b_mn=b_mn, cg=1, bn=256)


@pytest.mark.parametrize("prec,tol", [(2, 1e-4), (3, 2e-3)])   # fp32_tc (np = 3), bf16x2 (np = 2)
def test_dw_256_wide_tiles_split_precision_step(sb, prec, tol):
    """W_0 = 2000 x 1024 at 2048 rows: 128-wide tiles give 128 CTAs x 1 split, 256-wide 64 tiles x 2 splits of >= 32
    k-blocks of the extended K axis - the planner takes the 256-wide tile.  Gradients against the fp32 oracle: fp32 tolerance
    for np = 3, relative 2e-3 for np = 2 (~2^-17 per product)."""
    rows = 2048
    net, params, cfg, desc = make_pair(sb, 2000, [1024, 64], [so.ACT_RELU, so.ACT_RELU], optimizer=so.OPT_SGD, lr=0.01,
                                       max_batch=rows, precision=prec)
    X, y, w = so.synth_batch(rows, 2000, 5, weights="mixed")
    ref = so.CleanTrainer(net, params, cfg)
    ref.step([(X, y, w)])
    with sb.Trainer(desc) as t:
        t.set_params(so.flatten_params(params))
        t.step(X, y, w)
        g = t.get_grads()
    rg = ref.last_grads
    if prec == 2:
        assert np.abs(g - rg).max() <= tol
    else:
        assert np.abs(g - rg).max() <= tol * np.abs(rg).max()


OPT_SHAPES = [
    # W_0 1001 x 40: 16-byte runs and a short last run; W_1 40 x 37 and b_1 (37): out_dim and run lengths not multiples of
    # 4; W_2 starts unaligned
    (1001, [40, 37, 8]),
]


@pytest.mark.parametrize("optimizer", [so.OPT_ADADELTA, so.OPT_ADAM, so.OPT_SGD, so.OPT_MOMENTUM])
@pytest.mark.parametrize("F,hidden", OPT_SHAPES)
def test_optimizer_pass_against_oracle(sb, F, hidden, optimizer):
    """fp32_tc: the master and state after three steps match the oracle (the state enters every later update), and the
    three-part bf16 shadow the pass wrote equals the one refreshed from the master (same scores, bit for bit)"""
    rows = 96
    acts = [so.ACT_TANH] * len(hidden)
    # Adam moves a coordinate by ~lr * m / sqrt(v) however small its gradient, so a summation-order difference in a ~1e-8
    # gradient can move it by a good part of lr: a smaller step keeps the master comparison at the same tolerance
    lr = 0.01 if optimizer == so.OPT_ADAM else 0.05
    net, params, cfg, desc = make_pair(sb, F, hidden, acts, optimizer=optimizer, lr=lr, max_batch=rows, precision=2)
    ref = so.CleanTrainer(net, params, cfg)
    Xs, _, _ = so.synth_batch(rows, F, 99)
    with sb.Trainer(desc) as t:
        t.set_params(so.flatten_params(params))
        for s in range(3):
            X, y, w = so.synth_batch(rows, F, 200 + s, weights="mixed")
            rl = ref.step([(X, y, w)])[0]
            assert abs(t.step(X, y, w) - rl) <= 1e-4, "step %d" % s
            tol_p = 5e-4 if optimizer == so.OPT_ADAM else 2e-5
            assert np.abs(t.get_params() - ref.theta).max() <= tol_p, "step %d" % s
        theta = t.get_params()
        scores = t.predict(Xs)
    with sb.Trainer(desc) as t2:
        t2.set_params(theta)
        np.testing.assert_array_equal(scores, t2.predict(Xs))


@pytest.mark.parametrize("optimizer", [so.OPT_ADAM, so.OPT_MOMENTUM])
def test_optimizer_pass_bf16_shadow(sb, optimizer):
    """plain bf16: the shadow written by the pass (16-byte runs and element runs) equals bf16 of the new master"""
    F, hidden, rows = 1001, [40, 37, 8], 96
    net, params, cfg, desc = make_pair(sb, F, hidden, [so.ACT_RELU] * 3, optimizer=optimizer, lr=0.05, max_batch=rows,
                                       precision=1)
    Xs, _, _ = so.synth_batch(rows, F, 98)
    with sb.Trainer(desc) as t:
        t.set_params(so.flatten_params(params))
        for s in range(2):
            X, y, w = so.synth_batch(rows, F, 300 + s, weights="mixed")
            t.step(X, y, w)
        theta = t.get_params()
        scores = t.predict(Xs)
    with sb.Trainer(desc) as t2:
        t2.set_params(theta)
        np.testing.assert_array_equal(scores, t2.predict(Xs))
