"""Wide+deep on the GPU (BASELINE.json configs[3]: 5000 one-hot + 500 dense columns, MLP [1024, 512]): the sparse step
(sb_trainer_step_sparse: embedding gather in the forward, scatter-add in the backward) against
  * the sparse restatement oracle/wide_deep.py (== the dense oracle on the materialised one-hot matrix,
    tests/test_wide_deep_oracle.py), fp32 parity mode <= 1e-4 / bf16 mode vs the bf16-emulating dense oracle;
  * the repo's own DENSE step on the materialised one-hot matrix (same parameters, same update)."""
import numpy as np
import pytest

from oracle import shifu_oracle as so
from oracle import wide_deep as wd

pytestmark = pytest.mark.gpu


def _setup(sb, n_dense, vocab, hidden, acts, rows, prec, opt=so.OPT_SGD, lr=0.1, seed=2):
    n_onehot = int(sum(vocab))
    F = n_dense + n_onehot
    net = so.NetDesc(F, hidden, acts)
    params = so.xavier_init(net, seed)
    Xd, idx, y, w = wd.synth_wide_deep_batch(rows, n_dense, vocab, seed)
    desc = sb.make_desc(F, hidden, acts, optimizer=opt, learning_rate=lr, max_batch=rows, precision=prec)
    return net, params, desc, (Xd, idx, y, w), n_onehot


@pytest.mark.parametrize("prec", [0, 2, 1])
@pytest.mark.parametrize("shape", ["small", "cfg4", "one_layer"])
def test_sparse_step_matches_oracle_and_dense_step(sb, prec, shape):
    if shape == "small":
        n_dense, vocab, hidden, acts, rows = 21, [5, 9, 3, 17], [40, 24], [so.ACT_TANH, so.ACT_RELU], 130
    elif shape == "cfg4":   # BASELINE config 4: 500 dense + 5000 one-hot (50 categorical columns x 100 values), [1024, 512]
        n_dense, vocab, hidden, acts, rows = 500, [100] * 50, [1024, 512], [so.ACT_RELU, so.ACT_RELU], 2048
    else:       # one hidden layer: its GEMM adds the embedding sums, so the output layer is not fused (out_layer_rows_kernel<1>)
        n_dense, vocab, hidden, acts, rows = 21, [5, 9, 3, 17], [48], [so.ACT_RELU], 130
    # the sparse step fuses the output layer into the last hidden GEMM only when that GEMM is not the first layer's
    sparse_fused = hidden[-1] <= 256 and len(hidden) > 1
    net, params, desc, (Xd, idx, y, w), n_onehot = _setup(sb, n_dense, vocab, hidden, acts, rows, prec)
    Xfull = np.concatenate([Xd, wd.onehot_matrix(idx, n_onehot)], axis=1)
    L, g, yhat = wd.loss_and_grads_sparse(net, params, Xd, idx, y, w)
    g = so.flatten_params(g)
    with sb.Trainer(desc) as ts, sb.Trainer(desc) as tdense:
        for t in (ts, tdense):
            t.set_params(so.flatten_params(params))
        ts.set_sparse(n_dense, n_onehot, len(vocab))
        pred = ts.predict_sparse(Xd, idx)
        pred_dense = tdense.predict(Xfull)
        loss = ts.step_sparse(Xd, idx, y, w)
        grads, theta = ts.get_grads(), ts.get_params()
        loss_d = tdense.step(Xfull, y, w)
        grads_d, theta_d = tdense.get_grads(), tdense.get_params()
    gmax = np.abs(g).max()
    if prec in (0, 2):        # the two fp32-class parity modes: north-star tolerances
        assert abs(loss - L) <= 1e-4 and np.abs(grads - g).max() <= 1e-4
        assert np.abs(pred - yhat.ravel()).max() <= 1e-5
        assert np.abs(grads - grads_d).max() <= 1e-5 + 1e-4 * gmax and abs(loss - loss_d) <= 1e-5
    else:                     # bf16: against the dense bf16-emulating oracle on the one-hot matrix (0/1 are exact in bf16)
        Lb, gb, yb = so.loss_and_grads_bf16(net, params, Xfull, y, w, fused_out=sparse_fused)
        gb = so.flatten_params(gb)
        assert abs(loss - Lb) <= 2e-5 and np.abs(grads - gb).max() <= 2e-3 * np.abs(gb).max()
        if sparse_fused == (hidden[-1] <= 256):
            assert abs(loss - loss_d) <= 2e-5 and np.abs(grads - grads_d).max() <= 2e-3 * gmax
        else:   # the dense step keeps A_L in fp32 where the sparse one rounds it: each against the oracle of its own rounding
            Ld, gd, _ = so.loss_and_grads_bf16(net, params, Xfull, y, w, fused_out=True)
            gd = so.flatten_params(gd)
            assert abs(loss_d - Ld) <= 2e-5 and np.abs(grads_d - gd).max() <= 2e-3 * np.abs(gd).max()
    assert np.abs(pred - pred_dense).max() <= (1e-6 if prec != 1 else 2e-3)
    assert np.abs(theta - theta_d).max() <= (1e-5 if prec != 1 else 2e-3)
    # rows of the embedding block nobody selected keep a zero gradient
    W0g = so.unflatten_params(net, grads)[0]
    unused = np.setdiff1d(np.arange(n_onehot), idx[idx >= 0])
    if len(unused):
        assert np.abs(W0g[n_dense + unused]).max() == 0.0


def test_sparse_argument_checks(sb):
    net, params, desc, (Xd, idx, y, w), n_onehot = _setup(sb, 8, [4, 4], [8], [so.ACT_RELU], 16, 0)
    with sb.Trainer(desc) as t:
        with pytest.raises(sb.ShifuB200Error):
            t.set_sparse(8, n_onehot + 1, 2)          # n_dense + n_onehot != n_features
        t.set_sparse(8, n_onehot, 2)
        bad = idx.copy(); bad[0, 0] = n_onehot
        with pytest.raises(sb.ShifuB200Error):
            t.step_sparse(Xd, bad, y, w)
        # -1 is the only "missing" index: any other negative one is refused by every sparse entry point
        for j in (-2, -2 ** 31):
            bad = idx.copy(); bad[-1, 1] = j
            for call in (lambda: t.step_sparse(Xd, bad, y, w), lambda: t.predict_sparse(Xd, bad),
                         lambda: t.eval_loss_sparse(Xd, bad, y, w)):
                with pytest.raises(sb.ShifuB200Error) as e:
                    call()
                assert e.value.code == sb.capi.SB_ERR_INVALID and "outside [-1," in str(e.value)
