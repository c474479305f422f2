"""Parity of the batched scorer (sb_model_*) and of eval/predict against the oracle, through the C-ABI.
Contract (BASELINE.json): eval scores within 1e-5 of the reference-equivalent CPU path (fp32 parity mode)."""
import os

import numpy as np
import pytest

from oracle import shifu_oracle as so
from util import make_pair

GOLDEN_HEAD = os.path.join(os.path.dirname(__file__), "golden", "dummydl_head.npz")


@pytest.mark.gpu
@pytest.mark.parametrize("hidden", [[100, 50], [64, 300], [64, 700], [64, 1100]], ids=["h50", "h300", "h700", "h1100"])
@pytest.mark.parametrize("precision,tol", [(0, 1e-5), (2, 1e-5), (3, 1e-5), (1, 2e-2)])
def test_model_score_matches_oracle(sb, precision, tol, hidden):
    """1e-5 (north star) must hold in both parity modes: fp32 on the CUDA cores (0) and fp32-class on the tensor cores
    (2 = three bf16 parts); the two-part mode (3) meets it as well on these nets; plain bf16 (1) is the performance mode.
    A last hidden layer of 300 / 700 / 1100 scores through out_layer_rows_kernel<2> / <4> / out_layer_kernel<bf16> on
    the tensor cores and through out_layer_kernel<float>'s column chunks on the CUDA cores."""
    net, params, cfg, desc = make_pair(sb, 200, hidden, [so.ACT_RELU, so.ACT_TANH], precision=precision)
    X, _, _ = so.synth_batch(1000, 200, 3)
    m = sb.Model.create(desc, so.flatten_params(params))
    got = m.score(X)
    want = so.score_rows(net, params, X.astype(np.float64))
    assert np.abs(got - want).max() <= tol
    if precision == 1:   # bf16 mode: tight against the bf16-emulating oracle
        yb = so.loss_and_grads_bf16(net, params, X, np.zeros((len(X), 1), np.float32), np.ones((len(X), 1), np.float32), fused_out=False)[2]
        assert np.abs(got - yb.ravel()).max() <= 1e-3   # one bf16 ulp flip of an activation moves a score by ~2e-4
    # compute(MLData): one row of doubles (TensorflowModel.java:53-94)
    r = m.score_row_f64(X[7].astype(np.float64))
    assert abs(r - want[7]) <= tol
    with pytest.raises(sb.ShifuB200Error):
        m.score_row_f64(np.zeros(199))
    m.close()


@pytest.mark.gpu
def test_model_score_many_chunks_and_ragged_tail(sb):
    """more rows than one internal chunk (16384) and a ragged tail; every row must be scored exactly once"""
    net, params, cfg, desc = make_pair(sb, 40, [24], [so.ACT_SIGMOID])
    rows = 16384 * 2 + 77
    X, _, _ = so.synth_batch(rows, 40, 9)
    m = sb.Model.create(desc, so.flatten_params(params))
    got = m.score(X)
    want = so.score_rows(net, params, X.astype(np.float64))
    assert np.abs(got - want).max() <= 1e-5
    m.close()


@pytest.mark.gpu
def test_scorer_on_reference_fixture_weights(sb):
    """kernels vs the REAL weights of the reference's SavedModel fixture (dummydl; first 3 + last layer, committed
    as tests/golden/dummydl_head.npz by tests/golden/make_golden.py)."""
    g = np.load(GOLDEN_HEAD)
    hidden = [g["W0"].shape[1], g["W1"].shape[1], g["W2"].shape[1]]
    flat = np.concatenate([np.concatenate([g["W%d" % i].ravel(), g["b%d" % i].ravel()]) for i in range(4)])
    for prec in (sb.PREC_FP32, sb.PREC_FP32_TC):
        desc = sb.make_desc(1522, hidden, [so.ACT_RELU] * 3, precision=prec)
        m = sb.Model.create(desc, flat)
        assert np.abs(m.score(g["X"]) - g["Y"].ravel()).max() <= 1e-5
        m.close()


@pytest.mark.gpu
def test_cfg2_net_scores_within_1e5_on_tensor_cores(sb):
    """the eval-path net (BASELINE config 5: 2000 cols, [1024, 512, 256]) scored in SB_PREC_FP32_TC: <= 1e-5 from the oracle"""
    net, params, cfg, desc = make_pair(sb, 2000, [1024, 512, 256], [so.ACT_RELU] * 3, precision=sb.PREC_FP32_TC)
    X, _, _ = so.synth_batch(4096, 2000, 3)
    m = sb.Model.create(desc, so.flatten_params(params))
    got = m.score(X)
    want = so.score_rows(net, params, X.astype(np.float64))
    err = np.abs(got - want).max()
    m.close()
    assert err <= 1e-5, err


@pytest.mark.gpu
def test_savedmodel_export_then_load_scores_identically(sb, tmp_path):
    net, params, cfg, desc = make_pair(sb, 30, [16, 8], [so.ACT_LEAKYRELU, so.ACT_TANH], max_batch=64)
    X, y, w = so.synth_batch(64, 30, 1, weights="mixed")
    d = str(tmp_path / "final_model")
    with sb.Trainer(desc) as t:
        t.set_params(so.flatten_params(params))
        t.step(X, y, w)
        trained = t.get_params()
        pred = t.predict(X)
        t.export_savedmodel(d)
    m = sb.Model.load(d, "shifu_input_0", "shifu_output_0", tag="serve")
    got = m.score(X)
    np.testing.assert_allclose(got, pred, atol=1e-7)
    want = so.score_rows(net, so.unflatten_params(net, trained), X.astype(np.float64))
    assert np.abs(got - want).max() <= 1e-5
    m.close()


@pytest.mark.gpu
def test_eval_loss_is_one_big_batch(sb):
    """validation pass (ssgd_monitor.py:281-284): the whole valid set in ONE sess.run, i.e. sum over all rows /
    count of non-zero weights over all rows - also when it is processed in several max_batch chunks."""
    net, params, cfg, desc = make_pair(sb, 25, [12], [so.ACT_TANH], max_batch=50)
    X, y, w = so.synth_batch(173, 25, 4, weights="mixed")
    ref = so.CleanTrainer(net, params, cfg)
    with sb.Trainer(desc) as t:
        t.set_params(so.flatten_params(params))
        assert abs(t.eval_loss(X, y, w) - ref.eval_loss(X, y, w)) <= 1e-6
        np.testing.assert_allclose(t.predict(X), so.score_rows(net, params, X.astype(np.float64)), atol=1e-6)


@pytest.mark.gpu
def test_checkpoint_roundtrip_resumes_identically(sb, tmp_path):
    net, params, cfg, desc = make_pair(sb, 20, [10], [so.ACT_RELU], optimizer=so.OPT_ADAM, max_batch=32)
    batches = [so.synth_batch(32, 20, s, weights="mixed") for s in range(4)]
    ck = str(tmp_path / "model.ckpt")
    with sb.Trainer(desc) as a:
        a.set_params(so.flatten_params(params))
        a.step(*batches[0]); a.step(*batches[1])
        a.save_checkpoint(ck)
        a.step(*batches[2]); a.step(*batches[3])
        want = a.get_params()
    with sb.Trainer(desc) as b:
        b.load_checkpoint(ck)
        assert b.global_step == 2
        b.step(*batches[2]); b.step(*batches[3])
        np.testing.assert_array_equal(b.get_params(), want)


@pytest.mark.gpu
def test_model_score_is_reentrant_across_threads(sb):
    """Computable.compute may be called from several scorer threads at once (TensorflowModel has no locking,
    TensorflowModel.java:53-94; Session.run is thread-safe) -> sb_model_score / score_row_f64 on ONE handle from 8
    threads must give exactly the single-threaded answers."""
    import threading
    net, params, cfg, desc = make_pair(sb, 120, [64, 32], [so.ACT_RELU, so.ACT_TANH], max_batch=256, precision=sb.PREC_FP32)
    flat = so.flatten_params(params)
    rng = np.random.RandomState(9)
    Xs = [rng.standard_normal((rows, 120)).astype(np.float32) for rows in (1, 7, 256, 300, 1000, 33, 512, 2)]
    with sb.Model.create(desc, flat) as m:
        want = [m.score(X) for X in Xs]
        want_row = m.score_row_f64(Xs[3][5].astype(np.float64))
        got, errs = [None] * len(Xs), []

        def work(i):
            try:
                for _ in range(20):
                    got[i] = m.score(Xs[i])
                    if i == 3:
                        assert m.score_row_f64(Xs[3][5].astype(np.float64)) == want_row
            except Exception as e:      # noqa: BLE001 - surfaced below
                errs.append(e)

        th = [threading.Thread(target=work, args=(i,)) for i in range(len(Xs))]
        [t.start() for t in th]; [t.join() for t in th]
        assert not errs, errs
        for a, b in zip(got, want):
            np.testing.assert_array_equal(a, b)
