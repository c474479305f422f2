"""Adagrad, RMSProp and FTRL on the H100, in every precision mode and through every place an update happens: the single-GPU
optimizer pass (optimizer_kernel), the owner update of the peer exchange (xchg_update_kernel, xchg_ll_kernel), the
wide+deep step and the worker.  Checked against oracle/tf_optimizers.py (the TF 1.x training_ops.cc forms):

  state start       s1 / s2 after creation, init_xavier and set_params (Adagrad / FTRL accum = initial_accumulator,
                    RMSProp ms = 1, the rest 0)
  one step          at the full cfg1 / cfg2 shapes: the oracle update applied to the step's own gradient (get_grads) gives
                    the step's theta, s1 and s2 (an element-wise fp32 rule on the same inputs: <= 1e-4 in every mode)
  loss curves       sb_trainer_run_resident at cfg1 over 24 steps: fp32 modes vs CleanTrainer per step <= 1e-4, bf16 vs
                    Bf16Trainer <= 5e-4 (the bounds of tests/test_benchmarked_paths.py)
  checkpoint        deterministic mode: save after k steps, load into a fresh trainer, continue = an uninterrupted run, bit
                    for bit; two deterministic runs are bit-identical
  peer exchange     W = 2, 4 in-process replicas: only the owner of a run changes its state, every rank ends with the same
                    bits, and the run matches CleanTrainer.step([shards]) (fp32 <= 1e-4)"""
import numpy as np
import pytest

from oracle import shifu_oracle as so
from oracle import tf_optimizers as tfo
from oracle import wide_deep as wd

pytestmark = pytest.mark.gpu

FP32, BF16, FP32_TC, BF16X2 = 0, 1, 2, 3
PRECS = [FP32, BF16, FP32_TC, BF16X2]
OPTS = {"adagrad": tfo.OPT_ADAGRAD, "rmsprop": tfo.OPT_RMSPROP, "ftrl": tfo.OPT_FTRL}
# learning rates of each rule's usual scale; FTRL with both penalties on, so that l1 / l2 reach the kernels
LR = {tfo.OPT_ADAGRAD: 0.01, tfo.OPT_RMSPROP: 0.001, tfo.OPT_FTRL: 0.05}
FTRL_PARAMS = dict(initial_accumulator=0.1, l1=1e-3, l2=1e-2)


def _cfg(kind, lr=None):
    kw = dict(FTRL_PARAMS) if kind == tfo.OPT_FTRL else {}
    return tfo.tf_config(kind, LR[kind] if lr is None else lr, **kw)


def _trainer(sb, kind, F, hidden, B, prec, lr=None, **kw):
    desc = sb.make_desc(F, hidden, [sb.ACT_RELU] * len(hidden), optimizer=kind, learning_rate=LR[kind] if lr is None else lr,
                        max_batch=B, precision=prec)
    if kind == tfo.OPT_FTRL:
        kw = dict(FTRL_PARAMS, **kw)
    return sb.Trainer(desc, **kw)


def _state(sb, t):
    return t.debug_buffer(sb.capi.DEBUG_BUF_S1), t.debug_buffer(sb.capi.DEBUG_BUF_S2)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("name", list(OPTS))
def test_state_starts_at_the_tf_slot_values(sb, name, prec):
    kind = OPTS[name]
    s1_0 = 1.0 if kind == tfo.OPT_RMSPROP else 0.1
    net = so.NetDesc(40, [24, 16], [so.ACT_RELU] * 2)
    with sb.Trainer(sb.make_desc(40, [24, 16], [sb.ACT_RELU] * 2, optimizer=kind, max_batch=32, precision=prec)) as t:
        for what in ("create", "init_xavier", "set_params"):
            if what == "init_xavier":
                t.init_xavier(3)
            elif what == "set_params":
                t.set_params(so.flatten_params(so.xavier_init(net, 4)))
            s1, s2 = _state(sb, t)
            assert np.all(s1 == np.float32(s1_0)) and np.all(s2 == 0), what
    if kind != tfo.OPT_RMSPROP:
        with sb.Trainer(sb.make_desc(40, [24, 16], [sb.ACT_RELU] * 2, optimizer=kind, max_batch=32, precision=prec),
                        initial_accumulator=0.375) as t:
            t.init_xavier(3)
            s1, s2 = _state(sb, t)
            assert np.all(s1 == np.float32(0.375)) and np.all(s2 == 0)


def test_optimizer_params_are_checked_before_device_work(sb):
    desc = lambda k: sb.make_desc(16, [8], [sb.ACT_RELU], optimizer=k, max_batch=16)
    with sb.Trainer(desc(sb.OPT_FTRL)) as t:
        for args in ((0.0, 0, 0), (-1.0, 0, 0), (float("nan"), 0, 0), (0.1, -1e-3, 0), (0.1, 0, -1e-3), (0.1, float("inf"), 0)):
            with pytest.raises(sb.ShifuB200Error) as e:
                t.set_optimizer_params(*args)
            assert e.value.code == sb.capi.SB_ERR_INVALID, args
        assert np.all(_state(sb, t)[0] == np.float32(0.1))   # a refused call changed nothing
        t.set_optimizer_params(0.2, 0.01, 0.02)
        X, y, w = so.synth_batch(16, 16, 1)
        t.step(X, y, w)
        with pytest.raises(sb.ShifuB200Error) as e:
            t.set_optimizer_params(0.2, 0.01, 0.02)
        assert e.value.code == sb.capi.SB_ERR_STATE
    with sb.Trainer(desc(sb.OPT_ADAGRAD)) as t:
        with pytest.raises(sb.ShifuB200Error) as e:
            t.set_optimizer_params(0.1, 0.01, 0.0)            # Adagrad has no l1 / l2
        assert e.value.code == sb.capi.SB_ERR_INVALID
    for k in (sb.OPT_RMSPROP, sb.OPT_ADAM, sb.OPT_MOMENTUM, sb.OPT_SGD, sb.OPT_ADADELTA):
        with sb.Trainer(desc(k)) as t:
            with pytest.raises(sb.ShifuB200Error) as e:
                t.set_optimizer_params(0.1, 0.0, 0.0)
            assert e.value.code == sb.capi.SB_ERR_INVALID


CFG = {"cfg1": dict(F=1000, hidden=[512, 256, 128], batch=4096),
       "cfg2": dict(F=2000, hidden=[1024, 512, 256], batch=8192)}


def _dataset(F, rows, seed=7):
    rng = np.random.default_rng(seed)
    X = np.clip(rng.standard_normal((rows, F), dtype=np.float32), -4, 4)
    beta = rng.standard_normal(F).astype(np.float32) / np.sqrt(F)
    p = 1.0 / (1.0 + np.exp(-(2.5 * (X @ beta) - 1.2)))
    y = (rng.random(rows) < p).astype(np.float32)
    w = rng.choice(np.array([0.0, 1.0, 2.5], np.float32), size=rows, p=[0.1, 0.7, 0.2]).astype(np.float32)
    return X, y, w


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("cfg", ["cfg1", "cfg2"])
@pytest.mark.parametrize("name", list(OPTS))
def test_one_resident_step_is_the_oracle_update_of_its_gradient(sb, name, cfg, prec):
    kind, c = OPTS[name], CFG[cfg]
    net = so.NetDesc(c["F"], c["hidden"], [so.ACT_RELU] * len(c["hidden"]))
    theta0 = so.flatten_params(so.xavier_init(net, 4))
    X, y, w = _dataset(c["F"], c["batch"])
    with _trainer(sb, kind, c["F"], c["hidden"], c["batch"], prec) as t:
        t.set_params(theta0)
        t.load_dataset(X, y, w)
        t.step_resident(0, c["batch"])
        g, theta = t.get_grads(), t.get_params()
        s1, s2 = _state(sb, t)
    opt = tfo.Optimizer(_cfg(kind), theta0.size)
    want = opt.apply(theta0, g)
    assert np.abs(g).max() > 0
    assert np.abs(theta - want).max() <= 1e-4
    assert np.abs(s1 - opt.s1).max() <= 1e-4 * max(1.0, np.abs(opt.s1).max())
    assert np.abs(s2 - opt.s2).max() <= 1e-4 * max(1.0, np.abs(opt.s2).max())
    if kind == tfo.OPT_FTRL:    # the l1 ball: exact zeros where the oracle has them
        assert np.array_equal(theta == 0, want == 0) and (want == 0).any()


_CURVE_REF = {}


@pytest.mark.parametrize("prec", [FP32, FP32_TC, BF16])
@pytest.mark.parametrize("name", list(OPTS))
def test_cfg1_loss_curve_through_run_resident(sb, name, prec):
    kind, c, steps, n_batches = OPTS[name], CFG["cfg1"], 24, 5
    B = c["batch"]
    net = so.NetDesc(c["F"], c["hidden"], [so.ACT_RELU] * len(c["hidden"]))
    params = so.xavier_init(net, 4)
    X, y, w = _dataset(c["F"], n_batches * B)
    offs = [(i % n_batches) * B for i in range(steps)]
    key = (name, prec == BF16)
    if key not in _CURVE_REF:
        ref = (tfo.Bf16Trainer(net, params, _cfg(kind), fused_out=True) if prec == BF16
               else tfo.CleanTrainer(net, params, _cfg(kind)))
        want = [float(ref.step([(X[o:o + B], y[o:o + B].reshape(-1, 1), w[o:o + B].reshape(-1, 1))])[0]) for o in offs]
        _CURVE_REF[key] = (np.array(want), ref.theta.copy())
    want, ref_theta = _CURVE_REF[key]
    with _trainer(sb, kind, c["F"], c["hidden"], B, prec) as t:
        t.set_params(so.flatten_params(params))
        t.load_dataset(X, y, w)
        t.run_resident(offs, B)
        got = t.loss_history(1, steps)
        theta = t.get_params()
    assert abs(want[0] - want[-1]) > 1e-3, "the planted signal must move the loss"
    if prec == BF16:
        assert np.abs(got - want).max() <= 5e-4, (got, want)
    else:
        assert np.abs(got - want).max() <= 1e-4, (got, want)
        assert np.abs(theta - ref_theta).max() <= 1e-4


def _small(sb, kind, prec, det=True):
    return _trainer(sb, kind, 96, [64, 32], 128, prec, deterministic=det)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("name", list(OPTS))
def test_checkpoint_resume_and_deterministic_runs_are_bit_identical(sb, tmp_path, name, prec):
    kind = OPTS[name]
    net = so.NetDesc(96, [64, 32], [so.ACT_RELU] * 2)
    theta0 = so.flatten_params(so.xavier_init(net, 9))
    X, y, w = so.synth_batch(4 * 128, 96, 5, weights="mixed")
    offs = [(i % 4) * 128 for i in range(10)]
    ck = str(tmp_path / "opt.ckpt")

    def run(t, o):
        for off in o:
            t.step_resident(off, 128)

    results = []
    for _ in range(2):                                     # two uninterrupted runs
        with _small(sb, kind, prec) as t:
            t.set_params(theta0); t.load_dataset(X, y, w)
            run(t, offs)
            results.append((t.get_params(), *_state(sb, t), t.loss_history(1, 10)))
    with _small(sb, kind, prec) as t:                      # k = 4 steps, checkpoint
        t.set_params(theta0); t.load_dataset(X, y, w)
        run(t, offs[:4])
        t.save_checkpoint(ck)
    with _small(sb, kind, prec) as t:                      # a fresh trainer continues from it
        t.load_checkpoint(ck)
        t.load_dataset(X, y, w)
        assert t.global_step == 4
        run(t, offs[4:])
        resumed = (t.get_params(), *_state(sb, t))
    for a, b in zip(results[0], results[1]):
        np.testing.assert_array_equal(a, b)
    for a, b in zip(results[0][:3], resumed):
        np.testing.assert_array_equal(a, b)
    other = tfo.OPT_ADAGRAD if kind != tfo.OPT_ADAGRAD else tfo.OPT_FTRL
    with _small(sb, other, prec) as t:                     # another optimizer's state does not apply
        with pytest.raises(sb.ShifuB200Error) as e:
            t.load_checkpoint(ck)
        assert e.value.code == sb.capi.SB_ERR_FORMAT


def _owner_of_each_param(lay, W, n):
    own = np.full(n, -1, np.int64)
    for s in range(lay["slots"]):
        b, e = lay["begin"][s], lay["end"][s]
        for r in range(W):
            for k in range(b + ((e - b) * r) // W, b + ((e - b) * (r + 1)) // W):
                wk = lay["work"][k]
                own[wk["off"]:wk["off"] + wk["count"]] = r
    return own


@pytest.mark.parametrize("W,prec", [(2, FP32), (4, FP32), (2, BF16), (2, FP32_TC), (2, BF16X2)])
@pytest.mark.parametrize("name", list(OPTS))
def test_replicas_on_one_gpu_update_on_the_owner_only(sb, monkeypatch, name, W, prec):
    monkeypatch.setenv("SB_XCHG_BLOCKS", "8")
    monkeypatch.setenv("SB_XCHG_TIMEOUT_S", "60")
    kind = OPTS[name]
    F, hidden, B, n_batches, n_steps = 256, [192, 128, 64], 512, 3, 8
    acts = [so.ACT_RELU, so.ACT_TANH, so.ACT_LEAKYRELU]
    net = so.NetDesc(F, hidden, acts)
    params = so.xavier_init(net, 4)
    desc = sb.make_desc(F, hidden, acts, optimizer=kind, learning_rate=LR[kind], max_batch=B, precision=prec)
    kw = dict(FTRL_PARAMS) if kind == tfo.OPT_FTRL else {}
    ts = [sb.Trainer(desc, device=0, nccl_id=None, rank=r, world=W, **kw) for r in range(W)]
    try:
        bases = [t.exchange_base for t in ts]
        for t in ts:
            t.set_peer_pointers(bases)
            t.set_params(so.flatten_params(params))
        shards = []
        for r in range(W):
            X, y, w = so.synth_batch(n_batches * B, F, 100 + 17 * r, weights="mixed")
            rng = np.random.RandomState(100 + r)
            beta = rng.randn(F).astype(np.float32) / np.sqrt(F)
            y = (rng.uniform(size=(len(X), 1)) < 1 / (1 + np.exp(-2 * (X @ beta).reshape(-1, 1)))).astype(np.float32)
            shards.append((X, y, w))
        for t, (X, y, w) in zip(ts, shards):
            t.load_dataset(X, y, w)
        offs = [(s % n_batches) * B for s in range(n_steps)]
        for s0 in range(0, n_steps, 4):
            for t in ts:
                t.run_resident(offs[s0:s0 + 4], B)
        for t in ts:
            t.sync()
        # raw state before anything gathers it: a run's state changed on its owner only
        lay = ts[0].debug_exchange_layout()
        own = _owner_of_each_param(lay, W, ts[0].n_params)
        assert np.all(own >= 0)
        s1_0 = np.float32(1.0 if kind == tfo.OPT_RMSPROP else 0.1)
        for r, t in enumerate(ts):
            s1 = t.debug_buffer(sb.capi.DEBUG_BUF_S1)
            assert np.all(s1[own != r] == s1_0), "rank %d changed state it does not own" % r
            assert np.mean(s1[own == r] != s1_0) > 0.5
        losses = np.stack([t.loss_history(1, n_steps) for t in ts], axis=1)
        thetas = [t.get_params() for t in ts]
        grads = [t.get_grads() for t in ts]
        preds = [t.predict(shards[0][0][:200]) for t in ts]
    finally:
        for t in ts:
            t.close()
    for r in range(1, W):
        np.testing.assert_array_equal(thetas[0], thetas[r])
        np.testing.assert_array_equal(grads[0], grads[r])
        np.testing.assert_array_equal(preds[0], preds[r])
    ref = tfo.Bf16Trainer(net, params, _cfg(kind), fused_out=True) if prec == BF16 else tfo.CleanTrainer(net, params, _cfg(kind))
    want = np.array([ref.step([(X[o:o + B], y[o:o + B], w[o:o + B]) for (X, y, w) in shards]) for o in offs])
    if prec in (FP32, FP32_TC):
        assert np.abs(losses - want).max() <= 1e-4
        assert np.abs(thetas[0] - ref.theta).max() <= 1e-4
    else:       # bf16 (vs the bf16-emulating oracle) and bf16x2 (vs fp32): the bounds of test_data_parallel_one_gpu.py
        assert np.abs(losses - want).max() <= 1e-3
        assert np.abs(thetas[0] - ref.theta).max() <= 5e-3


@pytest.mark.parametrize("prec", [FP32, FP32_TC])
@pytest.mark.parametrize("name", ["adagrad", "ftrl"])
def test_wide_deep_sparse_step(sb, name, prec):
    kind = OPTS[name]
    n_dense, vocab, hidden, acts, rows = 21, [5, 9, 3, 17], [40, 24], [so.ACT_TANH, so.ACT_RELU], 130
    n_onehot = sum(vocab)
    net = so.NetDesc(n_dense + n_onehot, hidden, acts)
    params = so.xavier_init(net, 2)
    Xd, idx, y, w = wd.synth_wide_deep_batch(rows, n_dense, vocab, 2)
    desc = sb.make_desc(n_dense + n_onehot, hidden, acts, optimizer=kind, learning_rate=LR[kind], max_batch=rows, precision=prec)
    kw = dict(FTRL_PARAMS) if kind == tfo.OPT_FTRL else {}
    ref = tfo.Optimizer(_cfg(kind), net.n_params)
    theta0 = so.flatten_params(params)
    with sb.Trainer(desc, **kw) as t:
        t.set_params(theta0)
        t.set_sparse(n_dense, n_onehot, len(vocab))
        theta = theta0
        for step in range(3):
            P = so.unflatten_params(net, theta)
            L, g, _ = wd.loss_and_grads_sparse(net, P, Xd, idx, y, w)
            g = so.flatten_params(g)
            loss = t.step_sparse(Xd, idx, y, w)
            assert abs(loss - L) <= 1e-4
            assert np.abs(t.get_grads() - g).max() <= 1e-4
            theta = ref.apply(theta, t.get_grads())
            assert np.abs(t.get_params() - theta).max() <= 1e-4
            theta = t.get_params()


@pytest.mark.parametrize("name", list(OPTS))
def test_worker_end_to_end_matches_the_sync_replicas_oracle(sb, tmp_path, name):
    """Optimizer: adagrad | rmsprop | ftrl in ModelConfig (TF defaults) through the whole worker, against
    SyncReplicasTrainer driven by the reference's loop (as tests/test_host_mirrors.py does for Adadelta)"""
    from test_host_mirrors import _run_worker, _Seq
    from shifu_tensorflow_b200 import trainer as tr
    kind = OPTS[name]
    lr = 0.05
    rc, lines, env, (X, y, w, F, conf) = _run_worker(sb, tmp_path, 1000, 4, {"Optimizer": name, "LearningRate": lr})
    assert rc == 0
    ctx = tr.load_data(env["TRAINING_DATA_PATH"], list(range(1, F + 1)), 0, -1, 0.2, rng=_Seq(5))
    tx = np.asarray(ctx["train_data"], np.float32); ty = np.asarray(ctx["train_target"], np.float32)
    tw = np.asarray(ctx["train_data_sample_weight"], np.float32)
    vx = np.asarray(ctx["valid_data"], np.float32); vy = np.asarray(ctx["valid_target"], np.float32)
    vw = np.asarray(ctx["valid_data_sample_weight"], np.float32)
    net = so.NetDesc(F, [8, 4], [so.ACT_TANH, so.ACT_RELU])
    with sb.Trainer(tr.model(F, conf, 128)) as t0:
        assert t0.desc.optimizer == kind
        t0.init_xavier(11)
        theta = t0.get_params()
    R = so.replicas_to_aggregate(1000, 0.2, 100)
    ref = tfo.SyncReplicasTrainer(net, so.unflatten_params(net, theta), tfo.tf_config(kind, lr), R)
    batches = so.split_batches(len(tx), 100)
    want = []
    while ref.global_step < 4:
        for bi in batches:
            L, gs = ref.run(tx[bi], ty[bi], tw[bi])
            if gs >= 4:
                break
        A, z, yh = so.forward(net, so.unflatten_params(net, ref.theta), vx)
        want.append((gs, float(L), float(so.loss_value(z, yh, vy, vw, so.LOSS_MSE)[0])))
    got = [(int(l.split("current_epoch:")[1].split(",")[0]), float(l.split("training_loss:")[1].split(",")[0]),
            float(l.split("valid_loss:")[1])) for l in lines]
    assert [g[0] for g in got] == [x[0] for x in want]
    assert np.abs(np.array(got)[:, 1:] - np.array(want)[:, 1:]).max() <= 1e-4
