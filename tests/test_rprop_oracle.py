"""CPU checks of RPROP (SB_OPT_RPROP, iRPROP-): the float32 restatement (tests/rprop_ref.py) against torch.optim.Rprop bit
for bit, the oracle's sync_replicas trainer with it, the full-batch training it is meant for, the worker's ModelConfig
name, and the C-ABI's descriptor check."""
import os

import numpy as np
import pytest

import rprop_ref as rr
from oracle import shifu_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def _gradients(n, steps, seed):
    """float32 gradients over `steps` updates whose columns exercise every branch of the rule:
      [0, n/8)       sign alternates every update (repeated flips: the step halves every second update, to 1e-6)
      [n/8, n/4)     constant sign (the step grows by 1.2 per update, to 50)
      [n/4, 3n/8)    magnitudes around 1e-25: products of consecutive gradients underflow to +-0
      [3n/8, n/2)    exact zeros and -0 mixed with ordinary values
      [n/2, n)       random sign and magnitude 1e-30 .. 1e2"""
    rng = np.random.default_rng(seed)
    q = n // 8
    sign0 = rng.choice([-1.0, 1.0], n)
    out = []
    for s in range(steps):
        g = rng.choice([-1.0, 1.0], n) * 10.0 ** rng.uniform(-30, 2, n)
        g[:q] = sign0[:q] * (-1.0) ** s * 10.0 ** rng.uniform(-3, 1, q)
        g[q:2 * q] = sign0[q:2 * q] * 10.0 ** rng.uniform(-3, 1, q)
        g[2 * q:3 * q] = rng.choice([-1.0, 1.0], q) * 10.0 ** rng.uniform(-26, -24, q)
        z = g[3 * q:4 * q]
        k = rng.integers(0, 3, q)
        z[k == 0] = 0.0
        z[k == 1] = -0.0
        out.append(g.astype(np.float32))
    return out


def test_gradients_reach_every_branch():
    n, steps = 4096, 60
    gs = _gradients(n, steps, 1)
    prev, step = rr.start_state(0.01, n)
    theta = np.zeros(n, np.float32)
    seen_flip = seen_underflow = False
    for g in gs:
        p = g * prev
        seen_flip |= bool(np.any(p < 0))
        seen_underflow |= bool(np.any((p == 0) & (g != 0) & (prev != 0)))
        theta, prev, step = rr.rprop_update(theta, g, prev, step)
    assert seen_flip and seen_underflow
    assert np.any(step == rr.STEP_MIN) and np.any(step == rr.STEP_MAX)
    assert np.any(_bits(gs[0]) == 0x80000000) and np.any(_bits(gs[0]) == 0)


@pytest.mark.parametrize("lr", [0.01, 1e-8, 100.0, 0.003])
def test_rule_matches_torch_rprop_bit_for_bit(lr):
    """60 updates; lr 1e-8 and 100 lie outside [1e-6, 50], so torch clamps the step on the first update"""
    torch = pytest.importorskip("torch")
    n, steps = 4096, 60
    theta0 = (np.random.default_rng(2).standard_normal(n) * 0.5).astype(np.float32)
    p = torch.nn.Parameter(torch.tensor(theta0))
    topt = torch.optim.Rprop([p], lr=lr, etas=(0.5, 1.2), step_sizes=(1e-6, 50), foreach=False)
    theta = theta0.copy()
    prev, step = rr.start_state(lr, n)
    for s, g in enumerate(_gradients(n, steps, 3)):
        p.grad = torch.tensor(g)
        topt.step()
        theta, prev, step = rr.rprop_update(theta, g, prev, step)
        st = topt.state[p]
        for what, got, want in (("theta", theta, p.detach().numpy()), ("prev", prev, st["prev"].numpy()),
                                ("step", step, st["step_size"].numpy())):
            bad = np.flatnonzero(_bits(got) != _bits(want))
            assert bad.size == 0, "update %d: %s differs at %s: %r vs torch %r" % (s + 1, what, bad[:8], got[bad[:8]],
                                                                                  want[bad[:8]])
    if lr > 50 or lr < 1e-6:
        assert np.all(step >= rr.STEP_MIN) and np.all(step <= rr.STEP_MAX)


def test_zero_gradient_keeps_theta_bits_and_flip_skips_one_update():
    theta = np.array([0.5, -0.0, 0.0, 1.0, 2.0], np.float32)
    prev = np.array([1.0, 1.0, -1.0, 1.0, 1.0], np.float32)
    step = np.full(5, 0.25, np.float32)
    g = np.array([0.0, -0.0, -0.0, -3.0, 3.0], np.float32)
    t2, p2, s2 = rr.rprop_update(theta, g, prev, step)
    assert np.array_equal(_bits(t2[:3]), _bits(theta[:3]))              # +-0 gradients: theta keeps its bits
    assert t2[3] == np.float32(1.0) and p2[3] == 0 and s2[3] == np.float32(0.125)   # a flip: no move, prev = 0
    assert t2[4] == np.float32(2.0) - np.float32(0.3) and s2[4] == np.float32(0.25) * np.float32(1.2)
    t3, p3, s3 = rr.rprop_update(t2, g, p2, s2)                          # after a flip the next update never shrinks
    assert s3[3] == s2[3] and t3[3] == t2[3] + s2[3]


def _synthetic(rows, F, seed):
    rng = np.random.default_rng(seed)
    X = np.clip(rng.standard_normal((rows, F)), -3, 3).astype(np.float32)
    beta = rng.standard_normal(F) / np.sqrt(F)
    pr = 1.0 / (1.0 + np.exp(-(3.0 * (X @ beta) - 0.5)))
    y = (rng.random(rows) < pr).astype(np.float32).reshape(-1, 1)
    return X, y, np.ones((rows, 1), np.float32)


def _run_epochs(tr, X, y, w, epochs):
    batches = so.split_batches(len(X), 100)
    while tr.global_step < epochs:
        for bi in batches:
            _, gs = tr.run(X[bi], y[bi], w[bi])
            if gs >= epochs:
                break


def _train_loss(net, theta, X, y, w):
    A, z, yh = so.forward(net, so.unflatten_params(net, theta), X)
    return float(so.loss_value(z, yh, y, w, so.LOSS_MSE)[0])


def test_sync_replicas_oracle_is_the_restatement_fed_its_gradients():
    F, hidden = 12, [8, 4]
    net = so.NetDesc(F, hidden, [so.ACT_TANH, so.ACT_RELU])
    X, y, w = _synthetic(1000, F, 4)
    params = so.xavier_init(net, 11)
    lr = 0.01
    R = so.replicas_to_aggregate(1000, 0.0, 100)
    tr = rr.SyncReplicasTrainer(net, params, so.OptConfig(kind=rr.RPROP, lr=lr), R)
    applied = []
    apply = tr.opt.apply
    tr.opt.apply = lambda theta, g: (applied.append(np.array(g, np.float32)), apply(theta, g))[1]
    _run_epochs(tr, X, y, w, 6)
    assert len(applied) == 6 and tr.global_step == 6
    theta = so.flatten_params(params).astype(np.float32)
    prev, step = rr.start_state(lr, theta.size)
    for g in applied:
        theta, prev, step = rr.rprop_update(theta, g, prev, step)
    assert np.array_equal(_bits(theta), _bits(tr.theta))
    assert np.array_equal(_bits(prev), _bits(tr.opt.s1)) and np.array_equal(_bits(step), _bits(tr.opt.s2))
    assert np.any(step != np.float32(lr))


def test_rprop_trains_full_batch_where_adadelta_barely_moves():
    """30 sync_replicas epochs (one update each, from the whole set's mean gradient) at the reference's LearningRate
    0.003: RPROP ends at a lower training loss than Adadelta with the reference's defaults"""
    F, hidden = 12, [8, 4]
    net = so.NetDesc(F, hidden, [so.ACT_TANH, so.ACT_RELU])
    X, y, w = _synthetic(1000, F, 6)
    params = so.xavier_init(net, 3)
    R = so.replicas_to_aggregate(1000, 0.0, 100)
    start = _train_loss(net, so.flatten_params(params), X, y, w)
    final = {}
    for kind in (so.OPT_ADADELTA, rr.RPROP):
        tr = rr.SyncReplicasTrainer(net, params, so.OptConfig(kind=kind, lr=0.003), R)
        _run_epochs(tr, X, y, w, 30)
        final[kind] = _train_loss(net, tr.theta, X, y, w)
    assert abs(final[so.OPT_ADADELTA] - start) < 1e-3, (start, final)
    assert final[rr.RPROP] < final[so.OPT_ADADELTA] - 0.01, (start, final)


def test_worker_model_maps_rprop_in_any_case(sb):
    from shifu_tensorflow_b200 import trainer as tr
    for name in ("rprop", "RPROP", "Rprop", "RProp"):
        conf = {"train": {"params": {"NumHiddenLayers": 1, "NumHiddenNodes": [8], "ActivationFunc": ["relu"],
                                     "LearningRate": 0.02, "Optimizer": name}}}
        d = tr.model(6, conf, 32)
        assert d.optimizer == sb.OPT_RPROP == sb.capi.OPT_RPROP == 8
        assert d.learning_rate == np.float32(0.02)


def test_header_exposes_rprop():
    hdr = open(os.path.join(ROOT, "include", "shifu_b200.h")).read()
    assert "SB_OPT_RPROP = 8" in hdr and "= 7" not in hdr.split("sb_optimizer;")[0].split("SB_OPT_ADADELTA")[-1]


def test_descriptor_check_accepts_rprop(sb):
    """optimizer 8 passes the descriptor check: without a device the trainer is then refused for the missing device
    (SB_ERR_CUDA), with one it is created"""
    d = sb.make_desc(8, [4], [2], optimizer=sb.OPT_RPROP, learning_rate=0.01)
    if sb.capi.device_count() > 0:
        sb.Trainer(d).close()
        return
    with pytest.raises(sb.ShifuB200Error) as e:
        sb.Trainer(d)
    assert e.value.code == sb.capi.SB_ERR_CUDA, str(e.value)


@pytest.mark.parametrize("kind", [7, 9, -1])
def test_descriptor_check_refuses_the_values_around_rprop(sb, kind):
    with pytest.raises(sb.ShifuB200Error) as e:
        sb.Trainer(sb.make_desc(8, [4], [2], optimizer=kind))
    assert e.value.code == sb.capi.SB_ERR_INVALID
