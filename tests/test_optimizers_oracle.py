"""CPU checks of Adagrad, RMSProp and FTRL (TF 1.x training_ops.cc forms): the oracle's rules (oracle/tf_optimizers.py)
against torch and against a float64 restatement written here, their slot start values, the worker's ModelConfig names,
make_desc's per-optimizer defaults and the descriptor checks the C-ABI makes before it looks for a device."""
import ctypes
import math
import os

import numpy as np
import pytest

from oracle import shifu_oracle as so
from oracle import tf_optimizers as tfo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _grads(n, steps, seed):
    rng = np.random.default_rng(seed)
    return [rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 1, n) for _ in range(steps)]


def test_adagrad_matches_torch_in_float64():
    torch = pytest.importorskip("torch")
    n, lr = 257, 0.05
    theta0 = np.random.default_rng(1).standard_normal(n)
    p = torch.nn.Parameter(torch.tensor(theta0, dtype=torch.float64))
    topt = torch.optim.Adagrad([p], lr=lr, lr_decay=0, initial_accumulator_value=0.1, eps=0)
    opt = tfo.Optimizer(tfo.tf_config(tfo.OPT_ADAGRAD, lr), n, np.float64)
    theta = theta0.copy()
    for g in _grads(n, 5, 2):
        p.grad = torch.tensor(g, dtype=torch.float64)
        topt.step()
        theta = opt.apply(theta, g)
        assert np.abs(theta - p.detach().numpy()).max() <= 1e-12
        assert np.abs(opt.s1 - topt.state[p]["sum"].numpy()).max() <= 1e-12


def _rmsprop_ref(theta, grads, lr, decay, momentum, eps):
    """ApplyRMSProp element by element in float64; ms starts at 1 (TF's ones initializer), mom at 0"""
    theta = [float(v) for v in theta]
    ms, mom = [1.0] * len(theta), [0.0] * len(theta)
    for g in grads:
        for i, gi in enumerate(g):
            ms[i] = ms[i] + (gi * gi - ms[i]) * (1.0 - decay)
            mom[i] = momentum * mom[i] + lr * gi / math.sqrt(ms[i] + eps)
            theta[i] -= mom[i]
    return np.array(theta), np.array(ms), np.array(mom)


def _ftrl_ref(theta, grads, lr, l1, l2, acc0):
    """ApplyFtrl with learning_rate_power = -0.5 element by element in float64"""
    theta = [float(v) for v in theta]
    acc, lin = [acc0] * len(theta), [0.0] * len(theta)
    for g in grads:
        for i, gi in enumerate(g):
            new_acc = acc[i] + gi * gi
            lin[i] += gi - (math.sqrt(new_acc) - math.sqrt(acc[i])) / lr * theta[i]
            quad = math.sqrt(new_acc) / lr + 2.0 * l2
            theta[i] = (math.copysign(l1, lin[i]) - lin[i]) / quad if abs(lin[i]) > l1 else 0.0
            acc[i] = new_acc
    return np.array(theta), np.array(acc), np.array(lin)


@pytest.mark.parametrize("momentum", [0.0, 0.7])
def test_rmsprop_matches_float64_restatement(momentum):
    n, lr = 129, 0.01
    theta0 = np.random.default_rng(3).standard_normal(n)
    grads = _grads(n, 3, 4)
    cfg = tfo.tf_config(tfo.OPT_RMSPROP, lr, momentum=momentum)
    assert (cfg.rho, cfg.eps) == (0.9, 1e-10)
    opt = tfo.Optimizer(cfg, n, np.float64)
    theta = theta0.copy()
    for g in grads:
        theta = opt.apply(theta, g)
    want, ms, mom = _rmsprop_ref(theta0, grads, lr, 0.9, momentum, 1e-10)
    assert np.abs(theta - want).max() <= 1e-12
    assert np.abs(opt.s1 - ms).max() <= 1e-12 and np.abs(opt.s2 - mom).max() <= 1e-12


@pytest.mark.parametrize("l1,l2", [(0.0, 0.0), (0.01, 0.0), (0.0, 0.5), (0.02, 0.3)])
def test_ftrl_matches_float64_restatement(l1, l2):
    n, lr = 129, 0.05
    theta0 = np.random.default_rng(5).standard_normal(n)
    grads = _grads(n, 3, 6)
    opt = tfo.Optimizer(tfo.tf_config(tfo.OPT_FTRL, lr, l1=l1, l2=l2), n, np.float64)
    theta = theta0.copy()
    for g in grads:
        theta = opt.apply(theta, g)
    want, acc, lin = _ftrl_ref(theta0, grads, lr, l1, l2, 0.1)
    assert np.abs(theta - want).max() <= 1e-12
    assert np.abs(opt.s1 - acc).max() <= 1e-12 and np.abs(opt.s2 - lin).max() <= 1e-12


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_ftrl_zeroes_parameters_inside_the_l1_ball(dtype):
    n, lr, l1 = 4096, 0.1, 0.05
    rng = np.random.default_rng(7)
    theta = rng.standard_normal(n).astype(dtype)
    opt = tfo.Optimizer(tfo.tf_config(tfo.OPT_FTRL, lr, l1=l1), n, dtype)
    for _ in range(3):
        theta = opt.apply(theta, (rng.standard_normal(n) * 0.05).astype(dtype))
        inside = np.abs(opt.s2) <= dtype(l1)
        assert inside.any() and (~inside).any()
        assert np.all(theta[inside] == 0) and np.all(theta[~inside] != 0)
        assert theta.dtype == dtype
    # l1 = 0: a parameter whose gradient is exactly 0 from the start is set to 0 (linear stays 0) - TF's arithmetic
    opt = tfo.Optimizer(tfo.tf_config(tfo.OPT_FTRL, lr), 3, dtype)
    out = opt.apply(np.array([0.7, -0.2, 1.5], dtype), np.array([0.0, 0.3, 0.0], dtype))
    assert out[0] == 0 and out[2] == 0 and out[1] != 0


def test_initial_slot_values():
    n = 11
    for kind, s1, s2 in ((tfo.OPT_ADAGRAD, 0.1, 0.0), (tfo.OPT_FTRL, 0.1, 0.0), (tfo.OPT_RMSPROP, 1.0, 0.0),
                         (so.OPT_ADAM, 0.0, 0.0), (so.OPT_ADADELTA, 0.0, 0.0), (so.OPT_MOMENTUM, 0.0, 0.0)):
        opt = tfo.Optimizer(tfo.tf_config(kind, 0.01), n)
        assert np.all(opt.s1 == np.float32(s1)) and np.all(opt.s2 == np.float32(s2)), kind
    opt = tfo.Optimizer(tfo.tf_config(tfo.OPT_FTRL, 0.01, initial_accumulator=0.25), n)
    assert np.all(opt.s1 == np.float32(0.25))
    off = tfo.OptConfig(kind=tfo.OPT_RMSPROP, rmsprop_ms_starts_at_one=False)
    assert np.all(tfo.Optimizer(off, n).s1 == 0)


def test_reference_optimizers_unchanged_by_the_extension():
    """tf_optimizers.Optimizer runs the reference's four through shifu_oracle.Optimizer: same bits"""
    n = 300
    rng = np.random.default_rng(8)
    theta0 = rng.standard_normal(n).astype(np.float32)
    grads = [g.astype(np.float32) for g in _grads(n, 4, 9)]
    for kind in (so.OPT_ADADELTA, so.OPT_ADAM, so.OPT_SGD, so.OPT_MOMENTUM):
        a, b = so.Optimizer(so.OptConfig(kind=kind, lr=0.01), n), tfo.Optimizer(tfo.OptConfig(kind=kind, lr=0.01), n)
        ta, tb = theta0.copy(), theta0.copy()
        for g in grads:
            ta, tb = a.apply(ta, g), b.apply(tb, g)
        assert np.array_equal(ta, tb) and np.array_equal(a.s1, b.s1) and np.array_equal(a.s2, b.s2)


def _conf(opt):
    return {"train": {"params": {"NumHiddenLayers": 1, "NumHiddenNodes": [8], "ActivationFunc": ["relu"],
                                 "LearningRate": 0.02, "Optimizer": opt}}}


def test_worker_model_maps_optimizer_names_with_tf_defaults(sb):
    from shifu_tensorflow_b200 import trainer as tr
    f32 = lambda v: float(np.float32(v))
    for name, kind in (("adagrad", sb.OPT_ADAGRAD), ("rmsprop", sb.OPT_RMSPROP), ("ftrl", sb.OPT_FTRL),
                       ("RMSProp", sb.OPT_RMSPROP), ("Adagrad", sb.OPT_ADAGRAD), ("FTRL", sb.OPT_FTRL)):
        d = tr.model(6, _conf(name), 32)
        assert d.optimizer == kind
        if kind == sb.OPT_RMSPROP:
            assert (d.rho, d.epsilon, d.momentum) == (f32(0.9), f32(1e-10), 0.0)
        else:
            assert (d.rho, d.epsilon, d.momentum) == (f32(0.95), f32(1e-8), f32(0.9))
    assert (sb.OPT_ADAGRAD, sb.OPT_RMSPROP, sb.OPT_FTRL) == (4, 5, 6)
    assert sb.capi.INITIAL_ACCUMULATOR == 0.1 and sb.capi.L1 == 0.0 and sb.capi.L2 == 0.0


def test_make_desc_leaves_the_reference_optimizers_fields_bit_identical(sb):
    """the defaults every existing optimizer got before RMSProp's were added, spelled out"""
    for kind in (sb.OPT_ADADELTA, sb.OPT_ADAM, sb.OPT_SGD, sb.OPT_MOMENTUM):
        got = sb.make_desc(10, [6, 4], [2, 1], optimizer=kind, learning_rate=0.3, max_batch=64)
        want = sb.make_desc(10, [6, 4], [2, 1], optimizer=kind, learning_rate=0.3, rho=0.95, epsilon=1e-8, beta1=0.9,
                            beta2=0.999, momentum=0.9, max_batch=64)
        assert bytes(got) == bytes(want)
        assert (got.rho, got.epsilon, got.momentum) == tuple(float(np.float32(v)) for v in (0.95, 1e-8, 0.9))
    # explicit values win over the per-optimizer defaults
    d = sb.make_desc(10, [6], [2], optimizer=sb.OPT_RMSPROP, rho=0.5, epsilon=1e-3, momentum=0.25)
    assert (d.rho, d.epsilon, d.momentum) == (0.5, float(np.float32(1e-3)), 0.25)


def test_descriptor_layout_is_unchanged(sb):
    assert ctypes.sizeof(sb.NetDesc) == (2 + 2 * sb.capi.SB_MAX_HIDDEN + 2 + 6 + 2) * 4
    hdr = open(os.path.join(ROOT, "include", "shifu_b200.h")).read()
    for name, v in (("SB_OPT_ADAGRAD", 4), ("SB_OPT_RMSPROP", 5), ("SB_OPT_FTRL", 6)):
        assert "%s = %d" % (name, v) in hdr


@pytest.mark.parametrize("field,value", [("rho", -0.1), ("rho", 1.5), ("rho", float("nan")), ("momentum", -0.5),
                                         ("epsilon", -1e-9)])
def test_capi_rejects_invalid_rmsprop_hyperparameters_before_device_work(sb, field, value):
    d = sb.make_desc(8, [4], [2], optimizer=sb.OPT_RMSPROP, **{field: value})
    with pytest.raises(sb.ShifuB200Error) as e:
        sb.Trainer(d)
    assert e.value.code == sb.capi.SB_ERR_INVALID and "RMSProp" in str(e.value), str(e.value)


def test_capi_rejects_unknown_optimizer(sb):
    d = sb.make_desc(8, [4], [2], optimizer=7)
    with pytest.raises(sb.ShifuB200Error) as e:
        sb.Trainer(d)
    assert e.value.code == sb.capi.SB_ERR_INVALID


def test_tf_golden_optimizers_when_present():
    """TF's own three steps of each new optimizer (oracle/tf_golden_optimizers.py writes them on a machine with TF)"""
    path = os.path.join(ROOT, "tests", "golden", "tf_golden_optimizers.npz")
    if not os.path.exists(path):
        pytest.skip("tests/golden/tf_golden_optimizers.npz has not been generated (needs TensorFlow)")
    z = np.load(path)
    from oracle.tf_golden_optimizers import CASES
    for name, kind, kw in CASES:
        theta = z["theta0"].astype(np.float32)
        opt = tfo.Optimizer(tfo.tf_config(kind, float(z["lr"]), **kw), theta.size)
        for step in range(3):
            theta = opt.apply(theta, z["grad%d" % step].astype(np.float32))
            want = z["%s_step%d" % (name, step + 1)]
            assert np.abs(theta - want).max() <= 1e-6 * max(1.0, np.abs(want).max()), (name, step)
