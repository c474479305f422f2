"""Fine-tuning with frozen layers (sb_trainer_set_fixed_layers / Trainer(fixed_layers=...) / ModelConfig `FixedLayers`,
`FixedBias`).

Layers are numbered from 1 as in Shifu's NN trainer: hidden layers 1..L, the output layer L + 1.  A frozen parameter keeps
its bits - value, optimizer state and bf16 shadow - whatever the optimizer (Adam, Momentum, RMSProp and FTRL would move a
parameter whose gradient is zero), its get_grads entry is 0, and every parameter that trains gets the gradient it gets
without frozen layers.  A step skips the dW GEMM of a frozen weight matrix and the dA GEMMs nothing below needs."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from oracle import shifu_oracle as so
from util import make_pair

OPTS = [so.OPT_SGD, so.OPT_MOMENTUM, so.OPT_ADAM, so.OPT_ADADELTA, 4, 5, 6]   # + SB_OPT_ADAGRAD, RMSPROP, FTRL
PRECS = [0, 1, 2, 3]   # SB_PREC_FP32, SB_PREC_BF16, SB_PREC_FP32_TC, SB_PREC_BF16X2


def _layout(F, hidden):
    """-> [(w_off, w_n, b_off, b_n)] of layers 1..L+1 in the flat parameter vector"""
    out, off, prev = [], 0, F
    for h in list(hidden) + [1]:
        out.append((off, prev * h, off + prev * h, h))
        off += prev * h + h
        prev = h
    return out


def frozen_mask(F, hidden, layers, fix_bias=True):
    """bool [n_params]: the parameters FixedLayers = layers (1-based) / FixedBias = fix_bias freeze"""
    lay = _layout(F, hidden)
    m = np.zeros(lay[-1][2] + lay[-1][3], bool)
    for x in layers:
        wo, wn, bo, bn = lay[x - 1]
        m[wo:wo + wn] = True
        if fix_bias:
            m[bo:bo + bn] = True
    return m


class FrozenOracle:
    """An oracle trainer (CleanTrainer / Bf16Trainer) whose update skips the frozen parameters: their values and optimizer
    state are put back after every step"""

    def __init__(self, ref, mask):
        self.ref, self.mask = ref, mask

    def step(self, shards):
        r, m = self.ref, self.mask
        keep = (r.theta[m].copy(), r.opt.s1[m].copy(), r.opt.s2[m].copy())
        out = r.step(shards)
        r.theta[m], r.opt.s1[m], r.opt.s2[m] = keep
        return out


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


# ---------------------------------------------------------------- no GPU ----
def test_fixed_layers_key_parsing():
    from shifu_tensorflow_b200 import trainer as tr
    p = {"NumHiddenLayers": 3}
    assert tr.fixed_layers_requested(p) == ([], True)
    assert tr.fixed_layers_requested(dict(p, FixedLayers=[2, 1])) == ([1, 2], True)
    assert tr.fixed_layers_requested(dict(p, FixedLayers=["1", " 4 "], FixedBias="false")) == ([1, 4], False)
    assert tr.fixed_layers_requested(dict(p, FixedLayers=[4], FixedBias=True)) == ([4], True)
    # every layer but the biases: still something to train
    assert tr.fixed_layers_requested(dict(p, FixedLayers=[1, 2, 3, 4], FixedBias=False)) == ([1, 2, 3, 4], False)
    for bad in ([0], [5], [-1], [1, 1], ["x"], [1.5], [True], "1", [1, 2, 3, 4]):
        with pytest.raises(ValueError):
            tr.fixed_layers_requested(dict(p, FixedLayers=bad))
    with pytest.raises(ValueError):
        tr.fixed_layers_requested(dict(p, FixedLayers=[1], FixedBias="maybe"))


def _worker_env(tmp_path):
    return {"CLUSTER_SPEC": json.dumps({"ps": ["127.0.0.1:1"], "worker": ["127.0.0.1:2"]}), "WORKER_CNT": "1", "JOB_NAME": "worker",
            "TASK_ID": "0", "SOCKET_SERVER_PORT": "1", "SB_REQUIRE_SOCKET": "0", "TOTAL_TRAINING_DATA_NUMBER": "10",
            "SELECTED_COLUMN_NUMS": "1 2 3", "WEIGHT_COLUMN_NUM": "-1", "TARGET_COLUMN_NUM": "0",
            "TMP_MODEL_PATH": str(tmp_path / "t"), "FINAL_MODEL_PATH": str(tmp_path / "f"),
            "TRAINING_DATA_PATH": str(tmp_path / "none.gz")}


@pytest.mark.parametrize("fixed", [[0], [4], [1, 1], [1, 2, 3], ["one"]])
def test_worker_bad_fixed_layers_raise_before_any_device_call(tmp_path, monkeypatch, fixed):
    from shifu_tensorflow_b200 import _capi, trainer as tr

    def no_device(*a, **k):
        raise AssertionError("device call before the configuration check")
    monkeypatch.setattr(_capi, "lib", no_device)
    monkeypatch.setattr(tr, "load_data_gpu", no_device)
    monkeypatch.setattr(tr, "load_data", no_device)
    conf = {"train": {"params": {"NumHiddenLayers": 2, "NumHiddenNodes": [8, 4], "ActivationFunc": ["relu", "relu"],
                                 "LearningRate": 0.1, "FixedLayers": fixed}, "numTrainEpochs": 1, "validSetRate": 0.2}}
    cwd = os.getcwd()
    os.chdir(tmp_path)
    json.dump(conf, open("ModelConfig.json", "w"))
    try:
        with pytest.raises(ValueError, match="FixedLayers"):
            tr.main(env=_worker_env(tmp_path))
    finally:
        os.chdir(cwd)


def test_init_model_topology_mismatch_names_both(sb, tmp_path):
    from shifu_tensorflow_b200 import trainer as tr
    acts = [so.ACT_RELU, so.ACT_TANH]
    saved = sb.make_desc(12, [16, 8], acts)
    net = so.NetDesc(12, [16, 8], acts)
    flat = so.flatten_params(so.xavier_init(net, 1))
    d = str(tmp_path / "model")
    sb.capi.savedmodel_write(d, saved, flat)
    got = tr.read_init_model(d, sb.make_desc(12, [16, 8], acts))
    assert np.array_equal(_bits(got), _bits(flat))
    for other in (sb.make_desc(12, [16, 4], acts), sb.make_desc(13, [16, 8], acts), sb.make_desc(12, [16, 8], [so.ACT_RELU] * 2)):
        with pytest.raises(ValueError) as e:
            tr.read_init_model(d, other)
        msg = str(e.value)
        assert "[16, 8]" in msg and "SB_INIT_MODEL" in msg and "ModelConfig" in msg


def test_set_fixed_layers_null_arguments(sb):
    lib = sb.capi.lib()
    one = (C.c_int32 * 1)(1)
    assert lib.sb_trainer_set_fixed_layers(None, one, 1, 1) == sb.capi.SB_ERR_INVALID
    # a null layer list with n > 0 is refused before the trainer is looked at (the handle is never dereferenced)
    dummy = C.create_string_buffer(64)
    assert lib.sb_trainer_set_fixed_layers(C.cast(dummy, C.c_void_p), None, 1, 1) == sb.capi.SB_ERR_INVALID
    assert lib.sb_trainer_set_fixed_layers(C.cast(dummy, C.c_void_p), one, -1, 1) == sb.capi.SB_ERR_INVALID


@pytest.mark.parametrize("kind", [so.OPT_ADAM, so.OPT_MOMENTUM])
def test_frozen_oracle_skips_only_the_frozen_parameters(kind):
    F, hidden = 10, [6, 4]
    net = so.NetDesc(F, hidden, [so.ACT_RELU, so.ACT_TANH])
    params = so.xavier_init(net, 3)
    cfg = so.OptConfig(kind=kind, lr=0.05)
    X, y, w = so.synth_batch(32, F, 1, weights="mixed")
    m = frozen_mask(F, hidden, [1], True)
    plain, none = so.CleanTrainer(net, params, cfg), FrozenOracle(so.CleanTrainer(net, params, cfg), np.zeros_like(m))
    frozen = FrozenOracle(so.CleanTrainer(net, params, cfg), m)
    start = frozen.ref.theta.copy()
    first = plain.theta.copy()
    for k in range(3):
        assert plain.step([(X, y, w)]) == none.step([(X, y, w)])
        frozen.step([(X, y, w)])
        if k == 0:
            first = plain.theta.copy()
            # one step: the trainable parameters take the plain update (the gradient does not depend on what is frozen)
            assert np.array_equal(frozen.ref.theta[~m], first[~m])
    assert np.array_equal(plain.theta, none.ref.theta)
    assert np.array_equal(_bits(frozen.ref.theta[m]), _bits(start[m]))
    assert not np.any(frozen.ref.opt.s1[m]) and not np.any(frozen.ref.opt.s2[m])
    assert not np.array_equal(frozen.ref.theta[~m], start[~m])


# ---------------------------------------------------------------- GPU ----
HID = [256, 128, 96, 64]    # layers 1..4 hidden, 5 the output layer
FROZEN_SETS = [([1], True), ([2], True), ([5], True), ([1, 2], True), ([1], False), ([3], True)]


def _state(sb, t, precision, F, hidden):
    c = sb.capi
    st = [t.debug_buffer(c.DEBUG_BUF_THETA), t.debug_buffer(c.DEBUG_BUF_S1), t.debug_buffer(c.DEBUG_BUF_S2)]
    sh = []
    if precision != 0:
        prev = F
        for l, h in enumerate(hidden):
            sh.append(t.debug_buffer(c.DEBUG_BUF_SHADOW + l, n=c.PARTS[precision] * prev * (-(-h // 8) * 8)))
            prev = h
    return st, sh


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECS)
@pytest.mark.parametrize("optimizer", OPTS)
def test_frozen_bits_stay_put(sb, optimizer, precision):
    """8 steps through run_resident: every frozen value, optimizer-state word and bf16 shadow keeps its bits, the frozen
    entries of get_grads are 0, and the parameters that train move"""
    F, rows = 192, 512
    X, y, w = so.synth_batch(2 * rows, F, 7, weights="mixed")
    for layers, fix_bias in FROZEN_SETS:
        _, params, _, desc = make_pair(sb, F, HID, [so.ACT_RELU, so.ACT_TANH, so.ACT_RELU, so.ACT_SIGMOID], optimizer=optimizer,
                                       lr=0.01, max_batch=rows, precision=precision, seed=5)
        m = frozen_mask(F, HID, layers, fix_bias)
        with sb.Trainer(desc, fixed_layers=layers, fixed_bias=fix_bias) as t:
            t.set_params(so.flatten_params(params))
            (th0, s10, s20), sh0 = _state(sb, t, precision, F, HID)
            t.load_dataset(X, y, w)
            t.run_resident([(k % 2) * rows for k in range(8)], rows)
            t.sync()
            (th1, s11, s21), sh1 = _state(sb, t, precision, F, HID)
            g = t.get_grads()
        what = (layers, fix_bias)
        assert np.array_equal(_bits(th1)[m], _bits(th0)[m]), what
        assert np.array_equal(_bits(s11)[m], _bits(s10)[m]) and np.array_equal(_bits(s21)[m], _bits(s20)[m]), what
        assert not np.any(g[m]), what
        assert np.isfinite(th1).all() and not np.array_equal(th1[~m], th0[~m]), what
        for l in range(len(sh0)):     # tensor-core modes: the bf16 shadow of every hidden layer
            if (l + 1) in layers:
                assert np.array_equal(sh1[l], sh0[l]), (what, l)
            else:
                assert not np.array_equal(sh1[l], sh0[l]), (what, l)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECS)
def test_trainable_gradients_unchanged(sb, precision):
    """one deterministic step from the same parameters and batch, with and without frozen layers: fp32 mode gives the
    trainable gradients bit for bit, the tensor-core modes within the deterministic gradient's tolerances
    (tests/test_deterministic.py)"""
    F, rows = 300, 1000
    acts = [so.ACT_RELU, so.ACT_TANH, so.ACT_RELU]
    hidden = [200, 128, 77]
    X, y, w = so.synth_batch(rows, F, 4, weights="mixed")
    _, params, _, desc = make_pair(sb, F, hidden, acts, optimizer=so.OPT_SGD, lr=0.01, max_batch=rows, precision=precision)
    with sb.Trainer(desc, deterministic=True) as t:
        t.set_params(so.flatten_params(params))
        t.step(X, y, w)
        g_all = t.get_grads()
    for layers, fix_bias in [([1], True), ([1, 2], True), ([2], False), ([4], True), ([1, 2, 3], True)]:
        m = frozen_mask(F, hidden, layers, fix_bias)
        with sb.Trainer(desc, deterministic=True, fixed_layers=layers, fixed_bias=fix_bias) as t:
            t.set_params(so.flatten_params(params))
            t.step(X, y, w)
            g = t.get_grads()
        assert not np.any(g[m])
        if precision == 0:
            assert np.array_equal(_bits(g)[~m], _bits(g_all)[~m]), layers
        else:
            # fp32_tc 1e-4 absolute, bf16 2e-3 of max|g|, bf16x2 max(1e-4, 1e-3 of max|g|)
            gmax = float(np.abs(g_all).max())
            tol = {1: 2e-3 * gmax, 2: 1e-4, 3: max(1e-4, 1e-3 * gmax)}[precision]
            assert np.abs(g[~m] - g_all[~m]).max() <= tol, layers


@pytest.mark.gpu
def test_refusals(sb):
    F, hidden, rows = 64, [32, 16], 128
    X, y, w = so.synth_batch(rows, F, 1, weights="ones")
    _, _, _, desc = make_pair(sb, F, hidden, [so.ACT_RELU] * 2, max_batch=rows, precision=sb.PREC_BF16)
    c = sb.capi
    with sb.Trainer(desc) as t:
        for layers, fb in (([0], True), ([4], True), ([-1], True), ([1, 1], True), ([2, 1, 2], False), ([1, 2, 3], True)):
            with pytest.raises(sb.ShifuB200Error) as e:
                t.set_fixed_layers(layers, fb)
            assert e.value.code == c.SB_ERR_INVALID, layers
        t.set_fixed_layers([1, 2, 3], False)       # only the biases train
        t.set_fixed_layers([1])
        t.step(X, y, w)
        with pytest.raises(sb.ShifuB200Error) as e:
            t.set_fixed_layers([2])
        assert e.value.code == c.SB_ERR_STATE
    ts = [sb.Trainer(desc, rank=r, world=2) for r in range(2)]
    try:
        bases = [t.exchange_base for t in ts]
        for t in ts:
            t.set_peer_pointers(bases)
        with pytest.raises(sb.ShifuB200Error) as e:
            ts[0].set_fixed_layers([1])
        assert e.value.code == c.SB_ERR_STATE and "peer" in str(e.value)
    finally:
        for t in ts:
            t.close()


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECS)
def test_losses_match_oracle(sb, precision):
    """per-step losses against an oracle trainer whose update skips the frozen parameters, within the oracle bounds of
    tests/test_deterministic.py: 1e-4 for fp32 / fp32_tc, 5e-4 for bf16 (Bf16Trainer) and bf16x2"""
    F, hidden, rows, steps = 1000, [512, 256, 128], 2048, 8
    acts = [so.ACT_RELU] * 3
    net, params, cfg, desc = make_pair(sb, F, hidden, acts, optimizer=so.OPT_ADAM, lr=0.01, max_batch=rows, precision=precision,
                                       seed=3)
    X, y, w = so.synth_batch(2 * rows, F, 21, weights="mixed")
    offs = [(k % 2) * rows for k in range(steps)]
    for layers in ([1], [1, 2]):
        m = frozen_mask(F, hidden, layers)
        ref = FrozenOracle(so.Bf16Trainer(net, params, cfg, fused_out=True) if precision == 1 else so.CleanTrainer(net, params, cfg), m)
        want = np.asarray([ref.step([(X[o:o + rows], y[o:o + rows], w[o:o + rows])])[0] for o in offs], np.float64)
        with sb.Trainer(desc, fixed_layers=layers) as t:
            t.set_params(so.flatten_params(params))
            t.load_dataset(X, y, w)
            t.run_resident(offs, rows)
            got = t.loss_history(1, steps).astype(np.float64)
        tol = 1e-4 if precision in (0, 2) else 5e-4
        assert np.abs(got - want).max() <= tol, (layers, got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cfg1", "cfg2"])
def test_fewer_launches(sb, name):
    """bf16 resident step: [1] drops dW_0, dA_1 and layer 0's optimizer pass; [1, 2] also dW_1 and dA_2"""
    F, hidden, rows = {"cfg1": (1000, [512, 256, 128], 4096), "cfg2": (2000, [1024, 512, 256], 8192)}[name]
    X, y, w = so.synth_batch(rows, F, 3, weights="mixed")
    _, params, _, desc = make_pair(sb, F, hidden, [so.ACT_RELU] * 3, optimizer=so.OPT_ADAM, max_batch=rows, precision=sb.PREC_BF16)
    kps = {}
    for layers in ((), (1,), (1, 2)):
        with sb.Trainer(desc, fixed_layers=layers) as t:
            t.set_params(so.flatten_params(params))
            t.load_dataset(X, y, w)
            t.step_resident(0, rows)
            kps[layers] = t.kernels_per_step(rows)
    assert kps[(1,)] == kps[()] - 3 and kps[(1, 2)] == kps[()] - 5, kps


@pytest.mark.gpu
def test_sync_replicas_apply_keeps_frozen_bits(sb):
    F, hidden, rows = 200, [128, 64], 256
    _, params, _, desc = make_pair(sb, F, hidden, [so.ACT_RELU] * 2, optimizer=so.OPT_ADADELTA, lr=1.0, max_batch=rows,
                                   precision=sb.PREC_BF16)
    m = frozen_mask(F, hidden, [1, 3], True)
    with sb.Trainer(desc, fixed_layers=[1, 3]) as t:
        t.set_params(so.flatten_params(params))
        p0 = t.get_params()
        for k in range(2):
            for s in range(3):
                t.accumulate(*so.synth_batch(rows, F, 10 * k + s, weights="mixed"))
            t.apply_accumulated()
        p1 = t.get_params()
        s1 = t.debug_buffer(sb.capi.DEBUG_BUF_S1)
    assert np.array_equal(_bits(p1)[m], _bits(p0)[m]) and not np.any(s1[m])
    assert not np.array_equal(p1[~m], p0[~m])


@pytest.mark.gpu
def test_wide_deep_frozen_layer0_keeps_embedding(sb):
    from oracle import wide_deep as wd
    n_dense, vocab, hidden, acts, rows = 21, [5, 9, 3, 17], [40, 24], [so.ACT_TANH, so.ACT_RELU], 130
    n_onehot = sum(vocab)
    F = n_dense + n_onehot
    params = so.xavier_init(so.NetDesc(F, hidden, acts), 2)
    for prec in (0, 1):
        desc = sb.make_desc(F, hidden, acts, optimizer=so.OPT_ADAM, learning_rate=0.05, max_batch=rows, precision=prec)
        m = frozen_mask(F, hidden, [1])
        with sb.Trainer(desc, fixed_layers=[1]) as t:
            t.set_params(so.flatten_params(params))
            t.set_sparse(n_dense, n_onehot, len(vocab))
            p0 = t.get_params()
            for s in range(4):
                Xd, idx, y, w = wd.synth_wide_deep_batch(rows, n_dense, vocab, s)
                t.step_sparse(Xd, idx, y, w)
            p1 = t.get_params()
        assert np.array_equal(_bits(p1)[m], _bits(p0)[m]) and not np.array_equal(p1[~m], p0[~m])


@pytest.mark.gpu
@pytest.mark.parametrize("precision", [0, 1])
def test_deterministic_with_frozen_layers_bit_identical(sb, precision):
    F, hidden, rows, steps = 500, [256, 128, 64], 1024, 8
    X, y, w = so.synth_batch(2 * rows, F, 13, weights="mixed")
    _, params, _, desc = make_pair(sb, F, hidden, [so.ACT_RELU] * 3, optimizer=so.OPT_ADAM, lr=0.01, max_batch=rows,
                                   precision=precision)
    out = []
    for _ in range(2):
        with sb.Trainer(desc, deterministic=True, fixed_layers=[1]) as t:
            t.set_params(so.flatten_params(params))
            t.load_dataset(X, y, w)
            t.run_resident([(k % 2) * rows for k in range(steps)], rows)
            out.append((t.get_params(), t.loss_history(1, steps), t.get_grads()))
    for a, b in zip(*out):
        assert np.array_equal(_bits(a), _bits(b))


@pytest.mark.gpu
def test_replicas_with_frozen_layers(sb, monkeypatch):
    """two in-process fp32 replicas with peer pointers (as test_replicas_bit_identical_across_runs_and_ranks): the ranks
    agree bit for bit and keep the frozen bits; replicas that freeze different layers are refused when the peer table is
    set, not left to hang"""
    monkeypatch.setenv("SB_XCHG_BLOCKS", "8")
    monkeypatch.setenv("SB_XCHG_TIMEOUT_S", "60")
    F, hidden, B, steps = 300, [256, 64], 512, 8
    net = so.NetDesc(F, hidden, [so.ACT_RELU, so.ACT_TANH])
    params = so.flatten_params(so.xavier_init(net, 4))
    desc = sb.make_desc(F, hidden, [so.ACT_RELU, so.ACT_TANH], optimizer=so.OPT_MOMENTUM, learning_rate=0.05, max_batch=B,
                        precision=sb.PREC_FP32)
    shards = [so.synth_batch(2 * B, F, 30 + r, weights="mixed") for r in range(2)]
    m = frozen_mask(F, hidden, [1])
    ts = [sb.Trainer(desc, rank=r, world=2, deterministic=True, fixed_layers=[1]) for r in range(2)]
    try:
        assert ts[0].debug_exchange_layout()["slots"] == 1      # no layer-0 chunk slots
        bases = [t.exchange_base for t in ts]
        for t, (X, y, w) in zip(ts, shards):
            t.set_peer_pointers(bases)
            t.set_params(params)
            t.load_dataset(X, y, w)
        for s0 in range(0, steps, 4):
            for t in ts:
                t.run_resident([((s0 + k) % 2) * B for k in range(4)], B)
        for t in ts:
            t.sync()
        got = [t.get_params() for t in ts]
    finally:
        for t in ts:
            t.close()
    assert np.array_equal(_bits(got[0]), _bits(got[1]))
    assert np.array_equal(_bits(got[0])[m], _bits(params)[m]) and not np.array_equal(got[0][~m], params[~m])
    ts = [sb.Trainer(desc, rank=r, world=2, fixed_layers=[[1], [2]][r]) for r in range(2)]
    try:
        bases = [t.exchange_base for t in ts]
        for t in ts:
            with pytest.raises(sb.ShifuB200Error) as e:
                t.set_peer_pointers(bases)
            assert e.value.code == sb.capi.SB_ERR_INVALID and "fixes other parameters" in str(e.value)
    finally:
        for t in ts:
            t.close()


@pytest.mark.gpu
def test_worker_fine_tunes_from_init_model(sb, tmp_path):
    """a second worker run with FixedLayers [1] from the first run's SavedModel (SB_INIT_MODEL) exports layer 1's tensors
    byte for byte as the first run did, and new values for every other tensor"""
    from oracle import tf_formats as tff
    from test_deterministic import _worker
    rc, lines, env = _worker(tmp_path / "first", {"Optimizer": "adam"})
    assert rc == 0 and lines
    first = env["FINAL_MODEL_PATH"]
    rc, lines, env = _worker(tmp_path / "second", {"Optimizer": "adam", "FixedLayers": ["1"]}, extra_env={"SB_INIT_MODEL": first})
    assert rc == 0 and lines
    a, _ = tff.extract_mlp(first, "shifu_input_0", "shifu_output_0")
    b, _ = tff.extract_mlp(env["FINAL_MODEL_PATH"], "shifu_input_0", "shifu_output_0")
    assert len(a) == len(b) == 3
    assert a[0][0].tobytes() == b[0][0].tobytes() and a[0][1].tobytes() == b[0][1].tobytes()
    for (wa, ba, _), (wb, bb, _) in zip(a[1:], b[1:]):
        assert wa.tobytes() != wb.tobytes() and ba.tobytes() != bb.tobytes()
