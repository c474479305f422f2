"""Deterministic training (sb_trainer_set_deterministic / Trainer(deterministic=True) / ModelConfig `Deterministic`).

With the flag on, every reduction over the CTAs of a training launch is added in a fixed order (slots + the last CTA's
ordered sum; dW split-K capped at two addends), so two runs from the same seed and data give the same bits: parameters,
optimizer state, gradients, every loss and the exported files.  The default path is untouched; the deterministic one
must stay within the tolerances the default path is held to."""
import gzip
import json
import os
import socket
import threading

import numpy as np
import pytest

from oracle import shifu_oracle as so
from util import make_pair

FULL = {
    "cfg1": dict(F=1000, hidden=[512, 256, 128], rows=4096),   # dW split-K 4 by default -> capped at 2
    "cfg2": dict(F=2000, hidden=[1024, 512, 256], rows=8192),  # dW_0 on 128 x 256 tiles, split 2; 64 row tiles per column
}


def _trainer(sb, F, hidden, rows, precision, optimizer, det, lr=0.01, acts=None, seed=3, oracle=False):
    acts = acts or [so.ACT_RELU] * len(hidden)
    net, params, cfg, desc = make_pair(sb, F, hidden, acts, optimizer=optimizer, lr=lr, max_batch=rows, precision=precision, seed=seed)
    t = sb.Trainer(desc, deterministic=det)
    t.set_params(so.flatten_params(params))
    return (t, net, params, cfg) if oracle else t


PRECS = [0, 1, 2, 3]   # SB_PREC_FP32, SB_PREC_BF16, SB_PREC_FP32_TC, SB_PREC_BF16X2
_ORACLE = {}


def _oracle_losses(net, params, cfg, data, rows, steps, bf16):
    """per-step losses of oracle.CleanTrainer (fp32) or oracle.Bf16Trainer (the kernels' bf16 roundings) on the batches
    _run feeds, cached per configuration"""
    key = (tuple(net.hidden), net.n_features, cfg.kind, cfg.lr, bf16, rows, steps, id(data))
    if key not in _ORACLE:
        X, y, w, offs = data
        ref = (so.Bf16Trainer(net, params, cfg, fused_out=net.hidden[-1] <= 256) if bf16 else so.CleanTrainer(net, params, cfg))
        out = []
        for i in range(steps):
            o = offs[i % len(offs)]
            out.append(float(ref.step([(X[o:o + rows], y[o:o + rows], w[o:o + rows])])[0]))
        _ORACLE[key] = np.asarray(out)
    return _ORACLE[key]


def _resident_set(F, rows, n_batches, seed):
    X, y, w = so.synth_batch(rows * n_batches, F, seed, weights="mixed")
    return X, y, w, [i * rows for i in range(n_batches)]


def _run(t, data, rows, steps):
    X, y, w, offs = data
    t.load_dataset(X, y, w)
    t.run_resident([offs[i % len(offs)] for i in range(steps)], rows)
    t.sync()
    return t.get_params(), t.loss_history(1, steps), t.get_grads()


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same(a, b):
    return np.array_equal(_bits(a), _bits(b))


@pytest.mark.gpu
@pytest.mark.parametrize("optimizer", [so.OPT_MOMENTUM, so.OPT_ADAM])
@pytest.mark.parametrize("precision", PRECS)
@pytest.mark.parametrize("name", ["cfg1", "cfg2"])
def test_full_size_run_to_run_bit_identical(sb, name, precision, optimizer):
    """two fresh deterministic trainers, 12 steps through one run_resident call: same bits, even though the second run
    shares the GPU with another trainer stepping on its own stream; every step's loss within the oracle bounds of
    tests/test_benchmarked_paths.py (fp32-class modes vs oracle.CleanTrainer, bf16 vs oracle.Bf16Trainer)"""
    c = FULL[name]
    steps = 12
    data = _DATA.setdefault(name, _resident_set(c["F"], c["rows"], 3, 21))
    ta, net, params, cfg = _trainer(sb, c["F"], c["hidden"], c["rows"], precision, optimizer, True, oracle=True)
    with ta:
        pa, la, ga = _run(ta, data, c["rows"], steps)
    # the second run with a default trainer stepping beside it, so CTA timing differs between the runs
    other = _trainer(sb, c["F"], c["hidden"], c["rows"], precision, optimizer, False)
    Xo, yo, wo = so.synth_batch(c["rows"], c["F"], 5, weights="mixed")
    stop = threading.Event()

    def noise():
        while not stop.is_set():
            other.step(Xo, yo, wo)

    tb = _trainer(sb, c["F"], c["hidden"], c["rows"], precision, optimizer, True)
    th = threading.Thread(target=noise)
    th.start()
    try:
        with tb:
            pb, lb, gb = _run(tb, data, c["rows"], steps)
    finally:
        stop.set()
        th.join()
        other.close()
    assert np.isfinite(la).all() and np.abs(pa).max() > 0
    assert _same(pa, pb) and _same(la, lb) and _same(ga, gb)
    bf16 = precision == 1
    want = _oracle_losses(net, params, cfg, data, c["rows"], steps, bf16)
    # fp32 / fp32_tc: 1e-4 (test_benchmarked_paths); bf16 vs its emulating oracle: 5e-4 (that file's cfg1 bound);
    # bf16x2 (about 2^-17 per product) against the fp32 oracle: 5e-4
    tol = 1e-4 if precision in (0, 2) else 5e-4
    assert np.abs(la.astype(np.float64) - want).max() <= tol, (la, want)


_DATA = {}


# (F, hidden, rows, precision): ragged N, output layer not fused (h_L > 256: out_layer_rows_kernel; h_L > 1024:
# out_layer_kernel), several row tiles per column, fp32 mode (gemm_f32, out_layer_kernel<float>)
SHAPES = [
    (300, [200, 77], 1000, 1),
    (256, [384, 300], 777, 1),
    (128, [1100], 640, 1),
    (300, [200, 77], 1000, 0),
    (200, [130, 300], 700, 0),
    (300, [200, 77], 1000, 2),     # split-precision dA (gemm_tc_kernel, 64- and 128-wide tiles), fused output layer
    (256, [384, 300], 777, 3),     # split-precision, output layer not fused
]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "%dx%s@%d-p%d" % (s[0], "-".join(map(str, s[1])), s[2], s[3]))
def test_every_reduction_kind_bit_identical_and_paths_agree(sb, shape):
    """run_resident == the same steps through step_resident, bit for bit; two trainers agree bit for bit; eval_loss and
    loss_resident repeat their bits; the deterministic gradient is within the default path's tolerance"""
    F, hidden, rows, prec = shape
    steps = 8
    data = _resident_set(F, rows, 2, 9)
    acts = [so.ACT_RELU, so.ACT_TANH, so.ACT_SIGMOID][:len(hidden)]
    with _trainer(sb, F, hidden, rows, prec, so.OPT_ADAM, True, acts=acts) as ta, \
            _trainer(sb, F, hidden, rows, prec, so.OPT_ADAM, True, acts=acts) as tb:
        pa, la, ga = _run(ta, data, rows, steps)
        X, y, w, offs = data
        tb.load_dataset(X, y, w)
        lb = [tb.step_resident(offs[i % len(offs)], rows) for i in range(steps)]
        assert _same(pa, tb.get_params()) and _same(ga, tb.get_grads())
        assert _same(la, tb.loss_history(1, steps)) and _same(la, np.asarray(lb, np.float32))
        # the set is two max_batch chunks: eval_loss runs its forward launches twice per call
        e1, e2 = ta.eval_loss(X, y, w), ta.eval_loss(X, y, w)
        assert len(X) > rows and e1 == e2 == tb.eval_loss(X, y, w)
        r1, r2 = ta.loss_resident(0, rows), tb.loss_resident(0, rows)
        assert r1 == r2
    # one gradient against the oracle, with the tolerances the tests state for the default path: fp32-class modes 1e-4
    # abs (bf16x2: 1e-3 of max|g|, two parts per value), bf16 vs the bf16-emulating oracle 2e-5 on the loss and
    # 2e-3 max|g| on the gradient
    t1, net, params, cfg = _trainer(sb, F, hidden, rows, prec, so.OPT_SGD, True, acts=acts, oracle=True)
    with t1:
        Xb, yb, wb = so.synth_batch(rows, F, 4, weights="mixed")
        L1 = t1.accumulate(Xb, yb, wb)
        g1 = t1.get_grads()
    if prec == 1:
        L, g, _ = so.loss_and_grads_bf16(net, params, Xb, yb, wb, fused_out=hidden[-1] <= 256)
        g = so.flatten_params(g)
        assert abs(L1 - L) <= 2e-5 and np.abs(g1 - g).max() <= 2e-3 * np.abs(g).max()
    else:
        ref = so.CleanTrainer(net, params, cfg)
        L = float(ref.step([(Xb, yb, wb)])[0])
        g = ref.last_grads
        gt = 1e-4 if prec != 3 else max(1e-4, 1e-3 * float(np.abs(g).max()))
        assert abs(L1 - L) <= 1e-4 and np.abs(g1 - g).max() <= gt


@pytest.mark.gpu
def test_epoch_sync_schedule_bit_identical(sb):
    """accumulate_resident R times, a stale loss_resident, apply_accumulated_mean: identical over two runs"""
    F, hidden, rows = 500, [256, 128], 1024
    data = _resident_set(F, rows, 3, 13)
    out = []
    for _ in range(2):
        with _trainer(sb, F, hidden, rows, 1, so.OPT_ADADELTA, True, lr=1.0) as t:
            X, y, w, offs = data
            t.load_dataset(X, y, w)
            losses = []
            for epoch in range(3):
                for o in offs:
                    losses.append(t.accumulate_resident(o, rows))
                losses.append(t.loss_resident(offs[0], rows))
                t.apply_accumulated(total_pushes=len(offs))
            out.append((t.get_params(), np.asarray(losses, np.float32)))
    assert _same(out[0][0], out[1][0]) and _same(out[0][1], out[1][1])


@pytest.mark.gpu
@pytest.mark.parametrize("W", [2, 4])
def test_replicas_bit_identical_across_runs_and_ranks(sb, W, monkeypatch):
    """W in-process replicas on one GPU with peer pointers (the peer-memory exchange adds ranks in order).  fp32 mode: four
    bf16 replicas on one device do not make progress together (tests/test_data_parallel_one_gpu.py)"""
    monkeypatch.setenv("SB_XCHG_BLOCKS", "8")
    monkeypatch.setenv("SB_XCHG_TIMEOUT_S", "60")
    F, hidden, B, steps = 300, [256, 64], 512, 8
    net = so.NetDesc(F, hidden, [so.ACT_RELU, so.ACT_TANH])
    params = so.flatten_params(so.xavier_init(net, 4))
    desc = sb.make_desc(F, hidden, [so.ACT_RELU, so.ACT_TANH], optimizer=so.OPT_MOMENTUM, learning_rate=0.05, max_batch=B,
                        precision=sb.PREC_FP32)
    shards = [so.synth_batch(2 * B, F, 30 + r, weights="mixed") for r in range(W)]
    runs = []
    for _ in range(2):
        ts = [sb.Trainer(desc, device=0, nccl_id=None, rank=r, world=W, deterministic=True) for r in range(W)]
        try:
            bases = [t.exchange_base for t in ts]
            for t, (X, y, w) in zip(ts, shards):
                t.set_peer_pointers(bases)
                t.set_params(params)
                t.load_dataset(X, y, w)
            # replicas on one device: queue a few steps on every rank before any rank waits
            for s0 in range(0, steps, 4):
                for t in ts:
                    t.run_resident([((s0 + k) % 2) * B for k in range(4)], B)
            for t in ts:
                t.sync()
            runs.append([(t.get_params(), t.loss_history(1, steps)) for t in ts])
        finally:
            for t in ts:
                t.close()
    for r in range(W):
        assert _same(runs[0][r][0], runs[1][r][0]) and _same(runs[0][r][1], runs[1][r][1])
        assert _same(runs[0][r][0], runs[0][0][0])


@pytest.mark.gpu
def test_rejections(sb):
    F, hidden, rows = 64, [32, 16], 128
    X, y, w = so.synth_batch(rows, F, 1, weights="ones")
    with _trainer(sb, F, hidden, rows, 1, so.OPT_SGD, True) as t:
        with pytest.raises(sb.ShifuB200Error) as e:
            t.set_sparse(32, 32, 4)
        assert e.value.code == sb.capi.SB_ERR_STATE and "deterministic" in str(e.value)
    with _trainer(sb, F, hidden, rows, 1, so.OPT_SGD, False) as t:
        t.step(X, y, w)
        with pytest.raises(sb.ShifuB200Error) as e:
            t.set_deterministic(True)
        assert e.value.code == sb.capi.SB_ERR_STATE
    # world 2, no peer table: refused at the first step (no NCCL all-reduce, no hang)
    _, _, _, desc = make_pair(sb, F, hidden, [so.ACT_RELU] * 2, max_batch=rows, precision=sb.PREC_BF16)
    with sb.Trainer(desc, rank=0, world=2, deterministic=True) as t:
        with pytest.raises(sb.ShifuB200Error) as e:
            t.step(X, y, w)
        assert e.value.code == sb.capi.SB_ERR_STATE and "peer" in str(e.value)


# ---- worker (trainer.main) ----
class _Seq:
    def __init__(self, seed):
        self.r = np.random.RandomState(seed)

    def random(self):
        return float(self.r.rand())


def _write_gz(path, X, y):
    with gzip.open(path, "wb") as f:
        for i in range(len(X)):
            f.write(("|".join([str(int(y[i]))] + [repr(float(v)) for v in X[i]]) + "\n").encode())


def _worker(tmp_path, params, n_rows=1200, F=12, extra_env=None):
    from shifu_tensorflow_b200 import trainer as tr
    X, y, _ = so.synth_batch(n_rows, F, 2, weights="ones")
    tmp_path.mkdir(parents=True, exist_ok=True)
    data = str(tmp_path / "part-00000.gz")
    _write_gz(data, X, y.ravel())
    conf = {"train": {"params": dict({"NumHiddenLayers": 2, "NumHiddenNodes": [16, 8], "ActivationFunc": ["tanh", "relu"],
                                      "LearningRate": 0.1, "MiniBatchs": 200, "Schedule": "batch"}, **params),
                      "numTrainEpochs": 3, "validSetRate": 0.2}}
    cwd = os.getcwd()
    os.chdir(tmp_path)
    json.dump(conf, open("ModelConfig.json", "w"))
    srv = socket.socket(); srv.bind(("127.0.0.1", 0)); srv.listen(1)
    lines = []

    def serve():
        try:
            c, _ = srv.accept()
        except OSError:
            return
        buf = b""
        while True:
            d = c.recv(4096)
            if not d:
                break
            buf += d
        lines.extend(buf.decode().splitlines())

    th = threading.Thread(target=serve); th.start()
    env = {"CLUSTER_SPEC": json.dumps({"ps": ["127.0.0.1:1"], "worker": ["127.0.0.1:2"]}), "WORKER_CNT": "1", "JOB_NAME": "worker",
           "TASK_ID": "0", "SOCKET_SERVER_PORT": str(srv.getsockname()[1]), "SB_REQUIRE_SOCKET": "0",
           "TOTAL_TRAINING_DATA_NUMBER": str(n_rows), "SELECTED_COLUMN_NUMS": " ".join(str(i) for i in range(1, F + 1)),
           "WEIGHT_COLUMN_NUM": "-1", "TARGET_COLUMN_NUM": "0", "TMP_MODEL_PATH": str(tmp_path / "tmp_model"),
           "FINAL_MODEL_PATH": str(tmp_path / "final_model"), "TRAINING_DATA_PATH": data, "SB_SEED": "11"}
    env.update(extra_env or {})
    try:
        rc = tr.main(env=env, rng=_Seq(5))
    finally:
        os.chdir(cwd)
        srv.close()
        th.join(10)
    return rc, lines, env


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_worker_deterministic_runs_write_identical_models(sb, tmp_path, precision):
    out = []
    for k in range(2):
        rc, lines, env = _worker(tmp_path / ("run%d" % k), {"Deterministic": True, "Precision": precision, "Optimizer": "adam"})
        assert rc == 0 and lines
        var = os.path.join(env["FINAL_MODEL_PATH"], "variables", "variables.data-00000-of-00001")
        # the socket lines without their wall-clock field: epoch, training and validation loss
        out.append((open(var, "rb").read(), [",".join(f for f in ln.split(",") if not f.startswith("time:")) for ln in lines]))
    assert out[0][0] == out[1][0]
    assert out[0][1] == out[1][1]


def test_worker_deterministic_with_wide_deep_columns_raises_before_any_device_call(tmp_path, monkeypatch):
    from shifu_tensorflow_b200 import _capi, trainer as tr

    def no_device(*a, **k):
        raise AssertionError("device call before the configuration check")
    monkeypatch.setattr(_capi, "lib", no_device)
    monkeypatch.setattr(tr, "load_data_gpu", no_device)
    monkeypatch.setattr(tr, "load_data", no_device)
    conf = {"train": {"params": {"NumHiddenLayers": 1, "NumHiddenNodes": [8], "ActivationFunc": ["relu"], "LearningRate": 0.1,
                                 "Deterministic": "true"}, "numTrainEpochs": 1, "validSetRate": 0.2}}
    cwd = os.getcwd()
    os.chdir(tmp_path)
    json.dump(conf, open("ModelConfig.json", "w"))
    env = {"CLUSTER_SPEC": json.dumps({"ps": ["127.0.0.1:1"], "worker": ["127.0.0.1:2"]}), "WORKER_CNT": "1", "JOB_NAME": "worker",
           "TASK_ID": "0", "SOCKET_SERVER_PORT": "1", "SB_REQUIRE_SOCKET": "0", "TOTAL_TRAINING_DATA_NUMBER": "10",
           "SELECTED_COLUMN_NUMS": "", "SELECTED_NUMERIC_COLUMN_NUMS": "1 2", "SELECTED_CATEGORY_COLUMN_NUMS": "3",
           "WEIGHT_COLUMN_NUM": "-1", "TARGET_COLUMN_NUM": "0", "TMP_MODEL_PATH": str(tmp_path / "t"),
           "FINAL_MODEL_PATH": str(tmp_path / "f"), "TRAINING_DATA_PATH": str(tmp_path / "none.gz")}
    try:
        with pytest.raises(ValueError, match="Deterministic"):
            tr.main(env=env, rng=_Seq(1))
    finally:
        os.chdir(cwd)


def test_deterministic_key_parsing():
    from shifu_tensorflow_b200 import trainer as tr
    assert tr.deterministic_requested({}) is False
    assert tr.deterministic_requested({"Deterministic": True}) is True
    assert tr.deterministic_requested({"Deterministic": "TRUE"}) is True
    assert tr.deterministic_requested({"Deterministic": "false"}) is False
    with pytest.raises(ValueError):
        tr.deterministic_requested({"Deterministic": "yes"})
