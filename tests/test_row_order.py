"""Reading the resident set through a row order (sb_trainer_set_row_order / Trainer.set_row_order / ModelConfig `Shuffle`).

An ordered step gathers its batch's rows of the resident set into the step's batch buffer (gather_batch_kernel) and then
runs the host-batch launches.  The order changes which rows form a batch, never what a step computes from them: with
deterministic training, a trainer reading the set through an order pi must match, bit for bit, a trainer that loaded the
physically permuted set X[pi]."""
import ctypes as C
import gzip
import json
import os
import socket
import threading

import numpy as np
import pytest

from oracle import shifu_oracle as so
from util import make_pair

PRECS = [0, 1, 2, 3]   # SB_PREC_FP32, SB_PREC_BF16, SB_PREC_FP32_TC, SB_PREC_BF16X2
# (F, hidden, rows): ragged widths, a batch that is not a multiple of 64; cfg1's widths at a reduced row count
SHAPES = {"ragged": (300, [200, 77], 333), "cfg1": (1000, [512, 256, 128], 1000)}


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same(a, b):
    return np.array_equal(_bits(a), _bits(b))


def _trainer(sb, F, hidden, rows, precision, optimizer=so.OPT_ADAM, det=True, lr=0.01, seed=3):
    acts = [so.ACT_RELU, so.ACT_TANH, so.ACT_SIGMOID][:len(hidden)]
    net, params, cfg, desc = make_pair(sb, F, hidden, acts, optimizer=optimizer, lr=lr, max_batch=rows, precision=precision,
                                       seed=seed)
    t = sb.Trainer(desc, deterministic=det)
    t.set_params(so.flatten_params(params))
    return t


def _state(t, tmp_path, tag):
    """parameters, gradients and the checkpoint's bytes (theta, optimizer state, global_step)"""
    path = str(tmp_path / ("%s.ckpt" % tag))
    t.save_checkpoint(path)
    return t.get_params(), t.get_grads(), open(path, "rb").read()


def _assert_same_state(a, b, tmp_path):
    pa, ga, ca = _state(a, tmp_path, "a")
    pb, gb, cb = _state(b, tmp_path, "b")
    assert _same(pa, pb) and _same(ga, gb) and ca == cb


def _drive(t, rows, n_logical):
    """every resident entry point, at logical offsets inside [0, n_logical): returns the losses they report"""
    out = [t.step_resident(0, rows), t.step_resident(n_logical - rows, rows)]
    # 6 steps: one graph of four, then two single steps; offsets anywhere in the order
    offs = [(i * 97) % (n_logical - rows + 1) for i in range(6)]
    t.run_resident(offs, rows)
    out += list(t.loss_history(3, 6))
    t.run_resident([5, n_logical - 1, 0, 11, 3], 1)       # one-row batches
    out += list(t.loss_history(9, 5))
    out.append(t.accumulate_resident(rows // 2, rows))
    out.append(t.accumulate_resident(1, rows - 1))
    t.apply_accumulated()
    out.append(t.loss_resident(n_logical - rows, rows))
    out.append(t.step_resident(2, rows))
    return np.asarray(out, np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECS)
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_ordered_equals_physically_permuted(sb, tmp_path, shape, precision):
    F, hidden, rows = SHAPES[shape]
    n = 3 * rows + 17
    X, y, w = so.synth_batch(n, F, 5, weights="mixed")
    pi = np.random.default_rng(1).permutation(n)
    with _trainer(sb, F, hidden, rows, precision) as a, _trainer(sb, F, hidden, rows, precision) as b:
        a.load_dataset(X, y, w)
        a.set_row_order(pi)
        b.load_dataset(X[pi], y[pi], w[pi])
        la, lb = _drive(a, rows, n), _drive(b, rows, n)
        assert np.isfinite(la).all() and _same(la, lb)
        _assert_same_state(a, b, tmp_path)
        assert a.kernels_per_step(rows) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECS)
def test_identity_repeated_and_short_orders(sb, tmp_path, precision):
    """the identity order == no order; an order with repeated rows, shorter than the set == the set it materialises"""
    F, hidden, rows = SHAPES["ragged"]
    n = 4 * rows
    X, y, w = so.synth_batch(n, F, 6, weights="mixed")
    with _trainer(sb, F, hidden, rows, precision) as a, _trainer(sb, F, hidden, rows, precision) as b:
        a.load_dataset(X, y, w)
        a.set_row_order(np.arange(n))
        b.load_dataset(X, y, w)
        assert _same(_drive(a, rows, n), _drive(b, rows, n))
        _assert_same_state(a, b, tmp_path)
    idx = np.random.default_rng(2).integers(0, n, size=2 * rows + 5)
    idx[:40] = idx[40]                                      # repeats inside one batch
    assert len(np.unique(idx)) < len(idx) < n
    with _trainer(sb, F, hidden, rows, precision) as a, _trainer(sb, F, hidden, rows, precision) as b:
        a.load_dataset(X, y, w)
        a.set_row_order(idx)
        b.load_dataset(X[idx], y[idx], w[idx])
        assert _same(_drive(a, rows, len(idx)), _drive(b, rows, len(idx)))
        _assert_same_state(a, b, tmp_path)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", [0, 1])
def test_reorder_between_calls_and_reload_drops_the_order(sb, tmp_path, precision):
    F, hidden, rows = SHAPES["ragged"]
    n = 3 * rows
    X, y, w = so.synth_batch(n, F, 7, weights="mixed")
    rng = np.random.default_rng(3)
    offs = [0, rows, 2 * rows, rows, 0, 2 * rows, 0, rows]   # two graphs of four steps per call
    with _trainer(sb, F, hidden, rows, precision) as a, _trainer(sb, F, hidden, rows, precision) as b:
        a.load_dataset(X, y, w)
        for k in range(4):
            pi = rng.permutation(n)
            a.set_row_order(pi if k != 2 else None)           # and back to the physical order once
            b.load_dataset(*((X[pi], y[pi], w[pi]) if k != 2 else (X, y, w)))
            a.run_resident(offs, rows)
            b.run_resident(offs, rows)
            s = 1 + k * len(offs)
            assert _same(a.loss_history(s, len(offs)), b.loss_history(s, len(offs)))
            assert _same(a.get_params(), b.get_params())
        # a shorter order, then a new set: the order is gone and offsets reach the whole new set again
        a.set_row_order(np.arange(rows))
        a.load_dataset(X, y, w)
        b.load_dataset(X, y, w)
        assert _same(a.step_resident(n - rows, rows), b.step_resident(n - rows, rows))
        _assert_same_state(a, b, tmp_path)


def _planted(n, F, seed):
    """labels from a planted logistic model, so that the loss curve moves (tests/test_benchmarked_paths.py)"""
    rng = np.random.default_rng(seed)
    X = np.clip(rng.standard_normal((n, F), dtype=np.float32), -4, 4)
    beta = rng.standard_normal(F).astype(np.float32) / np.sqrt(F)
    p = 1.0 / (1.0 + np.exp(-(2.5 * (X @ beta) - 1.2)))
    y = (rng.random(n) < p).astype(np.float32)
    w = rng.choice(np.array([0.0, 1.0, 2.5], np.float32), size=n, p=[0.1, 0.7, 0.2]).astype(np.float32)
    return X, y, w


@pytest.mark.gpu
@pytest.mark.parametrize("precision", [0, 1, 2])
def test_loss_curve_over_reshuffled_epochs_against_the_oracle(sb, precision):
    """cfg1's shape and optimizer, three epochs of three batches, a new order per epoch, one run_resident call per epoch.
    Bounds of tests/test_benchmarked_paths.py: fp32 / fp32_tc <= 1e-4 per step from oracle.CleanTrainer, bf16 <= 5e-4
    from oracle.Bf16Trainer"""
    F, hidden, B, lr = 1000, [512, 256, 128], 4096, 0.001
    nb, epochs = 3, 3
    X, y, w = _planted(nb * B, F, 7)
    net = so.NetDesc(F, hidden, [so.ACT_RELU] * 3)
    params = so.xavier_init(net, 4)
    cfg = so.OptConfig(kind=so.OPT_ADAM, lr=lr)
    ref = (so.Bf16Trainer(net, params, cfg, fused_out=True) if precision == 1 else so.CleanTrainer(net, params, cfg))
    desc = sb.make_desc(F, hidden, [sb.ACT_RELU] * 3, loss=sb.LOSS_MSE, optimizer=so.OPT_ADAM, learning_rate=lr, max_batch=B,
                        precision=precision)
    rng = np.random.default_rng(11)
    want = []
    with sb.Trainer(desc) as t:
        t.set_params(so.flatten_params(params))
        t.load_dataset(X, y, w)
        for _ in range(epochs):
            pi = rng.permutation(len(X))
            t.set_row_order(pi)
            t.run_resident([i * B for i in range(nb)], B)
            for i in range(nb):
                r = pi[i * B:(i + 1) * B]
                want.append(float(ref.step([(X[r], y[r].reshape(-1, 1), w[r].reshape(-1, 1))])[0]))
        got = t.loss_history(1, nb * epochs)
    tol = 5e-4 if precision == 1 else 1e-4
    assert abs(want[0] - want[-1]) > 1e-3
    assert np.abs(got - np.asarray(want)).max() <= tol, (got, want)


@pytest.mark.gpu
def test_two_replicas_each_with_its_own_order(sb, monkeypatch):
    """W = 2 in-process replicas on one GPU (peer pointers), each rank permutes its own shard: the replicas hold the same
    bits, and follow oracle.CleanTrainer.step over the permuted shards within 1e-4 (fp32 mode: see
    tests/test_deterministic.py on bf16 replicas sharing one device)"""
    monkeypatch.setenv("SB_XCHG_BLOCKS", "8")
    monkeypatch.setenv("SB_XCHG_TIMEOUT_S", "60")
    W, F, hidden, B = 2, 300, [256, 64], 512
    net = so.NetDesc(F, hidden, [so.ACT_RELU, so.ACT_TANH])
    params = so.xavier_init(net, 4)
    cfg = so.OptConfig(kind=so.OPT_MOMENTUM, lr=0.05)
    desc = sb.make_desc(F, hidden, [so.ACT_RELU, so.ACT_TANH], optimizer=so.OPT_MOMENTUM, learning_rate=0.05, max_batch=B,
                        precision=sb.PREC_FP32)
    shards = [so.synth_batch(2 * B, F, 30 + r, weights="mixed") for r in range(W)]
    ref = so.CleanTrainer(net, params, cfg)
    want = []
    ts = [sb.Trainer(desc, device=0, nccl_id=None, rank=r, world=W, deterministic=True) for r in range(W)]
    try:
        bases = [t.exchange_base for t in ts]
        for t, (X, y, w) in zip(ts, shards):
            t.set_peer_pointers(bases)
            t.set_params(so.flatten_params(params))
            t.load_dataset(X, y, w)
        for epoch in range(2):
            pis = [np.random.default_rng((epoch, r)).permutation(2 * B) for r in range(W)]
            for t, pi in zip(ts, pis):
                t.set_row_order(pi)
            for t in ts:                       # replicas on one device: queue every rank's steps before any rank waits
                t.run_resident([0, B, 0, B], B)
            for k in range(4):
                o = (k % 2) * B
                want.append(ref.step([(X[pi[o:o + B]], y[pi[o:o + B]], w[pi[o:o + B]])
                                      for (X, y, w), pi in zip(shards, pis)]))
            for t in ts:
                t.sync()
        got = [(t.get_params(), t.loss_history(1, 8)) for t in ts]
    finally:
        for t in ts:
            t.close()
    assert _same(got[0][0], got[1][0])
    assert np.abs(got[0][0] - ref.theta).max() <= 1e-4
    for r in range(W):
        assert np.abs(got[r][1] - np.asarray([s[r] for s in want], np.float32)).max() <= 1e-4


@pytest.mark.gpu
def test_argument_checks(sb):
    F, hidden, rows = 64, [32, 16], 128
    X, y, w = so.synth_batch(4 * rows, F, 1, weights="ones")
    lib, err = sb.capi.lib(), sb.ShifuB200Error
    with _trainer(sb, F, hidden, rows, 1) as t:
        with pytest.raises(err) as e:
            t.set_row_order([0, 1])
        assert e.value.code == sb.capi.SB_ERR_STATE
        t.load_dataset(X, y, w)
        for bad in ([0, 4 * rows], [3, -1], []):
            with pytest.raises(err) as e:
                t.set_row_order(bad)
            assert e.value.code == sb.capi.SB_ERR_INVALID
        one = (C.c_int64 * 1)(0)
        for n in (0, -1, 1 << 31):                     # n is checked before the list is read
            assert lib.sb_trainer_set_row_order(t._h, one, n) == sb.capi.SB_ERR_INVALID
        assert lib.sb_trainer_set_row_order(t._h, None, 1) == sb.capi.SB_ERR_INVALID
        # a rejected order leaves the one in effect; offsets are positions in the order
        t.set_row_order(np.arange(2 * rows)[::-1])
        with pytest.raises(err):
            t.set_row_order([5, 4 * rows + 3])
        for call in (lambda: t.step_resident(rows + 1, rows), lambda: t.step_resident_async(2 * rows, 1),
                     lambda: t.run_resident([0, rows + 1], rows), lambda: t.accumulate_resident(rows + 1, rows),
                     lambda: t.loss_resident(rows + 1, rows), lambda: t.step_resident(-1, rows)):
            with pytest.raises(err) as e:
                call()
            assert e.value.code == sb.capi.SB_ERR_INVALID
        assert t.global_step == 0
        assert np.isfinite(t.step_resident(rows, rows))   # the last logical batch of the order still runs
        t.set_row_order(None)
        t.step_resident(3 * rows, rows)                   # back to the whole set


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


def _worker(tmp_path, params, epochs=3, n_rows=1200, F=12, extra_env=None):
    from shifu_tensorflow_b200 import trainer as tr
    X, y, _ = so.synth_batch(n_rows, F, 2, weights="ones")
    tmp_path.mkdir(parents=True, exist_ok=True)
    data = str(tmp_path / "part-00000.gz")
    if not os.path.exists(data):
        _write_gz(data, X, y.ravel())
    conf = {"train": {"params": dict({"NumHiddenLayers": 2, "NumHiddenNodes": [16, 8], "ActivationFunc": ["tanh", "relu"],
                                      "LearningRate": 0.1, "MiniBatchs": 200, "Schedule": "batch", "Optimizer": "sgd"}, **params),
                      "numTrainEpochs": epochs, "validSetRate": 0.2}}
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
           "FINAL_MODEL_PATH": str(tmp_path / "final_model"), "TRAINING_DATA_PATH": data, "SB_SEED": "11",
           "SB_HOST_LOADER": "1"}
    env.update(extra_env or {})
    try:
        rc = tr.main(env=env, rng=_Seq(5))
    finally:
        os.chdir(cwd)
        srv.close()
        th.join(10)
    return rc, lines, env


def _recording(base, log):
    """a Trainer class that logs the calls the worker's training loop makes"""
    class Rec(base):
        def init_xavier(self, seed):
            super().init_xavier(seed)
            log.append(("init", self.get_params()))

        def load_dataset(self, X, y, w=None):
            log.append(("data", np.array(X), np.array(y).reshape(-1), np.array(w).reshape(-1)))
            super().load_dataset(X, y, w)

        def set_row_order(self, rows=None):
            log.append(("order", self.global_step, np.array(rows)))
            super().set_row_order(rows)

        def run_resident(self, row_offsets, rows):
            log.extend(("step", int(o), rows) for o in row_offsets)
            super().run_resident(row_offsets, rows)

        def accumulate_resident(self, row_offset, rows):
            log.append(("acc", int(row_offset), rows))
            return super().accumulate_resident(row_offset, rows)

        def apply_accumulated(self, total_pushes=None):
            log.append(("apply", total_pushes))
            super().apply_accumulated(total_pushes)

        def close(self):
            if self._h:
                log.append(("final", self.get_params()))
            super().close()
    return Rec


@pytest.mark.gpu
@pytest.mark.parametrize("schedule", ["batch", "sync_replicas"])
def test_worker_shuffle_against_the_oracle(sb, tmp_path, monkeypatch, schedule):
    """fp32 worker with Shuffle: every pass reads its rows through pass_order(SB_SEED, rank, global_step); the oracle
    replays the same calls on the permuted rows (plain SGD) and ends within 1e-4 of the worker's parameters"""
    from shifu_tensorflow_b200 import trainer as tr
    log = []
    monkeypatch.setattr(tr.capi, "Trainer", _recording(tr.capi.Trainer, log))
    rc, lines, _ = _worker(tmp_path, {"Shuffle": True, "Precision": "fp32", "Schedule": schedule}, epochs=12)
    assert rc == 0 and lines
    ev = dict((e[0], e) for e in log if e[0] in ("init", "data", "final"))
    _, X, y, w = ev["data"]
    net = so.NetDesc(X.shape[1], [16, 8], [so.ACT_TANH, so.ACT_RELU])
    theta = ev["init"][1].astype(np.float32)
    opt = so.Optimizer(so.OptConfig(kind=so.OPT_SGD, lr=0.1), theta.size)
    pi, acc, orders = None, None, []

    def grad(o, r):
        rr = pi[o:o + r]
        _, g, _ = so.loss_and_grads(net, so.unflatten_params(net, theta), X[rr], y[rr].reshape(-1, 1), w[rr].reshape(-1, 1))
        return so.flatten_params(g)
    for e in log:
        if e[0] == "order":
            orders.append(e[1])
            pi = e[2]
            assert np.array_equal(pi, tr.pass_order(11, 0, e[1], len(X)))
        elif e[0] == "step":
            theta = opt.apply(theta, grad(e[1], e[2]))
        elif e[0] == "acc":
            g = grad(e[1], e[2])
            acc = g if acc is None else acc + g
        elif e[0] == "apply":
            theta = opt.apply(theta, acc / np.float32(e[1]))
            acc = None
    assert len(set(orders)) >= 2
    assert np.abs(ev["final"][1] - theta).max() <= 1e-4


@pytest.mark.gpu
def test_worker_shuffle_deterministic_runs_write_identical_models(sb, tmp_path):
    out = []
    for k in range(2):
        rc, lines, env = _worker(tmp_path / ("run%d" % k), {"Shuffle": "true", "Deterministic": True, "Optimizer": "adam"})
        assert rc == 0 and lines
        var = os.path.join(env["FINAL_MODEL_PATH"], "variables", "variables.data-00000-of-00001")
        out.append((open(var, "rb").read(), [",".join(f for f in ln.split(",") if not f.startswith("time:")) for ln in lines]))
    assert out[0] == out[1]


# ---- CPU: the worker's orders through a stand-in trainer ----
class _FakeTrainer:
    """the device calls of the worker's training loop, with global_step bookkeeping only"""
    calls = []

    def __init__(self, desc, device=0, nccl_id=None, rank=0, world=1):
        self.global_step = 0

    def set_deterministic(self, on=True):
        pass

    def init_xavier(self, seed):
        pass

    def load_checkpoint(self, path):
        self.global_step = int(open(path).read())

    def save_checkpoint(self, path):
        open(path, "w").write(str(self.global_step))

    def load_dataset(self, X, y, w=None):
        _FakeTrainer.n_rows = len(X)

    def set_row_order(self, rows=None):
        _FakeTrainer.calls.append((self.global_step, np.array(rows)))

    def run_resident(self, offs, rows):
        self.global_step += len(offs)

    def accumulate_resident(self, off, rows):
        return 0.0

    def loss_resident(self, off, rows):
        return 0.0

    def apply_accumulated(self, pushes=None):
        self.global_step += 1

    def last_loss(self):
        return 0.0

    def eval_loss(self, X, y, w=None):
        return 0.0

    def close(self):
        pass


def _fake_run(tmp_path, monkeypatch, params, epochs):
    from shifu_tensorflow_b200 import trainer as tr
    monkeypatch.setattr(tr.capi, "Trainer", _FakeTrainer)
    monkeypatch.setattr(tr, "simple_save", lambda trainer, path: None)
    _FakeTrainer.calls = []
    rc, _, env = _worker(tmp_path, params, epochs=epochs)
    assert rc == 0
    return list(_FakeTrainer.calls)


@pytest.mark.parametrize("schedule", ["batch", "sync_replicas"])
def test_worker_orders_per_pass_and_on_resume(tmp_path, monkeypatch, schedule):
    from shifu_tensorflow_b200 import trainer as tr
    p = {"Shuffle": True, "Schedule": schedule}
    full = _fake_run(tmp_path / "full", monkeypatch, p, epochs=12)
    n = _FakeTrainer.n_rows            # about 960 of the 1200 rows (validSetRate 0.2): 4 batches per pass
    assert len(full) >= 3
    for gs, perm in full:
        assert np.array_equal(np.sort(perm), np.arange(n))
        assert np.array_equal(perm, tr.pass_order(11, 0, gs, n))
    if schedule != "batch":
        return      # (a sync-replicas pass may end without an update: its passes need not start where a resumed run does)
    # stopped after the second pass, resumed from its checkpoint: the resumed run draws the uninterrupted run's orders
    first = _fake_run(tmp_path / "resume", monkeypatch, p, epochs=full[2][0])
    rest = _fake_run(tmp_path / "resume", monkeypatch, p, epochs=12)
    assert [g for g, _ in first + rest] == [g for g, _ in full]
    assert all(np.array_equal(a, b) for (_, a), (_, b) in zip(first + rest, full))


def test_worker_without_shuffle_sets_no_order(tmp_path, monkeypatch):
    for k, params in enumerate(({}, {"Shuffle": False}, {"Shuffle": "false"})):
        assert _fake_run(tmp_path / ("off%d" % k), monkeypatch, params, epochs=8) == []
    assert _fake_run(tmp_path / "on", monkeypatch, {"Shuffle": True}, epochs=8)


def test_pass_order_is_keyed_by_seed_rank_and_step():
    from shifu_tensorflow_b200 import trainer as tr
    a = tr.pass_order(11, 0, 0, 100)
    assert np.array_equal(a, tr.pass_order(11, 0, 0, 100))
    for other in (tr.pass_order(12, 0, 0, 100), tr.pass_order(11, 1, 0, 100), tr.pass_order(11, 0, 4, 100)):
        assert not np.array_equal(a, other)


def test_shuffle_key_parsing():
    from shifu_tensorflow_b200 import trainer as tr
    assert tr.shuffle_requested({}) is False
    assert tr.shuffle_requested({"Shuffle": True}) is True
    assert tr.shuffle_requested({"Shuffle": "TRUE"}) is True
    assert tr.shuffle_requested({"Shuffle": "false"}) is False
    assert tr.shuffle_requested({"Shuffle": False}) is False
    with pytest.raises(ValueError, match="Shuffle"):
        tr.shuffle_requested({"Shuffle": "yes"})
