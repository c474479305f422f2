"""Wide+deep training and validation through the entry points the worker calls (trainer.py: step_sparse for every
mini-batch, eval_loss_sparse after every pass), against float64 in every precision mode:

  validation     Trainer.predict_sparse and Trainer.eval_loss_sparse run the forward in max_batch pieces
                 (forward_chunks): at 1, B - 1, B, B + 1 and 2.5 B + a ragged tail rows, every prediction within its
                 row bound (wide_deep_ref.py) and the loss within the sum of the pieces' output-unit loss bounds
                 (score_ref.validation_loss); a set whose weights are all 0 has loss 0; the predictions of a call over
                 many pieces are, bit for bit, those of one call per piece
  steps          12 momentum steps at B and B - 1 rows (two captured step graphs, as np.array_split's batches give the
                 worker) with a validation pass after every fourth: FP32 / FP32_TC against the float64 sparse oracle
                 (oracle/wide_deep.py) within 1e-4; BF16X2 against it and BF16 against Bf16Trainer on the one-hot
                 matrix within 1e-3 (loss) / 5e-3 (parameters); every validation call within its bound at the trainer's
                 parameters of that moment
  peer exchange  W = 2 replicas on one GPU (SB_XCHG_BLOCKS=8, set_peer_pointers), each driven from its own thread
                 (step_sparse waits until its exchange is done): layer 0's gradient in two slot chunks, in one, one
                 hidden layer (the single exchange launch) and FP32 mode, against CleanTrainer / Bf16Trainer.step
                 ([shard_0, shard_1]) on the one-hot matrices; the replicas' parameters, gradients and predictions
                 bit-identical.  With two GPUs, the same with one rank per device (dW_1 in front of dW_0)
  worker         a wide+deep worker reporting to a local socket: every epoch line's training_loss and valid_loss
                 within 1e-4 of the dense oracle's replay
Without a GPU: the sparse reference equals score_ref on the materialised matrix [Xd | one-hot], and its bounds reject
an index off by one, a dropped categorical column, a missing index read as 0 and a loss divided by the row count."""
import gzip
import json
import os
import socket
import sys
import threading

import numpy as np
import pytest

from oracle import shifu_oracle as so
from oracle import wide_deep as wd
from out_layer_ref import ACTS
from score_ref import BF16, BF16X2, FP32, FP32_TC, hidden_forward, scores, unflatten, validation_loss
from wide_deep_ref import hidden_forward_sparse

PRECS = {"fp32": FP32, "bf16": BF16, "fp32_tc": FP32_TC, "bf16x2": BF16X2}
SMALL = (21, [5, 9, 3, 17])
SHAPES = {   # n_dense, vocab, hidden, acts, max_batch
    "small": SMALL + ([40, 24], ["tanh", "relu"], 130),
    "one_layer": SMALL + ([48], ["relu"], 130),
    "cfg4": (500, [100] * 50, [1024, 512], ["relu", "relu"], 2048),      # BASELINE config 4
}

_worst = {}
_notes = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(_worst):
        print("worst error / bound, %s: %.3g" % (k, _worst[k]))
    for k in sorted(_notes):
        print("%s: %s" % (k, _notes[k]))


def _name(prec):
    return [k for k, v in PRECS.items() if v == prec][0]


def _codes(acts):
    return [ACTS[a] for a in acts]


def _counts(B):
    return [1, B - 1, B, B + 1, 5 * B // 2 + 7]


def _rows(n, n_dense, vocab, seed, hot=True):
    """n rows (dense block, indices, labels, weights in {0, 1, 2.5}): one hot embedding row chosen by every row in
    column 0, and row 3 with every category missing"""
    Xd, idx, y, w = wd.synth_wide_deep_batch(n, n_dense, vocab, seed, missing=0.1)
    if hot:
        idx[:, 0] = 1
    idx[min(3, n - 1)] = -1
    return Xd, idx.astype(np.int32), y.ravel(), w.ravel()


def _params(F, hidden, seed):
    """a flat parameter vector: Xavier weights, biases N(0, 0.1^2)"""
    net = so.NetDesc(F, hidden, [so.ACT_RELU] * len(hidden))
    P = so.xavier_init(net, seed)
    rng = np.random.RandomState(seed + 1)
    for k in range(1, len(P), 2):
        P[k] = (rng.standard_normal(P[k].shape) * 0.1).astype(np.float32)
    return so.flatten_params(P)


def _held(got, want, what, key):
    """values got [M] against (value, bound) [M]: every one within its bound"""
    yh, e = want
    err = np.abs(np.asarray(got, np.float64) - yh)
    r = float(np.max(err / e))
    _worst[key] = max(_worst.get(key, 0.0), r)
    bad = np.flatnonzero(err > e)
    assert bad.size == 0, "%s: %d rows off, first row %d: %r vs %r (bound %.3g), worst %.3g x its bound" % (
        what, bad.size, bad[0], got[bad[0]], yh[bad[0]], e[bad[0]], r)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _eval_route_depth(prec, H_L):
    from test_out_layer import _depth, expected_route
    route = expected_route(prec, H_L, False, "eval")
    return lambda m: _depth(route, m, 0)


def _check_validation(t, prec, Xd, idx, y, w, layers, acts, B, what):
    """predict_sparse and eval_loss_sparse of trainer t on the rows against the reference at parameters `layers`"""
    a, e_a = hidden_forward_sparse(Xd, idx, layers, _codes(acts), prec)
    pred = t.predict_sparse(Xd, idx)
    _held(pred, scores(a, e_a, layers, _codes(acts)), "%s predict_sparse" % what, "predict_sparse " + _name(prec))
    loss = t.eval_loss_sparse(Xd, idx, y, w)
    want, tol = validation_loss(a, e_a, layers[-1][0], layers[-1][1], y, w, ACTS[acts[-1]], B,
                                _eval_route_depth(prec, layers[-2][0].shape[1]))
    _held(np.array([loss]), (np.array([want]), np.array([tol])), "%s eval_loss_sparse" % what, "eval_loss_sparse " + _name(prec))
    return pred


# ---------------------------------------------------------------------------------------------- validation entry points
@pytest.mark.gpu
@pytest.mark.parametrize("prec", sorted(PRECS))
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_validation_entry_points(sb, shape, prec):
    p = PRECS[prec]
    n_dense, vocab, hidden, acts, B = SHAPES[shape]
    n_onehot = int(sum(vocab))
    F = n_dense + n_onehot
    flat = _params(F, hidden, 5)
    layers = unflatten(flat, F, hidden)
    counts = _counts(B)
    N = counts[-1]
    Xd, idx, y, w = _rows(N, n_dense, vocab, 6)
    a, e_a = hidden_forward_sparse(Xd, idx, layers, _codes(acts), p)
    yh, e = scores(a, e_a, layers, _codes(acts))
    depth = _eval_route_depth(p, hidden[-1])
    with sb.Trainer(sb.make_desc(F, hidden, _codes(acts), max_batch=B, precision=p)) as t:
        t.set_params(flat)
        t.set_sparse(n_dense, n_onehot, len(vocab))
        for n in counts:
            what = "%s %s %d rows" % (shape, prec, n)
            pred = t.predict_sparse(Xd[:n], idx[:n])
            _held(pred, (yh[:n], e[:n]), what + " predict_sparse", "predict_sparse " + prec)
            loss = t.eval_loss_sparse(Xd[:n], idx[:n], y[:n], w[:n])
            want, tol = validation_loss(a[:n], e_a[:n], layers[-1][0], layers[-1][1], y[:n], w[:n], ACTS[acts[-1]], B, depth)
            if np.count_nonzero(w[:n]) == 0:
                assert loss == 0.0, what
            else:
                _held(np.array([loss]), (np.array([want]), np.array([tol])), what + " eval_loss_sparse", "eval_loss_sparse " + prec)
        # weights all 0: no row counts, the loss is 0 (not 0 / 0)
        assert t.eval_loss_sparse(Xd, idx, y, np.zeros_like(w)) == 0.0
        # rows never interact: one call over many pieces gives the bits of one call per piece
        pieces = np.concatenate([t.predict_sparse(Xd[r0:r0 + B], idx[r0:r0 + B]) for r0 in range(0, N, B)])
        np.testing.assert_array_equal(_bits(pieces), _bits(pred))
    if p != BF16:
        _notes["%s %s max |predict_sparse - float64|" % (shape, prec)] = "%.3g" % float(np.abs(pred - yh).max())


# ---------------------------------------------------------------------------------------------- steps in the worker's order
@pytest.mark.gpu
@pytest.mark.parametrize("prec", sorted(PRECS))
def test_steps_with_validation_in_the_workers_order(sb, prec):
    p = PRECS[prec]
    n_dense, vocab, hidden, acts, B = SHAPES["small"]
    n_onehot = int(sum(vocab))
    F = n_dense + n_onehot
    net = so.NetDesc(F, hidden, _codes(acts))
    params = so.xavier_init(net, 3)
    lr, n_steps = 0.05, 12
    sizes = [B - (s % 2) for s in range(n_steps)]
    Xd, idx, y, w = _rows(sum(sizes), n_dense, vocab, 11, hot=False)
    Xfull = np.concatenate([Xd, wd.onehot_matrix(idx, n_onehot)], axis=1)
    V = _rows(5 * B // 2 + 7, n_dense, vocab, 12)
    cfg = so.OptConfig(kind=so.OPT_MOMENTUM, lr=lr)
    theta = so.flatten_params(params)
    opt = so.Optimizer(cfg, theta.size)
    # the sparse step fuses the output layer into the last hidden GEMM only when that GEMM is not the first layer's
    bf = so.Bf16Trainer(net, params, cfg, fused_out=hidden[-1] <= 256 and len(hidden) > 1)
    got, want = [], []
    desc = sb.make_desc(F, hidden, _codes(acts), optimizer=so.OPT_MOMENTUM, learning_rate=lr, max_batch=B, precision=p)
    with sb.Trainer(desc) as t:
        t.set_params(theta)
        t.set_sparse(n_dense, n_onehot, len(vocab))
        o = 0
        for s, r in enumerate(sizes):
            sl = slice(o, o + r)
            o += r
            got.append(t.step_sparse(Xd[sl], idx[sl], y[sl], w[sl]))
            if p == BF16:
                want.append(bf.step([(Xfull[sl], y[sl, None], w[sl, None])])[0])
            else:
                L, g, _ = wd.loss_and_grads_sparse(net, so.unflatten_params(net, theta), Xd[sl], idx[sl], y[sl, None], w[sl, None])
                want.append(L)
                theta = opt.apply(theta, so.flatten_params(g))
            if s % 4 == 3:
                # the validation pass at the trainer's own parameters, between two captured steps
                layers = unflatten(t.get_params(), F, hidden)
                _check_validation(t, p, *V, layers, acts, B, "%s after step %d" % (prec, s + 1))
        theta_got = t.get_params()
    if p == BF16:
        theta = bf.theta
    dl, dp = float(np.abs(np.array(got) - np.array(want)).max()), float(np.abs(theta_got - theta).max())
    _notes["steps %s max |loss - oracle|, |theta - oracle|" % prec] = "%.3g, %.3g" % (dl, dp)
    tol_l, tol_p = (1e-4, 1e-4) if p in (FP32, FP32_TC) else (1e-3, 5e-3)
    assert dl <= tol_l, (got, want)
    assert dp <= tol_p


# ---------------------------------------------------------------------------------------------- replicas, peer exchange
REPLICAS = {   # precision, n_dense, vocab, hidden, acts
    "fp32_tc_two_chunks": (FP32_TC, 64, [100] * 5, [128, 64], ["relu", "tanh"]),    # layers[0].in = 564, out % 8 == 0
    "bf16_two_chunks": (BF16, 64, [100] * 5, [128, 64], ["relu", "tanh"]),
    "fp32_tc_one_chunk": (FP32_TC,) + SMALL + ([40, 24], ["tanh", "relu"]),         # layers[0].in = 55
    "bf16_one_chunk": (BF16,) + SMALL + ([40, 24], ["tanh", "relu"]),
    "fp32_tc_one_layer": (FP32_TC,) + SMALL + ([48], ["relu"]),                     # one exchange launch
    "bf16_one_layer": (BF16,) + SMALL + ([48], ["relu"]),
    "fp32": (FP32,) + SMALL + ([40, 24], ["tanh", "relu"]),
}


def _in_threads(n, fn):
    """fn(r) for r < n, each in its own thread; their results, or the first error"""
    out, errs = [None] * n, []

    def run(r):
        try:
            out[r] = fn(r)
        except Exception as e:      # noqa: BLE001
            errs.append(e)

    th = [threading.Thread(target=run, args=(r,)) for r in range(n)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    if errs:
        raise errs[0]
    return out


W_REPLICAS, B_REPLICAS, REPLICA_STEPS, REPLICA_LR = 2, 130, 6, 0.05


def _replica_case(sb, case):
    """-> (desc, flat parameters, the step sizes, every rank's rows) of a replica case"""
    p, n_dense, vocab, hidden, acts = REPLICAS[case]
    F = n_dense + int(sum(vocab))
    params = so.xavier_init(so.NetDesc(F, hidden, _codes(acts)), 4)
    sizes = [B_REPLICAS - (s % 2) for s in range(REPLICA_STEPS)]
    shards = [_rows(sum(sizes), n_dense, vocab, 20 + 7 * r, hot=False) for r in range(W_REPLICAS)]
    desc = sb.make_desc(F, hidden, _codes(acts), optimizer=so.OPT_MOMENTUM, learning_rate=REPLICA_LR, max_batch=B_REPLICAS,
                        precision=p)
    return desc, so.flatten_params(params), sizes, shards


def _set_sparse(t, case):
    _, n_dense, vocab, _, _ = REPLICAS[case]
    t.set_sparse(n_dense, int(sum(vocab)), len(vocab))


def _replica_steps(t, sizes, rows):
    """rank t's sparse steps on its rows -> its losses"""
    Xd, idx, y, w = rows
    losses, o = [], 0
    for n in sizes:
        losses.append(t.step_sparse(Xd[o:o + n], idx[o:o + n], y[o:o + n], w[o:o + n]))
        o += n
    return losses


def _check_replicas(case, flat, sizes, shards, got, thetas, grads, preds, where):
    """got [step, rank] losses, every rank's parameters, last gradient and predictions of rank 0's first rows: the replicas
    bit-identical, and the run against CleanTrainer.step([shard_0, shard_1]) (BF16: Bf16Trainer) on the one-hot matrices"""
    p, n_dense, vocab, hidden, acts = REPLICAS[case]
    for r in range(1, len(thetas)):
        np.testing.assert_array_equal(thetas[0], thetas[r])
        np.testing.assert_array_equal(grads[0], grads[r])
        np.testing.assert_array_equal(preds[0], preds[r])
    n_onehot = int(sum(vocab))
    net = so.NetDesc(n_dense + n_onehot, hidden, _codes(acts))
    params = so.unflatten_params(net, flat)
    cfg = so.OptConfig(kind=so.OPT_MOMENTUM, lr=REPLICA_LR)
    ref = (so.Bf16Trainer(net, params, cfg, fused_out=hidden[-1] <= 256 and len(hidden) > 1) if p == BF16
           else so.CleanTrainer(net, params, cfg))
    full = [(np.concatenate([Xd, wd.onehot_matrix(idx, n_onehot)], axis=1), y[:, None], w[:, None]) for Xd, idx, y, w in shards]
    want, o = [], 0
    for n in sizes:
        want.append(ref.step([(X[o:o + n], y[o:o + n], w[o:o + n]) for X, y, w in full]))
        o += n
    dl, dp = float(np.abs(got - np.array(want)).max()), float(np.abs(thetas[0] - ref.theta).max())
    dg = float(np.abs(grads[0] - ref.last_grads).max() / np.abs(ref.last_grads).max())
    _notes["replicas %s %s max |loss - oracle|, |theta - oracle|, |grad - oracle| / max |grad|" % (where, case)] = (
        "%.3g, %.3g, %.3g" % (dl, dp, dg))
    tol_l, tol_p, tol_g = (1e-4, 1e-4, 1e-3) if p != BF16 else (1e-3, 5e-3, 5e-2)
    assert dl <= tol_l, (got, want)
    assert dp <= tol_p
    assert dg <= tol_g


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(REPLICAS))
def test_replicas_through_the_peer_exchange(sb, monkeypatch, case):
    monkeypatch.setenv("SB_XCHG_BLOCKS", "8")          # the exchange kernels spin: leave SMs to the other replica
    monkeypatch.setenv("SB_XCHG_TIMEOUT_S", "60")
    desc, flat, sizes, shards = _replica_case(sb, case)
    ts = [sb.Trainer(desc, device=0, nccl_id=None, rank=r, world=W_REPLICAS) for r in range(W_REPLICAS)]
    try:
        for t in ts:
            t.set_peer_pointers([x.exchange_base for x in ts])
            t.set_params(flat)
            _set_sparse(t, case)
        got = np.array(_in_threads(W_REPLICAS, lambda r: _replica_steps(ts[r], sizes, shards[r]))).T
        thetas = [t.get_params() for t in ts]
        grads = [t.get_grads() for t in ts]
        preds = [t.predict_sparse(shards[0][0][:300], shards[0][1][:300]) for t in ts]
    finally:
        for t in ts:
            t.close()
    _check_replicas(case, flat, sizes, shards, got, thetas, grads, preds, "one GPU")


def _two_gpu_rank_main(rank, world, port, out_dir, case):
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import torch.distributed as dist
    import shifu_tensorflow_b200 as sb
    from shifu_tensorflow_b200 import dist_util as du
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ.setdefault("SB_XCHG_TIMEOUT_S", "60")
    dist.init_process_group("gloo", rank=rank, world_size=world)
    desc, flat, sizes, shards = _replica_case(sb, case)
    t = sb.Trainer(desc, device=rank, nccl_id=None, rank=rank, world=world)
    du.enable_peer_exchange(dist, t, world)
    t.set_params(flat)
    _set_sparse(t, case)
    losses = _replica_steps(t, sizes, shards[rank])
    theta, grads = t.get_params(), t.get_grads()
    pred = t.predict_sparse(shards[0][0][:300], shards[0][1][:300])
    dist.barrier()
    np.savez(os.path.join(out_dir, "r%d.npz" % rank), losses=np.array(losses), theta=theta, grads=grads, pred=pred)
    t.close()
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["fp32_tc_two_chunks", "bf16_two_chunks"])
def test_replicas_on_two_gpus(sb, tmp_path, case):
    """two ranks on two devices over CUDA-IPC peer memory: dW_1 in front of dW_0, the placement of ranks that do not
    share a device"""
    if sb.capi.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    from test_host_mirrors import _free_port
    mp.spawn(_two_gpu_rank_main, args=(W_REPLICAS, _free_port(), str(tmp_path), case), nprocs=W_REPLICAS, join=True)
    r = [np.load(str(tmp_path / ("r%d.npz" % k))) for k in range(W_REPLICAS)]
    desc, flat, sizes, shards = _replica_case(sb, case)
    _check_replicas(case, flat, sizes, shards, np.stack([x["losses"] for x in r], axis=1), [x["theta"] for x in r],
                    [x["grads"] for x in r], [x["pred"] for x in r], "two GPUs")


# ---------------------------------------------------------------------------------------------- the worker
@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "fp32_tc"])
def test_worker_reports_the_oracles_losses(sb, tmp_path, precision):
    """SELECTED_COLUMN_NUMS blank + SELECTED_NUMERIC_/CATEGORY_COLUMN_NUMS: the wide+deep worker's epoch lines (training
    loss of the last mini-batch, eval_loss_sparse of the validation rows, global step) against CleanTrainer on the
    one-hot matrix, driven as the worker drives its steps"""
    from shifu_tensorflow_b200 import trainer as tr
    from test_host_mirrors import _Seq
    n_dense, vocab, n_rows, epochs = 6, [4, 7, 3], 900, 21
    Xd, idx, y, _ = wd.synth_wide_deep_batch(n_rows, n_dense, vocab, 3)
    offs = np.concatenate([[0], np.cumsum(vocab)[:-1]])
    codes = np.where(idx >= 0, idx - offs[None, :], -1)
    data = str(tmp_path / "part-00000.gz")
    with gzip.open(data, "wb") as f:
        for i in range(n_rows):
            cols = [str(int(y[i, 0]))] + [repr(float(v)) for v in Xd[i]] + [str(int(c)) for c in codes[i]]
            f.write(("|".join(cols) + "\n").encode())
    hidden, acts = [16, 8], [so.ACT_RELU, so.ACT_TANH]
    conf = {"train": {"params": {"NumHiddenLayers": 2, "NumHiddenNodes": hidden, "ActivationFunc": ["relu", "tanh"],
                                 "LearningRate": 0.1, "Optimizer": "sgd", "Precision": precision, "MiniBatchs": 100},
                      "numTrainEpochs": epochs, "validSetRate": 0.2}}
    srv = socket.socket()
    srv.bind(("127.0.0.1", 0))
    srv.listen(1)
    lines = []

    def serve():
        c, _ = srv.accept()
        buf = b""
        while True:
            d = c.recv(4096)
            if not d:
                break
            buf += d
        lines.extend(buf.decode().splitlines())

    th = threading.Thread(target=serve)
    th.start()
    env = {"CLUSTER_SPEC": json.dumps({"ps": ["127.0.0.1:1"], "worker": ["127.0.0.1:2"]}), "WORKER_CNT": "1", "JOB_NAME": "worker",
           "TASK_ID": "0", "SOCKET_SERVER_PORT": str(srv.getsockname()[1]), "TOTAL_TRAINING_DATA_NUMBER": str(n_rows),
           "SELECTED_COLUMN_NUMS": "", "SELECTED_NUMERIC_COLUMN_NUMS": " ".join(str(1 + i) for i in range(n_dense)),
           "SELECTED_CATEGORY_COLUMN_NUMS": " ".join(str(1 + n_dense + i) for i in range(len(vocab))),
           "SB_CATEGORY_VOCAB": " ".join(str(v) for v in vocab), "WEIGHT_COLUMN_NUM": "-1", "TARGET_COLUMN_NUM": "0",
           "TMP_MODEL_PATH": str(tmp_path / "tmp_model"), "FINAL_MODEL_PATH": str(tmp_path / "final_model"),
           "TRAINING_DATA_PATH": data, "SB_SEED": "11"}
    cwd = os.getcwd()
    os.chdir(tmp_path)
    try:
        json.dump(conf, open("ModelConfig.json", "w"))
        rc = tr.main(env=env, rng=_Seq(5))
    finally:
        os.chdir(cwd)
        th.join(10)
        srv.close()
    assert rc == 0
    # the dense replay: the worker's split (one coin per row), its init, one SGD update per np.array_split mini-batch
    seq = _Seq(5)
    coins = np.array([seq.random() >= 0.2 for _ in range(n_rows)])
    Xfull = np.concatenate([Xd, wd.onehot_matrix(idx, sum(vocab))], axis=1).astype(np.float32)
    tx, ty, vx, vy = Xfull[coins], y[coins], Xfull[~coins], y[~coins]
    F = Xfull.shape[1]
    net = so.NetDesc(F, hidden, acts)
    with sb.Trainer(sb.make_desc(F, hidden, acts, max_batch=128)) as t0:
        t0.init_xavier(11)
        theta = t0.get_params()
    ref = so.CleanTrainer(net, so.unflatten_params(net, theta), so.OptConfig(kind=so.OPT_SGD, lr=0.1))
    want, steps = [], 0
    while steps < epochs:
        for b in so.split_batches(len(tx), 100):
            L = ref.step([(tx[b], ty[b], np.ones((len(b), 1), np.float32))])[0]
            steps += 1
            if steps >= epochs:
                break
        want.append((steps, float(L), float(ref.eval_loss(vx, vy, np.ones((len(vx), 1), np.float32)))))
    got = [(int(l.split("current_epoch:")[1].split(",")[0]), float(l.split("training_loss:")[1].split(",")[0]),
            float(l.split("valid_loss:")[1])) for l in lines]
    assert [g[0] for g in got] == [x[0] for x in want], lines
    d = np.abs(np.array(got)[:, 1:] - np.array(want)[:, 1:])
    _notes["worker %s max |training_loss - oracle|, |valid_loss - oracle|" % precision] = "%.3g, %.3g" % tuple(d.max(axis=0))
    assert d.max() <= 1e-4, (got, want)


# ---------------------------------------------------------------------------------------------- no GPU
def _ref_case(prec, seed=7):
    n_dense, vocab, hidden, acts, _ = SHAPES["small"]
    F = n_dense + sum(vocab)
    layers = unflatten(_params(F, hidden, seed), F, hidden)
    Xd, idx, y, w = _rows(400, n_dense, vocab, seed, hot=False)
    return n_dense, vocab, hidden, acts, layers, Xd, idx, y, w


@pytest.mark.parametrize("prec", sorted(PRECS))
def test_sparse_reference_is_the_dense_one_on_the_onehot_matrix(prec):
    p = PRECS[prec]
    n_dense, vocab, hidden, acts, layers, Xd, idx, _, _ = _ref_case(p)
    Xfull = np.concatenate([Xd, wd.onehot_matrix(idx, sum(vocab))], axis=1)
    ys, es = scores(*hidden_forward_sparse(Xd, idx, layers, _codes(acts), p), layers, _codes(acts))
    yd, ed = scores(*hidden_forward(Xfull, layers, _codes(acts), p), layers, _codes(acts))
    if p != BF16:       # the same exact model on the fp32 parameters
        assert np.abs(ys - yd).max() <= 1e-12
    # two enclosures of what the kernels compute meet, and the sparse one is no looser than the dense one, whose
    # contraction runs over every one-hot column
    assert (np.abs(ys - yd) <= es + ed).all()
    assert np.median(es / ed) <= 1.0


def _mutated(idx, vocab, kind):
    """idx with one fault of the kind a gather could make; and the rows it changes"""
    offs = np.concatenate([[0], np.cumsum(vocab)[:-1]])
    m = idx.copy()
    if kind == "off_by_one":            # the last column's code one off, inside its vocabulary
        c = len(vocab) - 1
        code = m[:, c] - offs[c]
        m[:, c] = np.where(m[:, c] < 0, -1, offs[c] + np.where(code + 1 < vocab[c], code + 1, code - 1))
    elif kind == "column_dropped":
        m[:, 1] = -1
    else:                               # "missing_as_0": -1 read as embedding row 0
        m[m < 0] = 0
    return m, (m != idx).any(axis=1)


@pytest.mark.parametrize("kind", ["off_by_one", "column_dropped", "missing_as_0"])
@pytest.mark.parametrize("prec", sorted(PRECS))
def test_bounds_reject_wrong_indices(prec, kind):
    """the reference of the wrong indices misses the right model on most of the rows the fault changes: a kernel within
    its bound of the right rows (|k - y| <= e) is outside the bound of the wrong ones wherever |y - y'| > e + e'"""
    p = PRECS[prec]
    n_dense, vocab, hidden, acts, layers, Xd, idx, _, _ = _ref_case(p)
    codes = _codes(acts)
    y, e = scores(*hidden_forward_sparse(Xd, idx, layers, codes, p), layers, codes)
    bad, changed = _mutated(idx, vocab, kind)
    y2, e2 = scores(*hidden_forward_sparse(Xd, bad, layers, codes, p), layers, codes)
    assert changed.sum() >= 20
    caught = float(np.mean((np.abs(y - y2) > e + e2)[changed]))
    _notes["%s %s: changed rows the bound rejects" % (prec, kind)] = "%.3f" % caught
    assert caught >= 0.9, caught


@pytest.mark.parametrize("prec", sorted(PRECS))
def test_loss_bound_rejects_division_by_the_row_count(prec):
    p = PRECS[prec]
    n_dense, vocab, hidden, acts, layers, Xd, idx, y, w = _ref_case(p)
    a, e_a = hidden_forward_sparse(Xd, idx, layers, _codes(acts), p)
    want, tol = validation_loss(a, e_a, layers[-1][0], layers[-1][1], y, w, ACTS[acts[-1]], 130, lambda m: 64)
    nnz = np.count_nonzero(w)
    assert 0 < nnz < len(w)
    wrong = want * nnz / len(w)
    assert abs(wrong - want) > 2 * tol, (want, wrong, tol)
