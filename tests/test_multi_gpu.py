"""2-GPU data-parallel parity (needs a machine with two GPUs): two processes, NCCL inside libshifu_b200.so, each rank steps on its
own shard; parameters after the steps must equal the oracle's data-parallel trainer (mean of per-rank gradients)."""
import os
import socket

import numpy as np
import pytest

from oracle import shifu_oracle as so

torch = pytest.importorskip("torch")


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close()
    return p


def _rank_main(rank, world, port, out_dir, precision, exchange="nccl"):
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import torch.distributed as dist
    import shifu_tensorflow_b200 as sb
    from shifu_tensorflow_b200 import dist_util as du
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    uid = du.broadcast_bytes(dist, sb.capi.nccl_unique_id, sb.capi.SB_NCCL_ID_BYTES, rank)
    net = so.NetDesc(96, [64, 32], [so.ACT_RELU, so.ACT_TANH])
    params = so.xavier_init(net, 4)
    desc = sb.make_desc(96, [64, 32], net.acts, optimizer=so.OPT_MOMENTUM, learning_rate=0.1, max_batch=128, precision=precision)
    t = sb.Trainer(desc, device=rank, nccl_id=uid, rank=rank, world=world)
    if exchange == "p2p":
        du.enable_peer_exchange(dist, t, world)
    t.set_params(so.flatten_params(params))
    losses = []
    for s in range(3):
        X, y, w = so.synth_batch(256, 96, 20 + s, weights="mixed")
        idx = du.shard_rows(256, rank, world)
        losses.append(t.step(X[idx], y[idx], w[idx]))
    theta, grads = t.get_params(), t.get_grads()      # (sharded exchange: gathered from the owner ranks)
    dist.barrier()                                    # nobody frees its arena while a peer still reads it
    np.savez(os.path.join(out_dir, "r%d.npz" % rank), theta=theta, grads=grads, losses=np.array(losses))
    t.close()
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize("exchange", ["nccl", "p2p"])
@pytest.mark.parametrize("precision", [0, 1])
def test_two_gpu_data_parallel_matches_oracle(sb, tmp_path, precision, exchange):
    if sb.capi.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    world, port = 2, _free_port()
    mp.spawn(_rank_main, args=(world, port, str(tmp_path), precision, exchange), nprocs=world, join=True)
    r = [np.load(str(tmp_path / ("r%d.npz" % i))) for i in range(world)]
    np.testing.assert_array_equal(r[0]["theta"], r[1]["theta"])      # replicas stay bit-identical
    np.testing.assert_array_equal(r[0]["grads"], r[1]["grads"])
    net = so.NetDesc(96, [64, 32], [so.ACT_RELU, so.ACT_TANH])
    ref = so.CleanTrainer(net, so.xavier_init(net, 4), so.OptConfig(kind=so.OPT_MOMENTUM, lr=0.1))
    for s in range(3):
        X, y, w = so.synth_batch(256, 96, 20 + s, weights="mixed")
        want = ref.step([(X[i::2], y[i::2], w[i::2]) for i in range(2)])
        if precision == 0:
            assert abs(want[0] - r[0]["losses"][s]) <= 1e-5 and abs(want[1] - r[1]["losses"][s]) <= 1e-5
    tol = 1e-5 if precision == 0 else 5e-3
    assert np.abs(r[0]["theta"] - ref.theta).max() <= tol


RES_F, RES_HIDDEN, RES_B, RES_STEPS = 96, [64, 48, 32], 128, 14      # 3 graphs of 4 steps + 2 single steps


def _resident_rank_main(rank, world, port, out_dir, precision):
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import torch.distributed as dist
    import shifu_tensorflow_b200 as sb
    from shifu_tensorflow_b200 import dist_util as du
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    os.environ.setdefault("SB_XCHG_TIMEOUT_S", "60")
    dist.init_process_group("gloo", rank=rank, world_size=world)
    acts = [so.ACT_RELU, so.ACT_TANH, so.ACT_RELU]
    net = so.NetDesc(RES_F, RES_HIDDEN, acts)
    desc = sb.make_desc(RES_F, RES_HIDDEN, acts, optimizer=so.OPT_MOMENTUM, learning_rate=0.05, max_batch=RES_B, precision=precision)
    t = sb.Trainer(desc, device=rank, nccl_id=None, rank=rank, world=world)
    du.enable_peer_exchange(dist, t, world)
    t.set_params(so.flatten_params(so.xavier_init(net, 4)))
    X, y, w = so.synth_batch(world * RES_B * RES_STEPS, RES_F, 31, weights="mixed")
    mine = np.concatenate([np.arange(s * world * RES_B + rank, (s + 1) * world * RES_B, world) for s in range(RES_STEPS)])
    t.load_dataset(X[mine], y[mine], w[mine])
    t.run_resident([s * RES_B for s in range(RES_STEPS)], RES_B)
    hist = t.loss_history(1, RES_STEPS)
    theta, grads = t.get_params(), t.get_grads()
    dist.barrier()
    np.savez(os.path.join(out_dir, "r%d.npz" % rank), theta=theta, grads=grads, losses=np.array(hist))
    t.close()
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize("precision", [1, 2])
def test_two_gpu_resident_run_matches_oracle(sb, tmp_path, precision):
    """sb_trainer_run_resident on two REAL GPUs over CUDA-IPC peer memory (no NCCL communicator at all): multi-step graphs
    with three hidden layers, i.e. the schedule bench.py times - dW_0 in chunks with their exchanges beside the next GEMMs,
    slot 0's exchange on the side stream behind dW_1 (bf16: the LL kernel; fp32_tc: the flag-and-pull kernel)."""
    if sb.capi.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    world, port = 2, _free_port()
    mp.spawn(_resident_rank_main, args=(world, port, str(tmp_path), precision), nprocs=world, join=True)
    r = [np.load(str(tmp_path / ("r%d.npz" % i))) for i in range(world)]
    np.testing.assert_array_equal(r[0]["theta"], r[1]["theta"])      # replicas stay bit-identical
    np.testing.assert_array_equal(r[0]["grads"], r[1]["grads"])
    acts = [so.ACT_RELU, so.ACT_TANH, so.ACT_RELU]
    net = so.NetDesc(RES_F, RES_HIDDEN, acts)
    ref = so.CleanTrainer(net, so.xavier_init(net, 4), so.OptConfig(kind=so.OPT_MOMENTUM, lr=0.05))
    X, y, w = so.synth_batch(world * RES_B * RES_STEPS, RES_F, 31, weights="mixed")
    for s in range(RES_STEPS):
        rows = [np.arange(s * world * RES_B + k, (s + 1) * world * RES_B, world) for k in range(world)]
        want = ref.step([(X[i], y[i], w[i]) for i in rows])
        tol_l = 1e-4 if precision == 2 else 2e-2
        for k in range(world):
            assert abs(want[k] - r[k]["losses"][s]) <= tol_l, (s, k, want[k], r[k]["losses"][s])
    # fp32_tc (3 x bf16 split, fp32 accumulate): the fp32 bound of the single-GPU parity tests; bf16: the bound of the NCCL test above
    tol = 1e-4 if precision == 2 else 5e-3
    assert np.abs(r[0]["theta"] - ref.theta).max() <= tol


@pytest.mark.gpu
@pytest.mark.parametrize("schedule", ["batch", "sync_replicas"])
def test_launcher_with_two_real_ranks(sb, tmp_path, schedule):
    """the per-node launcher (launcher.py) with REAL workers on 2 GPUs: env rewriting -> two `trainer.py` processes ->
    rendezvous on the CLUSTER_SPEC address -> NCCL communicator + state broadcast from worker 0 -> CUDA-IPC peer exchange
    -> training -> one aggregated metrics line per epoch upstream -> chief exports the SavedModel -> exit code 0.
    No SB_SEED: every rank would draw its own initial weights without the broadcast."""
    if sb.capi.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import gzip
    import json
    import sys
    import threading
    from shifu_tensorflow_b200 import launcher as la
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    F, n_rows = 24, 4000
    X, y, w = so.synth_batch(n_rows, F, 2)
    data = str(tmp_path / "part-00000.gz")
    with gzip.open(data, "wb") as f:
        for i in range(n_rows):
            f.write(("|".join([str(int(y[i, 0]))] + [repr(float(v)) for v in X[i]]) + "\n").encode())
    conf = {"train": {"params": {"NumHiddenLayers": 2, "NumHiddenNodes": [32, 16], "ActivationFunc": ["relu", "tanh"], "LearningRate": 0.05,
                                 "Optimizer": "momentum", "Schedule": schedule, "MiniBatchs": 200, "Precision": "bf16"},
                      "numTrainEpochs": 12 if schedule == "batch" else 3, "validSetRate": 0.2}}
    work = tmp_path / "cwd"; work.mkdir()
    json.dump(conf, open(work / "ModelConfig.json", "w"))
    srv = socket.socket(); srv.bind(("127.0.0.1", 0)); srv.listen(1)
    got = []

    def serve():
        c, _ = srv.accept()
        buf = b""
        while True:
            d = c.recv(4096)
            if not d:
                break
            buf += d
        got.extend(buf.decode().splitlines())

    th = threading.Thread(target=serve, daemon=True); th.start()
    env = dict(os.environ)
    env.update({"JOB_NAME": "worker", "TASK_ID": "0", "WORKER_CNT": "1",
                "CLUSTER_SPEC": json.dumps({"ps": ["127.0.0.1:1"], "worker": ["127.0.0.1:%d" % _free_port()]}),
                "SOCKET_SERVER_PORT": str(srv.getsockname()[1]), "TRAINING_DATA_PATH": data, "TOTAL_TRAINING_DATA_NUMBER": str(n_rows),
                "SELECTED_COLUMN_NUMS": " ".join(str(i) for i in range(1, F + 1)), "WEIGHT_COLUMN_NUM": "-1", "TARGET_COLUMN_NUM": "0",
                "TMP_MODEL_PATH": str(tmp_path / "tmp_model"), "FINAL_MODEL_PATH": str(tmp_path / "final_model"),
                "SB_LOCAL_GPUS": "2", "PYTHONPATH": root + os.pathsep + env.get("PYTHONPATH", ""), "SB_XCHG_TIMEOUT_S": "60"})
    cwd = os.getcwd()
    os.chdir(work)
    try:
        rc = la.main(env=env, worker_cmd=[sys.executable, "-c", "import sys, shifu_tensorflow_b200.trainer as t; sys.exit(t.main())"])
    finally:
        os.chdir(cwd)
    th.join(20); srv.close()
    assert rc == 0
    assert got and all(l.startswith("worker_index:0,") for l in got)
    last = la.parse_metrics_line(got[-1])
    assert int(last["current_epoch"]) == conf["train"]["numTrainEpochs"] and np.isfinite(last["valid_loss"]) and 0 < last["valid_loss"] < 1
    final = str(tmp_path / "final_model")
    assert sorted(os.listdir(final)) == ["GenericModelConfig.json", "saved_model.pb", "variables"]
    Fn, hidden, acts, out_act, flat = sb.capi.savedmodel_read(final, "shifu_input_0", "shifu_output_0")
    assert (Fn, hidden) == (F, [32, 16]) and np.isfinite(flat).all()
