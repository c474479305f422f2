"""Launch order of a training step (enqueue_step_backward, csrc/capi.cu), read from the in-graph step trace
(SB_STEP_TRACE=1): the names of the GEMM, optimizer and exchange launches of the last captured step, in the order they
were enqueued.  Dense steps are captured by kernels_per_step, which only captures and instantiates the graph; the sparse
(wide+deep) step is captured by one step_sparse.

Where dW_1 runs depends on the SM count (plan_dw1), so the expected orders are those of a 132-SM H100 SXM."""
import numpy as np
import pytest

from oracle import shifu_oracle as so
from oracle import wide_deep as wd

pytestmark = pytest.mark.gpu

CASES = {
    # cfg1's shape on one GPU: every dW_l beside the dA chain, dW_0 behind the last dA GEMM, split optimizer tail
    "cfg1": dict(F=1000, hidden=[512, 256, 128], B=4096, prec=1, names=[
        "fwd0@4096x512x1000", "fwd1@4096x256x512", "fwd_out2@4096x128x256",
        "dW2@256x128x4096", "dA2@4096x256x128", "dW1@512x256x4096", "dA1@4096x512x256", "dW0@1000x512x4096",
        "opt", "opt_side"]),
    # dW_0 alone fills every SM: dW_1 moves in front of it on the main stream
    "dw0_fills_sms": dict(F=2000, hidden=[1280, 512], B=4096, prec=1, names=[
        "fwd0@4096x1280x2000", "fwd1@4096x512x1280", "out_layer",
        "dA1@4096x1280x512", "dW1@1280x512x4096", "dW0@2000x1280x4096", "opt", "opt_side"]),
    "bf16x2": dict(F=256, hidden=[192, 128, 64], B=512, prec=3, names=[
        "fwd0@512x192x256", "fwd1@512x128x192", "fwd_out2@512x64x128",
        "dW2@128x64x512", "dA2@512x128x64", "dW1@192x128x512", "dA1@512x192x128", "dW0@256x192x512",
        "opt", "opt_side"]),
    # two bf16 replicas that share a device: dW_0 cut into the exchange slot chunks with each chunk's exchange behind it,
    # dW_1 behind dW_0, slot A's exchange last
    "two_replicas_one_device": dict(F=1000, hidden=[512, 256, 128], B=4096, prec=1, world=2, names=[
        "fwd0@4096x512x1000", "fwd1@4096x256x512", "fwd_out2@4096x128x256",
        "dW2@256x128x4096", "dA2@4096x256x128", "dA1@4096x512x256",
        "dW0.0@512x512x4096", "xchg_B0", "dW0.1@488x512x4096", "xchg_B1", "dW1@512x256x4096", "xchg_A"]),
}

SPARSE_CASES = {
    "wide_deep_small": dict(n_dense=21, vocab=[5, 9, 3, 17], hidden=[40, 24], rows=130, names=[
        "fwd0@130x40x21", "fwd_out1@130x24x40", "dW1@40x24x130", "dA1@130x40x24", "dW0@21x40x130", "opt", "opt_side"]),
    # BASELINE config 4: dW_0 (planned over all 5500 rows of W_0) fills every SM, so dW_1 runs in front of it
    "wide_deep_cfg4": dict(n_dense=500, vocab=[100] * 50, hidden=[1024, 512], rows=2048, names=[
        "fwd0@2048x1024x500", "fwd1@2048x512x1024", "out_layer",
        "dA1@2048x1024x512", "dW1@1024x512x2048", "dW0@500x1024x2048", "opt", "opt_side"]),
}


@pytest.fixture(autouse=True)
def _h100_sxm(sb, monkeypatch):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if sms != 132:
        pytest.skip("the expected launch orders are those of a 132-SM H100 SXM; where dW_1 runs depends on the SM count "
                    "(this device has %d SMs)" % sms)
    monkeypatch.setenv("SB_STEP_TRACE", "1")


def _desc(sb, F, hidden, B, prec):
    return sb.make_desc(F, hidden, [so.ACT_RELU] * len(hidden), optimizer=so.OPT_MOMENTUM, learning_rate=0.01, max_batch=B,
                        precision=prec)


@pytest.mark.parametrize("case", sorted(CASES))
def test_dense_step_launch_order(sb, monkeypatch, case):
    c = CASES[case]
    desc = _desc(sb, c["F"], c["hidden"], c["B"], c["prec"])
    world = c.get("world", 1)
    if world > 1:
        monkeypatch.setenv("SB_XCHG_BLOCKS", "8")
    ts = [sb.Trainer(desc, device=0, nccl_id=None, rank=r, world=world) for r in range(world)]
    try:
        if world > 1:
            for t in ts:
                t.set_peer_pointers([x.exchange_base for x in ts])
        ts[0].kernels_per_step(c["B"])          # captured and instantiated, never launched
        names, _ = ts[0].debug_step_trace()
    finally:
        for t in ts:
            t.close()
    assert names == c["names"]


# Which kernel runs the output layer: the fused output-layer GEMM (fwd_out, last hidden layer <= 256 wide and not a
# wide+deep first layer) or the output-layer kernel of its own (out_layer).  Pins the route of the parity tests that exist
# for one of them (test_trainer_parity.py, test_wide_deep_gpu.py): out_layer_rows_kernel<1 / 2 / 4> up to 256 / 512 /
# 1024 columns, out_layer_kernel<bf16> beyond.
ROUTES = {
    # name: (hidden, precision, sparse, kernel)
    "h256_bf16": ([96, 256], 1, False, "fwd_out"),
    "h257_bf16": ([96, 257], 1, False, "out_layer"),
    "h256_fp32tc": ([96, 256], 2, False, "fwd_out"),
    "h300_bf16x2": ([96, 300], 3, False, "out_layer"),
    "h700_bf16": ([96, 700], 1, False, "out_layer"),
    "h700_fp32tc": ([96, 700], 2, False, "out_layer"),
    "h1100_bf16": ([96, 1100], 1, False, "out_layer"),
    "h1100_bf16x2": ([96, 1100], 3, False, "out_layer"),
    "wide_deep_one_layer": ([48], 1, True, "out_layer"),
}


@pytest.mark.parametrize("case", sorted(ROUTES))
def test_output_layer_route(sb, case):
    hidden, prec, sparse, kernel = ROUTES[case]
    rows, n_dense, vocab = 300, 21, [5, 9, 3, 17]
    F = n_dense + sum(vocab) if sparse else 120
    with sb.Trainer(_desc(sb, F, hidden, rows, prec)) as t:
        if sparse:
            Xd, idx, y, w = wd.synth_wide_deep_batch(rows, n_dense, vocab, 2)
            t.init_xavier(1)
            t.set_sparse(n_dense, sum(vocab), len(vocab))
            assert np.isfinite(t.step_sparse(Xd, idx, y, w))
        else:
            t.kernels_per_step(rows)
        names, _ = t.debug_step_trace()
    fused = [n for n in names if n.startswith("fwd_out")]
    own = [n for n in names if n == "out_layer"]
    if kernel == "fwd_out":
        assert fused == ["fwd_out%d@%dx%dx%d" % (len(hidden) - 1, rows, hidden[-1], hidden[-2])] and not own, names
    else:
        assert own == ["out_layer"] and not fused, names


@pytest.mark.parametrize("case", sorted(SPARSE_CASES))
def test_sparse_step_launch_order(sb, case):
    c = SPARSE_CASES[case]
    n_onehot = int(sum(c["vocab"]))
    desc = _desc(sb, c["n_dense"] + n_onehot, c["hidden"], c["rows"], 1)
    Xd, idx, y, w = wd.synth_wide_deep_batch(c["rows"], c["n_dense"], c["vocab"], 2)
    with sb.Trainer(desc) as t:
        t.init_xavier(1)
        t.set_sparse(c["n_dense"], n_onehot, len(c["vocab"]))
        assert np.isfinite(t.step_sparse(Xd, idx, y, w))
        names, _ = t.debug_step_trace()
    assert names == c["names"]
