"""Where a training step gets its batch (its feed): a host batch, the bf16 or fp32 resident set, the resident set through a
row order, a bf16 set in host memory streamed batch by batch, or a wide+deep sparse batch.

Every entry point describes its batch once and hands that description to the one descriptor writer, the one descriptor
ring and the one graph cache of csrc/capi.cu.  These tests pin what that must keep:
  - per feed, the launches of a captured step (kernels_per_step and the SB_STEP_TRACE names, of a single step and of an
    interior step of a run_resident graph), as recorded before the feeds shared that code;
  - in deterministic mode, a mixed sequence of entry points gives the same bits whether the calls queue behind each other
    or each one is waited for: a descriptor set rewritten while a queued step still reads it would change them.

The launch names depend on the SM count through plan_dw1, so they are those of a 132-SM H100 SXM."""
import numpy as np
import pytest

from oracle import shifu_oracle as so
from oracle import wide_deep as wd

pytestmark = pytest.mark.gpu

F, HIDDEN, B = 120, [96, 64], 256
N_ROWS = 16 * B
SPARSE = dict(n_dense=21, vocab=[5, 9, 3, 17], hidden=[40, 24], rows=130)

# feed -> (kernels_per_step(B), names of a single step, names of an interior step of a run_resident graph)
EXPECTED = {
    "host": (9,
        ['fwd0@256x96x120', 'fwd_out1@256x64x96', 'dW1@96x64x256', 'dA1@256x96x64', 'dW0@120x96x256', 'opt', 'opt_side'],
        None),
    "resident_bf16": (8,
        ['fwd0@256x96x120', 'fwd_out1@256x64x96', 'dW1@96x64x256', 'dA1@256x96x64', 'dW0@120x96x256', 'opt', 'opt_side'],
        ['fwd0@256x96x120', 'fwd_out1@256x64x96', 'dW1@96x64x256', 'dA1@256x96x64', 'dW0@120x96x256', 'opt', 'opt_side']),
    "resident_fp32": (9,
        ['out_layer', 'opt'],
        ['out_layer', 'opt']),
    "ordered_bf16": (9,
        ['gather_batch', 'fwd0@256x96x120', 'fwd_out1@256x64x96', 'dW1@96x64x256', 'dA1@256x96x64', 'dW0@120x96x256', 'opt', 'opt_side'],
        ['gather_batch', 'fwd0@256x96x120', 'fwd_out1@256x64x96', 'dW1@96x64x256', 'dA1@256x96x64', 'dW0@120x96x256', 'opt', 'opt_side']),
    "ordered_fp32": (9,
        ['gather_batch', 'out_layer', 'opt'],
        ['gather_batch', 'out_layer', 'opt']),
    "streamed_bf16": (9,
        ['fwd0@256x96x120', 'fwd_out1@256x64x96', 'dW1@96x64x256', 'dA1@256x96x64', 'dW0@120x96x256', 'opt', 'opt_side'],
        ['fwd0@256x96x120', 'fwd_out1@256x64x96', 'dW1@96x64x256', 'dA1@256x96x64', 'dW0@120x96x256', 'opt', 'opt_side']),
    "sparse": (None,
        ['fwd0@130x40x21', 'fwd_out1@130x24x40', 'dW1@40x24x130', 'dA1@130x40x24', 'dW0@21x40x130', 'opt', 'opt_side'],
        None),
}


def _desc(sb, prec, hidden=HIDDEN, F=F, B=B):
    return sb.make_desc(F, hidden, [so.ACT_RELU] * len(hidden), optimizer=so.OPT_MOMENTUM, learning_rate=0.01, max_batch=B,
                        precision=prec)


def observe(sb, feed):
    """-> (kernels_per_step(B) or None, trace names of a single step, trace names of a run_resident step or None)"""
    if feed == "sparse":
        n_onehot = int(sum(SPARSE["vocab"]))
        Xd, idx, y, w = wd.synth_wide_deep_batch(SPARSE["rows"], SPARSE["n_dense"], SPARSE["vocab"], 2)
        with sb.Trainer(_desc(sb, 1, SPARSE["hidden"], SPARSE["n_dense"] + n_onehot, SPARSE["rows"])) as t:
            t.init_xavier(1)
            t.set_sparse(SPARSE["n_dense"], n_onehot, len(SPARSE["vocab"]))
            assert np.isfinite(t.step_sparse(Xd, idx, y, w))
            return None, t.debug_step_trace()[0], None
    prec = 0 if feed.endswith("fp32") else 1
    with sb.Trainer(_desc(sb, prec)) as t:
        t.init_xavier(1)
        if feed != "host":
            X, y, w = so.synth_batch(N_ROWS, F, 3, weights="mixed")
            if feed.startswith("streamed"):
                t.debug_force_host_set(True)
            t.load_dataset(X, y, w)
            if feed.startswith("ordered"):
                t.set_row_order(np.random.RandomState(5).permutation(N_ROWS))
        kps = t.kernels_per_step(B)
        names = t.debug_step_trace()[0]
        run_names = None
        if feed != "host":
            t.run_resident([k * B for k in range(4)], B)
            t.sync()
            run_names = t.debug_step_trace()[0]
        return kps, names, run_names


@pytest.fixture
def _h100_sxm(sb, monkeypatch):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if sms != 132:
        pytest.skip("the expected launches are those of a 132-SM H100 SXM (this device has %d SMs)" % sms)
    monkeypatch.setenv("SB_STEP_TRACE", "1")


@pytest.mark.parametrize("feed", ["host", "resident_bf16", "resident_fp32", "ordered_bf16", "ordered_fp32", "streamed_bf16",
                                  "sparse"])
def test_step_launches_per_feed(sb, _h100_sxm, feed):
    kps, names, run_names = observe(sb, feed)
    assert (kps, names, run_names) == EXPECTED[feed]


def _run_mixed(sb, tmp_path, prec, world, sync_each, monkeypatch):
    """the sequence of entry points, each call queued on every replica before the next call, without waiting or
    (sync_each) waiting for every replica after each call -> per replica (checkpoint bytes, loss history, last loss, the
    losses the calls returned)"""
    if world > 1:
        monkeypatch.setenv("SB_XCHG_BLOCKS", "8")
        monkeypatch.setenv("SB_XCHG_TIMEOUT_S", "60")
    net = so.NetDesc(F, HIDDEN, [so.ACT_RELU] * len(HIDDEN))
    params = so.flatten_params(so.xavier_init(net, 4))
    shards = [so.synth_batch(N_ROWS, F, 6 + r, weights="mixed") for r in range(world)]
    ts = [sb.Trainer(_desc(sb, prec), device=0, nccl_id=None, rank=r, world=world, deterministic=True) for r in range(world)]
    try:
        for t, (X, y, w) in zip(ts, shards):
            if world > 1:
                t.set_peer_pointers([x.exchange_base for x in ts])
            t.set_params(params)
            t.load_dataset(X, y, w)

        def each(fn, *args):
            out = [fn(t)(*args) for t in ts]
            if sync_each:
                for t in ts:
                    t.sync()
            return out

        if world > 1:
            # fp32 replicas read the set through a row order from the start, so that every resident step is an ordered one
            # and takes its descriptors from the ring like a bf16-resident step
            each(lambda t: t.set_row_order, np.random.RandomState(9).permutation(N_ROWS))
        for k in range(3):
            each(lambda t: t.step_resident_async, k * B + 11 * k, B)
        each(lambda t: t.run_resident, [(k % 12) * B + 3 * k for k in range(9)], B)     # two graphs of four steps + one step
        losses = each(lambda t: t.loss_resident, 2 * B + 5, B)
        for k in range(2):
            losses += each(lambda t: t.accumulate_resident, (4 + k) * B, B)
        each(lambda t: t.apply_accumulated)
        each(lambda t: t.set_row_order, np.random.RandomState(8).permutation(N_ROWS))
        each(lambda t: t.run_resident, [(k * 5 % 14) * B + k for k in range(8)], B)
        n = 21
        if world == 1:      # (step() waits for its own exchange: replicas on one device would wait for each other)
            for k in range(2):
                each(lambda t: t.step_async, *(a[o:o + B] for a in shards[0] for o in [(3 + 2 * k) * B + 7]))
            losses += each(lambda t: t.step, *(a[9 * B + 2:10 * B + 2] for a in shards[0]))
            n = 24
        out = []
        for r, t in enumerate(ts):
            t.sync()
        for r, t in enumerate(ts):
            assert t.global_step == n
            path = str(tmp_path / ("ckpt_%d_%d" % (r, sync_each)))
            t.save_checkpoint(path)
            with open(path, "rb") as f:
                out.append((f.read(), t.loss_history(1, n).tobytes(), np.float32(t.last_loss()).tobytes(),
                            np.float32(losses[r::world]).tobytes()))
        return out
    finally:
        for t in ts:
            t.close()


@pytest.mark.parametrize("prec,world", [(1, 1), (0, 1), (0, 2)], ids=["bf16", "fp32", "fp32_two_replicas_ordered"])
def test_mixed_entry_points_queued_equal_synced(sb, tmp_path, monkeypatch, prec, world):
    queued = _run_mixed(sb, tmp_path, prec, world, False, monkeypatch)
    synced = _run_mixed(sb, tmp_path, prec, world, True, monkeypatch)
    for r in range(world):
        assert queued[r] == synced[r], "replica %d" % r
