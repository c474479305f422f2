"""Every trainer, scorer and kernel test hook gives back the device memory it allocated.

Rounds of: a trainer created, used on each of its paths (resident set + multi-step graphs, pipelined host steps,
accumulation, prediction) and closed; two in-process replicas joined by their peer tables, stepped and closed; a scorer
created, used and closed, and one refused for a wrong parameter count; each kernel test hook once.  After the rounds, the
device's free memory must be back at what it was after the first (which also loads every kernel the rounds launch).

Device memory only: leaked events and pinned host memory are not visible here, and neither are failure paths."""
import numpy as np
import pytest

from oracle import shifu_oracle as so

pytestmark = pytest.mark.gpu

MB = 1 << 20
F, HIDDEN, ACTS, B = 2048, [512, 256], [2, 1], 2048
ROWS = 16 * B                     # resident set: 128 MB as bf16 (and a 256 MB fp32 conversion window while loading)
TOL = 32 * MB                     # well under one round's footprint (a single trainer's is asserted below)


def _free(torch):
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info(0)[0]


def _trainer_round(sb, X, y, w):
    desc = sb.make_desc(F, HIDDEN, ACTS, optimizer=sb.OPT_ADAM, learning_rate=1e-3, max_batch=B, precision=sb.PREC_BF16)
    with sb.Trainer(desc) as t:
        t.init_xavier(1)
        t.load_dataset(X, y, w)
        t.run_resident([k * B for k in range(8)], B)        # two 4-step graphs on the alternating descriptor sets
        t.step_async(X[:B], y[:B], w[:B])                      # second staging slot and copy stream
        t.step_async(X[B:2 * B], y[B:2 * B], w[B:2 * B])
        t.accumulate(X[:B], y[:B], w[:B])
        t.apply_accumulated()
        p = t.predict(X[:B])
        assert np.isfinite(p).all() and np.isfinite(t.last_loss())


def _replica_round(sb, X, y, w, monkeypatch):
    monkeypatch.setenv("SB_XCHG_BLOCKS", "8")
    monkeypatch.setenv("SB_XCHG_TIMEOUT_S", "60")
    desc = sb.make_desc(F, HIDDEN, ACTS, optimizer=sb.OPT_MOMENTUM, learning_rate=0.01, max_batch=B, precision=sb.PREC_BF16)
    ts = [sb.Trainer(desc, device=0, nccl_id=None, rank=r, world=2) for r in range(2)]
    try:
        bases = [t.exchange_base for t in ts]
        for t in ts:
            t.set_peer_pointers(bases)
            t.init_xavier(2)
        for r, t in enumerate(ts):
            t.load_dataset(X[r * 4 * B:(r + 1) * 4 * B], y[r * 4 * B:(r + 1) * 4 * B], w[r * 4 * B:(r + 1) * 4 * B])
        for t in ts:
            t.run_resident([k * B for k in range(4)], B)
        for t in ts:
            t.sync()
        assert np.allclose(ts[0].get_params(), ts[1].get_params())
    finally:
        for t in ts:
            t.close()


def _model_round(sb, X):
    desc = sb.make_desc(F, HIDDEN, ACTS, precision=sb.PREC_BF16)
    net = so.NetDesc(F, HIDDEN, ACTS)
    flat = so.flatten_params(so.xavier_init(net, 3))
    m = sb.Model.create(desc, flat)
    try:
        assert np.isfinite(m.score(X[:B])).all()
    finally:
        m.close()
    with pytest.raises(sb.ShifuB200Error) as e:
        sb.Model.create(desc, flat[:-1])
    assert e.value.code == sb.capi.SB_ERR_INVALID


def _hook_round(sb):
    # shapes the kernel tests of each hook already cover
    rng = np.random.default_rng(0)
    A = rng.standard_normal((1000, 4096), dtype=np.float32)
    sb.capi.debug_gemm_bf16(A, rng.standard_normal((512, 4096), dtype=np.float32), split_k=4)
    sb.capi.debug_gemm_bench(1000, 512, 4096, a_mn=True, b_mn=True, cg=1, bn=256, iters=2)
    A = rng.standard_normal((4096, 1000), dtype=np.float32)
    sb.capi.debug_gemm_split(A, rng.standard_normal((512, 1000), dtype=np.float32), 3)
    sb.capi.debug_gemm_epilogue(A, rng.standard_normal((1000, 512), dtype=np.float32), sb.capi.ACT_RELU,
                                bias=np.zeros(512, np.float32), iters=2)
    sb.capi.debug_gemm_epilogue(A, rng.standard_normal((512, 1000), dtype=np.float32), sb.capi.ACT_TANH,
                                aux=np.tanh(rng.standard_normal((4096, 512), dtype=np.float32)))
    A = rng.standard_normal((1000, 512), dtype=np.float32)
    sb.capi.debug_gemm_fwd_out(A, rng.standard_normal((512, 200), dtype=np.float32), np.zeros(200, np.float32),
                               rng.standard_normal(200, dtype=np.float32), 0.1, (rng.uniform(size=1000) < 0.3).astype(np.float32),
                               np.ones(1000, np.float32), sb.capi.ACT_RELU, sb.LOSS_SIGMOID_CE, np_parts=2)


def test_rounds_give_back_device_memory(sb, monkeypatch):
    torch = pytest.importorskip("torch")
    X, y, w = so.synth_batch(ROWS, F, 5, weights="mixed")

    def one_round():
        _trainer_round(sb, X, y, w)
        _replica_round(sb, X, y, w, monkeypatch)
        _model_round(sb, X)
        _hook_round(sb)

    one_round()
    base = _free(torch)
    desc = sb.make_desc(F, HIDDEN, ACTS, max_batch=B, precision=sb.PREC_BF16)
    with sb.Trainer(desc) as t:                    # for scale: what one trainer with its resident set holds
        t.load_dataset(X, y, w)
        one_trainer = base - _free(torch)
    print("one trainer with its resident set: %.1f MB" % (one_trainer / MB))
    assert one_trainer > TOL, "the tolerance must be well under what a round allocates"
    for _ in range(3):
        one_round()
        print("free after a round: %+.1f MB against the baseline" % ((_free(torch) - base) / MB))
    end = _free(torch)
    assert end >= base - TOL, "device memory not given back: %.1f MB less free than after the first round" % ((base - end) / MB)
