"""The scorer's small-batch and compute() paths give the bits of the batched path.

- An fp32 model scores a batch of up to SMALL_ROWS rows in one launch (score_rows_kernel): every score must equal, bit
  for bit, the same row's score in a batch of more than SMALL_ROWS rows (the layer-by-layer launches).
- Concurrent compute() calls (sb_model_score_row_f64) on one handle share device batches of up to 128 rows: every result
  must equal the same row's lone call, in every precision mode, and reach its own caller.
The debug hooks (batch stats, hold) confirm which path ran and that batches are really shared."""
import ctypes
import os
import threading

import numpy as np
import pytest

from oracle import shifu_oracle as so

GOLDEN_HEAD = os.path.join(os.path.dirname(__file__), "golden", "dummydl_head.npz")
SIG, TANH, RELU, LEAKY, NONE = so.ACT_SIGMOID, so.ACT_TANH, so.ACT_RELU, so.ACT_LEAKYRELU, -1
MODES = [0, 1, 2, 3]        # PREC_FP32, PREC_BF16, PREC_FP32_TC, PREC_BF16X2


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _model(sb, F, hidden, acts, precision=0, seed=0):
    """a model with seeded weights of ~ unit-variance activations (scores spread over (0, 1))"""
    rng = np.random.default_rng(seed)
    parts, prev = [], F
    for h in list(hidden) + [1]:
        parts.append(rng.standard_normal((prev, h)).astype(np.float32) * np.float32(1.5 / np.sqrt(prev)))
        parts.append(rng.standard_normal(h).astype(np.float32) * np.float32(0.1))
        prev = h
    flat = np.concatenate([p.ravel() for p in parts])
    return sb.Model.create(sb.make_desc(F, hidden, acts, precision=precision), flat)


def _rows(F, n, seed):
    X = np.random.default_rng(seed).standard_normal((n, F)).astype(np.float32)
    X[0] = -0.0                 # signed zeros and a sparse row: the zero-padded K tail of the fp32 GEMM
    X[1] = 0.0
    X[2, ::3] = 0.0
    return X


# (F, hidden, acts): every activation, F in {37, 1000, 1522}, widths 1 .. 1100, 1 to 21 dense layers
NETS = {
    "f37_w1": (37, [1], [NONE]),
    "f37_mixed": (37, [7, 33, 1, 100], [SIG, TANH, RELU, LEAKY]),
    "f1000_wide": (1000, [1100, 300], [LEAKY, NONE]),
    "f1000_deep": (1000, [300, 7, 100, 1100, 1, 33], [RELU, TANH, SIG, NONE, LEAKY, RELU]),
    "f1522_dummydl": (1522, [100] * 20, [RELU, TANH, SIG, LEAKY, NONE] * 4),
}
COUNTS = sorted({1, 2, 17, 64, 127, 128, 96})


@pytest.mark.gpu
@pytest.mark.parametrize("net", list(NETS), ids=list(NETS))
def test_small_fp32_batches_score_the_bits_of_the_batched_path(sb, net):
    F, hidden, acts = NETS[net]
    counts = sorted(set(COUNTS) | {sb.capi.SMALL_ROWS})
    X_big = _rows(F, sb.capi.SMALL_ROWS + 172, 1)
    rng = np.random.default_rng(2)
    with _model(sb, F, hidden, acts, seed=3) as m:
        s0 = m.batch_stats()["small_launches"]
        big = m.score(X_big)
        assert m.batch_stats()["small_launches"] == s0, "a batch of more than SMALL_ROWS rows took the one-launch kernel"
        assert np.isfinite(big).all()
        for k, c in enumerate(counts):
            # one of the zero rows first, then c - 1 distinct others in random order
            idx = np.concatenate([[k % 3], 3 + rng.choice(len(X_big) - 3, c - 1, replace=False)])
            got = m.score(X_big[idx])
            assert m.batch_stats()["small_launches"] == s0 + k + 1, "%d rows did not take the one-launch kernel" % c
            np.testing.assert_array_equal(_bits(got), _bits(big[idx]), err_msg="%d rows" % c)


@pytest.mark.gpu
def test_small_fp32_batches_through_score_device(sb):
    torch = pytest.importorskip("torch")
    F, hidden, acts = NETS["f1000_deep"]
    X_big = _rows(F, 300, 4)
    with _model(sb, F, hidden, acts, seed=5) as m:
        big = m.score(X_big)
        for c in (1, 17, sb.capi.SMALL_ROWS):
            s0 = m.batch_stats()["small_launches"]
            dX = torch.from_numpy(X_big[5:5 + c].copy()).cuda()
            dOut = torch.full((c,), float("nan"), dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            m.score_device(dX.data_ptr(), c, dOut.data_ptr())
            m.sync()
            assert m.batch_stats()["small_launches"] == s0 + 1
            np.testing.assert_array_equal(_bits(dOut.cpu().numpy()), _bits(big[5:5 + c]))


@pytest.mark.gpu
@pytest.mark.parametrize("precision", MODES)
def test_concurrent_compute_calls_get_their_own_serial_bits(sb, precision):
    """64 threads each score their own 200 distinct rows through compute() while another thread scores 5000 rows in one
    batched call: every result equals the same row's lone compute() call, bit for bit."""
    F, hidden, acts = 120, [64, 300, 32], [RELU, TANH, SIG]
    n_threads, per = 64, 200
    X = np.random.default_rng(6).standard_normal((n_threads * per, F))     # float64: compute() casts to float32
    X_batch = _rows(F, 5000, 7)
    with _model(sb, F, hidden, acts, precision=precision, seed=8) as m:
        want = np.array([m.score_row_f64(x) for x in X])
        want_batch = m.score(X_batch)
        if precision == sb.PREC_FP32:        # (the tensor-core GEMM plans of 12 800 rows are not the 128-row plan)
            np.testing.assert_array_equal(_bits(want), _bits(m.score(X.astype(np.float32))))
        st0 = m.batch_stats()
        got = np.full(len(X), np.nan)
        got_batch, errs = [None], []
        go = threading.Barrier(n_threads + 1)

        def rows(t):
            try:
                go.wait()
                for i in range(t * per, (t + 1) * per):
                    got[i] = m.score_row_f64(X[i])
            except Exception as e:      # noqa: BLE001 - surfaced below
                errs.append(e)

        def batch():
            try:
                go.wait()
                got_batch[0] = m.score(X_batch)
            except Exception as e:      # noqa: BLE001
                errs.append(e)

        th = [threading.Thread(target=rows, args=(t,)) for t in range(n_threads)] + [threading.Thread(target=batch)]
        [t.start() for t in th]; [t.join() for t in th]
        assert not errs, errs
        wrong = np.flatnonzero(got != want)
        assert wrong.size == 0, "%d of %d results differ, first at row %d" % (wrong.size, len(X), wrong[0])
        np.testing.assert_array_equal(_bits(got_batch[0]), _bits(want_batch))
        st = m.batch_stats()
        assert st["rows"] - st0["rows"] == len(X)
        assert st["max_fill"] <= 128
        path = "graph" if precision != sb.PREC_FP32 else "small"
        assert st[path] - st0[path] == st["batches"] - st0["batches"]
        print("precision %d: %d compute() rows in %d device batches, largest %d" %
              (precision, len(X), st["batches"] - st0["batches"], st["max_fill"]))


@pytest.mark.gpu
@pytest.mark.parametrize("precision", [0, 2])
def test_compute_calls_share_one_batch_under_hold(sb, precision):
    F, hidden, acts = 50, [40, 20], [RELU, TANH]
    X = np.random.default_rng(9).standard_normal((32, F))
    with _model(sb, F, hidden, acts, precision=precision, seed=10) as m:
        want = np.array([m.score_row_f64(x) for x in X])          # lone calls: one row per batch
        st = m.batch_stats()
        assert (st["batches"], st["rows"], st["max_fill"]) == (32, 32, 1)
        m.hold(32, 20000)
        got = np.full(32, np.nan)
        go = threading.Barrier(32)

        def one(i):
            go.wait()
            got[i] = m.score_row_f64(X[i])

        th = [threading.Thread(target=one, args=(i,)) for i in range(32)]
        [t.start() for t in th]; [t.join() for t in th]
        st2 = m.batch_stats()
        assert (st2["batches"] - st["batches"], st2["rows"] - st["rows"], st2["max_fill"]) == (1, 32, 32)
        np.testing.assert_array_equal(got, want)
        m.score_row_f64(X[0])                                     # the hold applied to one batch only
        assert m.batch_stats()["batches"] == st2["batches"] + 1


@pytest.mark.gpu
def test_fixture_weights_through_compute(sb):
    """the reference fixture's real weights (dummydl head): compute() within 1e-5 of the stored answers and equal to
    score() bit for bit, in fp32 and fp32_tc"""
    g = np.load(GOLDEN_HEAD)
    hidden = [g["W0"].shape[1], g["W1"].shape[1], g["W2"].shape[1]]
    flat = np.concatenate([np.concatenate([g["W%d" % i].ravel(), g["b%d" % i].ravel()]) for i in range(4)])
    X = np.asarray(g["X"], np.float32)
    for prec in (sb.PREC_FP32, sb.PREC_FP32_TC):
        with sb.Model.create(sb.make_desc(1522, hidden, [RELU] * 3, precision=prec), flat) as m:
            got = np.array([m.score_row_f64(x.astype(np.float64)) for x in X])
            assert np.abs(got - g["Y"].ravel()).max() <= 1e-5
            np.testing.assert_array_equal(got, m.score(X).astype(np.float64))


@pytest.mark.gpu
def test_short_row_fails_only_its_own_call(sb):
    F, hidden, acts = 64, [32], [RELU]
    X = np.random.default_rng(11).standard_normal((16, F))
    with _model(sb, F, hidden, acts, seed=12) as m:
        want = np.array([m.score_row_f64(x) for x in X])
        m.hold(16, 2000)
        got, errs, short = np.full(16, np.nan), [], []
        go = threading.Barrier(17)

        def one(i):
            go.wait()
            got[i] = m.score_row_f64(X[i])

        def bad():
            go.wait()
            try:
                m.score_row_f64(X[0][:F - 1])
            except sb.ShifuB200Error as e:
                short.append(e)

        th = [threading.Thread(target=one, args=(i,)) for i in range(16)] + [threading.Thread(target=bad)]
        [t.start() for t in th]; [t.join() for t in th]
        assert len(short) == 1 and short[0].code == sb.capi.SB_ERR_INVALID and "expected %d features" % F in str(short[0])
        np.testing.assert_array_equal(got, want)


@pytest.mark.gpu
def test_models_used_by_threads_give_back_device_memory(sb):
    torch = pytest.importorskip("torch")
    F, hidden, acts = 1000, [512, 256], [RELU, TANH]
    X = np.random.default_rng(13).standard_normal((256, F))

    def one_round():
        for prec in (sb.PREC_FP32, sb.PREC_FP32_TC):
            m = _model(sb, F, hidden, acts, precision=prec, seed=14)
            try:
                th = [threading.Thread(target=lambda t=t: [m.score_row_f64(x) for x in X[t::16]]) for t in range(16)]
                [t.start() for t in th]; [t.join() for t in th]
                assert np.isfinite(m.score(X.astype(np.float32))).all()
            finally:
                m.close()

    def free():
        torch.cuda.synchronize()
        return torch.cuda.mem_get_info(0)[0]

    one_round()
    base = free()
    for _ in range(3):
        one_round()
    assert free() >= base - (8 << 20), "device memory not given back: %.1f MB" % ((base - free()) / (1 << 20))


def test_debug_hooks_reject_a_null_handle(sb):
    lib = sb.capi.lib()
    st = (ctypes.c_int64 * sb.capi.DEBUG_MSTAT_WORDS)()
    assert lib.sb_debug_model_batch_stats(None, st, sb.capi.DEBUG_MSTAT_WORDS) == sb.capi.SB_ERR_STATE
    assert lib.sb_debug_model_hold(None, 4, 10) == sb.capi.SB_ERR_STATE
    assert lib.sb_debug_model_routes(None, ctypes.create_string_buffer(64), 64) == sb.capi.SB_ERR_STATE
    assert b"not initialized" in lib.sb_last_error()
