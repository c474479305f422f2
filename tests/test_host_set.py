"""A training set in pinned host memory (sb_trainer_load_dataset when the set does not fit in HBM).

The library keeps a set that does not fit in HBM in mapped pinned host memory, in the layout the HBM set has.  Tensor-core
steps (Feed::STREAMED) fetch each batch's rows over PCIe into one of two batch buffers, inside a run_resident graph one
step ahead beside GEMMs planned for the remaining SMs; fp32 steps read the host rows through the host-batch load kernel.  What a step computes is
unchanged: with deterministic training a trainer whose set is in host memory (sb_debug_force_host_set, so that the sizes
fit) must match, bit for bit, the same trainer with the set in HBM."""
import numpy as np
import pytest

from oracle import shifu_oracle as so
from util import make_pair
from test_batch_load import NP, check_stage, fill_sentinels, ld8, values, weights, D, _ids

FP32, BF16, FP32_TC, BF16X2 = 0, 1, 2, 3
PRECS = [FP32, BF16, FP32_TC, BF16X2]


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same(a, b):
    return np.array_equal(_bits(a), _bits(b))


def _pair(sb, F, hidden, rows, precision, det=True, seed=3):
    """two trainers with the same parameters: (set in host memory, set in HBM)"""
    _ids(sb)
    acts = [so.ACT_RELU, so.ACT_TANH, so.ACT_SIGMOID][:len(hidden)]
    out = []
    for host in (True, False):
        net, params, cfg, desc = make_pair(sb, F, hidden, acts, optimizer=so.OPT_ADAM, lr=0.01, max_batch=rows,
                                           precision=precision, seed=seed)
        t = sb.Trainer(desc, deterministic=det)
        t.set_params(so.flatten_params(params))
        t.debug_force_host_set(host)
        out.append(t)
    return out


def _load(pair, X, y, w):
    for t, host in zip(pair, (True, False)):
        t.load_dataset(X, y, w)
        assert t.dataset_on_host == host


def _drive(t, rows, n):
    """run_resident over 7 steps (one graph of four, three single steps), accumulate_resident + apply_accumulated_mean,
    loss_resident and a step: the losses they report"""
    offs = [(i * 97) % (n - rows + 1) for i in range(7)]
    t.run_resident(offs, rows)
    out = list(t.loss_history(1, 7))
    out.append(t.accumulate_resident(rows // 2, rows))
    out.append(t.accumulate_resident(1, rows - 1))
    t.apply_accumulated(3)
    out.append(t.loss_resident(n - rows, rows))
    out.append(t.step_resident(2, rows))
    t.step_resident_async(n - rows, rows)
    t.sync()
    out.append(t.last_loss())
    return np.asarray(out, np.float32)


def _state(t, tmp_path, tag):
    path = str(tmp_path / ("%s.ckpt" % tag))
    t.save_checkpoint(path)
    return t.get_params(), t.get_grads(), open(path, "rb").read()


@pytest.mark.gpu
@pytest.mark.parametrize("order", ["physical", "shuffled"])
@pytest.mark.parametrize("precision", PRECS)
def test_host_set_trains_to_the_hbm_bits(sb, tmp_path, precision, order):
    F, hidden, rows = 300, [200, 77], 333
    n = 3 * rows + 17
    X, y, w = so.synth_batch(n, F, 5, weights="mixed")
    a, b = _pair(sb, F, hidden, rows, precision)
    with a, b:
        _load((a, b), X, y, w)
        if precision != FP32:
            m = NP[precision] * n * ld8(F)
            assert np.array_equal(a.debug_buffer(D.DS_X, n=m), b.debug_buffer(D.DS_X, n=m))
            assert np.array_equal(a.debug_buffer(D.DS_P, n=n + 1), b.debug_buffer(D.DS_P, n=n + 1))
        if order == "shuffled":
            pi = np.random.default_rng(1).permutation(n)
            a.set_row_order(pi)
            b.set_row_order(pi)
        la, lb = _drive(a, rows, n), _drive(b, rows, n)
        assert np.isfinite(la).all() and _same(la, lb), (la, lb)
        pa, ga, ca = _state(a, tmp_path, "a")
        pb, gb, cb = _state(b, tmp_path, "b")
        assert _same(pa, pb) and _same(ga, gb) and ca == cb


@pytest.mark.gpu
@pytest.mark.parametrize("precision", [BF16, FP32_TC])
def test_reordered_between_calls_over_many_graphs(sb, precision):
    """three run_resident calls of three graphs of four steps each, a new row order before every call and the physical
    order once: the host set's steps read the rows each call's order names"""
    F, hidden, rows = 256, [128, 64], 256
    n = 4 * rows
    X, y, w = so.synth_batch(n, F, 7, weights="mixed")
    rng = np.random.default_rng(3)
    offs = [(k * rows) % (n - rows + 1) for k in range(12)]
    a, b = _pair(sb, F, hidden, rows, precision)
    with a, b:
        _load((a, b), X, y, w)
        for k in range(4):
            pi = rng.permutation(n) if k != 2 else None
            a.set_row_order(pi)
            b.set_row_order(pi)
            a.run_resident(offs, rows)
            b.run_resident(offs, rows)
        got, want = a.loss_history(1, 48), b.loss_history(1, 48)
        assert _same(got, want) and _same(a.get_params(), b.get_params())


@pytest.mark.gpu
@pytest.mark.parametrize("precision", [BF16, FP32_TC])
def test_non_deterministic_host_set_within_tolerance(sb, precision):
    F, hidden, rows = 300, [200, 77], 333
    n = 3 * rows + 17
    X, y, w = so.synth_batch(n, F, 9, weights="mixed")
    a, b = _pair(sb, F, hidden, rows, precision, det=False)
    with a, b:
        _load((a, b), X, y, w)
        la, lb = _drive(a, rows, n), _drive(b, rows, n)
        tol = 5e-4 if precision == BF16 else 1e-4
        assert np.isfinite(la).all() and np.abs(la - lb).max() <= tol, (la, lb)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", [BF16, FP32_TC, BF16X2, FP32])
@pytest.mark.parametrize("F", [1, 7, 300, 2000])
def test_gather_from_host_bit_for_bit(sb, precision, F):
    """the first kernel of a step over the host set fills the batch operand (every part, +0 pad columns), y / w, n_nz and
    the cleared loss sum and gradient exactly as the numpy split says, and leaves every byte outside the batch alone"""
    rng = np.random.default_rng(F)
    max_batch = 8192 if F == 2000 else 600
    n = max_batch + 300
    X, y, w = values(rng, n, F), rng.standard_normal(n).astype(np.float32), weights(rng, n)
    with sb.Trainer(sb.make_desc(F, [8], [2], max_batch=max_batch, precision=precision)) as t:
        _ids(sb)
        t.debug_force_host_set(True)
        t.load_dataset(X, y, w)
        assert t.dataset_on_host
        pi = rng.permutation(n)
        cases = [(None, 0, 1), (None, n - max_batch, max_batch), (None, 17, 257), (pi, 5, max_batch), (pi, n - 1, 1)]
        for order, off, rows in cases:
            t.set_row_order(order)
            idx = (np.arange(n) if order is None else order)[off:off + rows]
            fill_sentinels(t, precision, max_batch, ld8(F))
            route = t.debug_first_kernel(row_offset=off, rows=rows, clear=True)
            # fp32 mode reads the host rows through the host-batch load kernel, an order through the gather
            want_route = ("gather_batch<fp32>" if order is not None else "load_batch<fp32>") if precision == FP32 \
                else "gather_batch<bf16>"
            assert route == want_route
            check_stage(t, precision, max_batch, X[idx], y[idx], w[idx], yw_written=(precision != FP32 or order is not None))


@pytest.mark.gpu
def test_errors(sb):
    F, hidden, rows = 64, [32, 16], 128
    X, y, w = so.synth_batch(4 * rows, F, 1, weights="ones")
    err = sb.ShifuB200Error
    with sb.Trainer(sb.make_desc(F, hidden, [2, 2], max_batch=rows, precision=BF16)) as t:
        for bad in (2, -1):
            with pytest.raises(err) as e:
                sb.capi.check(sb.capi.lib().sb_debug_force_host_set(t._h, bad))
            assert e.value.code == sb.capi.SB_ERR_INVALID
        t.debug_force_host_set(True)
        with pytest.raises(err) as e:
            t.step_resident(0, rows)
        assert e.value.code == sb.capi.SB_ERR_STATE
        assert not t.dataset_on_host
        t.load_dataset(X, y, w)
        assert t.dataset_on_host
        with pytest.raises(err) as e:
            t.set_row_order([0, 4 * rows])
        assert e.value.code == sb.capi.SB_ERR_INVALID
        for call in (lambda: t.step_resident(3 * rows + 1, rows), lambda: t.run_resident([0, 3 * rows + 1], rows),
                     lambda: t.accumulate_resident(-1, rows), lambda: t.loss_resident(4 * rows, 1)):
            with pytest.raises(err) as e:
                call()
            assert e.value.code == sb.capi.SB_ERR_INVALID
        assert t.global_step == 0
        assert np.isfinite(t.step_resident(3 * rows, rows))
        t.debug_force_host_set(False)
        t.load_dataset(X, y, w)                  # small enough for HBM again
        assert not t.dataset_on_host


@pytest.mark.gpu
def test_pinned_allocation_failure_names_the_bytes(sb):
    """a set far larger than any host's address space: the pinned allocation fails at once, the error names the bytes it
    asked for, and no set is loaded (nothing of the set is read before the allocation)"""
    F, n_rows = 100000, (1 << 31) - 1
    want = n_rows * ld8(F) * 2 * 3
    X, y = np.zeros((1, F), np.float32), np.zeros(1, np.float32)
    with sb.Trainer(sb.make_desc(F, [4], [2], max_batch=64, precision=FP32_TC)) as t:
        rc = sb.capi.lib().sb_trainer_load_dataset(t._h, sb.capi._ptr(X), sb.capi._ptr(y), None, n_rows)
        assert rc == sb.capi.SB_ERR_CUDA
        assert str(want) in sb.capi.lib().sb_last_error().decode()
        assert not t.dataset_on_host
        with pytest.raises(sb.ShifuB200Error) as e:
            t.step_resident(0, 1)
        assert e.value.code == sb.capi.SB_ERR_STATE


# ---- CPU: the worker's footprint estimate and its choice of loader ----
def test_footprint_estimate():
    from shifu_tensorflow_b200 import trainer as tr, _capi as capi
    text, lines, F = 10 ** 9, 10 ** 6, 2000
    parsed = lines * (F + 2) * 4
    assert tr.gpu_load_footprint(text, lines, F, capi.PREC_BF16) == text + parsed + lines * 2000 * 2
    assert tr.gpu_load_footprint(text, lines, F, capi.PREC_FP32_TC) == text + parsed + lines * 2000 * 6
    assert tr.gpu_load_footprint(text, lines, F, capi.PREC_BF16X2) == text + parsed + lines * 2000 * 4
    assert tr.gpu_load_footprint(text, lines, F, capi.PREC_FP32) == text + parsed + lines * 2000 * 4
    assert tr.gpu_load_footprint(0, 10, 3, capi.PREC_BF16) == 10 * 5 * 4 + 10 * 8 * 2    # pitch round_up(3, 8)
    assert tr.parse_on_host_side(101, 100) and not tr.parse_on_host_side(100, 100)
    # four local ranks: each parses the whole text, but keeps a quarter of the rows
    assert tr.gpu_load_footprint(text, lines, F, capi.PREC_BF16, 4) == text + parsed + lines // 4 * 2000 * 2


def _write_gz(path, X, y, wcol=None):
    import gzip
    with gzip.open(path, "wb") as f:
        for i in range(len(X)):
            cells = [str(int(y[i]))] + [repr(float(v)) for v in X[i]] + ([repr(float(wcol[i]))] if wcol is not None else [])
            f.write(("|".join(cells) + "\n").encode())


class _Seq:
    def __init__(self, seed):
        self.r = np.random.RandomState(seed)

    def random(self):
        return float(self.r.rand())


@pytest.mark.parametrize("free", [10 ** 12, 1000])
def test_worker_loader_choice(tmp_path, monkeypatch, free):
    """with a stubbed free-memory figure: enough -> the device parse (sb_text_parse_device); too little -> host parse in
    line-aligned pieces (sb_text_parse, here stood in for by the host state machine), the same coins per line, and the
    same rows, labels and weights as the reference loader"""
    from shifu_tensorflow_b200 import trainer as tr, _capi as capi
    rng = np.random.default_rng(0)
    n, F = 500, 6
    X = np.round(rng.standard_normal((n, F)), 3).astype(np.float32)
    y = (rng.random(n) < 0.5).astype(np.float32)
    wc = np.round(rng.uniform(-1, 3, n), 2).astype(np.float32)
    X[7, 2] = 1e-45                                  # a cell the fast path declines
    path = str(tmp_path / "part-00000.gz")
    _write_gz(path, X, y, wc)
    calls = []
    monkeypatch.setattr(capi, "device_mem_info", lambda device=0: (free, 2 * free))
    monkeypatch.setattr(tr, "HOST_PARSE_CHUNK", 997)          # many pieces, cut at line ends

    parse = capi.text_parse

    def host_parse(text, col_map, n_feat, delim="|", device=0):
        calls.append(len(text))
        assert text.endswith(b"\n")
        return parse(text, col_map, n_feat, delim, host_debug=True)

    def device_parse(*a, **k):
        calls.append("device")
        raise RuntimeError("device parse")
    monkeypatch.setattr(capi, "text_parse", host_parse)
    monkeypatch.setattr(capi, "text_parse_device", device_parse)
    cols = list(range(1, F + 1))
    if free > 10 ** 9:
        with pytest.raises(RuntimeError, match="device parse"):
            tr.load_data_gpu(path, cols, 0, F + 1, 0.2, rng=_Seq(5))
        assert calls == ["device"]
        return
    got = tr.load_data_gpu(path, cols, 0, F + 1, 0.2, rng=_Seq(5))
    assert len(calls) > 5 and all(c <= 997 for c in calls)
    want = tr.load_data(path, cols, 0, F + 1, 0.2, rng=_Seq(5))
    assert got["feature_count"] == F
    for pre in ("train", "valid"):
        np.testing.assert_array_equal(got[pre + "_data"], np.asarray(want[pre + "_data"], np.float32))
        np.testing.assert_array_equal(got[pre + "_target"], np.asarray(want[pre + "_target"], np.float32).reshape(-1))
        np.testing.assert_array_equal(got[pre + "_data_sample_weight"],
                                      np.asarray(want[pre + "_data_sample_weight"], np.float32).reshape(-1))


def test_header_and_prototypes_have_the_host_set_calls(sb):
    import os
    import re
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "shifu_b200.h")).read()
    for name in ("sb_debug_force_host_set", "sb_trainer_dataset_on_host", "sb_device_mem_info"):
        assert re.search(r"\b%s\s*\(" % name, hdr) and name in sb.capi.PROTOTYPES
