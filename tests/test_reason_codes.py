"""Per-row reason codes (sb_model_reason_codes, Model.reason_codes) against column sensitivity and float64.

The property the GPU tests lean on: every returned delta is bit-identical to sb_model_sensitivity's delta at the
returned position, and the positions are reason_ref's top k of those deltas, for k in {1, 5, 32} and every order, in
all four precision modes: on the eval net (2000 columns) over rows enough for several row chunks of several pieces, and
on the small net of test_score_paths over every row and column.  Besides: the deltas and base scores against their
float64 bounds (sensitivity_ref.py) with no unselected position able to beat the k-th, planted cells, ties of repeated
columns, bit-identical repeats across host / device pointers, sentinels around device outputs, calls beside compute()
threads, the launches of each precision, argument errors before any device work, and TensorflowModel.computeReasonCodes.

The CPU tests check the reference ranking itself against a plain Python sort, and that merging top-k lists block by
block gives the top k of the whole row."""
import ctypes as C
import math
import threading

import numpy as np
import pytest

from out_layer_ref import ACTS, U
from reason_ref import ORDERS, keys, merged_topk, topk
from score_ref import BF16, BF16X2, FP32, FP32_TC, unflatten
from sensitivity_ref import pair_scores
from test_score_paths import EVAL_ACTS, EVAL_F, EVAL_GAINS, EVAL_HIDDEN, SMALL_ACTS, SMALL_F, SMALL_HIDDEN, _acts, _device_sms, _model, \
    _rows, _seeded
from test_sensitivity import chunk_rows, expected_sens_routes

PRECS = {"fp32": FP32, "bf16": BF16, "fp32_tc": FP32_TC, "bf16x2": BF16X2}
SENTINEL = 0x7FCDCDCD


def expected_reason_routes(prec, F, hidden, rows, n_cols, sms):
    """the launches of a call's last row chunk's z0 and last piece (score.cu sens_forward, then sens_topk_kernel)"""
    r = expected_sens_routes(prec, F, hidden, rows, n_cols, sms)
    assert r.endswith("+sens_reduce")
    return r[:-len("sens_reduce")] + "sens_topk"


# ------------------------------------------------------------------ the reference (CPU)
def _python_order(d, order):
    """one row's positions sorted by a plain Python sort of (NaN, -key, position)"""
    ks = [float(x) for x in keys(d, order)]
    return sorted(range(len(ks)), key=lambda j: (math.isnan(ks[j]), 0.0 if math.isnan(ks[j]) else -ks[j], j))


def _awkward_rows():
    rng = np.random.default_rng(5)
    rows = [rng.standard_normal(40).astype(np.float32),
            np.zeros(40, np.float32),                                     # all equal
            np.full(40, np.float32(0.25)),
            np.array([0.0, -0.0] * 20, np.float32),                       # +-0 compare equal
            np.full(40, np.nan, np.float32)]
    r = rng.standard_normal(40).astype(np.float32)
    r[[3, 9, 17]] = np.nan                                                 # NaN among numbers
    r[[4, 11]] = -np.inf
    r[[5, 6]] = np.inf
    r[[20, 21, 22]] = -0.0
    r[[23, 24]] = 0.0
    r[30:36] = r[7]                                                       # repeated positions: equal deltas
    r[36:40] = -r[8]                                                      # equal magnitudes of opposite sign
    rows.append(r)
    return np.stack(rows)


@pytest.mark.parametrize("order", ORDERS)
def test_reference_order_equals_python_sort(order):
    d = _awkward_rows()
    for k in (1, 5, 32, 40):
        p, v = topk(d, k, order)
        for r in range(d.shape[0]):
            want = _python_order(d[r], order)[:k]
            assert p[r].tolist() == want, (order, k, r)
            assert v[r].tobytes() == d[r, want].tobytes()
    # NaN ranks last, -0 ties +0 by position, an all-equal row is positions 0 .. k-1
    p, _ = topk(d, 40, order)
    assert p[1].tolist() == list(range(40)) and p[2].tolist() == list(range(40)) and p[3].tolist() == list(range(40))
    assert p[4].tolist() == list(range(40))
    assert sorted(p[5, -3:].tolist()) == [3, 9, 17] and p[5, -3:].tolist() == [3, 9, 17]


@pytest.mark.parametrize("order", ORDERS)
def test_merging_blocks_equals_global_topk(order):
    rng = np.random.default_rng(11)
    d = rng.standard_normal((64, 300)).astype(np.float32)
    d[:, 100:140] = d[:, :40]                                              # ties across blocks
    d[::5, ::7] = np.nan
    d[1::5, 2::9] = 0.0
    d[2::5, 3::9] = -0.0
    d[3] = 0.5
    d = np.concatenate([d, _awkward_rows()[:, :1].repeat(300, 1)], 0)
    for k in (1, 5, 32):
        want = topk(d, k, order)
        for bounds in ([0, 300], [0, 1, 300], [0, 31, 32, 33, 200, 300], list(range(0, 301, 13)) + [300],
                       sorted(set([0, 300] + rng.integers(1, 300, 9).tolist()))):
            got = merged_topk(d, k, order, bounds)
            assert np.array_equal(got[0], want[0]), (k, bounds)
            assert got[1].tobytes() == want[1].tobytes(), (k, bounds)


def test_null_model_is_state_error(sb):
    lib = sb.capi.lib()
    X = np.zeros(4, np.float32)
    pos, d = np.zeros(4, np.int32), np.zeros(4, np.float32)
    st = lib.sb_model_reason_codes(None, X.ctypes.data_as(C.c_void_p), 1, None, 0, None, 1, 0, pos.ctypes.data_as(C.c_void_p),
                                   d.ctypes.data_as(C.c_void_p), None)
    assert st == sb.capi.SB_ERR_STATE
    assert "TF model not initialized." in lib.sb_last_error().decode()


# ------------------------------------------------------------------ the GPU path
def _small_net():
    flat = _seeded(SMALL_F, SMALL_HIDDEN, (1.4, 1.4, 1.4, 4.0), 9)
    return flat, unflatten(flat, SMALL_F, SMALL_HIDDEN), _acts(SMALL_ACTS) + [ACTS["sigmoid"]]


def _check_against_sensitivity(m, X, cols, values, ks, what):
    """every order and k: pos = the reference top k of the sensitivity deltas, d bit-identical to them"""
    deltas = m.sensitivity(X, cols=cols, values=values, deltas=True)["deltas"]
    for order in ORDERS:
        for k in ks:
            got = m.reason_codes(X, k, cols=cols, values=values, order=order)
            want_p, want_d = topk(deltas, k, order)
            bad = np.argwhere(got["pos"] != want_p)
            assert bad.size == 0, "%s %s k=%d: %d positions differ, first (r, i) %s: %d vs %d" % (
                what, order, k, len(bad), tuple(bad[0]), got["pos"][tuple(bad[0])], want_p[tuple(bad[0])])
            assert got["d"].tobytes() == want_d.tobytes(), (what, order, k)
            assert got["d"].tobytes() == np.take_along_axis(deltas, got["pos"], 1).tobytes(), (what, order, k)
    return deltas


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PRECS))
def test_eval_net_matches_sensitivity(sb, name):
    prec = PRECS[name]
    flat = _seeded(EVAL_F, EVAL_HIDDEN, EVAL_GAINS, 7)
    rows = 200                                      # several row chunks (R = 64), each of two to eight pieces
    assert chunk_rows(prec, EVAL_F) == 64
    X = _rows(EVAL_F, rows, 13)
    with _model(sb, EVAL_F, EVAL_HIDDEN, EVAL_ACTS, prec, flat) as m:
        _check_against_sensitivity(m, X, None, None, (1, 5, 32), "eval " + name)
        assert m.routes() == expected_reason_routes(prec, EVAL_F, EVAL_HIDDEN, rows, EVAL_F, _device_sms())
        for order in ORDERS:
            got = m.reason_codes(X, 32, order=order)
            assert got["pos"][0].tolist() == list(range(32))              # row 0 is all zeros: every delta +0
            assert np.all(got["d"][0].view(np.uint32) == 0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PRECS))
@pytest.mark.parametrize("cols_kind", ["all", "list"])
def test_small_net_matches_sensitivity(sb, name, cols_kind):
    prec = PRECS[name]
    flat, _, _ = _small_net()
    rng = np.random.default_rng(23)
    cols = None if cols_kind == "all" else np.array([30, 2, 17, 2, 36, 0, 30, 9], np.int32)
    n_cols = SMALL_F if cols is None else len(cols)
    values = None if cols is None else rng.standard_normal(n_cols).astype(np.float32)
    ks = (1, 5, 32) if cols is None else (1, 5, 8)
    R = chunk_rows(prec, n_cols)
    sms = _device_sms()
    with _model(sb, SMALL_F, SMALL_HIDDEN, SMALL_ACTS, prec, flat) as m:
        for rows in (1, 2 * R + 77):
            X = _rows(SMALL_F, rows, rows)
            if rows > 5:
                X[5, 9] = np.nan          # the small net's activations carry NaN through: every delta of the row is NaN
            deltas = _check_against_sensitivity(m, X, cols, values, ks, "small %s %s rows=%d" % (name, cols_kind, rows))
            assert m.routes() == expected_reason_routes(prec, SMALL_F, SMALL_HIDDEN, rows, n_cols, sms)
            if rows > 5:
                assert np.all(np.isnan(deltas[5]))
                for order in ORDERS:
                    assert m.reason_codes(X, ks[-1], cols=cols, values=values, order=order)["pos"][5].tolist() == list(range(ks[-1]))


def _check_bounds(got, ref, order, what):
    """returned deltas and base scores within their float64 bounds (ref: sensitivity_ref.pair_scores of the call's
    inputs); no unselected position's key can beat the k-th's"""
    (s0, e0), (s, e) = ref
    d_ref = (s0[None, :] - s).T                                             # [rows, K]
    e_d = (e0[None, :] + e).T + U * np.abs(d_ref)
    p = got["pos"].astype(np.int64)
    rr = np.arange(d_ref.shape[0])[:, None]
    err = np.abs(got["d"].astype(np.float64) - d_ref[rr, p])
    assert np.all(err <= e_d[rr, p]), "%s: %d deltas outside their bound" % (what, int(np.sum(err > e_d[rr, p])))
    assert np.all(np.abs(got["scores"].astype(np.float64) - s0) <= e0), what + ": base scores"
    if order == "raise":
        lo, hi = d_ref - e_d, d_ref + e_d
    elif order == "lower":
        lo, hi = -d_ref - e_d, -d_ref + e_d
    else:
        lo, hi = np.maximum(np.abs(d_ref) - e_d, 0.0), np.abs(d_ref) + e_d
    kth_hi = hi[rr[:, 0], p[:, -1]]
    unselected = np.ones(d_ref.shape, bool)
    unselected[rr, p] = False
    beats = unselected & (lo > kth_hi[:, None])
    assert not beats.any(), "%s: %d unselected positions certainly beat the k-th" % (what, int(beats.sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PRECS))
def test_against_float64(sb, name):
    prec = PRECS[name]
    flat, layers, acts = _small_net()
    rng = np.random.default_rng(31)
    values = rng.standard_normal(SMALL_F).astype(np.float32)
    cl = np.arange(SMALL_F)
    X = _rows(SMALL_F, 2 * chunk_rows(prec, SMALL_F) + 77, 17)
    ref = pair_scores(X, layers, acts, prec, cl, values)
    with _model(sb, SMALL_F, SMALL_HIDDEN, SMALL_ACTS, prec, flat) as m:
        for order in ORDERS:
            for k in (1, 5, 32):
                got = m.reason_codes(X, k, values=values, order=order, scores=True)
                _check_bounds(got, ref, order, "small %s %s k=%d" % (name, order, k))
    # the eval net over every column of a few rows
    flat = _seeded(EVAL_F, EVAL_HIDDEN, EVAL_GAINS, 7)
    layers = unflatten(flat, EVAL_F, EVAL_HIDDEN)
    acts = _acts(EVAL_ACTS) + [ACTS["sigmoid"]]
    X = _rows(EVAL_F, 8, 19)
    with _model(sb, EVAL_F, EVAL_HIDDEN, EVAL_ACTS, prec, flat) as m:
        got = {o: m.reason_codes(X, 5, order=o, scores=True) for o in ORDERS}
    ref = pair_scores(X, layers, acts, prec, np.arange(EVAL_F), np.zeros(EVAL_F, np.float32))
    for o in ORDERS:
        _check_bounds(got[o], ref, o, "eval %s %s" % (name, o))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PRECS))
def test_planted_cells_and_ties(sb, name):
    prec = PRECS[name]
    flat, _, _ = _small_net()
    cols = np.array([30, 2, 17, 2, 36, 0, 30, 9, 11, 12], np.int32)
    values = np.random.default_rng(3).standard_normal(len(cols)).astype(np.float32)
    values[3] = values[1]                                                  # repeated columns with the same value tie
    values[6] = values[0]
    X = _rows(SMALL_F, 300, 29)
    X[7, cols] = values                                                    # every listed cell already holds its value
    X[8, cols[4]] = values[4]                                              # one planted cell
    X[9, cols[5]] = values[5]
    with _model(sb, SMALL_F, SMALL_HIDDEN, SMALL_ACTS, prec, flat) as m:
        for order in ORDERS:
            got = m.reason_codes(X, len(cols), cols=cols, values=values, order=order)
            p, d = got["pos"], got["d"]
            assert p[7].tolist() == list(range(len(cols))), order
            assert np.all(d[7].view(np.uint32) == 0)
            for r, j in ((8, 4), (9, 5)):
                assert d[r, list(p[r]).index(j)].view(np.uint32) == 0, (order, r)
            for a, b in ((1, 3), (0, 6)):
                ia, ib = (p == a).argmax(1), (p == b).argmax(1)
                assert np.all(ia < ib), (order, a, b)
                assert np.take_along_axis(d, ia[:, None], 1).tobytes() == np.take_along_axis(d, ib[:, None], 1).tobytes()
            for k in range(1, len(cols)):                                  # at the cut, the lower position wins the tie
                pk = m.reason_codes(X, k, cols=cols, values=values, order=order)["pos"]
                for a, b in ((1, 3), (0, 6)):
                    assert np.all((pk == a).any(1)[(pk == b).any(1)]), (order, k, a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PRECS))
def test_repeat_pointers_and_sentinels(sb, name):
    torch = pytest.importorskip("torch")
    prec = PRECS[name]
    flat, _, _ = _small_net()
    rows, k, pad = 2 * chunk_rows(prec, SMALL_F) + 5, 5, 64
    X = _rows(SMALL_F, rows, 4)
    vals = np.random.default_rng(8).standard_normal(SMALL_F).astype(np.float32)

    def bits(r):
        return [np.asarray(r[key].cpu() if hasattr(r[key], "cpu") else r[key]).tobytes() for key in ("pos", "d")]

    with _model(sb, SMALL_F, SMALL_HIDDEN, SMALL_ACTS, prec, flat) as m:
        a = m.reason_codes(X, k, values=vals, order="magnitude", scores=True)
        b = m.reason_codes(X, k, values=vals, order="magnitude", scores=True)
        c = m.reason_codes(X, k, values=vals, order="magnitude")
        assert bits(a) == bits(b) == bits(c) and c["scores"] is None
        assert a["scores"].tobytes() == b["scores"].tobytes()
        dX = torch.from_numpy(X).cuda()
        sent = torch.tensor([SENTINEL], dtype=torch.int32).view(torch.float32).item()
        bp = torch.full((rows * k + 2 * pad,), SENTINEL, dtype=torch.int32, device="cuda")
        bd = torch.full((rows * k + 2 * pad,), sent, dtype=torch.float32, device="cuda")
        bs = torch.full((rows + 2 * pad,), sent, dtype=torch.float32, device="cuda")
        for x in (X, dX):
            for dev_out in (False, True):
                if dev_out:
                    r = m.reason_codes(x, k, values=vals, order="magnitude", scores=bs[pad:pad + rows], pos=bp[pad:pad + rows * k],
                                       d=bd[pad:pad + rows * k])
                    torch.cuda.synchronize()
                    got = {"pos": bp[pad:pad + rows * k].cpu().numpy().reshape(rows, k),
                           "d": bd[pad:pad + rows * k].cpu().numpy().reshape(rows, k)}
                    assert bs[pad:pad + rows].cpu().numpy().tobytes() == a["scores"].tobytes()
                    assert r["pos"].data_ptr() == bp.data_ptr() + 4 * pad
                else:
                    got = m.reason_codes(x, k, values=vals, order="magnitude", scores=True)
                    assert got["scores"].tobytes() == a["scores"].tobytes()
                assert bits(got) == bits(a), (x is dX, dev_out)
        for buf in (bp, bd.view(torch.int32), bs.view(torch.int32)):
            h = buf.cpu().numpy()
            assert np.all(h[:pad] == SENTINEL) and np.all(h[-pad:] == SENTINEL)
        # rows = 0 writes nothing
        lib = sb.capi.lib()
        bp.fill_(SENTINEL); bd.fill_(sent); bs.fill_(sent)
        st = lib.sb_model_reason_codes(m._h, C.c_void_p(dX.data_ptr()), 0, None, 0, None, k, 0, C.c_void_p(bp.data_ptr()),
                                       C.c_void_p(bd.data_ptr()), C.c_void_p(bs.data_ptr()))
        torch.cuda.synchronize()
        assert st == sb.capi.SB_OK
        for buf in (bp, bd.view(torch.int32), bs.view(torch.int32)):
            assert np.all(buf.cpu().numpy() == SENTINEL)
        hp = np.full(8, SENTINEL, np.int32)
        st = lib.sb_model_reason_codes(m._h, X.ctypes.data_as(C.c_void_p), 0, None, 0, None, 1, 0, hp.ctypes.data_as(C.c_void_p),
                                       hp.ctypes.data_as(C.c_void_p), hp.ctypes.data_as(C.c_void_p))
        assert st == sb.capi.SB_OK and np.all(hp == SENTINEL)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["bf16", "fp32"])
def test_beside_compute_threads(sb, name):
    prec = PRECS[name]
    flat, _, _ = _small_net()
    X = _rows(SMALL_F, 300, 6)
    with _model(sb, SMALL_F, SMALL_HIDDEN, SMALL_ACTS, prec, flat) as m:
        solo = m.reason_codes(X, 5, scores=True)
        solo_rows = [m.score_row_f64(X[i].astype(np.float64)) for i in range(64)]
        got, errs = {}, []

        def scorer(t):
            try:
                got[t] = [m.score_row_f64(X[i].astype(np.float64)) for i in range(64)]
            except Exception as ex:      # noqa: BLE001 - re-raised below
                errs.append(ex)

        ths = [threading.Thread(target=scorer, args=(t,)) for t in range(4)]
        for t in ths:
            t.start()
        busy = [m.reason_codes(X, 5, scores=True) for _ in range(3)]
        for t in ths:
            t.join()
        assert not errs, errs
        for r in busy:
            for key in ("pos", "d", "scores"):
                assert r[key].tobytes() == solo[key].tobytes(), key
        for t in range(4):
            assert got[t] == solo_rows


@pytest.mark.gpu
def test_argument_errors_before_device_work(sb):
    flat, _, _ = _small_net()
    lib = sb.capi.lib()
    X = _rows(SMALL_F, 4, 1)
    with _model(sb, SMALL_F, SMALL_HIDDEN, SMALL_ACTS, BF16, flat) as m:
        def call(X_=X, rows=4, cols=None, n_cols=0, values=None, k=1, order=0, pos=True, d=True):
            p, dd = np.full(4 * 40, 7, np.int32), np.full(4 * 40, 7.0, np.float32)
            cp = None if cols is None else np.ascontiguousarray(cols, np.int32).ctypes.data_as(C.POINTER(C.c_int32))
            vp = None if values is None else np.ascontiguousarray(values, np.float32).ctypes.data_as(C.POINTER(C.c_float))
            st = lib.sb_model_reason_codes(m._h, None if X_ is None else X_.ctypes.data_as(C.c_void_p), rows, cp, n_cols, vp, k,
                                           order, p.ctypes.data_as(C.c_void_p) if pos else None,
                                           dd.ctypes.data_as(C.c_void_p) if d else None, None)
            if st != sb.capi.SB_OK:
                assert np.all(p == 7) and np.all(dd == 7.0)
            return st

        INV = sb.capi.SB_ERR_INVALID
        assert call(X_=None) == INV and call(pos=False) == INV and call(d=False) == INV
        assert call(rows=-1) == INV
        assert call(cols=[1, 2], n_cols=0) == INV and call(cols=None, n_cols=3) == INV
        assert call(cols=[1, SMALL_F], n_cols=2) == INV and call(cols=[-1], n_cols=1) == INV
        assert call(cols=[3, 4], n_cols=2, values=[1.0, np.nan]) == INV and call(cols=[3], n_cols=1, values=[np.inf]) == INV
        assert call(k=0) == INV and call(k=-1) == INV
        assert call(k=33) == INV                                # more than 32 (SMALL_F = 37 columns)
        assert call(cols=[3, 4], n_cols=2, k=3) == INV          # more than the list
        assert call(order=3) == INV and call(order=-1) == INV
        assert m.routes() == "none"                             # no device work so far
        assert call(rows=0, cols=[3, 5], n_cols=2, k=2) == sb.capi.SB_OK
        assert m.routes() == "none"
        assert call(cols=[3, 4], n_cols=2, k=2, order=2) == sb.capi.SB_OK
        assert m.routes() != "none"


@pytest.mark.gpu
def test_scorer_compute_reason_codes(sb):
    from shifu_tensorflow_b200 import scorer
    flat, _, _ = _small_net()
    X = _rows(SMALL_F, 50, 2).astype(np.float64) + 1e-9          # doubles, cast to float as computeBatch casts them
    cols = [4, 1, 30, 1, 12]
    vals = [0.5, -1.0, 0.0, 2.0, 1.5]
    tm = scorer.TensorflowModel()
    with pytest.raises(scorer.IllegalStateException):
        tm.computeReasonCodes(X, 2)
    with _model(sb, SMALL_F, SMALL_HIDDEN, SMALL_ACTS, FP32, flat) as m:
        tm = scorer.TensorflowModel.__new__(scorer.TensorflowModel)
        tm.initiate, tm._model = True, m
        for order in ORDERS:
            r = tm.computeReasonCodes(X, 3, columns=cols, values=vals, order=order)
            want = m.reason_codes(X.astype(np.float32), 3, cols=cols, values=np.array(vals, np.float32), order=order, scores=True)
            assert np.array_equal(r["columns"], np.array(cols)[want["pos"]])
            assert r["deltas"].tobytes() == want["d"].tobytes() and r["scores"].tobytes() == want["scores"].tobytes()
        r = tm.computeReasonCodes(X, 2)
        want = m.reason_codes(X.astype(np.float32), 2)
        assert np.array_equal(r["columns"], want["pos"])
