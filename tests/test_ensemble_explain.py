"""Explaining a bagged model's score (sb_ensemble_sensitivity / sb_ensemble_reason_codes, Ensemble.sensitivity /
reason_codes) against float64 and against the single model.

- One member: every stat gives sb_model_sensitivity's / sb_model_reason_codes' bits.  Identical members: max, min and
  median (and the mean of two) give the single model's bits.
- Heterogeneous members (different widths, depths and activations; K = 2 .. 5, and K = 32 tiny nets): every delta within
  its bound from ensemble_explain_ref.py, every sum within the sum of its terms' bounds, every reason code a valid top k
  and bit-identical to the sensitivity delta at its position, exact +0 where a cell already holds the value; the eval
  net's shape over all 2000 columns in BF16 and FP32_TC.
- Host / device pointers, repeats, sentinels, the launches of a call, calls beside compute() threads, argument errors
  before any device work, and the scorer's TensorflowEnsemble methods.
The CPU tests check the reference: its statistics of point values against test_ensemble.stats_ref, and that its bounds
reject four wrong statistics."""
import ctypes as C
import threading

import numpy as np
import pytest

from ensemble_explain_ref import STATS, deltas, member_pair_scores, stat_interval
from out_layer_ref import ACTS, U
from reason_ref import ORDERS, keys, merged_topk
from score_ref import BF16, BF16X2, FP32, FP32_TC, unflatten
from test_ensemble import stats_ref
from test_score_paths import CHUNK, EVAL_ACTS, EVAL_F, EVAL_GAINS, EVAL_HIDDEN, _acts, _model, _rows, _seeded
from test_sensitivity import _planted, chunk_rows

PRECS = {"fp32": FP32, "bf16": BF16, "fp32_tc": FP32_TC, "bf16x2": BF16X2}
F = 37
# one F; different widths, depths and activations (output-layer routes of 1, 2 and 4 chunks in the tensor-core modes)
HETERO = [([33, 1, 100], ["sigmoid", "tanh", "leakyrelu"]), ([300], ["relu"]), ([600, 20], ["tanh", "none"]),
          ([7, 33, 64], ["leakyrelu", "sigmoid", "relu"]), ([40], ["tanh"])]
SENTINEL = 0x7FCDCDCD


def _net(hidden, acts, seed, f=F, gains=None):
    flat = _seeded(f, hidden, gains or (1.4,) * len(hidden) + (4.0,), seed)
    return flat, (unflatten(flat, f, hidden), _acts(acts) + [ACTS["sigmoid"]])


def _ensemble(sb, nets, prec, f=F):
    """nets: [(hidden, acts, flat)] -> an Ensemble"""
    descs = [sb.make_desc(f, h, _acts(a), precision=prec) for h, a, _ in nets]
    return sb.Ensemble.create(descs, [fl for _, _, fl in nets])


def _hetero(K, seed0=100):
    nets, refs = [], []
    for g in range(K):
        h, a = HETERO[g % len(HETERO)]
        flat, ref = _net(h, a, seed0 + g)
        nets.append((h, a, flat))
        refs.append(ref)
    return nets, refs


def _pieces(prec, C):
    """the list positions at which a row chunk's pieces start, and C (score.cu sens_forward)"""
    cp = CHUNK[prec] // chunk_rows(prec, C) - 1
    return list(range(0, C, cp)) + [C]


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("K", [1, 2, 3, 4, 5, 32])
def test_point_values_equal_stats_ref(K):
    rng = np.random.default_rng(K)
    S = rng.random((200, K)).astype(np.float32)
    S[0] = 0.5                                          # all tied
    S[1, : K // 2] = 0.25                               # half tied
    want = stats_ref(S)
    for i, stat in enumerate(STATS):
        c, h = stat_interval(S.T.astype(np.float64), np.zeros(S.T.shape), stat)
        assert np.all(np.abs(want[:, i] - c) <= h), stat
        if stat in ("max", "min") or (stat == "median" and K % 2):
            assert np.array_equal(c, want[:, i].astype(np.float64)), stat


def _rejected(bad, c, h):
    """the share of rows whose wrong value lies outside the interval"""
    return float(np.mean(np.abs(bad - c) > h))


@pytest.mark.parametrize("K", [2, 4, 5])
def test_bounds_reject_wrong_statistics(K):
    """member scores with bounds of a few 1e-7: the right fp32 statistics lie inside every interval, four wrong ones
    outside most"""
    rng = np.random.default_rng(7 + K)
    s = rng.random((K, 500)).astype(np.float32)
    e = np.full(s.shape, 3e-7)
    pair = rng.random((K, 500)).astype(np.float32)
    S, P = stats_ref(s.T), stats_ref(pair.T)
    for i, stat in enumerate(STATS):
        c, h = stat_interval(s, e, stat)
        assert np.all(np.abs(S[:, i] - c) <= h), stat
    c, h = stat_interval(s, e, "mean")
    assert _rejected(s.astype(np.float64).sum(0) / (K - 1), c, h) > 0.99
    c, h = stat_interval(s, e, "max")
    assert _rejected(s[0], c, h) > 0.3
    if K % 2 == 0:
        c, h = stat_interval(s, e, "median")
        assert _rejected(np.sort(s, axis=0)[(K - 1) // 2], c, h) > 0.99
    (d, bd), _ = deltas(((s, e), (pair[:, None, :], e[:, None, :])), "mean")
    assert np.all(np.abs((S[:, 0] - P[:, 0]).astype(np.float64) - d[:, 0]) <= bd[:, 0])
    assert _rejected((s[0] - P[:, 0]).astype(np.float64), d[:, 0], bd[:, 0]) > 0.99


def test_null_handle_and_symbols(sb):
    lib = sb.capi.lib()
    for n in ("sb_ensemble_sensitivity", "sb_ensemble_reason_codes"):
        assert n in sb.capi.PROTOTYPES and hasattr(lib, n)
    X = np.zeros(F, np.float32)
    f64 = C.POINTER(C.c_double)
    s2, s1, ws = np.zeros(1), np.zeros(1), C.c_double()
    for stat in (0, 7):
        assert lib.sb_ensemble_sensitivity(None, stat, X.ctypes.data_as(C.c_void_p), None, 1, None, 0, None,
                                           s2.ctypes.data_as(f64), s1.ctypes.data_as(f64), C.byref(ws), None) == sb.capi.SB_ERR_STATE
        assert "TF ensemble not initialized." in lib.sb_last_error().decode()
        pos, d = np.zeros(4, np.int32), np.zeros(4, np.float32)
        assert lib.sb_ensemble_reason_codes(None, stat, X.ctypes.data_as(C.c_void_p), 1, None, 0, None, 1, 0,
                                            pos.ctypes.data_as(C.c_void_p), d.ctypes.data_as(C.c_void_p), None) == sb.capi.SB_ERR_STATE


# ---------------------------------------------------------------------------------------------------------------- GPU
def _same_sens(a, b, what):
    for key in ("sum_sq", "sum"):
        assert a[key].tobytes() == b[key].tobytes(), (what, key)
    assert np.float64(a["w_sum"]).tobytes() == np.float64(b["w_sum"]).tobytes(), what
    if a["deltas"] is not None or b["deltas"] is not None:
        assert a["deltas"].tobytes() == b["deltas"].tobytes(), (what, "deltas")


def _same_reason(a, b, what):
    assert np.array_equal(a["pos"], b["pos"]), what
    assert a["d"].tobytes() == b["d"].tobytes(), what
    assert a["scores"].tobytes() == b["scores"].tobytes(), what


def _long_list(rng, n):
    """n list positions with repeats and non-zero values (one in five 0)"""
    cols = rng.integers(0, F, n).astype(np.int32)
    vals = rng.standard_normal(n).astype(np.float32)
    vals[::5] = 0.0
    return cols, vals


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PRECS))
def test_one_member_is_the_model(sb, name):
    """K = 1: every stat gives the model's sums, deltas, positions, reason-code deltas and base scores bit for bit, over
    three row chunks of two or more pieces each"""
    prec = PRECS[name]
    rng = np.random.default_rng(1)
    h, a = HETERO[0]
    flat, _ = _net(h, a, 5)
    cols, vals = _long_list(rng, 1100)
    R = chunk_rows(prec, len(cols))
    assert len(_pieces(prec, len(cols))) > 2
    rows = 2 * R + 37
    X = _rows(F, rows, 3)
    w = rng.uniform(0.0, 2.0, rows).astype(np.float32)
    with _model(sb, F, h, a, prec, flat) as m, _ensemble(sb, [(h, a, flat)], prec) as e:
        ms = m.sensitivity(X, w=w, cols=cols, values=vals, deltas=True)
        mr = {o: m.reason_codes(X, 5, cols=cols, values=vals, order=o, scores=True) for o in ORDERS}
        for stat in STATS:
            _same_sens(e.sensitivity(X, w=w, cols=cols, values=vals, deltas=True, stat=stat), ms, stat)
            for o in ORDERS:
                _same_reason(e.reason_codes(X, 5, cols=cols, values=vals, order=o, stat=stat, scores=True), mr[o], (stat, o))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PRECS))
def test_identical_members_are_the_model(sb, name):
    """K copies of one net: max, min and median are the model's bits at K = 2, 3, 5; the mean is at K = 2"""
    prec = PRECS[name]
    rng = np.random.default_rng(2)
    h, a = HETERO[2]
    flat, _ = _net(h, a, 6)
    cols, vals = _long_list(rng, 60)
    rows = chunk_rows(prec, len(cols)) + 13
    X = _rows(F, rows, 4)
    w = rng.uniform(0.0, 2.0, rows).astype(np.float32)
    with _model(sb, F, h, a, prec, flat) as m:
        ms = m.sensitivity(X, w=w, cols=cols, values=vals, deltas=True)
        mr = m.reason_codes(X, 4, cols=cols, values=vals, order="magnitude", scores=True)
        for K in (2, 3, 5):
            with _ensemble(sb, [(h, a, flat)] * K, prec) as e:
                for stat in STATS:
                    if stat == "mean" and K != 2:
                        continue
                    _same_sens(e.sensitivity(X, w=w, cols=cols, values=vals, deltas=True, stat=stat), ms, (K, stat))
                    _same_reason(e.reason_codes(X, 4, cols=cols, values=vals, order="magnitude", stat=stat, scores=True), mr,
                                 (K, stat))


def _check_sens(got, ref, w, what):
    """deltas within their bounds, sums within the sums of their terms' bounds; -> the worst error / bound"""
    (d_ref, e_d), _ = ref
    d = np.asarray(got["deltas"], np.float64)
    err = np.abs(d - d_ref)
    bad = np.argwhere(err > e_d)
    assert bad.size == 0, "%s: %d deltas outside their bound, first (r, k) = %s: %r vs %r (bound %.3g)" % (
        what, len(bad), tuple(bad[0]), d[tuple(bad[0])], d_ref[tuple(bad[0])], e_d[tuple(bad[0])])
    w64 = np.ones(d.shape[0]) if w is None else np.asarray(w, np.float64)
    aw = np.abs(w64)[:, None]
    b1 = (aw * e_d).sum(0)
    assert np.all(np.abs(got["sum"] - (w64[:, None] * d_ref).sum(0)) <= b1 * (1 + 1e-9)), what + ": sum"
    b2 = (aw * e_d * (2 * np.abs(d_ref) + e_d)).sum(0)
    assert np.all(np.abs(got["sum_sq"] - (w64[:, None] * d_ref * d_ref).sum(0)) <= b2 * (1 + 1e-9)), what + ": sum_sq"
    assert got["w_sum"] == pytest.approx(float(w64.sum()), rel=1e-15, abs=0)
    return float(np.max(err / np.maximum(e_d, 1e-300)))


def _check_reason(got, sens_d, ref, k, order, bounds, what):
    """positions = the merged top k of the sensitivity deltas, d bit-identical to them, base scores within their bound, and
    no unselected position certainly beats the k-th under the float64 bounds"""
    p, dd = merged_topk(sens_d, k, order, bounds)
    assert np.array_equal(got["pos"], p), what
    assert got["d"].tobytes() == dd.tobytes(), what
    (d_ref, e_d), (c0, h0) = ref
    assert np.all(np.abs(got["scores"].astype(np.float64) - c0) <= h0), what + ": base scores"
    kd = keys(d_ref, order).astype(np.float64)
    if order == "magnitude":
        lo, hi = np.maximum(kd - e_d, 0.0), kd + e_d
    else:
        lo, hi = kd - e_d, kd + e_d
    rr = np.arange(d_ref.shape[0])[:, None]
    pp = got["pos"].astype(np.int64)
    kth_hi = hi[rr[:, 0], pp[:, -1]]
    unselected = np.ones(d_ref.shape, bool)
    unselected[rr, pp] = False
    assert not (unselected & (lo > kth_hi[:, None])).any(), what + ": an unselected position certainly beats the k-th"


def _explain_case(sb, e, refs, prec, X, w, cols, vals, k, what, plant=None, orders=ORDERS):
    """every stat of one call against the reference; -> the worst delta error / bound"""
    cl = np.arange(X.shape[1], dtype=np.int32) if cols is None else cols
    vl = np.zeros(len(cl), np.float32) if vals is None else vals
    ms = member_pair_scores(X, refs, prec, cl, vl)
    worst = 0.0
    for stat in STATS:
        ref = deltas(ms, stat)
        got = e.sensitivity(X, w=w, cols=cols, values=vals, deltas=True, stat=stat)
        worst = max(worst, _check_sens(got, ref, w, "%s %s" % (what, stat)))
        if plant is not None:
            assert np.all(got["deltas"][plant].view(np.uint32) == 0), "%s %s: planted cells" % (what, stat)
        for o in orders:
            r = e.reason_codes(X, k, cols=cols, values=vals, order=o, stat=stat, scores=True)
            _check_reason(r, got["deltas"], ref, k, o, _pieces(prec, len(cl)), "%s %s %s" % (what, stat, o))
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PRECS))
@pytest.mark.parametrize("K", [2, 3, 4, 5])
def test_heterogeneous_members_against_float64(sb, name, K):
    """one row over every column; a ragged row count in one chunk; two row chunks of several pieces with planted cells"""
    prec = PRECS[name]
    rng = np.random.default_rng(10 + K)
    nets, refs = _hetero(K)
    cols, vals = _long_list(rng, 1100)
    R = chunk_rows(prec, len(cols))
    worst = 0.0
    with _ensemble(sb, nets, prec) as e:
        X = _rows(F, 1, 1) + 0.5
        worst = max(worst, _explain_case(sb, e, refs, prec, X, None, None, None, 3, "%s K=%d one row" % (name, K)))
        c40, v40 = cols[:40], vals[:40]
        X = _rows(F, chunk_rows(prec, 40) - 17, 2)
        w = rng.uniform(0.0, 2.0, len(X)).astype(np.float32)
        worst = max(worst, _explain_case(sb, e, refs, prec, X, w, c40, v40, 5, "%s K=%d ragged" % (name, K), orders=("raise",)))
        X, plant = _planted(_rows(F, R + 5, 3), cols, vals, 3)
        w = rng.uniform(0.0, 2.0, len(X)).astype(np.float32)
        w[::9] = 0.0
        worst = max(worst, _explain_case(sb, e, refs, prec, X, w, cols, vals, 5, "%s K=%d chunks" % (name, K), plant=plant))
    print("%s K=%d: worst delta error / bound %.3g" % (name, K, worst))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["bf16", "fp32_tc"])
def test_eval_shape_every_column(sb, name):
    prec = PRECS[name]
    nets, refs = [], []
    for g in range(2):
        flat, ref = _net(EVAL_HIDDEN, EVAL_ACTS, 7 + g, f=EVAL_F, gains=EVAL_GAINS)
        nets.append((EVAL_HIDDEN, EVAL_ACTS, flat))
        refs.append(ref)
    X = _rows(EVAL_F, 5, 11)
    with _ensemble(sb, nets, prec, f=EVAL_F) as e:
        worst = _explain_case(sb, e, refs, prec, X, None, None, None, 5, "eval " + name, orders=("raise", "magnitude"))
        d = e.sensitivity(X, deltas=True, stat="median")["deltas"]
    assert np.all(d[0].view(np.uint32) == 0)              # row 0 is all zeros: every column already holds 0
    print("eval %s: worst delta error / bound %.3g" % (name, worst))


@pytest.mark.gpu
def test_thirty_two_tiny_members(sb):
    prec = BF16
    hs = [([5], ["tanh"]), ([9, 3], ["relu", "sigmoid"]), ([17], ["leakyrelu"]), ([4, 4], ["none", "tanh"])]
    nets, refs = [], []
    for g in range(sb.capi.ENSEMBLE_MAX):
        h, a = hs[g % len(hs)]
        flat, ref = _net(h, a, 300 + g)
        nets.append((h, a, flat))
        refs.append(ref)
    rng = np.random.default_rng(32)
    cols, vals = _long_list(rng, 45)
    X = _rows(F, 70, 12)
    with _ensemble(sb, nets, prec) as e:
        _explain_case(sb, e, refs, prec, X, None, cols, vals, 4, "K=32", orders=("lower",))


def _dev(torch, n, dtype):
    """a device buffer of n words between 64 sentinel words each side -> (whole buffer, the middle)"""
    buf = torch.empty(n + 128, dtype=torch.int32, device="cuda")
    buf.fill_(SENTINEL)
    return buf, buf[64:64 + n].view(dtype)


def _sentinels_kept(buf):
    b = buf.cpu().numpy().view(np.uint32)
    return np.all(b[:64] == SENTINEL) and np.all(b[-64:] == SENTINEL)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PRECS))
def test_pointers_repeats_and_sentinels(sb, name):
    torch = pytest.importorskip("torch")
    prec = PRECS[name]
    nets, _ = _hetero(3, 40)
    rng = np.random.default_rng(5)
    cols, vals = _long_list(rng, 300)
    rows = 2 * chunk_rows(prec, len(cols)) + 3
    X = _rows(F, rows, 6)
    w = rng.uniform(0.0, 2.0, rows).astype(np.float32)
    C_ = len(cols)
    with _ensemble(sb, nets, prec) as e:
        for stat in ("mean", "median"):
            a = e.sensitivity(X, w=w, cols=cols, values=vals, deltas=True, stat=stat)
            _same_sens(a, e.sensitivity(X, w=w, cols=cols, values=vals, deltas=True, stat=stat), "repeat")
            nod = e.sensitivity(X, w=w, cols=cols, values=vals, stat=stat)
            assert nod["deltas"] is None
            _same_sens(dict(nod, deltas=None), dict(a, deltas=None), "without deltas")
            dX, dw = torch.from_numpy(X).cuda(), torch.from_numpy(w).cuda()
            buf, dd = _dev(torch, rows * C_, torch.float32)
            got = e.sensitivity(dX, w=dw, cols=cols, values=vals, deltas=dd, stat=stat)
            torch.cuda.synchronize()
            _same_sens(dict(got, deltas=None), dict(a, deltas=None), "device")
            assert dd.cpu().numpy().tobytes() == a["deltas"].tobytes() and _sentinels_kept(buf)
            r = e.reason_codes(X, 6, cols=cols, values=vals, order="lower", stat=stat, scores=True)
            _same_reason(r, e.reason_codes(X, 6, cols=cols, values=vals, order="lower", stat=stat, scores=True), "repeat")
            bp, dp = _dev(torch, rows * 6, torch.int32)
            bd, ddd = _dev(torch, rows * 6, torch.float32)
            bs, ds = _dev(torch, rows, torch.float32)
            e.reason_codes(dX, 6, cols=cols, values=vals, order="lower", stat=stat, scores=ds, pos=dp, d=ddd)
            torch.cuda.synchronize()
            assert np.array_equal(dp.cpu().numpy().reshape(rows, 6), r["pos"])
            assert ddd.cpu().numpy().tobytes() == r["d"].tobytes() and ds.cpu().numpy().tobytes() == r["scores"].tobytes()
            assert _sentinels_kept(bp) and _sentinels_kept(bd) and _sentinels_kept(bs)


def _parts(routes):
    return routes.split("+")


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PRECS))
def test_routes(sb, name):
    """one load, every member's z0 GEMM, per member its perturbation, layers and output unit, then the statistic and the
    reduction: each member's launches are the ones its model runs for the same call"""
    prec = PRECS[name]
    nets, _ = _hetero(3, 60)
    rng = np.random.default_rng(9)
    cols, vals = _long_list(rng, 1100)
    X = _rows(F, chunk_rows(prec, len(cols)) + 9, 7)
    z0, piece, load = [], [], None
    for h, a, flat in nets:
        with _model(sb, F, h, a, prec, flat) as m:
            m.sensitivity(X, cols=cols, values=vals)
            p = _parts(m.routes())
        assert p[-1] == "sens_reduce"
        load = p[0]
        z0.append(p[1])
        piece += p[2:-1]
    with _ensemble(sb, nets, prec) as e:
        assert e.routes() == "none"
        e.sensitivity(X, cols=cols, values=vals, stat="max")
        assert e.routes() == "+".join([load] + z0 + piece + ["ensemble_stat", "sens_reduce"])
        e.reason_codes(X, 3, cols=cols, values=vals, stat="min")
        assert e.routes() == "+".join([load] + z0 + piece + ["ensemble_stat", "sens_topk"])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["bf16", "fp32"])
def test_beside_compute_threads(sb, name):
    prec = PRECS[name]
    nets, _ = _hetero(3, 80)
    X = _rows(F, 300, 6)
    with _ensemble(sb, nets, prec) as e:
        solo = e.sensitivity(X, deltas=True, stat="median")
        solo_r = e.reason_codes(X, 5, stat="max", scores=True)
        solo_rows = [e.score_row_f64(X[i].astype(np.float64)).tobytes() for i in range(64)]
        got, errs = {}, []

        def scorer(t):
            try:
                got[t] = [e.score_row_f64(X[i].astype(np.float64)).tobytes() for i in range(64)]
            except Exception as ex:      # noqa: BLE001 - re-raised below
                errs.append(ex)

        ths = [threading.Thread(target=scorer, args=(t,)) for t in range(4)]
        for t in ths:
            t.start()
        busy = [(e.sensitivity(X, deltas=True, stat="median"), e.reason_codes(X, 5, stat="max", scores=True)) for _ in range(3)]
        for t in ths:
            t.join()
        assert not errs, errs
        for s, r in busy:
            _same_sens(s, solo, "busy")
            _same_reason(r, solo_r, "busy")
        for t in range(4):
            assert got[t] == solo_rows


@pytest.mark.gpu
def test_argument_errors_before_device_work(sb):
    nets, _ = _hetero(2, 90)
    lib = sb.capi.lib()
    f64 = C.POINTER(C.c_double)
    X = _rows(F, 4, 1)
    INV = sb.capi.SB_ERR_INVALID
    with _ensemble(sb, nets, BF16) as e:
        def sens(stat=0, X_=X, rows=4, cols=None, n_cols=0, values=None, s2=True):
            a2, a1, w = np.full(64, 7.0), np.full(64, 7.0), C.c_double(7.0)
            cp = None if cols is None else np.ascontiguousarray(cols, np.int32).ctypes.data_as(C.POINTER(C.c_int32))
            vp = None if values is None else np.ascontiguousarray(values, np.float32).ctypes.data_as(C.POINTER(C.c_float))
            st = lib.sb_ensemble_sensitivity(e._h, stat, None if X_ is None else X_.ctypes.data_as(C.c_void_p), None, rows, cp,
                                             n_cols, vp, a2.ctypes.data_as(f64) if s2 else None, a1.ctypes.data_as(f64),
                                             C.byref(w), None)
            return st, (a2, a1, w.value)

        def reason(stat=0, X_=X, rows=4, cols=None, n_cols=0, values=None, k=2, order=0):
            pos, d, s = np.full(64, 7, np.int32), np.full(64, 7.0, np.float32), np.full(8, 7.0, np.float32)
            cp = None if cols is None else np.ascontiguousarray(cols, np.int32).ctypes.data_as(C.POINTER(C.c_int32))
            vp = None if values is None else np.ascontiguousarray(values, np.float32).ctypes.data_as(C.POINTER(C.c_float))
            st = lib.sb_ensemble_reason_codes(e._h, stat, None if X_ is None else X_.ctypes.data_as(C.c_void_p), rows, cp, n_cols,
                                              vp, k, order, pos.ctypes.data_as(C.c_void_p), d.ctypes.data_as(C.c_void_p),
                                              s.ctypes.data_as(C.c_void_p))
            assert np.all(pos == 7) and np.all(d == 7.0) and np.all(s == 7.0)     # nothing written
            return st

        for bad in ({"stat": -1}, {"stat": 4}, {"X_": None}, {"rows": -1}, {"cols": [1, 2], "n_cols": 0}, {"n_cols": 3},
                    {"cols": [1, F], "n_cols": 2}, {"cols": [-1], "n_cols": 1}, {"cols": [3, 4], "n_cols": 2, "values": [1.0, np.nan]}):
            st, outs = sens(**bad)
            assert st == INV, bad
            assert reason(**bad) == INV, bad
        assert sens(s2=False)[0] == INV
        for bad in ({"k": 0}, {"k": 33}, {"k": 3, "cols": [1, 2], "n_cols": 2}, {"order": 3}, {"order": -1}):
            assert reason(**bad) == INV, bad
        reason(stat=4)
        assert "stat = 4" in lib.sb_last_error().decode()
        assert e.routes() == "none"                             # no device work so far
        st, (a2, a1, ws) = sens(rows=0, cols=[3, 5], n_cols=2)
        assert st == sb.capi.SB_OK and np.all(a2[:2] == 0) and np.all(a1[:2] == 0) and ws == 0.0
        assert reason(rows=0) == sb.capi.SB_OK
        assert e.routes() == "none"
        with pytest.raises(ValueError):
            e.sensitivity(X, stat="sum")
        with pytest.raises(ValueError):
            e.reason_codes(X, 2, stat="mode")


@pytest.mark.gpu
def test_scorer_compute_sensitivity_and_reason_codes(sb, tmp_path):
    from shifu_tensorflow_b200 import scorer
    nets, _ = _hetero(3, 120)
    configs = []
    for g, (h, a, flat) in enumerate(nets):
        d = str(tmp_path / ("model%d" % g))
        sb.capi.savedmodel_write(d, sb.make_desc(F, h, _acts(a)), flat)
        configs.append({"inputnames": ["shifu_input_0"],
                        "properties": {"modelpath": d, "outputnames": "shifu_output_0", "tags": ["serve"]}})
    ens = scorer.TensorflowEnsemble()
    ens.init(configs)
    try:
        e = ens._ensemble
        X = _rows(F, 50, 2).astype(np.float64) + 1e-9
        w = np.linspace(0.0, 1.0, 50)
        for stat in STATS:
            r = ens.computeSensitivity(X, weights=w, columns=[4, 1], values=[0.5, -1.0], score=stat)
            want = e.sensitivity(X.astype(np.float32), w=w.astype(np.float32), cols=[4, 1], values=np.array([0.5, -1.0], np.float32),
                                 stat=stat)
            assert r["sum_sq"].tobytes() == want["sum_sq"].tobytes() and r["sum"].tobytes() == want["sum"].tobytes()
            assert r["w_sum"] == want["w_sum"]
            assert np.array_equal(r["mse"], want["sum_sq"] / want["w_sum"]) and np.array_equal(r["mean"], want["sum"] / want["w_sum"])
            rc = ens.computeReasonCodes(X, 2, columns=[30, 2, 17], order="magnitude", score=stat)
            wr = e.reason_codes(X.astype(np.float32), 2, cols=[30, 2, 17], order="magnitude", stat=stat, scores=True)
            assert np.array_equal(rc["columns"], np.array([30, 2, 17], np.int32)[wr["pos"]])
            assert rc["deltas"].tobytes() == wr["d"].tobytes() and rc["scores"].tobytes() == wr["scores"].tobytes()
        for bad in ("sum", 0, None):
            with pytest.raises(ValueError):
                ens.computeSensitivity(X, score=bad)
            with pytest.raises(ValueError):
                ens.computeReasonCodes(X, 2, score=bad)
    finally:
        ens.releaseResource()
