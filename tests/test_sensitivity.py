"""Column sensitivity (sb_model_sensitivity, Model.sensitivity) against float64.

Every pair score s_k(r) is held to its bound from sensitivity_ref.py, every returned delta to the sum of its two scores'
bounds, in all four precision modes: on the eval net (2000 columns, [1024, 512, 256], relu, seeded as test_score_paths
seeds it) over every column of 48 rows, and on the small net of test_score_paths (37 -> [33, 1, 100]) over every row and
column.  Besides the bounds: exact +0 deltas where a cell already holds the value, fp64 sums against the float64 sums of
the returned deltas, bit-identical repeats across host / device pointers and with / without deltas, calls beside
compute() threads, the launches of each precision, and argument errors reported before any device work.

The CPU tests check the reference itself: its rank-1 path against brute-force re-scoring of modified rows."""
import ctypes as C
import threading

import numpy as np
import pytest

from out_layer_ref import ACTS, U
from score_ref import BF16, BF16X2, FP32, FP32_TC, unflatten
from sensitivity_ref import brute_scores, pair_scores, rank1_scores
from test_out_layer import expected_route
from test_score_paths import (CHUNK, EVAL_ACTS, EVAL_F, EVAL_GAINS, EVAL_HIDDEN, SMALL_ACTS, SMALL_F, SMALL_HIDDEN, _acts,
                              _device_sms, _model, _rows, _seeded, _wide)

PRECS = {"fp32": FP32, "bf16": BF16, "fp32_tc": FP32_TC, "bf16x2": BF16X2}
NPARTS = {FP32: 1, BF16: 1, FP32_TC: 3, BF16X2: 2}


def chunk_rows(prec, n_cols):
    """rows per row chunk (score.cu sens_chunk_rows)"""
    mb = CHUNK[prec]
    return min(mb // 2, max(64, mb // (n_cols + 1)))


def _next_prime(n):
    n += 1
    while any(n % p == 0 for p in range(2, int(n ** 0.5) + 1)):
        n += 1
    return n


def expected_sens_routes(prec, F, hidden, rows, n_cols, sms):
    """the launches of a call's last row chunk's z0 and last piece (score.cu sens_forward)"""
    R = chunk_rows(prec, n_cols)
    rc = rows - R * ((rows - 1) // R)
    cp = CHUNK[prec] // R - 1
    ck = n_cols - cp * ((n_cols - 1) // cp)
    pairs = rc * (ck + 1)
    r = ["load_batch<fp32>" if prec == FP32 else "load_batch<bf16>"]
    r.append("gemm_f32<FWD>" if prec == FP32 else "gemm_tc<%d,F32>" % (64 if hidden[0] <= 64 else 128))
    r.append({FP32: "sens_perturb<fp32>", BF16: "sens_perturb<bf16>", FP32_TC: "sens_perturb<bf16x3>",
              BF16X2: "sens_perturb<bf16x2>"}[prec])
    K = hidden[0]
    for N in hidden[1:]:
        if prec == FP32:
            r.append("gemm_f32<FWD>")
        elif prec == BF16:
            r.append("gemm_wide" if _wide(pairs, N, K, sms) else "gemm_pp<FWD>")
        else:
            r.append("gemm_tc<%d,FWD,GENERIC>" % (64 if N <= 64 else 128))
        K = N
    r.append(expected_route(prec, hidden[-1], False, "score"))
    return "+".join(r + ["sens_reduce"])


# ------------------------------------------------------------------ the reference (CPU)
@pytest.mark.parametrize("hidden,acts", [([9, 7], ["sigmoid", "tanh"]), ([9, 7], ["relu", "leakyrelu"]), ([8, 5], ["none", "relu"]),
                                         ([6, 1, 4], ["tanh", "sigmoid", "leakyrelu"])])
@pytest.mark.parametrize("prec", [FP32, BF16])
def test_reference_rank1_equals_brute_force(hidden, acts, prec):
    F = 11
    rng = np.random.default_rng(3)
    layers = unflatten(_seeded(F, hidden, [1.5] * (len(hidden) + 1), 5), F, hidden)
    X = rng.standard_normal((13, F)).astype(np.float32)
    cols = [0, 10, 4, 4, 7]
    values = rng.standard_normal(len(cols)).astype(np.float32)
    a = _acts(acts) + [ACTS["sigmoid"]]
    r1 = rank1_scores(X, layers, a, prec, cols, values)
    bf = brute_scores(X, layers, a, prec, cols, values)
    assert np.max(np.abs(r1 - bf)) <= 1e-12
    if prec == FP32:     # the bounded path carries the exact model's values
        (_, _), (s, _) = pair_scores(X, layers, a, prec, cols, values, block=2)
        assert np.max(np.abs(s - r1)) <= 1e-12


def test_null_model_is_state_error(sb):
    lib = sb.capi.lib()
    X = np.zeros(4, np.float32)
    s2, s1, ws = np.zeros(1), np.zeros(1), C.c_double()
    f64 = C.POINTER(C.c_double)
    st = lib.sb_model_sensitivity(None, X.ctypes.data_as(C.c_void_p), None, 1, None, 0, None, s2.ctypes.data_as(f64),
                                  s1.ctypes.data_as(f64), C.byref(ws), None)
    assert st == sb.capi.SB_ERR_STATE
    assert "TF model not initialized." in lib.sb_last_error().decode()


# ------------------------------------------------------------------ the GPU path
def _check_call(got, X, w, layers, acts, prec, cols, values, what):
    """deltas and sums of one call against the reference (module docstring); -> the worst error / bound"""
    d = np.asarray(got["deltas"], np.float64)                       # [rows, K]
    (s0, e0), (s, e) = pair_scores(X, layers, acts, prec, cols, values)
    d_ref = s0[None, :] - s                                         # [K, rows]
    e_d = e0[None, :] + e + U * np.abs(d_ref)
    err = np.abs(d.T - d_ref)
    bad = np.argwhere(err > e_d)
    assert bad.size == 0, "%s: %d deltas outside their bound, first (k, r) = %s: %r vs %r (bound %.3g)" % (
        what, len(bad), tuple(bad[0]), d.T[tuple(bad[0])], d_ref[tuple(bad[0])], e_d[tuple(bad[0])])
    w64 = np.ones(X.shape[0]) if w is None else np.asarray(w, np.float64)
    # fixed-order fp64 sums against float64 sums of the returned deltas, relative to the sum of magnitudes
    for key, terms in (("sum_sq", w64[:, None] * d * d), ("sum", w64[:, None] * d)):
        mag = np.abs(terms).sum(0)
        assert np.all(np.abs(got[key] - terms.sum(0)) <= 1e-12 * mag + 1e-300), (what, key)
    assert got["w_sum"] == pytest.approx(float(w64.sum()), rel=1e-15, abs=0)
    # against the exact sums, within the propagated bound
    ex1 = (w64[None, :] * d_ref).sum(1)
    b1 = (np.abs(w64)[None, :] * e_d).sum(1)
    assert np.all(np.abs(got["sum"] - ex1) <= b1 * (1 + 1e-9)), what
    ex2 = (w64[None, :] * d_ref * d_ref).sum(1)
    b2 = (np.abs(w64)[None, :] * e_d * (2 * np.abs(d_ref) + e_d)).sum(1)
    assert np.all(np.abs(got["sum_sq"] - ex2) <= b2 * (1 + 1e-9)), what
    return float(np.max(err / np.maximum(e_d, 1e-300)))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PRECS))
def test_eval_net_every_column(sb, name):
    prec = PRECS[name]
    flat = _seeded(EVAL_F, EVAL_HIDDEN, EVAL_GAINS, 7)
    layers = unflatten(flat, EVAL_F, EVAL_HIDDEN)
    acts = _acts(EVAL_ACTS) + [ACTS["sigmoid"]]
    X = _rows(EVAL_F, 48, 11)
    with _model(sb, EVAL_F, EVAL_HIDDEN, EVAL_ACTS, prec, flat) as m:
        got = m.sensitivity(X, deltas=True)
        routes = m.routes()
    cols = np.arange(EVAL_F)
    r = _check_call(got, X, None, layers, acts, prec, cols, np.zeros(EVAL_F, np.float32), "eval " + name)
    print("eval net %s: worst delta error / bound %.3g" % (name, r))
    # row 0 is all zeros: every column already holds 0
    assert np.all(got["deltas"][0].view(np.uint32) == 0)
    assert routes == expected_sens_routes(prec, EVAL_F, EVAL_HIDDEN, 48, EVAL_F, _device_sms())


def _small(sb, prec):
    flat = _seeded(SMALL_F, SMALL_HIDDEN, (1.4, 1.4, 1.4, 4.0), 9)
    return flat, unflatten(flat, SMALL_F, SMALL_HIDDEN), _acts(SMALL_ACTS) + [ACTS["sigmoid"]]


def _planted(X, cols, values, seed):
    """cells where X already holds the value: a few random ones per position, and -0 against a +0 value"""
    rng = np.random.default_rng(seed)
    X = X.copy()
    plant = np.zeros((X.shape[0], len(cols)), bool)
    for k, c in enumerate(cols):
        rs = rng.choice(X.shape[0], size=min(3, X.shape[0]), replace=False)
        X[rs, c] = values[k]
        if values[k] == 0:
            X[rs[:1], c] = np.float32(-0.0)
    for k, c in enumerate(cols):
        plant[:, k] = X[:, c] == values[k]
    return X, plant


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PRECS))
@pytest.mark.parametrize("cols_kind", ["one", "all", "list"])
def test_small_net_rows_and_columns(sb, name, cols_kind):
    prec = PRECS[name]
    flat, layers, acts = _small(sb, prec)
    rng = np.random.default_rng(21)
    cols = {"one": np.array([5], np.int32), "all": None,
            "list": np.array([30, 2, 17, 2, 36, 0, 30, 9], np.int32)}[cols_kind]
    cl = np.arange(SMALL_F, dtype=np.int32) if cols is None else cols
    values = None if cols_kind == "all" else rng.standard_normal(len(cl)).astype(np.float32)
    vl = np.zeros(len(cl), np.float32) if values is None else values
    if cols_kind == "list":
        vl[1] = 0.0
        values = vl
    R = chunk_rows(prec, len(cl))
    sms = _device_sms()
    with _model(sb, SMALL_F, SMALL_HIDDEN, SMALL_ACTS, prec, flat) as m:
        for rows in (1, _next_prime(R), 2 * R + 77):
            X, plant = _planted(_rows(SMALL_F, rows, rows), cl, vl, rows)
            w = rng.uniform(0.0, 2.0, rows).astype(np.float32)
            w[rng.random(rows) < 0.1] = 0.0
            got = m.sensitivity(X, w=w, cols=cols, values=values, deltas=True)
            assert m.routes() == expected_sens_routes(prec, SMALL_F, SMALL_HIDDEN, rows, len(cl), sms)
            _check_call(got, X, w, layers, acts, prec, cl, vl, "small %s %s rows=%d" % (name, cols_kind, rows))
            # exact +0 where the cell already holds the value
            assert np.all(got["deltas"][plant].view(np.uint32) == 0), "planted cells"


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PRECS))
def test_repeat_pointers_and_weights(sb, name):
    torch = pytest.importorskip("torch")
    prec = PRECS[name]
    flat, _, _ = _small(sb, prec)
    R = chunk_rows(prec, SMALL_F)
    rows = 2 * R + 5
    X = _rows(SMALL_F, rows, 4)
    rng = np.random.default_rng(8)
    w = rng.uniform(0.0, 2.0, rows).astype(np.float32)
    w[::7] = 0.0
    X[::7] = 1e3 * X[::7]          # zero-weight rows with wild scores add nothing
    vals = rng.standard_normal(SMALL_F).astype(np.float32)

    def bits(r):
        return [np.asarray(r[k]).tobytes() for k in ("sum_sq", "sum")] + [np.float64(r["w_sum"]).tobytes()]

    with _model(sb, SMALL_F, SMALL_HIDDEN, SMALL_ACTS, prec, flat) as m:
        a = m.sensitivity(X, w=w, values=vals, deltas=True)
        b = m.sensitivity(X, w=w, values=vals, deltas=True)
        c = m.sensitivity(X, w=w, values=vals)
        assert bits(a) == bits(b) == bits(c)
        assert a["deltas"].tobytes() == b["deltas"].tobytes()
        dX, dw = torch.from_numpy(X).cuda(), torch.from_numpy(w).cuda()
        dd = torch.full((rows, SMALL_F), float("nan"), dtype=torch.float32, device="cuda")
        e = m.sensitivity(dX, w=dw, values=vals, deltas=dd)
        torch.cuda.synchronize()
        assert bits(e) == bits(a)
        assert dd.cpu().numpy().tobytes() == a["deltas"].tobytes()
        ones = m.sensitivity(X, w=np.ones(rows, np.float32), values=vals)
        none = m.sensitivity(X, values=vals)
        assert bits(ones) == bits(none)
        # zero-weight rows: the same sums as the fp64 sums over the weighted rows only
        d = a["deltas"].astype(np.float64)
        keep = w != 0
        w64 = w.astype(np.float64)
        for key, t in (("sum_sq", w64[keep, None] * d[keep] ** 2), ("sum", w64[keep, None] * d[keep])):
            assert np.all(np.abs(a[key] - t.sum(0)) <= 1e-12 * np.abs(t).sum(0) + 1e-300), key
        assert np.all(np.isfinite(a["sum_sq"]))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["bf16", "fp32"])
def test_beside_compute_threads(sb, name):
    prec = PRECS[name]
    flat, _, _ = _small(sb, prec)
    X = _rows(SMALL_F, 300, 6)
    with _model(sb, SMALL_F, SMALL_HIDDEN, SMALL_ACTS, prec, flat) as m:
        solo = m.sensitivity(X, deltas=True)
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
        busy = [m.sensitivity(X, deltas=True) for _ in range(3)]
        for t in ths:
            t.join()
        assert not errs, errs
        for r in busy:
            assert r["deltas"].tobytes() == solo["deltas"].tobytes()
            assert r["sum_sq"].tobytes() == solo["sum_sq"].tobytes() and r["sum"].tobytes() == solo["sum"].tobytes()
        for t in range(4):
            assert got[t] == solo_rows


@pytest.mark.gpu
def test_argument_errors_before_device_work(sb):
    flat, _, _ = _small(sb, BF16)
    lib = sb.capi.lib()
    f64 = C.POINTER(C.c_double)
    X = _rows(SMALL_F, 4, 1)
    with _model(sb, SMALL_F, SMALL_HIDDEN, SMALL_ACTS, BF16, flat) as m:
        def call(X_=X, rows=4, cols=None, n_cols=0, values=None, s2=True, s1=True, ws=True):
            a2, a1, w = np.full(64, 7.0), np.full(64, 7.0), C.c_double(7.0)
            cp = None if cols is None else np.ascontiguousarray(cols, np.int32).ctypes.data_as(C.POINTER(C.c_int32))
            vp = None if values is None else np.ascontiguousarray(values, np.float32).ctypes.data_as(C.POINTER(C.c_float))
            st = lib.sb_model_sensitivity(m._h, None if X_ is None else X_.ctypes.data_as(C.c_void_p), None, rows, cp, n_cols, vp,
                                          a2.ctypes.data_as(f64) if s2 else None, a1.ctypes.data_as(f64) if s1 else None,
                                          C.byref(w) if ws else None, None)
            return st, a2, a1, w.value

        INV = sb.capi.SB_ERR_INVALID
        assert call(X_=None)[0] == INV
        assert call(s2=False)[0] == INV and call(s1=False)[0] == INV and call(ws=False)[0] == INV
        assert call(cols=[1, 2], n_cols=0)[0] == INV            # a list without a length
        assert call(cols=None, n_cols=3)[0] == INV              # a length without a list
        assert call(cols=[1, SMALL_F], n_cols=2)[0] == INV
        assert call(cols=[-1], n_cols=1)[0] == INV
        assert call(cols=[3, 4], n_cols=2, values=[1.0, np.nan])[0] == INV
        assert call(cols=[3], n_cols=1, values=[np.inf])[0] == INV
        assert call(rows=-1)[0] == INV
        assert m.routes() == "none"                             # no device work so far
        st, a2, a1, ws = call(rows=0, cols=[3, 5], n_cols=2)
        assert st == sb.capi.SB_OK and np.all(a2[:2] == 0) and np.all(a1[:2] == 0) and ws == 0.0
        assert m.routes() == "none"


@pytest.mark.gpu
def test_scorer_compute_sensitivity(sb):
    from shifu_tensorflow_b200 import scorer
    flat, _, _ = _small(sb, FP32)
    X = _rows(SMALL_F, 50, 2).astype(np.float64) + 1e-9          # doubles, cast to float as computeBatch casts them
    w = np.linspace(0.0, 1.0, 50)
    with _model(sb, SMALL_F, SMALL_HIDDEN, SMALL_ACTS, FP32, flat) as m:
        tm = scorer.TensorflowModel.__new__(scorer.TensorflowModel)
        tm.initiate, tm._model = True, m
        r = tm.computeSensitivity(X, weights=w, columns=[4, 1], values=[0.5, -1.0])
        want = m.sensitivity(X.astype(np.float32), w=w.astype(np.float32), cols=[4, 1], values=np.array([0.5, -1.0], np.float32))
        assert r["sum_sq"].tobytes() == want["sum_sq"].tobytes() and r["sum"].tobytes() == want["sum"].tobytes()
        assert r["w_sum"] == want["w_sum"]
        assert np.array_equal(r["mse"], want["sum_sq"] / want["w_sum"]) and np.array_equal(r["mean"], want["sum"] / want["w_sum"])
