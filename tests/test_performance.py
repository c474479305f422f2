"""Model performance over scored rows (sb_perf_*): exact ROC AUC, average precision, KS and operating points from one
radix sort of the scores on the GPU.

CPU: perf_ref (the header's definitions in float64 and exact integers) against independent computations - scipy's
Mann-Whitney U, O(P N) pair counts, brute-force threshold sweeps - and the C-ABI's argument errors, all found before any
device work.
GPU: the run table, the summary and the points against perf_ref, bit for bit where the header promises exact values and
within perf_ref's derived bounds elsewhere; the eval set's shape (100 M rows); invariance under splitting, pointer kind and
repeats; edge cases and invalid rows; scores straight from sb_model_score_device and an ensemble's outputs; memory."""
import ctypes
import itertools

import numpy as np
import pytest

import perf_ref as pr


def _set(n, seed, ties=None, weights=None, pos=0.3):
    rng = np.random.default_rng(seed)
    y = (rng.random(n) < pos).astype(np.float32)
    s = (rng.standard_normal(n) + 1.2 * y).astype(np.float32)            # logits: negative scores too
    if ties is not None:
        s = np.round(s * ties).astype(np.float32) / np.float32(ties)
    w = None
    if weights == "exact":
        w = rng.choice(np.array([0.0, 1.0, 2.5], np.float32), n)
    elif weights == "random":
        w = rng.random(n).astype(np.float32) * np.float32(3)
    return s, y, w


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_auc_is_mann_whitney_u():
    from scipy.stats import mannwhitneyu
    for seed, ties in ((1, None), (2, 4), (3, 1)):
        s, y, _ = _set(5000, seed, ties)
        r = pr.summary(pr.runs(s, y))
        u = mannwhitneyu(s[y == 1].astype(np.float64), s[y == 0].astype(np.float64)).statistic
        assert abs(r["auc"] - u / (r["pos"] * r["neg"])) < 1e-12


def test_weighted_auc_and_ks_are_pair_counts_and_sweeps():
    for seed, ties in ((4, None), (5, 3)):
        s, y, w = _set(600, seed, ties, weights="random")
        s[:5] = -0.0
        s[5:10] = 0.0
        s[10] = np.inf
        s[11] = -np.inf
        r = pr.runs(s, y, w)
        out = pr.summary(r)
        P, N = s[y == 1].astype(np.float64), s[y == 0].astype(np.float64)
        wP, wN = w[y == 1].astype(np.float64), w[y == 0].astype(np.float64)
        gt = (P[:, None] > N[None, :]) + 0.5 * (P[:, None] == N[None, :])
        assert abs(out["w_auc"] - (wP[:, None] * wN[None, :] * gt).sum() / (wP.sum() * wN.sum())) < 1e-12
        assert abs(out["auc"] - gt.mean()) < 1e-12
        ts = np.unique(s + np.float32(0))[::-1]
        assert np.array_equal(r["t"], ts) and len(ts) < len(s)
        ks, ks_t, wks, ap, wap = -1, None, -1, 0.0, 0.0
        prev_tp = prev_wtp = 0
        for t in ts:                                           # brute-force sweep
            f = s >= t
            tp, fp = int((f & (y == 1)).sum()), int((f & (y == 0)).sum())
            wtp, wfp = float(w[f & (y == 1)].astype(np.float64).sum()), float(w[f & (y == 0)].astype(np.float64).sum())
            d = abs(tp / len(P) - fp / len(N))
            if d > ks + 1e-15:
                ks, ks_t = d, t
            wks = max(wks, abs(wtp / wP.sum() - wfp / wN.sum()))
            ap += (tp - prev_tp) / len(P) * tp / (tp + fp)
            if wtp > prev_wtp:
                wap += (wtp - prev_wtp) / wP.sum() * wtp / (wtp + wfp)
            prev_tp, prev_wtp = tp, wtp
        assert abs(out["ks"] - ks) < 1e-12 and out["ks_score"] == ks_t
        assert abs(out["w_ks"] - wks) < 1e-12
        assert abs(out["ap"] - ap) < 1e-12 and abs(out["w_ap"] - wap) < 1e-12


def test_points_are_sweeps():
    s, y, w = _set(400, 6, 5, weights="exact")
    r = pr.runs(s, y, w)
    levels = [0.0, 0.05, 0.1, 0.5, 0.999, 1.0]
    for axis, weighted in itertools.product(("action_rate", "recall", "fpr"), (False, True)):
        got = pr.points(r, axis, levels, weighted)
        pos = (y == 1)
        wt = w if weighted else np.ones_like(w)
        for lv, (t, tp, fp, _, _) in zip(levels, got):
            num = {"action_rate": lambda f: wt[f].sum(), "recall": lambda f: wt[f & pos].sum(),
                   "fpr": lambda f: wt[f & ~pos].sum()}[axis]
            den = num(np.ones_like(pos))
            ok = [u for u in r["t"] if num(s >= u) / den >= lv]
            assert t == ok[0], (axis, weighted, lv)           # the highest threshold that reaches the level
            assert tp == int(((s >= t) & pos).sum()) and fp == int(((s >= t) & ~pos).sum())
    for lv, (t, tp, fp, _, _) in zip([-np.inf, -1.0, 0.0, 0.5, 100.0], pr.points(r, "score", [-np.inf, -1.0, 0.0, 0.5, 100.0])):
        below = [u for u in r["t"] if u >= lv]
        assert t == (below[-1] if below else np.inf) and tp == int(((s >= t) & (y == 1)).sum())


def test_single_class_and_empty_are_nan():
    s, y, w = _set(50, 7)
    one = pr.summary(pr.runs(s, np.ones_like(y), w))
    assert np.isnan(one["auc"]) and np.isnan(one["ks"]) and one["ap"] == 1.0
    z = pr.summary(pr.runs(s, y, np.zeros_like(s)))
    assert np.isnan(z["w_auc"]) and np.isnan(z["w_ap"]) and not np.isnan(z["auc"])
    e = pr.summary(pr.runs(np.zeros(0, np.float32), np.zeros(0, np.float32)))
    assert e["n_distinct"] == 0 and np.isnan(e["auc"])


def test_symbols_are_bound(sb):
    names = ["sb_perf_create", "sb_perf_destroy", "sb_perf_reset", "sb_perf_add", "sb_perf_summary_get", "sb_perf_points",
             "sb_perf_sync", "sb_perf_stream", "sb_debug_perf_runs", "sb_debug_perf_bytes"]
    lib = sb.capi.lib()
    for n in names:
        assert n in sb.capi.PROTOTYPES and hasattr(lib, n), n
    assert ctypes.sizeof(sb.capi.PerfSummary) == 4 * 8 + 8 * 8 + 8 and ctypes.sizeof(sb.capi.PerfPoint) == 40


def test_argument_errors_without_device_work(sb):
    lib = sb.capi.lib()
    INVALID, STATE = sb.capi.SB_ERR_INVALID, sb.capi.SB_ERR_STATE
    h = ctypes.c_void_p()
    assert lib.sb_perf_create(0, -1, ctypes.byref(h)) == INVALID
    assert lib.sb_perf_create(0, 2**31, ctypes.byref(h)) == INVALID
    assert lib.sb_perf_create(0, 0, None) == INVALID
    x = np.zeros(4, np.float32)
    xp = x.ctypes.data_as(ctypes.c_void_p)
    assert lib.sb_perf_add(None, xp, 1, xp, None, 4, None) == STATE
    assert lib.sb_perf_summary_get(None, ctypes.byref(sb.capi.PerfSummary())) == STATE
    lv = np.zeros(1)
    assert lib.sb_perf_points(None, 0, 0, lv.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), 1,
                              (sb.capi.PerfPoint * 1)()) == STATE
    assert lib.sb_perf_reset(None) == STATE and lib.sb_perf_sync(None) == STATE
    assert lib.sb_debug_perf_runs(None, None, None, None, None, None, 0, ctypes.byref(ctypes.c_int64())) == STATE
    assert lib.sb_debug_perf_bytes(None, ctypes.byref(ctypes.c_int64())) == STATE
    assert b"not initialized" in lib.sb_last_error()
    assert not lib.sb_perf_stream(None) and lib.sb_perf_destroy(None) == sb.capi.SB_OK


def test_no_device_is_a_cuda_error(sb):
    if sb.capi.device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(sb.ShifuB200Error) as e:
        sb.Performance()
    assert e.value.code == sb.capi.SB_ERR_CUDA


# ---------------------------------------------------------------------------------------------------------------- GPU
def _check_runs(got, want, weights_exact=True, n=1):
    np.testing.assert_array_equal(got["t"].view(np.uint32), want["t"].astype(np.float32).view(np.uint32))
    np.testing.assert_array_equal(got["tp"], want["tp"])
    np.testing.assert_array_equal(got["fp"], want["fp"])
    for k in ("w_tp", "w_fp"):
        if weights_exact:
            np.testing.assert_array_equal(got[k].view(np.uint64), want[k].view(np.uint64), err_msg=k)
        else:
            assert (np.abs(got[k] - want[k]) <= pr.weight_bound(n) * want[k]).all(), k
        assert (np.diff(got[k]) >= 0).all(), k                 # the device's cumulative sums never decrease


def _check_summary(got, r, n):
    want = pr.summary(r)
    for k in ("n_distinct", "pos", "neg"):
        assert got[k] == want[k], k
    for k in ("auc", "ks", "ks_score"):                        # exact: same bits (or both NaN)
        assert np.array_equal(np.float64(got[k]), np.float64(want[k]), equal_nan=True), (k, got[k], want[k])
    b = pr.metric_bounds(r, n)
    for k in ("w_auc", "ap", "w_ap", "w_ks"):
        if np.isnan(want[k]):
            assert np.isnan(got[k]), k
        else:
            assert abs(got[k] - want[k]) <= b[k], (k, got[k], want[k], b[k])
    if not np.isnan(want["w_ks"]):                             # the threshold of a maximum within the bound
        wd = np.abs(r["w_tp"] * want["w_neg"] - r["w_fp"] * want["w_pos"]) / (want["w_pos"] * want["w_neg"])
        j = int(np.nonzero(r["t"] == np.float32(got["w_ks_score"]))[0][0])
        assert wd[j] >= want["w_ks"] - b["w_ks"]
    return want


def _check_points(perf, r, n, weighted_exact=True):
    levels = np.array([0.0, 0.1, 0.25, 0.5, 0.75, 0.9, 1.0])
    for axis, wt in itertools.product(("action_rate", "recall", "fpr"), (False, True)):
        got = perf.points(axis, levels, weighted=wt)
        num, den = pr.axis_values(r, axis, wt)
        for i, lv in enumerate(levels):
            j = int(np.nonzero(r["t"] == got["threshold"][i])[0][0])
            if weighted_exact or not wt:
                assert num[j] / den >= lv and (j == 0 or num[j - 1] / den < lv), (axis, wt, lv)
            assert got["tp"][i] == r["tp"][j] and got["fp"][i] == r["fp"][j]
    sl = np.concatenate([[-np.inf, np.inf], r["t"][[0, len(r["t"]) // 2, -1]].astype(np.float64), [r["t"][0] + 1.0]])
    got = perf.points("score", sl)
    for i, (t, tp, fp, _, _) in enumerate(pr.points(r, "score", sl)):
        assert got["threshold"][i] == np.float32(t) and got["tp"][i] == tp and got["fp"][i] == fp


def _summ(p):
    return tuple(np.float64(v).tobytes() for v in p.summary().values())


@pytest.mark.gpu
def test_continuous_scores_at_16m_rows(sb):
    n = 16 * 2**20 + 12345
    s, y, w = _set(n, 11, weights="exact")
    r = pr.runs(s, y, w)
    with sb.Performance() as p:
        p.add(s, y, w)
        _check_runs(p.runs(), r)
        _check_summary(p.summary(), r, n)
        _check_points(p, r, n)
    s2, y2, w2 = _set(n, 12, weights="random")
    r2 = pr.runs(s2, y2, w2)
    with sb.Performance() as p:
        p.add(s2, y2, w2)
        _check_runs(p.runs(), r2, weights_exact=False, n=n)
        _check_summary(p.summary(), r2, n)
        _check_points(p, r2, n, weighted_exact=False)


@pytest.mark.gpu
def test_heavily_tied_scores(sb):
    for n, ties in ((3_000_000, 2), (1_000_003, 64), (70_000, 1000)):
        s, y, w = _set(n, 13 + ties, ties, weights="exact")
        r = pr.runs(s, y, w)
        with sb.Performance() as p:
            p.add(s, y, w)
            _check_runs(p.runs(), r)
            _check_summary(p.summary(), r, n)
            _check_points(p, r, n)


@pytest.mark.gpu
def test_eval_set_shape_100m_rows(sb):
    """100 M rows with scores k / 2^20: the restatement is a bincount over k"""
    n, K = 100_000_000, 2**20
    rng = np.random.default_rng(21)
    k = rng.integers(0, K + 1, n, dtype=np.int64)
    y = (rng.random(n, dtype=np.float32) < (k / K).astype(np.float32)).astype(np.float32)
    s = (k / K).astype(np.float32)
    w = rng.choice(np.array([0.0, 1.0, 2.5], np.float32), n)
    pos = y == 1
    cp = np.bincount(k[pos], minlength=K + 1)[::-1]
    cn = np.bincount(k[~pos], minlength=K + 1)[::-1]
    wp = np.bincount(k[pos], weights=w[pos], minlength=K + 1)[::-1]
    wn = np.bincount(k[~pos], weights=w[~pos], minlength=K + 1)[::-1]
    keep = (cp + cn) > 0
    t = (np.arange(K, -1, -1) / K).astype(np.float32)[keep]
    r = pr.runs_from_counts(t, cp[keep], cn[keep], wp[keep], wn[keep])
    del k
    with sb.Performance(reserve_rows=n) as p:
        p.add(s, y, w)
        _check_runs(p.runs(), r)
        got = _check_summary(p.summary(), r, n)
        _check_points(p, r, n)
        print("100M rows: %d runs, auc %.9f, ks %.9f" % (got["n_distinct"], got["auc"], got["ks"]))


@pytest.mark.gpu
def test_invariance_under_splits_pointers_and_repeats(sb):
    torch = pytest.importorskip("torch")
    n = 3_000_017
    s, y, w = _set(n, 31, 100, weights="random")
    with sb.Performance() as p:
        p.add(s, y, w)
        want_runs, want = p.runs(), _summ(p)
        p.reset()
        p.add(s, y, w)                                         # a repeat after reset
        assert _summ(p) == want
        p.reset()
        cuts = [0, 1, 17, 4096, 1_000_000, 1_000_001, 2_500_000, n]      # 7 uneven calls, a result asked midway
        for a, b in zip(cuts[:-1], cuts[1:]):
            p.add(s[a:b], y[a:b], w[a:b])
            if b == 1_000_000:
                p.summary()
        assert _summ(p) == want
        got = p.runs()
        for key in want_runs:
            np.testing.assert_array_equal(got[key], want_runs[key])
        p.reset()
        for a in range(0, n, 2**20):                           # 1 M-row calls
            p.add(s[a:a + 2**20], y[a:a + 2**20], w[a:a + 2**20])
        assert _summ(p) == want
        p.reset()
        ds, dy, dw = (torch.from_numpy(a).cuda() for a in (s, y, w))
        torch.cuda.synchronize()
        p.add_device(ds.data_ptr(), dy.data_ptr(), dw.data_ptr(), n)
        assert _summ(p) == want
        p.reset()
        p.add_device(ds.data_ptr(), y.ctypes.data, dw.data_ptr(), n)   # mixed: the staged path
        assert _summ(p) == want
    with sb.Performance(reserve_rows=n) as q:                  # a second handle
        q.add(s, y, w)
        assert _summ(q) == want


@pytest.mark.gpu
def test_edges(sb):
    with sb.Performance() as p:
        e = p.summary()
        assert e["rows"] == 0 and e["n_distinct"] == 0 and np.isnan(e["auc"]) and np.isnan(e["w_ks"])
        assert p.points("score", [0.5])["threshold"][0] == np.inf
        with pytest.raises(sb.ShifuB200Error) as err:
            p.points("recall", [0.5])
        assert err.value.code == sb.capi.SB_ERR_INVALID
        y = np.array([0, 1, 1, 0, 1, 0], np.float32)
        p.add(np.full(6, 0.25, np.float32), y)
        r = p.summary()
        assert r["auc"] == 0.5 and r["ks"] == 0.0 and r["n_distinct"] == 1
        p.reset()
        s = np.array([0.0, -0.0, np.inf, -np.inf, 1e-45, -1e-45, 1e-40, -3.0, 2.0, 0.0], np.float32)
        yy = np.array([1, 0, 1, 0, 1, 0, 1, 0, 0, 1], np.float32)
        p.add(s, yy)
        got = p.runs()
        want = pr.runs(s, yy)
        np.testing.assert_array_equal(got["t"].view(np.uint32), want["t"].view(np.uint32))
        np.testing.assert_array_equal(got["t"], s[[2, 8, 6, 4, 0, 5, 7, 3]])
        assert got["t"][4].view(np.uint32) == 0                     # +0, not -0
        assert got["tp"][4] == 5 and got["fp"][4] == 2              # +0 and -0 in one run of three rows
        _check_summary(p.summary(), want, len(s))
        p.reset()
        p.add(s, np.ones_like(s), np.zeros_like(s))                 # one class, zero total weight
        r = p.summary()
        assert np.isnan(r["auc"]) and np.isnan(r["ks"]) and np.isnan(r["w_auc"]) and np.isnan(r["w_ap"]) and r["ap"] == 1.0
        with pytest.raises(sb.ShifuB200Error):
            p.points("fpr", [0.5])
        with pytest.raises(sb.ShifuB200Error):
            p.points("recall", [0.5], weighted=True)
        p.points("recall", [0.5])


@pytest.mark.gpu
def test_invalid_rows_are_counted_until_reset(sb):
    lib = sb.capi.lib()
    with sb.Performance() as p:
        s = np.array([0.1, np.nan, 0.3, 0.4, 0.5, 0.6, np.nan], np.float32)
        y = np.array([0, 1, 0.5, -0.0, 2, 1, 1], np.float32)
        w = np.array([1, 1, 1, -1, np.inf, np.nan, -0.0], np.float32)
        p.add(s, y, w)
        for call in (p.summary, lambda: p.points("score", [0.5]), p.runs):
            with pytest.raises(sb.ShifuB200Error) as e:
                call()
            assert e.value.code == sb.capi.SB_ERR_INVALID
            assert "2 with a NaN score, 2 with a label other than 0 or 1, 3 with a negative or non-finite weight" in str(e.value)
        p.reset()
        p.add(s[[0, 3]], y[[0, 3]])                                 # -0 is a valid label
        assert p.summary()["neg"] == 2
        lv = np.array([np.nan])
        for axis, level in ((0, np.nan), (1, 1.5), (2, -0.1), (3, np.nan), (4, 0.5)):
            lv[0] = level
            assert lib.sb_perf_points(p._h, axis, 0, lv.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), 1,
                                      (sb.capi.PerfPoint * 1)()) == sb.capi.SB_ERR_INVALID, (axis, level)
        x = np.zeros(4, np.float32)
        xp = x.ctypes.data_as(ctypes.c_void_p)
        assert lib.sb_perf_add(p._h, xp, 0, xp, None, 4, None) == sb.capi.SB_ERR_INVALID
        assert lib.sb_perf_add(p._h, xp, 1, xp, None, -1, None) == sb.capi.SB_ERR_INVALID
        assert lib.sb_perf_add(p._h, None, 1, xp, None, 4, None) == sb.capi.SB_ERR_INVALID
        assert lib.sb_perf_add(p._h, xp, 1, xp, None, 2**31 - 2, None) == sb.capi.SB_ERR_INVALID   # 2 rows held
        assert lib.sb_perf_add(p._h, xp, 1, xp, None, 0, None) == sb.capi.SB_OK
        assert p.summary()["rows"] == 2


@pytest.mark.gpu
def test_model_scores_added_behind_the_model_stream(sb):
    torch = pytest.importorskip("torch")
    from oracle import shifu_oracle as so
    F, hidden = 2000, [1024, 512, 256]
    desc = sb.make_desc(F, hidden, [so.ACT_RELU] * 3, precision=sb.PREC_BF16)
    rng = np.random.default_rng(41)
    parts, prev = [], F
    for h in hidden + [1]:
        parts += [rng.standard_normal((prev, h)).astype(np.float32) * np.float32(1.5 / np.sqrt(prev)),
                  rng.standard_normal(h).astype(np.float32) * np.float32(0.1)]
        prev = h
    flat = np.concatenate([a.ravel() for a in parts])
    n = 200_000
    X = torch.randn(n, F, device="cuda", generator=torch.Generator("cuda").manual_seed(3))
    y = (torch.rand(n, device="cuda", generator=torch.Generator("cuda").manual_seed(4)) < 0.4).float()
    out = torch.full((n,), float("nan"), device="cuda")
    torch.cuda.synchronize()
    with sb.Model.create(desc, flat) as m, sb.Performance() as p:
        m.score_device(X.data_ptr(), n, out.data_ptr())
        p.add_device(out.data_ptr(), y.data_ptr(), None, n, after_stream=m.stream)   # no host synchronise in between
        got = _summ(p)
        m.sync()
        host = out.cpu().numpy()
        p.reset()
        p.add(host, y.cpu().numpy())
        assert _summ(p) == got
        assert not np.isnan(p.summary()["auc"])


@pytest.mark.gpu
def test_ensemble_columns_in_place_and_scorers(sb, tmp_path):
    torch = pytest.importorskip("torch")
    from shifu_tensorflow_b200 import scorer
    from oracle import shifu_oracle as so
    F = 37
    nets = [(F, [64, 16], [so.ACT_RELU, so.ACT_TANH]), (F, [300], [so.ACT_SIGMOID]), (F, [20], [so.ACT_LEAKYRELU])]
    configs, descs, flats = [], [], []
    for g, (f, h, a) in enumerate(nets):
        rng = np.random.default_rng(50 + g)
        parts, prev = [], f
        for hh in h + [1]:
            parts += [rng.standard_normal((prev, hh)).astype(np.float32) * np.float32(1.5 / np.sqrt(prev)),
                      rng.standard_normal(hh).astype(np.float32) * np.float32(0.1)]
            prev = hh
        flats.append(np.concatenate([x.ravel() for x in parts]))
        descs.append(sb.make_desc(f, h, a))
        d = str(tmp_path / ("model%d" % g))
        sb.capi.savedmodel_write(d, descs[-1], flats[-1])
        configs.append({"inputnames": ["shifu_input_0"],
                        "properties": {"modelpath": d, "outputnames": "shifu_output_0", "tags": ["serve"]}})
    n = 50_000
    rng = np.random.default_rng(60)
    X = rng.standard_normal((n, F)).astype(np.float32)
    y = (rng.random(n) < 0.3).astype(np.float32)
    w = rng.choice(np.array([0.0, 1.0, 2.5], np.float32), n)
    K = len(nets)
    with sb.Ensemble.create(descs, flats) as e, sb.Performance() as p:
        dX = torch.from_numpy(X).cuda()
        dS = torch.empty((n, K), device="cuda")
        dT = torch.empty((n, 4), device="cuda")
        dy, dw = torch.from_numpy(y).cuda(), torch.from_numpy(w).cuda()
        torch.cuda.synchronize()
        e.score_device(dX.data_ptr(), n, dS.data_ptr(), dT.data_ptr())
        S, T = e.score(X)
        for base, col, stride, host in [(dT, 0, 4, T[:, 0]), (dT, 3, 4, T[:, 3]), (dS, 1, K, S[:, 1])]:
            p.reset()
            p.add_device(base.data_ptr() + 4 * col, dy.data_ptr(), dw.data_ptr(), n, stride=stride, after_stream=e.stream)
            got = _summ(p)
            p.reset()
            p.add(np.ascontiguousarray(host), y, w)
            assert _summ(p) == got, (col, stride)
    ens = scorer.TensorflowEnsemble()
    ens.init(configs)
    for score, col in (("mean", None), ("median", None), (2, 2)):
        res = ens.computePerformance(X, y, w, buckets=10, score=score)
        _, T = ens._ensemble.score(X)
        sc = ens.computeBatch(X)["scores"][:, col].astype(np.float32) if col is not None else \
            T[:, sb.capi.ENSEMBLE_STATS.index(score)]
        r = pr.runs(sc, y, w)
        _check_summary(res["summary"], r, n)
        _check_tables(res, r)
    ens.releaseResource()
    m = scorer.TensorflowModel()
    m.init(configs[0])
    res = m.computePerformance(X.astype(np.float64), y, w, buckets=20)
    r = pr.runs(m.computeBatch(X).astype(np.float32), y, w)
    _check_summary(res["summary"], r, n)
    _check_tables(res, r, buckets=20)
    assert "weighted_gains" not in m.computePerformance(X, y)
    m.releaseResource()


def _check_tables(res, r, buckets=10):
    levels = np.arange(1, buckets + 1) / buckets
    s = pr.summary(r)
    for w in (False, True):
        for name, axis in (("gains", "action_rate"), ("roc", "fpr"), ("pr", "recall")):
            tab = res[("weighted_" if w else "") + name]
            want = pr.points(r, axis, levels, weighted=w)
            assert [np.float32(x[0]) for x in want] == list(tab["threshold"]), (name, w)
            assert [x[1] for x in want] == list(tab["tp"])
            P, N = (s["w_pos"], s["w_neg"]) if w else (s["pos"], s["neg"])
            tp = tab["w_tp"] if w else tab["tp"]
            fp = tab["w_fp"] if w else tab["fp"]
            np.testing.assert_allclose(tab["recall"], tp / P, rtol=1e-12)
            np.testing.assert_allclose(tab["lift"], tp / (tp + fp) / (P / (P + N)), rtol=1e-12)


@pytest.mark.gpu
def test_memory_within_the_header_bound(sb):
    fixed = 13 * 2**20
    with sb.Performance() as p:
        base = p.device_bytes()
        assert base < 2**20
        n = 5_000_000
        s, y, _ = _set(n, 71)
        p.add(s, y)
        p.summary()
        cap = 1.5 * n + 4096
        assert p.device_bytes() <= 53 * cap + fixed, (p.device_bytes(), cap)
    with sb.Performance(reserve_rows=n) as q:
        q.add(s, y)
        q.summary()
        b = q.device_bytes()
        assert b <= 53 * (n + 4096) + fixed and b >= 52 * n, b
        print("bytes per row held (every score distinct): %.2f" % ((b - 12 * 2**20) / n))
