"""Bagged-model scoring (sb_ensemble_*): K member models scored from one staged copy of the rows, with each row's mean,
max, min and median formed on the GPU.

- Each member's scores equal, bit for bit, what an sb_model_t of the same member computes from the same rows
  (score / score_device), in every precision mode, for eval nets and for a mixed set of small nets.
- The statistics equal stats_ref, a numpy float32 restatement of the header's definitions, bit for bit.
- The launches of a chunk: one load, each member's own launches without the load, then ensemble_stats.
- compute() calls from many threads give the bits of score(); the ensemble allocates one input staging.
The CPU tests check the argument errors (all found before any device work), the missing-device error and the reference
itself."""
import ctypes
import os
import threading

import numpy as np
import pytest

from oracle import shifu_oracle as so

SIG, TANH, RELU, LEAKY, NONE = so.ACT_SIGMOID, so.ACT_TANH, so.ACT_RELU, so.ACT_LEAKYRELU, -1
MODES = [0, 1, 2, 3]        # PREC_FP32, PREC_BF16, PREC_FP32_TC, PREC_BF16X2
QNAN = 0x7FC00000
EVAL = (2000, [1024, 512, 256], [RELU] * 3)
# one F, different widths, depths and activations (output-layer routes 1, 2 and 4 chunks in the tensor-core modes)
MIXED = [(37, [7, 33, 1, 100], [SIG, TANH, RELU, LEAKY]), (37, [300], [RELU]), (37, [600, 20], [TANH, NONE]),
         (37, [1000, 64, 8], [LEAKY, SIG, RELU])]
# activations that carry a NaN input through to the score
STATS_NETS = [(37, [7, 33], [SIG, TANH]), (37, [300], [TANH]), (37, [600, 20], [TANH, NONE]), (37, [100, 64], [SIG, NONE])]


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def stats_ref(S):
    """[rows, K] member scores -> [rows, 4] = mean, max, min, median as include/shifu_b200.h defines them, in float32"""
    S = np.ascontiguousarray(S, np.float32)
    K = S.shape[1]
    s, mx, mn = S[:, 0].copy(), S[:, 0].copy(), S[:, 0].copy()
    for g in range(1, K):
        s = (s + S[:, g]).astype(np.float32)
        mx = np.where(S[:, g] > mx, S[:, g], mx)
        mn = np.where(S[:, g] < mn, S[:, g], mn)
    mean = (s / np.float32(K)).astype(np.float32)
    srt = np.take_along_axis(S, np.argsort(S, axis=1, kind="stable"), axis=1)
    lo, hi = (K - 1) // 2, K // 2
    med = srt[:, lo] if lo == hi else ((srt[:, lo] + srt[:, hi]) * np.float32(0.5)).astype(np.float32)
    out = np.stack([mean, mx, mn, med], axis=1).astype(np.float32)
    out.view(np.uint32)[np.isnan(S).any(axis=1)] = QNAN
    return out


def _flat(F, hidden, seed):
    """seeded weights of ~ unit-variance activations (scores spread over (0, 1))"""
    rng = np.random.default_rng(seed)
    parts, prev = [], F
    for h in list(hidden) + [1]:
        parts.append(rng.standard_normal((prev, h)).astype(np.float32) * np.float32(1.5 / np.sqrt(prev)))
        parts.append(rng.standard_normal(h).astype(np.float32) * np.float32(0.1))
        prev = h
    return np.concatenate([p.ravel() for p in parts])


def _members(sb, nets, precision, seed0):
    descs = [sb.make_desc(F, h, a, precision=precision) for F, h, a in nets]
    flats = [_flat(F, h, seed0 + g) for g, (F, h, a) in enumerate(nets)]
    return descs, flats


def _rows(F, n, seed):
    X = np.random.default_rng(seed).standard_normal((n, F)).astype(np.float32)
    X[0] = -0.0
    if n > 2:
        X[2, ::3] = 0.0
    return X


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_stats_ref_matches_a_plain_sort():
    rng = np.random.default_rng(0)
    for K in (1, 2, 3, 4, 5, 32):
        S = rng.random((50, K)).astype(np.float32)
        S[0] = 0.5                                   # all tied
        S[1, : K // 2] = 0.25                        # half tied
        got = stats_ref(S)
        for r in range(len(S)):
            v = sorted(float(x) for x in S[r])
            med = v[(K - 1) // 2] if K % 2 else float((np.float32(v[K // 2 - 1]) + np.float32(v[K // 2])) * np.float32(0.5))
            assert got[r, 1] == max(v) and got[r, 2] == min(v) and got[r, 3] == np.float32(med)
            assert abs(got[r, 0] - np.mean(S[r].astype(np.float64))) <= 1e-6
    S = np.array([[0.1, np.nan, 0.3]], np.float32)
    assert (_bits(stats_ref(S)) == QNAN).all()


def test_ensemble_symbols_are_bound(sb):
    names = ["sb_ensemble_load", "sb_ensemble_create", "sb_ensemble_destroy", "sb_ensemble_size", "sb_ensemble_score",
             "sb_ensemble_score_device", "sb_ensemble_score_row_f64", "sb_ensemble_sync", "sb_ensemble_stream",
             "sb_debug_ensemble_routes", "sb_debug_ensemble_bytes", "sb_debug_model_bytes"]
    lib = sb.capi.lib()
    for n in names:
        assert n in sb.capi.PROTOTYPES and hasattr(lib, n), n
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "shifu_b200.h")).read()
    assert "#define SB_ENSEMBLE_MAX %d" % sb.capi.ENSEMBLE_MAX in hdr


def _create_raw(sb, descs, flats, k=None, n_params=None):
    lib = sb.capi.lib()
    k = len(descs) if k is None else k
    n = max(len(descs), 1)
    d_arr = (sb.NetDesc * n)(*descs)
    f_arr = (ctypes.POINTER(ctypes.c_float) * n)(*[f.ctypes.data_as(ctypes.POINTER(ctypes.c_float)) for f in flats])
    n_arr = (ctypes.c_int64 * n)(*(n_params if n_params is not None else [f.size for f in flats]))
    h = ctypes.c_void_p()
    return lib.sb_ensemble_create(d_arr, f_arr, n_arr, k, 0, ctypes.byref(h)), h


def test_create_argument_errors_without_device_work(sb):
    """every check is made before a device is looked at: without a GPU the call would otherwise fail with SB_ERR_CUDA"""
    lib = sb.capi.lib()
    INVALID = sb.capi.SB_ERR_INVALID
    descs, flats = _members(sb, MIXED[:2], 0, 1)
    assert _create_raw(sb, descs, flats, k=0)[0] == INVALID
    assert b"outside [1, 32]" in lib.sb_last_error()
    many_d, many_f = _members(sb, [MIXED[1]] * 33, 0, 1)
    assert _create_raw(sb, many_d, many_f)[0] == INVALID
    other_f = sb.make_desc(38, [7], [RELU])
    assert _create_raw(sb, [descs[0], other_f], [flats[0], _flat(38, [7], 0)])[0] == INVALID
    assert b"features" in lib.sb_last_error()
    other_p = sb.make_desc(37, [300], [RELU], precision=sb.PREC_BF16)
    assert _create_raw(sb, [descs[0], other_p], flats)[0] == INVALID
    assert b"precision" in lib.sb_last_error()
    assert _create_raw(sb, descs, flats, n_params=[flats[0].size, flats[1].size - 1])[0] == INVALID
    bad = sb.make_desc(37, [0], [RELU])
    assert _create_raw(sb, [descs[0], bad], [flats[0], flats[1]])[0] == INVALID
    h = ctypes.c_void_p()
    d_arr = (sb.NetDesc * 2)(*descs)
    assert lib.sb_ensemble_create(None, None, None, 2, 0, ctypes.byref(h)) == INVALID
    f_null = (ctypes.POINTER(ctypes.c_float) * 2)(flats[0].ctypes.data_as(ctypes.POINTER(ctypes.c_float)), None)
    n_arr = (ctypes.c_int64 * 2)(flats[0].size, flats[1].size)
    assert lib.sb_ensemble_create(d_arr, f_null, n_arr, 2, 0, ctypes.byref(h)) == INVALID
    assert lib.sb_ensemble_create(d_arr, f_null, n_arr, 2, 0, None) == INVALID


def test_load_argument_errors_without_device_work(sb, tmp_path):
    lib = sb.capi.lib()
    dirs = []
    for g, (F, h, a) in enumerate([(37, [7], [RELU]), (37, [9, 3], [TANH, SIG]), (38, [7], [RELU])]):
        d = str(tmp_path / ("model%d" % g))
        sb.capi.savedmodel_write(d, sb.make_desc(F, h, a), _flat(F, h, g))
        dirs.append(d)

    def load(ds, k=None, inp=b"shifu_input_0", out=b"shifu_output_0", tag=b"serve"):
        arr = (ctypes.c_char_p * max(len(ds), 1))(*[d if d is None else d.encode() for d in ds])
        h = ctypes.c_void_p()
        return lib.sb_ensemble_load(arr, len(ds) if k is None else k, inp, out, tag, 0, 0, ctypes.byref(h))

    INVALID = sb.capi.SB_ERR_INVALID
    assert load(dirs[:2], k=0) == INVALID
    assert load(dirs[:2], k=33) == INVALID
    assert lib.sb_ensemble_load(None, 2, b"a", b"b", b"serve", 0, 0, ctypes.byref(ctypes.c_void_p())) == INVALID
    assert load(dirs) == INVALID and b"features" in lib.sb_last_error()
    # a member's load errors are sb_model_load's, code and message
    for args in (dict(inp=None), dict(out=b""), dict(tag=None)):
        code = load(dirs[:2], **args)
        msg = lib.sb_last_error()
        h = ctypes.c_void_p()
        a = dict(dict(inp=b"shifu_input_0", out=b"shifu_output_0", tag=b"serve"), **args)
        assert lib.sb_model_load(dirs[0].encode(), a["inp"], a["out"], a["tag"], 0, 0, ctypes.byref(h)) == code == INVALID
        assert lib.sb_last_error() == msg
    missing = str(tmp_path / "missing")
    code = load([dirs[0], missing])
    msg = lib.sb_last_error()
    assert code == lib.sb_model_load(missing.encode(), b"shifu_input_0", b"shifu_output_0", b"serve", 0, 0,
                                     ctypes.byref(ctypes.c_void_p())) != sb.capi.SB_OK
    assert lib.sb_last_error() == msg
    code = load(["", dirs[0]])
    assert code == INVALID and b"Model path is null" in lib.sb_last_error()


def test_null_handle_is_a_state_error(sb):
    lib = sb.capi.lib()
    STATE = sb.capi.SB_ERR_STATE
    x = np.zeros((1, 4), np.float32)
    o = np.zeros(8, np.float32)
    xp, op = x.ctypes.data_as(ctypes.c_void_p), o.ctypes.data_as(ctypes.c_void_p)
    assert lib.sb_ensemble_score(None, xp, 1, op, op) == STATE
    assert lib.sb_ensemble_score_device(None, xp, 1, op, op) == STATE
    r = np.zeros(4)
    out = np.zeros(8)
    assert lib.sb_ensemble_score_row_f64(None, r.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), 4,
                                         out.ctypes.data_as(ctypes.POINTER(ctypes.c_double))) == STATE
    assert lib.sb_ensemble_sync(None) == STATE
    assert lib.sb_debug_ensemble_routes(None, ctypes.create_string_buffer(16), 16) == STATE
    assert lib.sb_debug_ensemble_bytes(None, ctypes.byref(ctypes.c_int64())) == STATE
    assert lib.sb_debug_model_bytes(None, ctypes.byref(ctypes.c_int64())) == STATE
    assert b"not initialized" in lib.sb_last_error()
    assert lib.sb_ensemble_size(None) == 0 and not lib.sb_ensemble_stream(None)
    assert lib.sb_ensemble_destroy(None) == sb.capi.SB_OK


def test_no_device_is_a_cuda_error(sb):
    if sb.capi.device_count() > 0:
        pytest.skip("a GPU is present")
    descs, flats = _members(sb, MIXED, 0, 1)
    with pytest.raises(sb.ShifuB200Error) as e:
        sb.Ensemble.create(descs, flats)
    assert e.value.code == sb.capi.SB_ERR_CUDA


# ---------------------------------------------------------------------------------------------------------------- GPU
def _check_against_models(sb, e, models, X, device=False):
    """scores bit-identical to each member model's, stats to stats_ref of them"""
    s, t = e.score(X)
    for g, m in enumerate(models):
        want = m.score(X)
        np.testing.assert_array_equal(_bits(s[:, g]), _bits(want), err_msg="member %d, %d rows" % (g, len(X)))
    np.testing.assert_array_equal(_bits(t), _bits(stats_ref(s)), err_msg="stats, %d rows" % len(X))
    if device:
        torch = pytest.importorskip("torch")
        dX = torch.from_numpy(X).cuda()
        dS = torch.full((len(X), e.k), float("nan"), device="cuda")
        dT = torch.full((len(X), 4), float("nan"), device="cuda")
        dO = torch.full((len(X),), float("nan"), device="cuda")
        torch.cuda.synchronize()
        e.score_device(dX.data_ptr(), len(X), dS.data_ptr(), dT.data_ptr())
        e.sync()
        np.testing.assert_array_equal(_bits(dS.cpu().numpy()), _bits(s))
        np.testing.assert_array_equal(_bits(dT.cpu().numpy()), _bits(t))
        for g, m in enumerate(models):
            m.score_device(dX.data_ptr(), len(X), dO.data_ptr())
            m.sync()
            np.testing.assert_array_equal(_bits(dS[:, g].cpu().numpy()), _bits(dO.cpu().numpy()), err_msg="device member %d" % g)
    return s, t


def _route_parts(r):
    return r.split("+")


def _check_routes(sb, e, models, rows, precision):
    er = e.routes()
    if precision == sb.PREC_FP32 and rows <= sb.capi.SMALL_ROWS:
        assert er == "+".join(["score_rows"] * len(models) + ["ensemble_stats"]), er
        return
    load = "load_batch<bf16>" if precision != sb.PREC_FP32 else "load_batch<fp32>"
    want = [load]
    for m in models:
        mr = _route_parts(m.routes())
        assert mr[0] == load
        want += mr[1:]
    assert er == "+".join(want + ["ensemble_stats"]), er


@pytest.mark.gpu
@pytest.mark.parametrize("precision", MODES)
def test_members_match_their_models_bit_for_bit(sb, precision):
    chunk = sb.capi.MODEL_CHUNK_ROWS[precision]
    for name, nets, counts in (("eval", [EVAL] * 5, (1, 128, 129, 2 * chunk + 777)),
                               ("mixed", MIXED, (1, 128, 129, 2 * chunk + 4099))):
        descs, flats = _members(sb, nets, precision, 10)
        models = [sb.Model.create(d, f) for d, f in zip(descs, flats)]
        try:
            with sb.Ensemble.create(descs, flats) as e:
                assert e.k == len(nets)
                X_all = _rows(nets[0][0], max(counts), 3)
                for c in counts:
                    _check_against_models(sb, e, models, X_all[:c], device=c in (129, max(counts)))
                    tail = (c - 1) % chunk + 1                  # the rows of the call's last chunk
                    for m in models:
                        m.score(X_all[:tail])                   # the member's own launches at that row count
                    _check_routes(sb, e, models, tail, precision)
                print("%s precision %d: %d members bit-identical at %s rows" % (name, precision, len(nets), counts))
        finally:
            for m in models:
                m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("precision", [0, 1])
def test_statistics_restate_bit_for_bit(sb, precision):
    F = 37
    X = _rows(F, 3000, 5)
    X[7, 4] = np.nan                                # this row's scores are NaN in every member
    for K in (1, 2, 3, 4, 5, 32):
        nets = [STATS_NETS[g % len(STATS_NETS)] for g in range(K)]
        descs, flats = _members(sb, nets, precision, 100 + K)
        if K >= 4:                                  # members 1 and 3 repeat member 0: tied scores on every row
            flats[1] = flats[0].copy(); descs[1] = descs[0]
            flats[3] = flats[0].copy(); descs[3] = descs[0]
        with sb.Ensemble.create(descs, flats) as e:
            for rows in (1, 100, 3000):
                s, t = e.score(X[:rows])
                np.testing.assert_array_equal(_bits(t), _bits(stats_ref(s)), err_msg="K=%d rows=%d" % (K, rows))
                if K == 1:                          # each statistic is the score (a NaN score: the quiet NaN)
                    ok = ~np.isnan(s[:, 0])
                    np.testing.assert_array_equal(_bits(t[ok]), _bits(np.repeat(s[ok], 4, axis=1)))
                    assert (_bits(t[~ok]) == QNAN).all()
                s2, _ = e.score(X[:rows], stats=False)
                _, t2 = e.score(X[:rows], scores=False)
                np.testing.assert_array_equal(_bits(s2), _bits(s))
                np.testing.assert_array_equal(_bits(t2), _bits(t))
            assert np.isnan(s[7]).any() and (_bits(t[7]) == QNAN).all()
            assert not np.isnan(t[8]).any()
            if K >= 4:
                assert (_bits(s[:, 1]) == _bits(s[:, 0])).all() and (_bits(s[:, 3]) == _bits(s[:, 0])).all()


@pytest.mark.gpu
def test_errors_and_empty_calls_on_a_live_handle(sb):
    descs, flats = _members(sb, MIXED, 0, 1)
    with sb.Ensemble.create(descs, flats) as e:
        lib = sb.capi.lib()
        x = np.zeros((2, 37), np.float32)
        xp = x.ctypes.data_as(ctypes.c_void_p)
        out = np.full((2, 8), 7, np.float32)
        assert lib.sb_ensemble_score(e._h, xp, 2, None, None) == sb.capi.SB_ERR_INVALID
        assert lib.sb_ensemble_score(e._h, None, 2, out.ctypes.data_as(ctypes.c_void_p), None) == sb.capi.SB_ERR_INVALID
        assert lib.sb_ensemble_score(e._h, xp, -1, out.ctypes.data_as(ctypes.c_void_p), None) == sb.capi.SB_ERR_INVALID
        assert lib.sb_ensemble_score_device(e._h, xp, 2, None, None) == sb.capi.SB_ERR_INVALID
        assert lib.sb_ensemble_score(e._h, xp, 0, out.ctypes.data_as(ctypes.c_void_p), None) == sb.capi.SB_OK
        assert (out == 7).all()
        assert e.routes() == "none"
        with pytest.raises(sb.ShifuB200Error) as err:
            e.score_row_f64(np.zeros(36))
        assert err.value.code == sb.capi.SB_ERR_INVALID and "expected 37 features" in str(err.value)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", MODES)
def test_compute_calls_from_many_threads(sb, precision):
    F = 120
    nets = [(F, [64, 300, 32], [RELU, TANH, SIG]), (F, [200], [LEAKY]), (F, [30, 30], [RELU, NONE])]
    descs, flats = _members(sb, nets, precision, 40)
    n_threads, per = 64, 40
    X = np.random.default_rng(6).standard_normal((n_threads * per, F))     # float64: compute() casts to float32
    X32 = X.astype(np.float32)
    with sb.Ensemble.create(descs, flats) as e:
        want_s = np.concatenate([e.score(X32[i:i + 128])[0] for i in range(0, len(X), 128)])
        want_t = stats_ref(want_s)
        lone = e.score_row_f64(X[0])                # a lone call returns at once
        np.testing.assert_array_equal(lone[:3], want_s[0].astype(np.float64))
        got = np.full((len(X), 3 + 4), np.nan)
        errs, short = [], []
        go = threading.Barrier(n_threads + 1)

        def rows(t):
            try:
                go.wait()
                for i in range(t * per, (t + 1) * per):
                    got[i] = e.score_row_f64(X[i])
            except Exception as ex:     # noqa: BLE001 - surfaced below
                errs.append(ex)

        def bad():
            go.wait()
            try:
                e.score_row_f64(X[0][:F - 1])
            except sb.ShifuB200Error as ex:
                short.append(ex)

        th = [threading.Thread(target=rows, args=(t,)) for t in range(n_threads)] + [threading.Thread(target=bad)]
        [t.start() for t in th]; [t.join() for t in th]
        assert not errs, errs
        assert len(short) == 1 and short[0].code == sb.capi.SB_ERR_INVALID
        np.testing.assert_array_equal(_bits(got[:, :3].astype(np.float32)), _bits(want_s))
        np.testing.assert_array_equal(_bits(got[:, 3:].astype(np.float32)), _bits(want_t))


@pytest.mark.gpu
def test_one_input_staging_per_ensemble(sb):
    """at the eval net in bf16, each added member costs less than one input staging (stX fp32 + Xb bf16 rows)"""
    F, hidden, acts = EVAL
    chunk = sb.capi.MODEL_CHUNK_ROWS[sb.PREC_BF16]
    staging = chunk * F * 4 + chunk * F * 2
    descs, flats = _members(sb, [EVAL] * 5, sb.PREC_BF16, 70)
    sizes = []
    for k in (1, 2, 5):
        with sb.Ensemble.create(descs[:k], flats[:k]) as e:
            sizes.append(e.device_bytes())
    with sb.Model.create(descs[0], flats[0]) as m:
        model = m.device_bytes()
    per_member = (sizes[2] - sizes[0]) / 4
    assert sizes[1] - sizes[0] < staging and per_member < staging, (sizes, staging)
    assert sizes[2] < 5 * model - 4 * staging + 5 * chunk * 4 * 3, (sizes, model)
    print("bytes: model %.0f MB; ensemble of 1 / 2 / 5: %.0f / %.0f / %.0f MB; input staging %.0f MB" %
          (model / 2**20, sizes[0] / 2**20, sizes[1] / 2**20, sizes[2] / 2**20, staging / 2**20))


@pytest.mark.gpu
def test_scorer_ensemble(sb, tmp_path):
    from shifu_tensorflow_b200 import scorer
    configs = []
    for g, (F, h, a) in enumerate(MIXED):
        d = str(tmp_path / ("model%d" % g))
        sb.capi.savedmodel_write(d, sb.make_desc(F, h, a), _flat(F, h, 200 + g))
        configs.append({"inputnames": ["shifu_input_0"],
                        "properties": {"modelpath": d, "outputnames": "shifu_output_0", "tags": ["serve"]}})
    ens = scorer.TensorflowEnsemble()
    with pytest.raises(scorer.IllegalStateException):
        ens.compute(np.zeros(37))
    with pytest.raises(RuntimeError, match="Model path is null"):
        scorer.TensorflowEnsemble().init([configs[0], {"inputnames": ["x"], "properties": {"outputnames": "y", "tags": ["s"]}}])
    with pytest.raises(scorer.IllegalArgumentException):
        bad = dict(configs[1], inputnames=["shifu_input_0", "keras_learning_phase"])
        bad["properties"] = dict(configs[1]["properties"], keras_learning_phase=True)
        scorer.TensorflowEnsemble().init([configs[0], bad])
    ens.init(configs)
    X = np.random.default_rng(9).standard_normal((300, 37))
    batch = ens.computeBatch(X)
    models = []
    for c in configs:
        m = scorer.TensorflowModel()
        m.init(c)
        models.append(m)
    for g, m in enumerate(models):
        np.testing.assert_array_equal(batch["scores"][:, g], m.computeBatch(X))
        m.releaseResource()
    one = ens.compute(X[5])
    np.testing.assert_array_equal(one["scores"], batch["scores"][5])
    for name in ("mean", "max", "min", "median"):
        assert one[name] == batch[name][5]
    ens.releaseResource()
    with pytest.raises(scorer.IllegalStateException):
        ens.computeBatch(X)
