"""Batch scoring against float64 through the entry points bench.py and the JVM use: Model.score_device, Model.score (from
pageable and from pinned host rows), Model.score_row_f64 (compute()), and the trainer's validation pass (Trainer.eval_loss,
Trainer.predict), in every precision mode.

Every score is held to its row's bound from score_ref.py: the exact model with the contraction and rounding bounds of the
step's GEMMs in FP32 / FP32_TC / BF16X2, and in BF16 the same roundings the kernels make (bf16 inputs, bf16 W shadows,
activations stored as bf16), so that most of a BF16 row's elements are known exactly and only the others carry a bound.
FP32 and FP32_TC eval-net scores are also held to the 1e-5 score contract against the exact model.  A model runs a call in forwards of at most max_batch rows (MODEL_CHUNK_ROWS: 65 536 in bf16, 32 768 in the split
modes, 16 384 in fp32); the row counts put several of them in one call, with a ragged tail, so that an offset wrong on
the second and later forwards is caught.  The eval net (2000 columns, [1024, 512, 256], relu, as bench.py scores it) is
checked on 128 rows each side of every forward's boundary and 2048 random rows; the small nets on every row.

sb_debug_model_routes names the launches of a model's last forward: every case asserts them, and the cases together
reach every forward and output-layer instantiation a score can launch."""
import zlib

import numpy as np
import pytest

from out_layer_ref import ACTS
from score_ref import BF16, BF16X2, FP32, FP32_TC, hidden_forward, score, unflatten, validation_loss
from test_out_layer import _depth, expected_route

PRECS = {"fp32": FP32, "bf16": BF16, "fp32_tc": FP32_TC, "bf16x2": BF16X2}
CHUNK = {FP32: 16384, BF16: 65536, FP32_TC: 32768, BF16X2: 32768}     # _capi.MODEL_CHUNK_ROWS
ACT_CYCLE = ["relu", "tanh", "sigmoid", "leakyrelu", "none"]
SMALL_ROWS = 128

EVAL_F, EVAL_HIDDEN, EVAL_ACTS = 2000, [1024, 512, 256], ["relu"] * 3
EVAL_ROWS = 2 * 65536 + 4099            # three bf16 forwards, five split-mode forwards, nine fp32 forwards
EVAL_GAINS = (1.4, 1.4, 1.4, 4.0)       # the seeded set: scores spread over (0, 1), some saturate
SMALL_F, SMALL_HIDDEN, SMALL_ACTS = 37, [33, 1, 100], ["sigmoid", "tanh", "leakyrelu"]
SENTINEL = 0x7FCDCDCD                   # a quiet NaN nothing computes

_worst = {}
_notes = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if _worst:
        print("\nworst error / bound: " + ", ".join("%s %.3g" % (p, _worst[p]) for p in PRECS if p in _worst))
    for k in sorted(_notes):
        print("%s: %s" % (k, _notes[k]))


def _name(prec):
    return [k for k, v in PRECS.items() if v == prec][0]


def _check(got, want, prec, what):
    """scores got [M] against the reference (y_hat, bound) [M]: every row within its bound"""
    yh, e = want
    err = np.abs(np.asarray(got, np.float64) - yh)
    r = float(np.max(err / e))
    _worst[_name(prec)] = max(_worst.get(_name(prec), 0.0), r)
    bad = np.flatnonzero(err > e)
    assert bad.size == 0, "%s: %d rows off, first row %d: %r vs %r (bound %.3g), worst %.3g x its bound" % (
        what, bad.size, bad[0], got[bad[0]], yh[bad[0]], e[bad[0]], r)
    return err


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _seeded(F, hidden, gains, seed):
    """a flat parameter vector: W_l ~ N(0, 1) gain_l / sqrt(in), b_l ~ N(0, 0.1^2)"""
    rng = np.random.default_rng(seed)
    parts, prev = [], F
    for h, g in zip(list(hidden) + [1], gains):
        parts.append(rng.standard_normal((prev, h)).astype(np.float32) * np.float32(g / np.sqrt(prev)))
        parts.append((rng.standard_normal(h) * 0.1).astype(np.float32))
        prev = h
    return np.concatenate([p.ravel() for p in parts])


def _wide(M, N, K, sms):
    """gemm_pp.cuh plan_gemm_pp(fwd = true) picks the 128x256 tile"""
    tiles_m, kb = -(-M // 128), -(-K // 64)
    wide, narrow = tiles_m * -(-N // 256), tiles_m * -(-N // 128)
    return N > 128 and 8 * wide >= 7 * sms and kb >= 16 and 2 * -(-wide // sms) <= -(-narrow // sms)


def expected_routes(prec, F, hidden, rows, sms):
    """the launches of a model's forward of `rows` rows (score.cu ScoreCore::forward, Net::enqueue_*)"""
    if prec == FP32 and rows <= SMALL_ROWS:
        return "score_rows"
    r = ["load_batch<fp32>" if prec == FP32 else "load_batch<bf16>"]
    K = F
    for N in hidden:
        if prec == FP32:
            r.append("gemm_f32<FWD>")
        elif prec == BF16:
            r.append("gemm_wide" if _wide(rows, N, K, sms) else "gemm_pp<FWD>")
        else:
            r.append("gemm_tc<%d,FWD,GENERIC>" % (64 if N <= 64 else 128))
        K = N
    return "+".join(r + [expected_route(prec, hidden[-1], False, "score")])


def _last_piece(prec, rows):
    return rows - CHUNK[prec] * ((rows - 1) // CHUNK[prec])


_sms = []


def _device_sms():
    if not _sms:
        import torch
        _sms.append(torch.cuda.get_device_properties(0).multi_processor_count)
    return _sms[0]


def _acts(names):
    return [ACTS[a] for a in names]


def _model(sb, F, hidden, acts, prec, flat):
    return sb.Model.create(sb.make_desc(F, hidden, _acts(acts), precision=prec), flat)


def _rows(F, n, seed):
    X = np.clip(np.random.default_rng(seed).standard_normal((n, F), dtype=np.float32), -4, 4)
    X[0] = 0.0                  # a zero row and a sparse row
    X[min(2, n - 1), ::3] = 0.0
    return X


# ------------------------------------------------------------------------------------------------------ the eval net
@pytest.fixture(scope="module")
def eval_params(sb):
    """the two weight sets of the eval net: 'trained' (the cfg2 net after 8 bf16 run_resident steps on the planted set
    test_benchmarked_paths.py trains on, as bench.py scores a trained net) and 'seeded' (EVAL_GAINS)"""
    from test_benchmarked_paths import _batches, _setup
    c, _, _, (X, y, w), t = _setup(sb, "cfg2", sb.PREC_BF16)
    assert c["F"] == EVAL_F and c["hidden"] == EVAL_HIDDEN
    t.run_resident([o for o, _ in _batches(c, X, y, w, 8)], c["batch"])
    trained = t.get_params()
    t.close()
    return {"trained": trained, "seeded": _seeded(EVAL_F, EVAL_HIDDEN, EVAL_GAINS, 21)}


@pytest.fixture(scope="module")
def eval_rows(sb):
    """EVAL_ROWS rows on the device as bench.py makes them (N(0, 1) clipped to +-4), followed by 64 NaN rows; the sampled
    rows (128 each side of every forward boundary of every precision, 2048 random rows, the last rows) on the host"""
    torch = pytest.importorskip("torch")
    N, F = EVAL_ROWS, EVAL_F
    buf = torch.full(((N + 64) * F,), float("nan"), dtype=torch.float32, device="cuda")
    g = torch.Generator(device="cuda")
    g.manual_seed(17)
    buf[:N * F].normal_(generator=g).clamp_(-4, 4)
    X = buf[:N * F].view(N, F)
    X[0] = 0.0
    idx = set(range(N - 128, N))
    for b in range(16384, N, 16384):
        idx |= set(range(b - 128, b + 128))
    idx |= set(np.random.default_rng(3).choice(N, 2048, replace=False).tolist())
    idx = np.array(sorted(idx))
    Xs = X[torch.from_numpy(idx).cuda()].cpu().numpy()
    torch.cuda.synchronize()
    return buf, idx, Xs


_eval_cache = {}


def _eval_scores(sb, eval_params, eval_rows, wset, prec):
    """score_device of every eval row into a buffer with 64 sentinel words each side; the sentinels keep their bits and
    the NaN rows behind the last row change no score.  A second call of one full forward gives that forward's bits and
    routes.  -> (scores [EVAL_ROWS], routes at a full forward)"""
    key = (wset, prec)
    if key in _eval_cache:
        return _eval_cache[key]
    import torch
    buf, _, _ = eval_rows
    N = EVAL_ROWS
    out = torch.empty(N + 128, dtype=torch.float32, device="cuda")
    out.view(torch.int32).fill_(SENTINEL)
    with _model(sb, EVAL_F, EVAL_HIDDEN, EVAL_ACTS, prec, eval_params[wset]) as m:
        torch.cuda.synchronize()
        m.score_device(buf.data_ptr(), N, out.data_ptr() + 64 * 4)
        m.sync()
        assert m.routes() == expected_routes(prec, EVAL_F, EVAL_HIDDEN, _last_piece(prec, N), _device_sms())
        got = out.cpu().numpy()
        c = CHUNK[prec]
        one = torch.empty(c, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        m.score_device(buf.data_ptr(), c, one.data_ptr())
        m.sync()
        routes = m.routes()
        np.testing.assert_array_equal(_bits(one.cpu().numpy()), _bits(got[64:64 + c]))
    w = got.view(np.uint32)
    assert (w[:64] == SENTINEL).all() and (w[64 + N:] == SENTINEL).all(), "a word outside dOut changed"
    scores = got[64:64 + N]
    assert np.isfinite(scores).all()
    _eval_cache[key] = (scores, routes)
    return _eval_cache[key]


@pytest.mark.gpu
@pytest.mark.parametrize("prec", sorted(PRECS))
@pytest.mark.parametrize("wset", ["trained", "seeded"])
def test_eval_net_at_bench_scale(sb, eval_params, eval_rows, wset, prec):
    p = PRECS[prec]
    scores, routes = _eval_scores(sb, eval_params, eval_rows, wset, p)
    assert routes == expected_routes(p, EVAL_F, EVAL_HIDDEN, CHUNK[p], _device_sms())
    if p == BF16 and _device_sms() == 132:      # the benchmarked plan on an H100 SXM
        assert routes == "load_batch<bf16>+gemm_wide+gemm_wide+gemm_pp<FWD>+out_layer_rows<1>"
    _, idx, Xs = eval_rows
    layers = unflatten(eval_params[wset], EVAL_F, EVAL_HIDDEN)
    exact = []
    want = score(Xs, layers, _acts(EVAL_ACTS), p, exact)
    got = scores[idx]
    err = _check(got, want, p, "eval net %s %s" % (wset, prec))
    if wset == "seeded":
        s = scores.astype(np.float64)
        assert s.min() < 1e-3 and s.max() > 1 - 1e-5 and np.mean((s > 0.1) & (s < 0.9)) > 0.2, "scores do not spread"
    if p != BF16:       # the reference value is the exact model
        dev = float(err.max())
        _notes["eval %s %s max |score - float64|" % (wset, prec)] = "%.3g" % dev
        # the 1e-5 score contract of the fp32 modes.  BF16X2 meets it on the trained net (3.5e-6 on an H100) but not on
        # the seeded one (2.4e-5: larger weights, saturating scores), so it is held to its bound alone (DESIGN §3)
        if p in (FP32, FP32_TC):
            assert dev <= 1e-5
    else:
        _notes["eval %s bf16 elements known exactly per layer" % wset] = ", ".join("%.4f" % f for f in exact)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["bf16", "fp32_tc"])
def test_eval_bound_catches_wrong_parameters(sb, eval_params, eval_rows, prec):
    """the checks are not vacuous: the reference of slightly wrong parameters misses the kernels' scores on rows the
    change affects.  W_0's last input row left out (a dropped K tail) falls outside the bound; a layer-0 bias element
    moved by one bf16 ulp falls outside fp32_tc's 1e-5 contract (in bf16 its rows are only reported)"""
    p = PRECS[prec]
    scores, _ = _eval_scores(sb, eval_params, eval_rows, "seeded", p)
    _, idx, Xs = eval_rows
    layers = unflatten(eval_params["seeded"], EVAL_F, EVAL_HIDDEN)
    acts = _acts(EVAL_ACTS)
    W0, b0 = layers[0]
    j = int(np.argmax(np.abs(b0)))
    b1 = b0.copy()
    b1[j] = np.float32(b0[j] + np.sign(b0[j]) * 2.0 ** (np.floor(np.log2(abs(b0[j]))) - 7))
    W1 = W0.copy()
    W1[-1] = 0.0
    for what, wrong in (("bias_ulp", [(W0, b1)] + layers[1:]), ("k_tail", [(W1, b0)] + layers[1:])):
        yh, e = score(Xs, wrong, acts, p)
        d = np.abs(scores[idx] - yh)
        n_bound, n_contract = int(np.sum(d > e)), int(np.sum(d > 1e-5))
        _notes["%s %s: rows outside the bound / the 1e-5 contract" % (prec, what)] = "%d / %d of %d" % (
            n_bound, n_contract, len(idx))
        if what == "k_tail":
            assert n_bound > 0, "the reference without W_0's last row still bounds every score"
        elif p == FP32_TC:
            assert n_contract > 0, "the reference with b_0[%d] one bf16 ulp off is still within 1e-5 of every score" % j


@pytest.mark.gpu
@pytest.mark.parametrize("prec", sorted(PRECS))
def test_eval_net_entry_points(sb, eval_params, eval_rows, prec):
    """score from pageable and from pinned host rows run the chunk plan score_device runs: the same bits; score_device of
    rows one float past a 16-byte boundary (the load's 4-byte path) gives the bits of the aligned rows; compute() of a
    few rows within the bound"""
    import torch
    p = PRECS[prec]
    scores, _ = _eval_scores(sb, eval_params, eval_rows, "trained", p)
    buf, idx, Xs = eval_rows
    N, F = EVAL_ROWS, EVAL_F
    Xh = buf[:N * F].view(N, F).cpu().numpy()
    pinned = torch.empty((N, F), dtype=torch.float32, pin_memory=True)
    pinned.numpy()[:] = Xh
    R = 65536                   # whole forwards in every precision
    mis = torch.empty(R * F + 4, dtype=torch.float32, device="cuda")
    mis[1:1 + R * F] = buf[:R * F]
    out = torch.empty(R, dtype=torch.float32, device="cuda")
    with _model(sb, F, EVAL_HIDDEN, EVAL_ACTS, p, eval_params["trained"]) as m:
        np.testing.assert_array_equal(_bits(m.score(Xh)), _bits(scores))
        np.testing.assert_array_equal(_bits(m.score(pinned.numpy())), _bits(scores))
        torch.cuda.synchronize()
        m.score_device(mis.data_ptr() + 4, R, out.data_ptr())
        m.sync()
        np.testing.assert_array_equal(_bits(out.cpu().numpy()), _bits(scores[:R]))
        pick = [0, 1, len(idx) // 2, len(idx) - 1]
        got = np.array([m.score_row_f64(Xs[i].astype(np.float64)) for i in pick])
    want = score(Xs[pick], unflatten(eval_params["trained"], F, EVAL_HIDDEN), _acts(EVAL_ACTS), p)
    _check(got, want, p, "eval net compute() %s" % prec)


# ------------------------------------------------------------------------------------------------------ small nets
_small_cache = {}


def _small_ref(prec):
    """every row of the small net's largest sweep count and its reference (rows are independent of the count)"""
    if prec not in _small_cache:
        n = 2 * CHUNK[BF16] + 4099
        X = _rows(SMALL_F, n, 5)
        flat = _seeded(SMALL_F, SMALL_HIDDEN, (1.5, 1.5, 1.5, 3.0), 6)
        _small_cache[prec] = (X, flat, score(X, unflatten(flat, SMALL_F, SMALL_HIDDEN), _acts(SMALL_ACTS), prec))
    return _small_cache[prec]


def _sweep_counts(prec):
    c = CHUNK[prec]
    return [1, 2, 127, 128, 129, c - 1, c, c + 1, 2 * c + 4099]


@pytest.mark.gpu
@pytest.mark.parametrize("prec", sorted(PRECS))
def test_row_sweep(sb, prec):
    """F = 37, [33, 1, 100]: every row of 1 .. 2 max_batch + 4099 rows against float64 (fp32 at <= 128 rows is
    score_rows_kernel); at the largest count score_device, score from pageable and from pinned rows give the same bits,
    the words around dOut keep theirs, and compute() of a few rows is within the bound"""
    import torch
    p = PRECS[prec]
    X, flat, (yh, e) = _small_ref(p)
    counts = _sweep_counts(p)
    with _model(sb, SMALL_F, SMALL_HIDDEN, SMALL_ACTS, p, flat) as m:
        for n in counts:
            got = m.score(X[:n])
            assert m.routes() == expected_routes(p, SMALL_F, SMALL_HIDDEN, _last_piece(p, n), _device_sms()), n
            _check(got, (yh[:n], e[:n]), p, "small net %s %d rows" % (prec, n))
        n = counts[-1]
        pinned = torch.empty((n, SMALL_F), dtype=torch.float32, pin_memory=True)
        pinned.numpy()[:] = X[:n]
        np.testing.assert_array_equal(_bits(m.score(pinned.numpy())), _bits(got))
        dX = torch.full((n + 64, SMALL_F), float("nan"), dtype=torch.float32, device="cuda")
        dX[:n] = torch.from_numpy(X[:n])
        out = torch.empty(n + 128 + 3, dtype=torch.float32, device="cuda")
        out.view(torch.int32).fill_(SENTINEL)
        torch.cuda.synchronize()
        m.score_device(dX.data_ptr(), n, out.data_ptr() + (64 + 3) * 4)
        m.sync()
        o = out.cpu().numpy()
        w = o.view(np.uint32)
        assert (w[:67] == SENTINEL).all() and (w[67 + n:] == SENTINEL).all(), "a word outside dOut changed"
        np.testing.assert_array_equal(_bits(o[67:67 + n]), _bits(got))
        pick = [0, 2, 5, n - 1]
        f64 = np.array([m.score_row_f64(X[i].astype(np.float64)) for i in pick])
    _check(f64, (yh[pick], e[pick]), p, "small net compute() %s" % prec)


WIDTHS = [1, 256, 257, 512, 513, 1024, 1025]


def _width_net(F, H):
    i = WIDTHS.index(H)
    hidden = [16, 1, H] if F == 37 else [24, H]           # F = 37: a 1-wide middle layer
    acts = [ACT_CYCLE[(i + k) % len(ACT_CYCLE)] for k in range(len(hidden))]
    return hidden, acts


@pytest.mark.gpu
@pytest.mark.parametrize("prec", sorted(PRECS))
@pytest.mark.parametrize("F", [37, 1999])
@pytest.mark.parametrize("H", WIDTHS)
def test_width_sweep(sb, H, F, prec):
    """last hidden widths across the out_layer_rows<1 | 2 | 4> / out_layer<bf16> boundaries, every activation, at 1, 129
    and 4099 rows"""
    p = PRECS[prec]
    hidden, acts = _width_net(F, H)
    X = _rows(F, 4099, 7 + H + F)
    flat = _seeded(F, hidden, (1.5,) * len(hidden) + (3.0,), zlib.crc32(repr((F, H)).encode()))
    yh, e = score(X, unflatten(flat, F, hidden), _acts(acts), p)
    with _model(sb, F, hidden, acts, p, flat) as m:
        for n in (1, 129, 4099):
            got = m.score(X[:n])
            assert m.routes() == expected_routes(p, F, hidden, n, _device_sms()), n
            _check(got, (yh[:n], e[:n]), p, "F=%d %s %s %d rows" % (F, hidden, prec, n))


@pytest.mark.gpu
@pytest.mark.parametrize("prec", sorted(PRECS))
def test_validation_pass(sb, prec):
    """Trainer.eval_loss and Trainer.predict run the same forward in max_batch pieces: over 2.5 max_batch rows with weights
    0 / 1 / 2.5, every prediction within its score bound, the loss within output_layer's loss bound summed over pieces"""
    p = PRECS[prec]
    F, hidden, acts, B = 120, [64, 300], ["relu", "tanh"], 1536
    n = 5 * B // 2
    X = _rows(F, n, 8)
    rng = np.random.default_rng(9)
    y = (rng.random(n) < 0.4).astype(np.float32)
    w = rng.choice(np.array([0.0, 1.0, 2.5], np.float32), size=n, p=[0.2, 0.6, 0.2]).astype(np.float32)
    flat = _seeded(F, hidden, (1.5, 1.5, 3.0), 10)
    layers = unflatten(flat, F, hidden)
    with sb.Trainer(sb.make_desc(F, hidden, _acts(acts), max_batch=B, precision=p)) as t:
        t.set_params(flat)
        pred = t.predict(X)
        loss = t.eval_loss(X, y, w)
    _check(pred, score(X, layers, _acts(acts), p), p, "predict %s" % prec)
    a, e_a = hidden_forward(X, layers, _acts(acts), p)
    route = expected_route(p, hidden[-1], False, "eval")
    want, tol = validation_loss(a, e_a, layers[-1][0], layers[-1][1], y, w, ACTS[acts[-1]], B, lambda m: _depth(route, m, 0))
    _notes["validation %s loss error / bound" % prec] = "%.3g" % (abs(loss - want) / tol)
    assert abs(loss - want) <= tol, (loss, want, tol)


# ------------------------------------------------------------------------------------------------------ no GPU
def test_cases_reach_every_instantiation():
    """the sweeps above reach every forward and output-layer launch a score can make (on an H100 SXM's 132 SMs)"""
    seen = set()
    for p in PRECS.values():
        for n in (CHUNK[p], _last_piece(p, EVAL_ROWS)):
            seen.update(expected_routes(p, EVAL_F, EVAL_HIDDEN, n, 132).split("+"))
        for n in _sweep_counts(p):
            seen.update(expected_routes(p, SMALL_F, SMALL_HIDDEN, _last_piece(p, n), 132).split("+"))
        for F in (37, 1999):
            for H in WIDTHS:
                for n in (1, 129, 4099):
                    seen.update(expected_routes(p, F, _width_net(F, H)[0], n, 132).split("+"))
    want = {"score_rows", "load_batch<fp32>", "load_batch<bf16>", "gemm_f32<FWD>", "gemm_wide", "gemm_pp<FWD>",
            "gemm_tc<64,FWD,GENERIC>", "gemm_tc<128,FWD,GENERIC>", "out_layer<float>", "out_layer<bf16>",
            "out_layer_rows<1>", "out_layer_rows<2>", "out_layer_rows<4>"}
    assert seen == want, seen ^ want


def test_chunk_sizes_match_the_library(sb):
    assert {int(k): v for k, v in sb.capi.MODEL_CHUNK_ROWS.items()} == CHUNK
