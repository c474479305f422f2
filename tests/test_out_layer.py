"""Kernel-level checks of the output layer's own kernels (kernels.cuh: out_layer_rows_kernel<1 / 2 / 4>, out_layer_kernel<bf16>
and out_layer_kernel<float>, each also in its deterministic form) through the sb_debug_out_layer hook, which launches
them with the step's own Net::enqueue_out on a Net whose last hidden layer holds A_L.

Oracle: float64 of the same operation on A_L as the kernel holds it, with the bounds of out_layer_ref.output_layer:
  a    FP32: A itself; BF16: bf16(A); BF16X2 / FP32_TC: the exact sum of A's 2 / 3 bf16 parts (the kernel rebuilds it in
       fp32: e_a = 2u |a|), plus 4u (|a| + 1) for the act' evaluation
  dZ   FP32 within e_g; BF16 within one bf16 ulp + e_g; split modes: the sum of the parts within e_g + 2^(1 - 8 np) |g|,
       each part below 2^-8 of the one before
  sums d = the depth of the kernel's reduction: rows a warp walks + its block's 8 warps + one addend per block (and row
       half) + a margin, so a dropped row or a shifted column misses by far more than its bound
The in/out sums start from non-zero values: the kernel must add into them, never store.  The hook fills A_L's pad
columns and the rows past the batch with NaN (y and w too on a score) and counts every write outside the outputs."""
import numpy as np
import pytest

from conftest import bf16_round
from out_layer_ref import ACTS, CE, LOSSES, MSE, U, activation, output_layer

FP32, BF16, FP32_TC, BF16X2 = 0, 1, 2, 3
PRECS = {"fp32": FP32, "bf16": BF16, "fp32tc": FP32_TC, "bf16x2": BF16X2}
NP = {FP32: 1, BF16: 1, FP32_TC: 3, BF16X2: 2}
MODES = {"step": (True, True), "eval": (True, False), "score": (False, False)}
WIDTHS = [1, 7, 8, 9, 255, 256, 257, 300, 511, 512, 513, 1000, 1024, 1025, 2048]
ROWS = [1, 7, 8, 9, 31, 32, 33, 257, 4099]
ACT_CYCLE = ["relu", "tanh", "sigmoid", "leakyrelu", "none"]
OUTS = ("yhat", "dZ", "db_L", "dw_o", "db_o", "loss")

_worst = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if _worst:
        print("\nworst error / bound: " + ", ".join("%s %.3g" % (k, _worst[k]) for k in OUTS if k in _worst))


def expected_route(prec, H, det, mode):
    """the instantiation Net::enqueue_out launches: the DET forms whenever something is summed"""
    d = ",DET" if det and mode != "score" else ""
    if prec == FP32:
        return "out_layer<float%s>" % d
    if H <= 1024:
        return "out_layer_rows<%d%s>" % (1 if H <= 256 else (2 if H <= 512 else 4), d)
    return "out_layer<bf16%s>" % d


_n_sm = []


def _device_sms():
    if not _n_sm:
        import torch
        _n_sm.append(torch.cuda.get_device_properties(0).multi_processor_count)
    return _n_sm[0]


def _depth(route, M, sms):
    if route.startswith("out_layer_rows"):
        # rows per block as enqueue_out plans them; a warp walks every 8th row of its block
        s = sms or _device_sms()
        rpb = max(8, (-(-M // (2 * s)) + 7) // 8 * 8)
        return -(-rpb // 8) + 8 + -(-M // rpb) + 4
    # 32-row blocks: 16 rows per thread and row half, 8 warps, two row halves per block
    return 16 + 8 + 2 * -(-M // 32) + 4


def _parts(x, n):
    """the step's split of fp32 x into n bf16 parts (bf16_residual)"""
    r, out = x.astype(np.float32), []
    for _ in range(n):
        p = bf16_round(r)
        out.append(p)
        r = (r - p).astype(np.float32)
    return out


def _operands(M, H, act, seed):
    rng = np.random.RandomState(seed * 7919 + M * 31 + H * 7 + ACTS[act])
    pre = (np.clip(rng.standard_normal((M, H)), -4, 4) * 1.5).astype(np.float32)
    A = activation(pre.astype(np.float64), ACTS[act]).astype(np.float32)
    wo = (rng.uniform(-1, 1, H) * np.sqrt(6.0 / (H + 1))).astype(np.float32)
    y = (rng.uniform(size=M) < 0.3).astype(np.float32)
    w = rng.choice(np.array([0.0, 1.0, 2.5], np.float32), size=M).astype(np.float32)
    init = dict(g_bL=(rng.standard_normal(H) * 0.1).astype(np.float32), g_wo=(rng.standard_normal(H) * 0.1).astype(np.float32),
                g_bo=0.37, loss_sum=1.25)
    return A, wo, np.float32(0.3), y, w, init


def _a_of(A, prec):
    """A_L as the kernel holds it (float64) and its bound"""
    if prec == FP32:
        a = A.astype(np.float64)
    else:
        a = np.sum([p.astype(np.float64) for p in _parts(A, NP[prec])], axis=0)
    e_a = 4 * U * (np.abs(a) + 1) + (2 * U * np.abs(a) if NP[prec] > 1 else 0.0)
    return a, e_a


def _note(name, err, tol):
    err, tol = np.broadcast_arrays(np.asarray(err, np.float64), np.asarray(tol, np.float64))
    pos = tol > 0                        # a zero bound (a row of weight 0) admits no error; the assertion checks it
    r = float(np.max(err[pos] / tol[pos])) if pos.any() else 0.0
    _worst[name] = max(_worst.get(name, 0.0), r)
    return r


def _check(got, ref, init, prec, mode, what):
    do_loss, do_bwd = MODES[mode]
    assert got["guard"] == 0, "%s: %d guard elements changed" % (what, got["guard"])
    yh, e_yh = ref["yhat"]
    err = np.abs(got["yhat"] - yh)
    r = _note("yhat", err, e_yh)
    assert (err <= e_yh).all(), "%s: y_hat off by %.3g x its bound (row %d)" % (what, r, np.argmax(err - e_yh))
    sums = [("loss", got["loss_sum"], init["loss_sum"])] if do_loss else []
    if do_bwd:
        dZ, g, e_g, ok = got["dZ"], ref["g"], ref["e_g"], ~ref["kink"]
        if prec == FP32:
            err, tol = np.abs(dZ[0] - g), e_g
        elif NP[prec] == 1:
            err, tol = np.abs(dZ[0] - g), 2.0 ** -7 * np.abs(g) + e_g
        else:
            n = NP[prec]
            err, tol = np.abs(dZ.astype(np.float64).sum(axis=0) - g), e_g + 2.0 ** (1 - 8 * n) * np.abs(g)
            for k in range(1, n):        # part k is the bf16 of what parts 0 .. k-1 leave: at most 2^-8 of part k-1
                assert (np.abs(dZ[k]) <= 2.0 ** -8 * np.abs(dZ[k - 1])).all(), "%s: part %d not below part %d" % (what, k, k - 1)
        bad = (err > tol) & ok
        _note("dZ", err[ok], tol[ok])
        assert not bad.any(), "%s: %d dZ_L elements off, first at %s: %r vs %r (bound %r)" % (
            what, bad.sum(), np.argwhere(bad)[0], dZ[0][bad][0], g[bad][0], tol[bad][0])
        sums += [("db_L", got["g_bL"], init["g_bL"]), ("dw_o", got["g_wo"], init["g_wo"]), ("db_o", got["g_bo"], init["g_bo"])]
    # in/out: the result minus the value passed in is the contribution (fp32 additions onto the initial value add d u |init|)
    for name, val, i0 in sums:
        want, tol = ref[name]
        val, i0 = np.asarray(val, np.float64), np.asarray(i0, np.float64)
        tol = tol + ref["d"] * U * (np.abs(i0) + np.abs(want))
        err = np.abs(val - i0 - want)
        r = _note(name, err, tol)
        assert (err <= tol).all(), "%s: %s off by %.3g x its bound (worst at %s)" % (what, name, r, np.argmax(err / tol))


def _run(sb, prec, M, H, act="relu", loss=MSE, mode="step", sms=0, det=False, seed=0, w=None, scale_wo=None):
    A, wo, bo, y, w0, init = _operands(M, H, act, seed)
    w = w0 if w is None else w
    if scale_wo is not None:
        wo = (wo * np.float32(scale_wo)).astype(np.float32)
    do_loss, do_bwd = MODES[mode]
    got = sb.capi.debug_out_layer(prec, A, wo, bo, ACTS[act], loss, y=y if do_loss else None, w=w if do_loss else None,
                                  do_loss=do_loss, do_bwd=do_bwd, det=det, sms=sms, **init)
    what = "prec=%d M=%d H=%d %s loss=%d %s sms=%d det=%d" % (prec, M, H, act, loss, mode, sms, det)
    route = expected_route(prec, H, det, mode)
    assert got["route"] == route, what
    a, e_a = _a_of(A, prec)
    ref = output_layer(a, e_a, wo, bo, y, w, ACTS[act], loss, _depth(route, M, sms))
    _check(got, ref, init, prec, mode, what)
    if det:
        assert got["repeat_same"] == 1, "%s: a second launch gave other bits" % what
    return got, ref, init


@pytest.mark.gpu
@pytest.mark.parametrize("loss", sorted(LOSSES))
@pytest.mark.parametrize("H", WIDTHS)
@pytest.mark.parametrize("prec", sorted(PRECS))
def test_widths(sb, prec, H, loss):
    # every route boundary (256 / 512 / 1024) and ragged 8-column pieces; the activation varies with the width
    _run(sb, PRECS[prec], 257, H, ACT_CYCLE[WIDTHS.index(H) % len(ACT_CYCLE)], LOSSES[loss])


@pytest.mark.gpu
@pytest.mark.parametrize("H", [100, 1100])
@pytest.mark.parametrize("sms", [0, 1, 3])
@pytest.mark.parametrize("M", ROWS)
@pytest.mark.parametrize("prec", sorted(PRECS))
def test_rows(sb, prec, M, sms, H):
    # sms = 1 / 3: rows per block up to half the batch, so one warp walks many rows and carries its column sums
    _run(sb, PRECS[prec], M, H, "relu", CE if M % 2 else MSE, sms=sms)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("loss", sorted(LOSSES))
@pytest.mark.parametrize("act", ACT_CYCLE)
@pytest.mark.parametrize("prec", sorted(PRECS))
def test_activations_and_modes(sb, prec, act, loss, mode):
    # eval: y_hat and the loss only; score: y_hat only, with y / w NaN - the gradient and the scalars stay as they were
    _run(sb, PRECS[prec], 300, 520 if PRECS[prec] != FP32 else 130, act, LOSSES[loss], mode=mode)


@pytest.mark.gpu
@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("H", [100, 600, 1100])
@pytest.mark.parametrize("prec", sorted(PRECS))
def test_no_nonzero_weight(sb, prec, H, det):
    # n_nz = 0: dz = 0 everywhere, so dZ_L is +-0 and every in/out value comes back with the bits it went in with
    M = 200
    for loss in (MSE, CE):
        got, _, init = _run(sb, PRECS[prec], M, H, "tanh", loss, det=det, w=np.zeros(M, np.float32))
        assert (got["dZ"] == 0).all()
        for k in ("g_bL", "g_wo"):
            assert got[k].tobytes() == init[k].tobytes()
        assert got["g_bo"] == np.float32(init["g_bo"]) and got["loss_sum"] == np.float32(init["loss_sum"])


@pytest.mark.gpu
@pytest.mark.parametrize("H", [256, 1100])
@pytest.mark.parametrize("act", ["relu", "sigmoid"])
@pytest.mark.parametrize("loss", sorted(LOSSES))
@pytest.mark.parametrize("prec", sorted(PRECS))
def test_saturated_logits(sb, prec, loss, act, H):
    # |z| up to ~90: the CE loss needs the softplus form max(z, 0) - z y + log1p(exp(-|z|)), MSE's dz vanishes in fp32,
    # y_hat of a very negative z is subnormal; nothing may turn non-finite
    M = 256
    A, wo, bo, _, _, _ = _operands(M, H, act, 0)
    a, _ = _a_of(A, PRECS[prec])
    z = a @ wo.astype(np.float64)
    got, ref, _ = _run(sb, PRECS[prec], M, H, act, LOSSES[loss], scale_wo=90.0 / np.abs(z).max())
    assert np.abs(ref["yhat"][0]).min() < 1e-30 or np.abs(1 - ref["yhat"][0]).min() < 1e-30
    assert all(np.isfinite(np.asarray(got[k])).all() for k in ("yhat", "dZ", "g_bL", "g_wo", "g_bo", "loss_sum"))


@pytest.mark.gpu
@pytest.mark.parametrize("sms", [0, 3])
@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("H", [9, 300, 700, 1100])
@pytest.mark.parametrize("prec", sorted(PRECS))
def test_deterministic(sb, prec, H, mode, sms):
    # the DET forms: slots summed in a fixed order by the last block, whose ticket goes back to 0 - a second launch on the
    # same net gives the same bits (a ticket left behind would drop its sums), within the float64 bound and within the
    # bound of the atomic form
    p = PRECS[prec]
    got, ref, init = _run(sb, p, 777, H, "leakyrelu", CE, mode=mode, sms=sms, det=True)
    free, _, _ = _run(sb, p, 777, H, "leakyrelu", CE, mode=mode, sms=sms)
    np.testing.assert_array_equal(got["yhat"], free["yhat"])
    do_loss, do_bwd = MODES[mode]
    if do_bwd:
        np.testing.assert_array_equal(got["dZ"], free["dZ"])
    for name, key in (("loss", "loss_sum"), ("db_L", "g_bL"), ("dw_o", "g_wo"), ("db_o", "g_bo")):
        if (name == "loss" and do_loss) or (name != "loss" and do_bwd):
            tol = 2 * (ref[name][1] + ref["d"] * U * (np.abs(init[key]) + np.abs(ref[name][0])))
            assert (np.abs(np.asarray(got[key], np.float64) - free[key]) <= tol).all(), name


CASES = ([(PRECS[p], H, False, "step") for p in PRECS for H in WIDTHS]
         + [(PRECS[p], H, True, m) for p in PRECS for H in (9, 300, 700, 1100) for m in MODES])


def test_cases_reach_every_instantiation():
    want = {"out_layer_rows<%d%s>" % (n, d) for n in (1, 2, 4) for d in ("", ",DET")}
    want |= {"out_layer<%s%s>" % (t, d) for t in ("bf16", "float") for d in ("", ",DET")}
    assert len(want) == 10
    assert {expected_route(*c) for c in CASES} == want


# ------------------------------------------------------------------------------------------------------------ no GPU
def _call(sb, prec=FP32_TC, det=0, do_loss=1, do_bwd=1, M=64, H=64, act=2, loss=MSE, sms=0, drop=(), route_cap=64):
    import ctypes as C
    buf = {k: np.ones(4 * 64 * 64, np.float32) for k in ("A", "wo", "y", "w", "yhat", "dZ", "g_bL", "g_wo", "g_bo", "loss_sum")}
    for k in drop:
        buf[k] = None
    guard, same = C.c_int32(-1), C.c_int32(-1)
    route = C.create_string_buffer(64)
    ptr = sb.capi._ptr
    return sb.capi.lib().sb_debug_out_layer(
        prec, det, do_loss, do_bwd, ptr(buf["A"]), ptr(buf["wo"]), 0.5, ptr(buf["y"]), ptr(buf["w"]), ptr(buf["yhat"]),
        ptr(buf["dZ"]), ptr(buf["g_bL"]), ptr(buf["g_wo"]), ptr(buf["g_bo"]), ptr(buf["loss_sum"]),
        None if "guard" in drop else C.byref(guard), C.byref(same), route, route_cap, M, H, act, loss, sms, 0)


INVALID = {
    "precision=4": dict(prec=4), "precision=-1": dict(prec=-1), "det=2": dict(det=2), "do_loss=2": dict(do_loss=2),
    "do_bwd=-1": dict(do_bwd=-1), "bwd_without_loss": dict(do_loss=0, do_bwd=1), "M=0": dict(M=0), "M=-5": dict(M=-5),
    "H=0": dict(H=0), "act=4": dict(act=4), "act=-2": dict(act=-2), "loss=2": dict(loss=2), "sms=-1": dict(sms=-1),
    "no_A": dict(drop=("A",)), "no_wo": dict(drop=("wo",)), "no_guard": dict(drop=("guard",)), "route_cap=0": dict(route_cap=0),
    "loss_no_y": dict(drop=("y",)), "loss_no_w": dict(drop=("w",)), "loss_no_loss_sum": dict(drop=("loss_sum",)),
    "bwd_no_dZ": dict(drop=("dZ",)), "bwd_no_g_bL": dict(drop=("g_bL",)), "bwd_no_g_wo": dict(drop=("g_wo",)),
    "bwd_no_g_bo": dict(drop=("g_bo",)), "score_no_yhat": dict(do_loss=0, do_bwd=0, drop=("yhat",)),
}


@pytest.mark.parametrize("case", sorted(INVALID))
def test_invalid_arguments_rejected_before_any_device_call(sb, case):
    # refused on a machine without a GPU, so no device work happens before the check
    assert _call(sb, **INVALID[case]) == sb.capi.SB_ERR_INVALID, sb.capi.lib().sb_last_error()


@pytest.mark.gpu
def test_sms_above_the_device_rejected(sb):
    assert _call(sb, sms=100000) == sb.capi.SB_ERR_INVALID
