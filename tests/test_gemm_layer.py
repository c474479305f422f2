"""Kernel-level checks of a training step's forward, dA and dW GEMMs through the sb_debug_gemm_layer hook, which builds a
network whose layer is the GEMM under test and launches it with the step's own Net::enqueue_* code: the step's plans,
tensor maps, part pairs and instantiations, in every precision mode the step runs them in.

Oracle: float64 of the same operation.  BF16 (np = 1) takes the operands rounded to bf16 (the kernel multiplies them
exactly and accumulates in fp32); BF16X2 / FP32_TC (np = 2 / 3) and FP32 take the fp32 inputs (the kernels split them
into bf16 parts, or multiply them in fp32).

Tolerances follow the arithmetic, with u = 2^-24 and S = |A| |B| (the sum of the magnitudes of a contraction's terms):
  contraction   e_c = c S: c = 3e-6 for np = 1 and 3, 2e-5 for np = 2 (the fp32-class bound of the tensor-core
                contraction, measured 0.7 - 1.4e-6 for np = 3); FP32: the FMA chain, c = (K + 2) u
  forward       e_pre = e_c + 4u (|pre| + |addend| + |bias|) for the two fp32 adds; e_a = e_pre + 4u (|a| + 1)
                (|act'| <= 1, a few ulp of expf / tanhf)
  dA            e_g = |act'| e_c + |pre| e_act' + 4u |g|, e_act' = 2 d |aux| + 4u where d is the error of the aux value
                the kernel reads (np = 2: 2^-16 |aux|; np = 3, FP32: 2^-24; np = 1: 0, the reference takes bf16(aux));
                |d act' / d aux| <= 2
  stored value  np = 1: e + 2^-8 (|v| + e) (round to nearest bf16); np = 2 / 3: the sum of the parts within
                e + 2^(1 - 8 np) |v|, and each part is the bf16 of the residual the parts before it leave:
                |p_(k+1)| <= 1/2 ulp(p_k); FP32: e
  sums          the column sums and dW (split-K, red.add into the values passed in) are held to the sum of their terms'
                bounds + d u (sum |terms| + |initial value|), d = the depth of the reduction: rows / 64 + 64 for the
                column sums, for dW the most splits the planner may cut K into (>= 8 k-blocks each) + 2
So an element is held relative to the magnitudes it is made of: a dropped lower part (2^-9 relative), a shifted column,
a tile stored twice or a sum flushed from the wrong buffer misses by far more than its bound.  relu / leakyrelu forward:
elements whose |pre| lies within e_pre of the kink are left out of the element check (act may flip there).

Every output is surrounded by a sentinel (the 64 rows past the batch in every part, the pad columns, the gradient outside
its in/out rows and a margin behind it, the cleared buffer's margin): the hook counts changed sentinel elements in
`guard`, which must be 0.  The in/out sums are pre-filled with non-zero values: the kernels must add into them."""
import zlib

import numpy as np
import pytest

from conftest import bf16_round
from score_ref import contraction_c

FP32, BF16, FP32_TC, BF16X2 = 0, 1, 2, 3
PREC = {"fp32": FP32, "bf16": BF16, "fp32_tc": FP32_TC, "bf16x2": BF16X2}
NPARTS = {FP32: 1, BF16: 1, FP32_TC: 3, BF16X2: 2}
ACTS = {"sigmoid": 0, "tanh": 1, "relu": 2, "leakyrelu": 3, "none": -1}
ALPHA = 0.2
U = 2.0 ** -24
FWD, DA, DW = 0, 1, 2
SPLIT = ["bf16x2", "fp32_tc", "fp32"]            # the precisions whose forward / dA GEMMs are the GENERIC / fp32 kernels
OUTS = ("out", "parts", "colsum", "dW", "guard")

_worst = {}
_cache = {}
_routes = set()


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if _worst:
        print("\nworst error / bound: " + ", ".join("%s %.3g" % (k, _worst[k]) for k in OUTS if k in _worst))
    if _routes:
        print("routes: " + ", ".join(sorted(_routes)))


def _note(name, err, tol):
    err, tol = np.broadcast_arrays(np.asarray(err, np.float64), np.asarray(tol, np.float64))
    r = float(np.max(err / tol)) if err.size else 0.0
    _worst[name] = max(_worst.get(name, 0.0), r)
    return r


def _c(prec, K):
    return contraction_c(prec, K)


def _act(z, act):
    if act == ACTS["sigmoid"]:
        return 1.0 / (1.0 + np.exp(-z))
    if act == ACTS["tanh"]:
        return np.tanh(z)
    if act == ACTS["relu"]:
        return np.maximum(z, 0.0)
    if act == ACTS["leakyrelu"]:
        return np.where(z > 0, z, ALPHA * z)
    return z


def _act_grad(a, act):
    if act == ACTS["sigmoid"]:
        return a * (1.0 - a)
    if act == ACTS["tanh"]:
        return 1.0 - a * a
    if act == ACTS["relu"]:
        return (a > 0).astype(np.float64)
    if act == ACTS["leakyrelu"]:
        return np.where(a > 0, 1.0, ALPHA)
    return np.ones_like(a)


def _parts(x, n):
    """the step's split of fp32 x into n bf16 parts (bf16_residual)"""
    out, r = [], np.asarray(x, np.float32)
    for _ in range(n):
        p = bf16_round(r)
        out.append(p)
        r = (r - p).astype(np.float32)
    return np.stack(out)


def _operands(key, shape_a, shape_b, scale_b):
    """A (standard normal, clipped, * 0.5) and B (uniform +-scale_b) for a key, with the float64 products the bounds need:
    (A B, |A| |B|) on the fp32 values and on the bf16-rounded ones (computed on first use, kept for the next case)"""
    if key not in _cache:
        rng = np.random.RandomState(zlib.crc32(repr(key).encode()))
        A = (np.clip(rng.standard_normal(shape_a), -4, 4) * 0.5).astype(np.float32)
        B = rng.uniform(-scale_b, scale_b, shape_b).astype(np.float32)
        if len(_cache) > 6:
            _cache.clear()
        _cache[key] = {"A": A, "B": B}
    return _cache[key]


def _products(ent, a, b, bf16, transpose_b=False, transpose_a=False):
    k = ("prod", bf16, transpose_a, transpose_b)
    if k not in ent:
        A = bf16_round(a) if bf16 else a
        B = bf16_round(b) if bf16 else b
        A64, B64 = A.astype(np.float64), B.astype(np.float64)
        if transpose_a:
            A64 = A64.T
        if transpose_b:
            B64 = B64.T
        ent[k] = (A64 @ B64, np.abs(A64) @ np.abs(B64))
    return ent[k]


def _check_stored(out, v, e, prec, what, skip=None):
    """out [np, M, N] against the float64 value v with bound e (module docstring)"""
    n = NPARTS[prec]
    ok = np.ones(v.shape, bool) if skip is None else ~skip
    if prec == FP32:
        err, tol = np.abs(out[0] - v), e
    elif n == 1:
        err, tol = np.abs(out[0] - v), e + 2.0 ** -8 * (np.abs(v) + e)
    else:
        err, tol = np.abs(out.astype(np.float64).sum(axis=0) - v), e + 2.0 ** (1 - 8 * n) * np.abs(v)
        for k in range(1, n):
            prev, cur = out[k - 1], out[k]
            _, ex = np.frexp(prev)
            half_ulp = np.where(prev != 0, np.ldexp(1.0, ex - 9), 0.0)
            bad = np.abs(cur) > half_ulp
            if bad.any():
                i = tuple(np.argwhere(bad)[0])
                raise AssertionError("%s: part %d not within half an ulp of part %d at %s: %r after %r" % (
                    what, k, k - 1, i, cur[i], prev[i]))
            _note("parts", np.abs(cur), np.where(half_ulp > 0, half_ulp, 1.0))
    bad = (err > tol) & ok
    _note("out", err[ok], tol[ok])
    if bad.any():
        i = tuple(np.argwhere(bad)[0])
        raise AssertionError("%s: %d elements off, first at %s: %r vs %r (bound %r)" % (
            what, bad.sum(), i, out[(slice(None),) + i].sum(), v[i], tol[i]))


def _check_sum(name, got, init, want, tol, d, mag, what):
    """got - init against want: tol (the terms' bounds) + d u (|init| + mag), mag = the sum of the terms' magnitudes"""
    got, init = np.asarray(got, np.float64), np.asarray(init, np.float64)
    tol = tol + d * U * (np.abs(init) + mag)
    err = np.abs(got - init - want)
    r = _note(name, err, tol)
    if not (err <= tol).all():
        i = np.unravel_index(np.argmax(err / tol), err.shape)
        raise AssertionError("%s: %s off by %.3g x its bound at %s: %r vs %r" % (what, name, r, i, got[i] - init[i], want[i]))


def _check_guard(guard, what):
    _worst["guard"] = max(_worst.get("guard", 0), guard)
    assert guard == 0, "%s: %d sentinel elements changed" % (what, guard)


# ------------------------------------------------------------------------------------------------------------ forward
def _fwd(sb, prec, M, N, K, act="relu", sms=0, row0=0, a_rows=None, addend=False, clear_n4=0, seed=0):
    a_rows = M if a_rows is None else a_rows
    ent = _operands(("fwd", M, N, K, a_rows, row0, seed), (a_rows, K), (K, N), np.sqrt(6.0 / (K + N)))
    A, W = ent["A"], ent["B"]
    if "bias" not in ent:
        rng = np.random.RandomState(N + seed)
        ent["bias"] = rng.uniform(-0.3, 0.3, N).astype(np.float32)
        ent["addend"] = rng.standard_normal((M, N)).astype(np.float32) * 0.5
        A[:row0] *= 100
        A[row0 + M:] *= 100
    bias, add = ent["bias"], (ent["addend"] if addend else None)
    code = ACTS[act]
    out, _, _, guard, route = sb.capi.debug_gemm_layer(FWD, prec, A, W, code, bias=bias, addend=add, M=M, row0=row0, sms=sms,
                                                       clear_n4=clear_n4)
    _routes.add(route)
    what = "fwd %dx%dx%d %s prec=%d sms=%d row0=%d addend=%s [%s]" % (M, N, K, act, prec, sms, row0, addend, route)
    _check_guard(guard, what)
    bf = NPARTS[prec] == 1 and prec != FP32
    pre, S = _products(ent, A[row0:row0 + M], W, bf) if (row0 == 0 and a_rows == M) else _products(
        {}, A[row0:row0 + M], W, bf)
    b64 = bias.astype(np.float64)
    add64 = add.astype(np.float64) if addend else 0.0
    z = pre + add64 + b64
    e_pre = _c(prec, K) * S + 4 * U * (np.abs(pre) + np.abs(add64) + np.abs(b64))
    a = _act(z, code)
    e_a = e_pre + 4 * U * (np.abs(a) + 1)
    kink = (np.abs(z) <= e_pre) if code in (ACTS["relu"], ACTS["leakyrelu"]) else None
    _check_stored(out, a, e_a, prec, what, kink)
    return out, route


FWD_SHAPES = [
    (100, 50, 200),          # cfg0 layer 0
    (130, 129, 72),          # ragged M / N / K
    (300, 40, 136),          # N <= 64: the 64-wide tile
    (300, 200, 136),
    (4096, 512, 1000),       # cfg1 forward 0
]


@pytest.mark.gpu
@pytest.mark.parametrize("prec", SPLIT)
@pytest.mark.parametrize("M,N,K", FWD_SHAPES)
def test_forward_shapes(sb, M, N, K, prec):
    _fwd(sb, PREC[prec], M, N, K, "relu")


@pytest.mark.gpu
@pytest.mark.parametrize("prec", SPLIT)
def test_forward_cfg2(sb, prec):
    _fwd(sb, PREC[prec], 8192, 1024, 2000, "relu")          # cfg2 forward 0


@pytest.mark.gpu
@pytest.mark.parametrize("prec", SPLIT)
@pytest.mark.parametrize("act", sorted(ACTS))
@pytest.mark.parametrize("M,N,K", [(130, 129, 72), (200, 40, 300)])
def test_forward_activations(sb, M, N, K, act, prec):
    _fwd(sb, PREC[prec], M, N, K, act)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["bf16x2", "fp32_tc"])
def test_forward_resident_row_offset(sb, prec):
    # the batch at row 77 of a larger set whose other rows are 100x larger: they must not leak into the first or last tile
    M, N, K, row0 = 300, 120, 72, 77
    _fwd(sb, PREC[prec], M, N, K, "tanh", row0=row0, a_rows=row0 + M + 50)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", SPLIT)
@pytest.mark.parametrize("N", [50, 200])
def test_forward_several_tiles_per_cta(sb, prec, N):
    # 8 x 1..2 tiles on 3 CTAs: the bias buffer of tile parity it & 1 is rewritten while the other tile's is still read
    _fwd(sb, PREC[prec], 1000, N, 136, "sigmoid", sms=3)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["bf16", "bf16x2", "fp32_tc"])
def test_forward_clears_the_buffer(sb, prec):
    # a resident step's layer-0 GEMM clears the gradient buffer with its idle producer warps: every float4 of the range
    # becomes +0, nothing behind it changes (the guard), on a small grid and on the full one
    for sms in (2, 0):
        _fwd(sb, PREC[prec], 300, 100, 200, "relu", row0=13, a_rows=400, clear_n4=10007, sms=sms)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["bf16", "bf16x2", "fp32_tc", "fp32"])
@pytest.mark.parametrize("N", [72, 100])
def test_forward_with_addend(sb, prec, N):
    # wide+deep layer 0: N = 72 / 100 ends inside a 32-column chunk (the scalar addend path); the chunks before it, and
    # N = 64 / 96 / 128 wholly, take the float4 path
    _fwd(sb, PREC[prec], 260, N, 136, "tanh", addend=True)
    _fwd(sb, PREC[prec], 260, N // 32 * 32, 136, "tanh", addend=True)


# ------------------------------------------------------------------------------------------------------------ dA
def _aux(rng, act, M, N, zeros=False):
    if act == ACTS["sigmoid"]:
        aux = rng.uniform(0.0, 1.0, (M, N))
    elif act == ACTS["tanh"]:
        aux = rng.uniform(-1.0, 1.0, (M, N))
    else:
        aux = rng.standard_normal((M, N))
        if zeros:
            aux[rng.uniform(size=(M, N)) < 0.25] = 0.0     # relu: act'(0) = 0
    return aux.astype(np.float32)


def _da(sb, prec, M, N, K, act="relu", sms=0, zeros=False, seed=0):
    ent = _operands(("da", M, N, K, seed), (M, K), (N, K), np.sqrt(6.0 / (K + N)))
    A, W = ent["A"], ent["B"]
    code = ACTS[act]
    rng = np.random.RandomState(M + N + code + seed)
    aux = _aux(rng, code, M, N, zeros)
    init = rng.standard_normal(N).astype(np.float32)
    out, cs, _, guard, route = sb.capi.debug_gemm_layer(DA, prec, A, W, code, aux=aux, colsum=init, sms=sms)
    _routes.add(route)
    what = "dA %dx%dx%d %s prec=%d sms=%d [%s]" % (M, N, K, act, prec, sms, route)
    _check_guard(guard, what)
    n = NPARTS[prec]
    bf = n == 1 and prec != FP32
    pre, S = _products(ent, A, W, bf, transpose_b=True)
    aux64 = (bf16_round(aux) if bf else aux).astype(np.float64)
    d = {1: 0.0, 2: 2.0 ** -16, 3: U}[n] if prec != FP32 else U
    ag = _act_grad(aux64, code)
    g = pre * ag
    e_g = np.abs(ag) * _c(prec, K) * S + np.abs(pre) * (2 * d * np.abs(aux64) + 4 * U) + 4 * U * np.abs(g)
    _check_stored(out, g, e_g, prec, what)
    _check_sum("colsum", cs, init, g.sum(axis=0), e_g.sum(axis=0), M // 64 + 64, np.abs(g).sum(axis=0), what)
    return out, cs, route


DA_SHAPES = [
    (100, 50, 200),          # cfg0 dA 1 layout (ragged)
    (130, 129, 72),
    (300, 40, 136),          # N <= 64
    (4096, 256, 128),        # cfg1 dA 2
    (4096, 512, 256),        # cfg1 dA 1
    (8192, 512, 256),        # cfg2 dA 2
]


@pytest.mark.gpu
@pytest.mark.parametrize("prec", SPLIT)
@pytest.mark.parametrize("M,N,K", DA_SHAPES)
def test_da_shapes(sb, M, N, K, prec):
    _da(sb, PREC[prec], M, N, K, "relu")


@pytest.mark.gpu
@pytest.mark.parametrize("prec", SPLIT)
def test_da_cfg2(sb, prec):
    _da(sb, PREC[prec], 8192, 1024, 512, "tanh")          # cfg2 dA 1


@pytest.mark.gpu
@pytest.mark.parametrize("prec", SPLIT)
@pytest.mark.parametrize("act", sorted(ACTS))
def test_da_activations(sb, act, prec):
    # sigmoid / tanh: the fp32 aux values have non-zero lower parts, which act' must read in the split modes
    _da(sb, PREC[prec], 260, 129, 100, act)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", SPLIT)
@pytest.mark.parametrize("act", ["relu", "leakyrelu"])
def test_da_relu_at_zero(sb, act, prec):
    _da(sb, PREC[prec], 260, 100, 72, act, zeros=True)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", SPLIT)
@pytest.mark.parametrize("N", [50, 300])
def test_da_several_tiles_per_cta(sb, prec, N):
    # 8 x 1..3 tiles on 3 CTAs: column sums accumulate in both shared buffers and are flushed from the one of their tile
    _da(sb, PREC[prec], 1000, N, 136, "tanh", sms=3)


# ------------------------------------------------------------------------------------------------------------ dW
def _dw(sb, prec, M, N, K, sms=0, r0=0, r1=None, row0=0, a_rows=None, seed=0):
    """grad[M, N] (rows r0 .. r1 - 1) += A^T dZ, A = rows row0 .. row0 + K - 1 of [a_rows, M], dZ [K, N]"""
    a_rows = K if a_rows is None else a_rows
    r1 = M if r1 is None else r1
    ent = _operands(("dw", M, N, K, a_rows, row0, seed), (a_rows, M), (K, N), 1.0)
    A, dZ = ent["A"], ent["B"]
    if "init" not in ent:
        ent["init"] = np.random.RandomState(M + N).standard_normal((M, N)).astype(np.float32)
        A[:row0] = 1e4
        A[row0 + K:] = -3e4
    init = ent["init"]
    _, _, g, guard, route = sb.capi.debug_gemm_layer(DW, prec, A, dZ, grad=init, row0=row0, r0=r0, r1=r1, sms=sms)
    _routes.add(route)
    what = "dW %dx%dx%d prec=%d sms=%d rows %d..%d row0=%d [%s]" % (M, N, K, prec, sms, r0, r1, row0, route)
    _check_guard(guard, what)
    n = NPARTS[prec]
    bf = n == 1 and prec != FP32
    batch = A[row0:row0 + K]
    pre, S = _products(ent if row0 == 0 and a_rows == K else {}, batch, dZ, bf, transpose_a=True)
    kb = -(-K // 64) * (1 if prec == FP32 else {1: 1, 2: 3, 3: 6}[n])
    d = (kb if prec == FP32 else kb // 8) + 2
    np.testing.assert_array_equal(g[:r0], init[:r0])
    np.testing.assert_array_equal(g[r1:], init[r1:])
    _check_sum("dW", g[r0:r1], init[r0:r1], pre[r0:r1], _c(prec, K) * S[r0:r1], d, S[r0:r1], what)
    return g, route


DW_SHAPES = [
    # (M = in, N = out, K = batch rows)
    (200, 100, 100),         # cfg0 dW 0
    (1000, 512, 4096),       # cfg1 dW 0
    (512, 256, 4096),        # cfg1 dW 1
    (256, 128, 4096),        # cfg1 dW 2
    (1024, 512, 8192),       # cfg2 dW 1
    (512, 256, 8192),        # cfg2 dW 2
    (300, 64, 500),          # N = 64: the 64-wide tile
    (300, 50, 500),          # N % 4 != 0: the scalar reds
    (130, 258, 200),         # everything ragged
]


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["bf16", "bf16x2", "fp32_tc", "fp32"])
@pytest.mark.parametrize("M,N,K", DW_SHAPES)
def test_dw_shapes(sb, M, N, K, prec):
    _dw(sb, PREC[prec], M, N, K)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["bf16", "bf16x2", "fp32_tc", "fp32"])
def test_dw_cfg2_layer0(sb, prec):
    _, route = _dw(sb, PREC[prec], 2000, 1024, 8192)     # cfg2 dW 0: 128 x 256 tiles in every tensor-core mode
    assert route == ("gemm_f32<DW>" if PREC[prec] == FP32 else "gemm_dw")


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["bf16", "bf16x2", "fp32_tc", "fp32"])
@pytest.mark.parametrize("sms", [44, 7])
def test_dw_grid_caps(sb, prec, sms):
    # a third of the SMs (plan_dw1's budget for dW_1 beside dW_0), and 7: several tiles and splits per CTA
    _dw(sb, PREC[prec], 512, 256, 4096, sms=sms)
    _dw(sb, PREC[prec], 130, 258, 200, sms=sms)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["bf16", "bf16x2", "fp32_tc"])
def test_dw_resident_row_offset(sb, prec):
    # the batch at row 77 of the resident set; the rows around it hold large finite values that must contribute nothing
    _dw(sb, PREC[prec], 200, 100, 300, row0=77, a_rows=77 + 300 + 90)
    _dw(sb, PREC[prec], 1000, 512, 1000, row0=77, a_rows=77 + 1000 + 90)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["bf16", "bf16x2", "fp32_tc"])
def test_dw_exchange_chunks(sb, prec):
    # cfg1's W_0 cut into the two exchange chunks at row 512: each launch adds into its rows only (the guard covers the
    # other chunk's rows and the bias behind the matrix)
    M, N, K = 1000, 512, 4096
    _dw(sb, PREC[prec], M, N, K, r0=0, r1=512)
    _dw(sb, PREC[prec], M, N, K, r0=512, r1=M)


# ------------------------------------------------------------------------------------------------------------ exact
@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["bf16", "bf16x2", "fp32_tc", "fp32"])
@pytest.mark.parametrize("kind", [FWD, DA])
def test_identity_is_exact(sb, kind, prec):
    # A = I: the output parts are W's (forward) or W^T's (dA) parts bit for bit - a swizzle, part order or part pair
    # mistake moves or changes elements
    p = PREC[prec]
    n = NPARTS[p]
    M, N = 200, 130
    W = np.random.RandomState(7).standard_normal((N, M) if kind == DA else (M, N)).astype(np.float32)
    I = np.eye(M, dtype=np.float32)
    if kind == FWD:
        out, _, _, guard, route = sb.capi.debug_gemm_layer(FWD, p, I, W, ACTS["none"], bias=np.zeros(N, np.float32))
        want = W
    else:
        out, _, _, guard, route = sb.capi.debug_gemm_layer(DA, p, I, W, ACTS["none"], aux=np.zeros((M, N), np.float32))
        want = W.T
    _routes.add(route)
    assert guard == 0
    if p == FP32:
        np.testing.assert_array_equal(out, want[None])
        return
    # the kernel's fp32 value is the sum of W's parts (exact); stored, it is split again.  np = 1 and 3: those are W's parts.
    # np = 2: where W's second part is a tie (exactly half an ulp of the first) the split rounds the sum to even instead,
    # the same value in other parts
    held = _parts(want, n).sum(axis=0, dtype=np.float32)
    np.testing.assert_array_equal(out, _parts(held, n))
    if n != 2:
        np.testing.assert_array_equal(out, _parts(want, n))


# ------------------------------------------------------------------------------------------------------------ routes
# every instantiation a step launches for these GEMMs, and a case that reaches it
ROUTES = {
    "gemm_tc<64,FWD,GENERIC>": (FWD, BF16X2, 130, 50, 72, 0),
    "gemm_tc<128,FWD,GENERIC>": (FWD, FP32_TC, 130, 129, 72, 0),
    "gemm_tc<64,DA,GENERIC>": (DA, FP32_TC, 130, 50, 72, 0),
    "gemm_tc<128,DA,GENERIC>": (DA, BF16X2, 130, 129, 72, 0),
    "gemm_tc<64,DW>": (DW, BF16, 300, 64, 500, 0),
    "gemm_tc<128,DW>": (DW, FP32_TC, 300, 200, 500, 0),
    "gemm_dw": (DW, BF16X2, 2000, 1024, 2048, 0),
    "gemm_f32<FWD>": (FWD, FP32, 130, 129, 72, 0),
    "gemm_f32<DA>": (DA, FP32, 130, 129, 72, 0),
    "gemm_f32<DW>": (DW, FP32, 130, 129, 72, 0),
    "gemm_pp<FWD>": (FWD, BF16, 130, 129, 72, 0),       # np = 1 goes where the step sends it
    "gemm_wide": (FWD, BF16, 1024, 256, 1024, 8),       # 8 wide tiles on 8 SMs
}


@pytest.mark.gpu
@pytest.mark.parametrize("route", sorted(ROUTES))
def test_routes(sb, route):
    kind, prec, M, N, K, sms = ROUTES[route]
    got = {FWD: lambda: _fwd(sb, prec, M, N, K, "relu", sms=sms)[-1],
           DA: lambda: _da(sb, prec, M, N, K, "relu", sms=sms)[-1],
           DW: lambda: _dw(sb, prec, M, N, K, sms=sms)[-1]}[kind]()
    assert got == route


def test_routes_cover_every_instantiation():
    want = {"gemm_tc<%d,%s,GENERIC>" % (bn, e) for bn in (64, 128) for e in ("FWD", "DA")}
    want |= {"gemm_tc<64,DW>", "gemm_tc<128,DW>", "gemm_dw", "gemm_f32<FWD>", "gemm_f32<DA>", "gemm_f32<DW>"}
    assert want <= set(ROUTES)
    assert any(r.startswith("gemm_pp") for r in ROUTES) and "gemm_wide" in ROUTES


# ------------------------------------------------------------------------------------------------------------ no GPU
def _call(sb, kind=FWD, prec=FP32_TC, M=64, N=64, K=64, a_rows=None, row0=0, act=2, r0=0, r1=None, sms=0, clear_n4=0,
          drop=(), addend=False):
    import ctypes as C
    rows = K if kind == DW else M
    a_rows = rows if a_rows is None else a_rows
    buf = {k: np.ones(max(1, 4 * 256 * 256), np.float32) for k in ("A", "W", "bias", "aux", "out", "colsum", "grad")}
    buf["addend"] = buf["A"] if addend else None
    for k in drop:
        buf[k] = None
    if kind != FWD and "bias" not in drop:
        buf["bias"] = None
    guard = C.c_int32(-1)
    ptr = sb.capi._ptr
    return sb.capi.lib().sb_debug_gemm_layer(
        kind, prec, ptr(buf["A"]), ptr(buf["W"]), ptr(buf["bias"]), ptr(buf["aux"]), ptr(buf["addend"]), ptr(buf["out"]),
        ptr(buf["colsum"]), ptr(buf["grad"]), C.byref(guard), None, 0, M, N, K, a_rows, row0, act, r0,
        (M if r1 is None else r1), sms, clear_n4, 0)


INVALID = {
    "kind=3": dict(kind=3), "kind=-1": dict(kind=-1), "precision=4": dict(prec=4), "act=4": dict(act=4),
    "act=-2": dict(act=-2), "M=0": dict(M=0), "N=0": dict(N=0), "K=0": dict(K=0),
    "no_A": dict(drop=("A",)), "no_W": dict(drop=("W",)), "fwd_no_bias": dict(drop=("bias",)),
    "fwd_no_out": dict(drop=("out",)), "da_no_aux": dict(kind=DA, drop=("aux",)), "da_no_colsum": dict(kind=DA, drop=("colsum",)),
    "dw_no_grad": dict(kind=DW, drop=("grad",)), "addend_with_da": dict(kind=DA, addend=True),
    "addend_with_dw": dict(kind=DW, addend=True), "row0=-1": dict(row0=-1), "past_a_rows": dict(row0=5, a_rows=66),
    "resident_fp32": dict(prec=FP32, row0=2, a_rows=80), "resident_da": dict(kind=DA, a_rows=80),
    "resident_addend": dict(addend=True, a_rows=80), "r0_unaligned": dict(kind=DW, r0=4),
    "r1_past_M": dict(kind=DW, r1=65), "r0_not_below_r1": dict(kind=DW, r0=32, r1=32),
    "fp32_dw_chunk": dict(kind=DW, prec=FP32, r1=32), "sms=-1": dict(sms=-1), "clear_n4=-1": dict(clear_n4=-1),
    "clear_fp32": dict(prec=FP32, clear_n4=16), "clear_da": dict(kind=DA, clear_n4=16),
}


@pytest.mark.parametrize("case", sorted(INVALID))
def test_invalid_arguments_rejected_before_any_device_call(sb, case):
    # refused on a machine without a GPU, so no device work happens before the check
    assert _call(sb, **INVALID[case]) == sb.capi.SB_ERR_INVALID, sb.capi.lib().sb_last_error()


@pytest.mark.gpu
def test_sms_above_the_device_rejected(sb):
    assert _call(sb, sms=100000) == sb.capi.SB_ERR_INVALID
