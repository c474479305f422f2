"""The step's input stage bit for bit: the kernels that build layer 0's operand and the step scalars, through the step's own
launch code (sb_debug_first_kernel: the descriptor write, then enqueue_first), against the split done in numpy.

  HOST / SPARSE   load_batch_kernel<bf16 | fp32>: fp32 rows -> np bf16 parts in Xb (or an fp32 copy in Xf), pad columns,
                  n_nz, the cleared loss sum and gradient buffer
  RESIDENT        cast_bf16_kernel over 32768-row windows into the resident set and the host prefix counts dsP at load time;
                  set_batch_kernel publishes n_nz = P[row0 + rows] - P[row0]
  ORDERED         gather_batch_kernel<bf16 | fp32>: rows through the row order, y / w gathered, n_nz counted

The split is p_0 = bf16(x), p_{k+1} = bf16(r_k - p_k) with r_0 = x, every residual exact in fp32, so every comparison is of
bits.  Before each call Xb / Xf, y / w, the slot's scalars and the gradient buffer hold sentinel bits: whatever the stage
does not own must keep them."""
import ctypes as C

import numpy as np
import pytest

from conftest import bf16_round

FP32, BF16, FP32_TC, BF16X2 = 0, 1, 2, 3
NP = {FP32: 1, BF16: 1, FP32_TC: 3, BF16X2: 2}
TC = (BF16, FP32_TC, BF16X2)
S16, S32 = np.uint16(0x7FC1), np.uint32(0x7FC00123)      # sentinel bits (NaN patterns no kernel writes)
WIN = 32768                                             # rows per conversion window of sb_trainer_load_dataset
ROUTES = {"load_batch<bf16>", "load_batch<fp32>", "gather_batch<bf16>", "gather_batch<fp32>", "none"}


def ld8(n):
    return (n + 7) // 8 * 8


def split_bits(X, np_parts):
    """[np, rows, ld8(F)] uint16: the bf16 parts of X, pad columns +0"""
    X = np.ascontiguousarray(X, np.float32)
    rows, F = X.shape
    out = np.zeros((np_parts, rows, ld8(F)), np.uint16)
    r = X.copy()
    for k in range(np_parts):
        p = bf16_round(r)
        out[k, :, :F] = (p.view(np.uint32) >> 16).astype(np.uint16)
        r = (r - p).astype(np.float32)
    return out


def values(rng, rows, F):
    """normal values with every edge the split can meet mixed in: +-0, bf16 round-to-even ties, subnormals, values whose
    residual parts are subnormal, large finite values whose bf16 rounding stays finite, and 60 decades of magnitudes"""
    X = rng.standard_normal((rows, F)).astype(np.float32)
    n = X.size
    u = X.reshape(-1).view(np.uint32)
    kind = rng.integers(0, 9, n)
    rnd = rng.integers(0, 1 << 31, n, dtype=np.uint64).astype(np.uint32)
    sign = (rng.integers(0, 2, n).astype(np.uint32) << 31)
    exp = rng.integers(1, 254, n).astype(np.uint32) << 23
    u[kind == 1] = sign[kind == 1]                                                           # +-0
    tie = (rnd & 0x007F0000) | 0x8000                                                        # low half exactly 0x8000
    u[kind == 2] = (sign | exp | tie)[kind == 2]
    u[kind == 3] = (sign | (rnd & 0x007FFFFF) | 1)[kind == 3]                                # subnormal
    u[kind == 4] = (sign | (np.uint32(3 << 23) + (rnd & 0x00FFFFFF)))[kind == 4]             # parts 1, 2 subnormal
    big = np.array([3.0e38, 3.3e38, 1e38, 2.5e37], np.float32).view(np.uint32)
    u[kind == 5] = (sign | big[rnd % 4])[kind == 5]
    mag = (rng.standard_normal(n) * 10.0 ** rng.uniform(-30, 30, n)).astype(np.float32).view(np.uint32)
    u[kind == 6] = mag[kind == 6]
    X = u.view(np.float32).reshape(rows, F)
    assert np.isfinite(X).all() and np.isfinite(bf16_round(X)).all()
    return X


def weights(rng, rows):
    w = rng.uniform(0.1, 3.0, rows).astype(np.float32)
    k = rng.integers(0, 5, rows)
    w[k == 0] = 0.0
    w[k == 1] = -0.0           # == 0: not counted
    w[k == 2] *= -1            # negative: counted
    return w


def fill_sentinels(t, prec, max_batch, xcols):
    """every buffer the input stage may write: batch operand, y / w, slot (0, 0)'s scalars, gradient"""
    c = t.debug_buffer
    if prec == FP32:
        c(D.BATCH_X, np.full(max_batch * t.n_features, S32, np.uint32).view(np.float32))
    else:
        c(D.BATCH_X, np.full(NP[prec] * max_batch * xcols, S16, np.uint16))
    for b in (D.BATCH_Y, D.BATCH_W):
        c(b, np.full(max_batch, S32, np.uint32).view(np.float32))
    c(D.SCAL, np.full(4, S32, np.uint32).view(np.float32))
    c(D.GRAD, np.full(t.n_params, S32, np.uint32).view(np.float32))


class D:
    """buffer ids (filled from the binding at import time of the first test)"""


def _ids(sb):
    cp = sb.capi
    D.GRAD, D.BATCH_X, D.BATCH_Y, D.BATCH_W, D.SCAL = cp.DEBUG_BUF_GRAD, cp.DEBUG_BUF_BATCH_X, cp.DEBUG_BUF_BATCH_Y, \
        cp.DEBUG_BUF_BATCH_W, cp.DEBUG_BUF_SCAL
    D.DS_X, D.DS_Y, D.DS_W, D.DS_P = cp.DEBUG_BUF_DS_X, cp.DEBUG_BUF_DS_Y, cp.DEBUG_BUF_DS_W, cp.DEBUG_BUF_DS_P


def trainer(sb, F, prec, max_batch, hidden=8):
    _ids(sb)
    return sb.Trainer(sb.make_desc(F, [hidden], [2], max_batch=max_batch, precision=prec))


def read_x(t, prec, max_batch, xcols):
    if prec == FP32:
        return t.debug_buffer(D.BATCH_X, n=max_batch * t.n_features).view(np.uint32).reshape(max_batch, t.n_features)
    return t.debug_buffer(D.BATCH_X, n=NP[prec] * max_batch * xcols).reshape(NP[prec], max_batch, xcols)


def check_stage(t, prec, max_batch, X, y, w, *, xcols=None, yw_written=True, clear=True, grad_cleared=True, x_written=True):
    """after one hook call on rows X [rows, F] (y, w as the descriptor sees them; w None = all ones)"""
    rows, F = X.shape
    xcols = ld8(F) if xcols is None else xcols
    got = read_x(t, prec, max_batch, xcols)
    if not x_written:
        want_sent = got == (S32 if prec == FP32 else S16)
        assert want_sent.all(), "the batch operand was written"
    elif prec == FP32:
        np.testing.assert_array_equal(got[:rows], X.view(np.uint32))
        assert (got[rows:] == S32).all(), "rows past the batch were written"
    else:
        want = split_bits(X, NP[prec])
        assert want.shape[2] == xcols
        for k in range(NP[prec]):
            np.testing.assert_array_equal(got[k, :rows], want[k], err_msg="part %d" % k)
        assert (got[:, :rows, F:] == 0).all(), "pad columns must be +0 in every part"
        assert (got[:, rows:] == S16).all(), "rows past the batch were written"
    scal = t.debug_buffer(D.SCAL, n=4)
    wv = np.ones(rows, np.float32) if w is None else np.asarray(w, np.float32)
    assert scal[1] == float(np.count_nonzero(wv)), (scal[1], np.count_nonzero(wv))
    assert scal[0].view(np.uint32) == 0, "the loss sum must be cleared to +0"
    assert (scal[2:].view(np.uint32) == S32).all()
    if yw_written:
        gy = t.debug_buffer(D.BATCH_Y, n=max_batch)
        np.testing.assert_array_equal(gy[:rows].view(np.uint32), np.asarray(y, np.float32).view(np.uint32))
        assert (gy[rows:].view(np.uint32) == S32).all()
        if w is not None:
            gw = t.debug_buffer(D.BATCH_W, n=max_batch)
            np.testing.assert_array_equal(gw[:rows].view(np.uint32), wv.view(np.uint32))
            assert (gw[rows:].view(np.uint32) == S32).all()
    g = t.debug_buffer(D.GRAD).view(np.uint32)
    if clear and grad_cleared:
        assert (g == 0).all(), "the gradient buffer was not cleared"
    else:
        assert (g == S32).all(), "the gradient buffer was written"


# ------------------------------------------------------------------------------------------------------------ cases
FS = (1, 7, 8, 13, 200, 1000, 2000)
HOST_CASES = [(p, F) for p in (FP32, BF16, FP32_TC, BF16X2) for F in FS]
SPARSE_CASES = [(p, nd) for p in (BF16, FP32_TC) for nd in (5, 16)]
RESIDENT_CASES = list(TC)
FP32_RESIDENT_CASES = [7, 13, 8]
ORDERED_CASES = [(p, F) for p in (FP32, BF16, FP32_TC, BF16X2) for F in (7, 8, 13, 200)]


def expected_route(feed, prec):
    if feed == "resident":
        return "none"
    kind = "gather_batch" if feed == "ordered" else "load_batch"
    return "%s<%s>" % (kind, "fp32" if prec == FP32 else "bf16")


def all_routes():
    r = {expected_route("host", p) for p, _ in HOST_CASES}
    r |= {expected_route("host", p) for p, _ in SPARSE_CASES}
    r |= {expected_route("resident", p) for p in RESIDENT_CASES}
    r |= {expected_route("host", FP32) for _ in FP32_RESIDENT_CASES}
    r |= {expected_route("ordered", p) for p, _ in ORDERED_CASES}
    return r


def test_cases_reach_every_instantiation():
    assert all_routes() == ROUTES
    assert {F % 8 != 0 for F in FS} == {True, False} and {F % 4 != 0 for _, F in ORDERED_CASES} == {True, False}


@pytest.mark.gpu
@pytest.mark.parametrize("prec,F", HOST_CASES)
def test_host_feed(sb, prec, F):
    mb = 300
    rng = np.random.default_rng(F * 10 + prec)
    with trainer(sb, F, prec, mb) as t:
        for rows, wmode, clear in ((1, "w", True), (255, "w", False), (256, None, True), (257, "w", True), (mb, "zero", True)):
            X = values(rng, rows, F)
            y = rng.standard_normal(rows).astype(np.float32)
            w = None if wmode is None else (np.zeros(rows, np.float32) if wmode == "zero" else weights(rng, rows))
            fill_sentinels(t, prec, mb, ld8(F))
            assert t.debug_first_kernel(X, y, w, clear=clear) == expected_route("host", prec)
            check_stage(t, prec, mb, X, y, w, clear=clear, yw_written=True)


@pytest.mark.gpu
@pytest.mark.parametrize("prec,n_dense", SPARSE_CASES)
def test_sparse_dense_block(sb, prec, n_dense):
    mb, n_onehot, n_cat = 64, 12, 3
    rng = np.random.default_rng(n_dense + prec)
    with trainer(sb, n_dense + n_onehot, prec, mb) as t:
        t.set_sparse(n_dense, n_onehot, n_cat)
        for rows in (1, 37, mb):
            X = values(rng, rows, n_dense)
            idx = rng.integers(-1, n_onehot, (rows, n_cat)).astype(np.int32)
            y = rng.standard_normal(rows).astype(np.float32)
            w = weights(rng, rows)
            fill_sentinels(t, prec, mb, ld8(n_dense))
            assert t.debug_first_kernel(X, y, w, idx=idx, clear=True) == expected_route("host", prec) + "+embed_gather"
            check_stage(t, prec, mb, X, y, w, xcols=ld8(n_dense))


def _resident_set(rng, n_rows, F):
    X = values(rng, n_rows, F)
    y = rng.standard_normal(n_rows).astype(np.float32)
    w = weights(rng, n_rows)
    w[-3:] = 0.0                               # n_nz of a batch at the very end of the set
    return X, y, w


@pytest.mark.gpu
@pytest.mark.parametrize("prec", RESIDENT_CASES)
def test_resident_set_and_nnz(sb, prec):
    F, mb, n_rows = 13, 512, 2 * WIN + 77
    rng = np.random.default_rng(prec)
    X, y, w = _resident_set(rng, n_rows, F)
    P = np.concatenate([[0], np.cumsum(w != 0)]).astype(np.int32)
    with trainer(sb, F, prec, mb) as t:
        t.load_dataset(X, y, w)
        got = t.debug_buffer(D.DS_X, n=NP[prec] * n_rows * ld8(F)).reshape(NP[prec], n_rows, ld8(F))
        want = split_bits(X, NP[prec])
        for k in range(NP[prec]):
            np.testing.assert_array_equal(got[k], want[k], err_msg="resident part %d" % k)
        np.testing.assert_array_equal(t.debug_buffer(D.DS_P, n=n_rows + 1), P)
        np.testing.assert_array_equal(t.debug_buffer(D.DS_Y, n=n_rows).view(np.uint32), y.view(np.uint32))
        np.testing.assert_array_equal(t.debug_buffer(D.DS_W, n=n_rows).view(np.uint32), w.view(np.uint32))
        for row0, rows in ((0, 1), (WIN - 1, 2), (WIN - 200, mb), (2 * WIN - 200, 256), (2 * WIN, 77), (n_rows - mb, mb),
                           (n_rows - 1, 1), (n_rows - 3, 3)):
            fill_sentinels(t, prec, mb, ld8(F))
            assert t.debug_first_kernel(row_offset=row0, rows=rows, clear=True) == "none"
            scal = t.debug_buffer(D.SCAL, n=4)
            assert scal[1] == float(P[row0 + rows] - P[row0]) == float(np.count_nonzero(w[row0:row0 + rows]))
            assert scal[0].view(np.uint32) == 0 and (scal[2:].view(np.uint32) == S32).all()
            # layer 0 reads the set in place: nothing else of the input stage is written, not even the gradient
            check_stage(t, prec, mb, X[row0:row0 + rows], None, w[row0:row0 + rows], yw_written=False, grad_cleared=False,
                        x_written=False)


@pytest.mark.gpu
def test_resident_set_from_device_arrays(sb):
    """w as a device array (what the GPU text ingest hands over) gives the same prefix counts and weights"""
    F, n_rows = 5, 2 * WIN + 77
    rng = np.random.default_rng(3)
    wtxt = rng.choice(["0", "-0", "2.5", "-1.25", "0.5", "1"], n_rows)
    feats = rng.integers(-999, 999, (n_rows, F))
    lines = ["%d|%s|%s" % (i & 1, "|".join(str(v) for v in feats[i]), wtxt[i]) for i in range(n_rows)]
    text = ("\n".join(lines) + "\n").encode()
    col_map = [sb.capi.COL_TARGET] + list(range(F)) + [sb.capi.COL_WEIGHT]
    Xd, yd, wd, fl, _, _ = sb.capi.text_parse_device(text, col_map, F)
    assert fl == []
    wh = wd.numpy()
    want_w = np.array([1.0 if float(s) < 0 else float(s) for s in wtxt], np.float32)
    np.testing.assert_array_equal(wh.view(np.uint32), want_w.view(np.uint32))
    P = np.concatenate([[0], np.cumsum(want_w != 0)]).astype(np.int32)
    with trainer(sb, F, BF16, 256) as a, trainer(sb, F, BF16, 256) as b:
        a.load_dataset(Xd, yd, wd)
        b.load_dataset(Xd.numpy(), yd.numpy(), wh)
        for t in (a, b):
            np.testing.assert_array_equal(t.debug_buffer(D.DS_P, n=n_rows + 1), P)
            np.testing.assert_array_equal(t.debug_buffer(D.DS_W, n=n_rows).view(np.uint32), want_w.view(np.uint32))
        np.testing.assert_array_equal(a.debug_buffer(D.DS_X, n=n_rows * 8), b.debug_buffer(D.DS_X, n=n_rows * 8))


@pytest.mark.gpu
@pytest.mark.parametrize("F", FP32_RESIDENT_CASES)
def test_fp32_resident_feed(sb, F):
    """the fp32 set is read in place through the host feed: odd offsets with odd F leave desc->X 16-byte misaligned"""
    mb, n_rows = 300, 1001
    rng = np.random.default_rng(F)
    X, y, w = _resident_set(rng, n_rows, F)
    with trainer(sb, F, FP32, mb) as t:
        t.load_dataset(X, y, w)
        np.testing.assert_array_equal(t.debug_buffer(D.DS_X, n=n_rows * F).view(np.uint32), X.reshape(-1).view(np.uint32))
        for off, rows in ((0, mb), (1, 257), (3, 256), (5, 1), (n_rows - mb, mb), (n_rows - 1, 1)):
            fill_sentinels(t, FP32, mb, F)
            assert t.debug_first_kernel(row_offset=off, rows=rows, clear=True) == "load_batch<fp32>"
            # y / w stay in the set (the staging buffers keep their sentinels)
            check_stage(t, FP32, mb, X[off:off + rows], None, w[off:off + rows], yw_written=False)
            assert (t.debug_buffer(D.BATCH_Y, n=mb).view(np.uint32) == S32).all()


@pytest.mark.gpu
@pytest.mark.parametrize("prec,F", ORDERED_CASES)
def test_ordered_feed_equals_host_feed(sb, prec, F):
    mb, n_rows = 260, 900
    rng = np.random.default_rng(100 * F + prec)
    X, y, w = _resident_set(rng, n_rows, F)
    order = rng.permutation(n_rows)
    order[7] = order[9] = order[400]                       # a repeated row
    with trainer(sb, F, prec, mb) as t:
        t.load_dataset(X, y, w)
        t.set_row_order(order)
        for off, rows, clear in ((0, mb, True), (5, 257, False), (123, 1, True), (n_rows - 256, 256, True)):
            sel = order[off:off + rows]
            fill_sentinels(t, prec, mb, ld8(F))
            assert t.debug_first_kernel(row_offset=off, rows=rows, clear=clear) == expected_route("ordered", prec)
            check_stage(t, prec, mb, X[sel], y[sel], w[sel], clear=clear)
            ordered = read_x(t, prec, mb, ld8(F)).copy()
            t.set_row_order(None)                          # the host feed of the same rows, through the staging buffers
            fill_sentinels(t, prec, mb, ld8(F))
            t.debug_first_kernel(X[sel], y[sel], w[sel], clear=clear)
            np.testing.assert_array_equal(read_x(t, prec, mb, ld8(F)), ordered)
            t.set_row_order(order)


@pytest.mark.gpu
@pytest.mark.parametrize("prec,feed", [(FP32_TC, "host"), (BF16, "ordered")])
def test_cfg2_batch(sb, prec, feed):
    """8192 x 2000: rows * ldF / 8 units are far more than the 16-blocks-per-SM grid, so every grid-stride loop turns"""
    F, mb = 2000, 8192
    rng = np.random.default_rng(2000 + prec)
    with trainer(sb, F, prec, mb, hidden=16) as t:
        if feed == "host":
            X = values(rng, mb, F)
            y = rng.standard_normal(mb).astype(np.float32)
            w = weights(rng, mb)
            fill_sentinels(t, prec, mb, F)
            assert t.debug_first_kernel(X, y, w, clear=True) == "load_batch<bf16>"
            check_stage(t, prec, mb, X, y, w)
        else:
            Xs, ys, ws = _resident_set(rng, mb + 100, F)
            order = rng.permutation(mb + 100)
            t.load_dataset(Xs, ys, ws)
            t.set_row_order(order)
            sel = order[50:50 + mb]
            fill_sentinels(t, prec, mb, F)
            assert t.debug_first_kernel(row_offset=50, rows=mb, clear=True) == "gather_batch<bf16>"
            check_stage(t, prec, mb, Xs[sel], ys[sel], ws[sel])


# ------------------------------------------------------------------------------------------------------------ arguments
def test_header_ids_match_binding(sb):
    import os
    import re
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "shifu_b200.h")).read()
    names = ("BATCH_Y", "BATCH_W", "SCAL", "DS_X", "DS_Y", "DS_W", "DS_P")
    assert re.search(r"#define SB_DEBUG_BUF_BATCH_X \(SB_DEBUG_BUF_SHADOW \+ SB_MAX_HIDDEN\)", hdr)
    assert sb.capi.DEBUG_BUF_BATCH_X == sb.capi.DEBUG_BUF_SHADOW + sb.capi.SB_MAX_HIDDEN
    for k, nm in enumerate(names, 1):
        assert "#define SB_DEBUG_BUF_%s (SB_DEBUG_BUF_BATCH_X + %d)" % (nm, k) in hdr
        assert getattr(sb.capi, "DEBUG_BUF_" + nm) == sb.capi.DEBUG_BUF_BATCH_X + k


def _buf_call(sb, which, n=4, write=0, t=None):
    buf = np.zeros(max(n, 1), np.float32)
    return sb.capi.lib().sb_debug_trainer_buffer(t, which, buf.ctypes.data_as(C.c_void_p), n, write)


def _err(sb):
    return sb.capi.lib().sb_last_error().decode()


@pytest.mark.parametrize("which", [-1, 4 + 32 + 8, 1000])
def test_buffer_bad_id(sb, which):
    assert _buf_call(sb, which) == sb.capi.SB_ERR_INVALID and "not a buffer id" in _err(sb)


@pytest.mark.parametrize("which", ["DS_X", "DS_Y", "DS_W", "DS_P"])
def test_buffer_resident_ids_are_read_only(sb, which):
    assert _buf_call(sb, getattr(sb.capi, "DEBUG_BUF_" + which), write=1) == sb.capi.SB_ERR_INVALID and "read-only" in _err(sb)


def test_buffer_write_modes_and_null_trainer(sb):
    cp = sb.capi
    assert _buf_call(sb, cp.DEBUG_BUF_SCAL, write=2) == cp.SB_ERR_INVALID and "write = 2" in _err(sb)
    assert _buf_call(sb, cp.DEBUG_BUF_BATCH_X, write=-1) == cp.SB_ERR_INVALID and "write = -1" in _err(sb)
    for which in (cp.DEBUG_BUF_BATCH_X, cp.DEBUG_BUF_SCAL, cp.DEBUG_BUF_DS_P):
        assert _buf_call(sb, which) == cp.SB_ERR_INVALID and "null argument" in _err(sb)


def _hook_call(sb, t=None, X=True, y=True, w=False, idx=False, row_offset=0, rows=4, clear=0, route_cap=64):
    a = np.zeros(64, np.float32)
    i = np.zeros(64, np.int32)
    ptr = sb.capi._ptr
    route = C.create_string_buffer(64)
    return sb.capi.lib().sb_debug_first_kernel(t, ptr(a) if X else None, ptr(a) if y else None, ptr(a) if w else None,
                                               i.ctypes.data_as(C.POINTER(C.c_int32)) if idx else None, row_offset, rows,
                                               clear, route if route_cap > 0 else None, route_cap)


@pytest.mark.parametrize("kw,msg", [
    (dict(clear=2), "clear = 2"), (dict(clear=-1), "clear = -1"), (dict(route_cap=-1), "route_cap -1"),
    (dict(X=False, y=True), "take no y"), (dict(X=False, y=False, w=True), "take no y"),
    (dict(X=False, y=False, idx=True), "take no y"), (dict(y=False), "need y"), (dict(row_offset=3), "row_offset"),
    (dict(), "null trainer"), (dict(X=False, y=False, row_offset=5), "null trainer")])
def test_first_kernel_arguments(sb, kw, msg):
    assert _hook_call(sb, **kw) == sb.capi.SB_ERR_INVALID and msg in _err(sb)


@pytest.mark.gpu
def test_buffer_sizes_and_states(sb):
    cp = sb.capi
    with trainer(sb, 13, FP32_TC, 32) as t, trainer(sb, 13, FP32, 32) as f:
        h = t._h
        assert _buf_call(sb, cp.DEBUG_BUF_BATCH_X, n=3 * 32 * 16, t=h) == cp.SB_OK
        for which, good in ((cp.DEBUG_BUF_BATCH_X, 3 * 32 * 16), (cp.DEBUG_BUF_BATCH_Y, 32), (cp.DEBUG_BUF_SCAL, 4)):
            for n in (good - 1, good + 1):
                assert _buf_call(sb, which, n=n, t=h) == cp.SB_ERR_INVALID and "expected %d values" % good in _err(sb)
        assert _buf_call(sb, cp.DEBUG_BUF_BATCH_X, n=32 * 13, t=f._h) == cp.SB_OK
        for which in (cp.DEBUG_BUF_DS_X, cp.DEBUG_BUF_DS_Y, cp.DEBUG_BUF_DS_W, cp.DEBUG_BUF_DS_P):
            assert _buf_call(sb, which, n=4, t=h) == cp.SB_ERR_STATE and "no resident dataset" in _err(sb)
        with pytest.raises(sb.ShifuB200Error) as e:
            t.debug_first_kernel(row_offset=0, rows=4)
        assert e.value.code == cp.SB_ERR_STATE
        with pytest.raises(sb.ShifuB200Error) as e:
            t.debug_first_kernel(np.zeros((33, 13), np.float32), np.zeros(33, np.float32))
        assert e.value.code == cp.SB_ERR_INVALID and "max_batch" in str(e.value)
        f.load_dataset(np.zeros((40, 13), np.float32), np.zeros(40, np.float32))
        assert _buf_call(sb, cp.DEBUG_BUF_DS_P, n=41, t=f._h) == cp.SB_ERR_STATE and "no prefix counts" in _err(sb)
        assert _buf_call(sb, cp.DEBUG_BUF_DS_W, n=41, t=f._h) == cp.SB_ERR_INVALID
        with pytest.raises(sb.ShifuB200Error) as e:
            f.debug_first_kernel(row_offset=30, rows=11)
        assert e.value.code == cp.SB_ERR_INVALID and "outside the resident set" in str(e.value)
