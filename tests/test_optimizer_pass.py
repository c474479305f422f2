"""Kernel-level checks of the single-GPU optimizer pass (optimizer_kernel<OPT_BASE / OPT_EXT> in csrc/kernels.cuh) and of the
bf16 shadow refresh (shadow_refresh_kernel), through the trainer's own launch code.

Each pass case builds a world-1 trainer, writes its raw arena buffers (sb_debug_trainer_buffer): theta, s1 and s2, every
part of every shadow filled with a sentinel, then, before each of three consecutive passes, a fresh gradient.
sb_debug_optimizer queues one update as the trainer does: the descriptor of the next update, then either one launch over
the whole work table (apply_accumulated, a step without the split tail) or the step's split tail (layer 0's runs on the
main stream, the others on the side stream, then the join).  After each pass every raw buffer is compared with a model
built here from a Python restatement of Net::build_work, not from anything the kernel reports:

  master and state   theta, s1, s2 of every run of the work table against opt_ref.reference (float64 evaluation of
                     opt_update on the float32 inputs, g = float32(grad * gscale)), within the bound derived there; FTRL's
                     l1 branch apart from the bound
  untouched          the state streams an optimizer does not have (s1 of SGD; s2 of SGD, Momentum and Adagrad), the raw
                     gradient, and theta / s1 / s2 / shadow of frozen parameters (fixed_layers) keep their bits
  operands           every part of every shadow-backed run is the bf16 (round to nearest even) of bf16_residual(new
                     theta, part), bit for bit, and the pad columns keep the sentinel
  lr_t, launches     lr_t is float32(lr), for Adam within 1e-6 of the float64 bias correction at steps 1, 2, 3; the
                     route names the instantiation, the stream and the run range of each launch
The exact case (SGD, lr = 2^-4, gscale = 1/4, dyadic theta and gradients) has no rounding anywhere and must match the
float64 result bit for bit.  The shadow-refresh cases check every part of every layer's shadow after
debug_buffer(theta, refresh_shadows=True), set_params and load_checkpoint, on values where bf16 rounding has edges."""
import zlib

import numpy as np
import pytest

from opt_ref import (ADADELTA, ADAGRAD, ADAM, BETA1, BETA2, BF16, BF16X2, C_BOUND, EPS, EXT, FP32, FP32_TC, FTRL, MOM,
                     MOMENTUM, NPARTS, ONAME, PNAME, RHO, RMSPROP, SGD, U, _bits_equal, check_l1_branch, lr_t_of, reference,
                     s1_start, shadow_bits, uses_s1, uses_s2)

# nets (features, hidden widths): the layouts of the work runs
NETS = {
    "m8": (200, [64, 48]),              # widths % 8 == 0: every run on the 16-byte path
    "odd": (150, [45, 30, 7]),          # widths = 1, 2, 3 mod 4: shadow-backed runs on the element path; fp32: unaligned runs
    "tiny": (8, [8]),                   # one hidden layer; with W_out frozen a run of one element (b_out)
    "cfg2": (2000, [1024, 512, 256]),   # the benchmark's cfg2 shape
}
# frozen sets (fixed_layers, fixed_bias): layers numbered from 1, the output layer is n_hidden + 1
FROZEN = {"none": ((), True), "l1": ((1,), True), "l2b": ((2,), False)}
LR = {SGD: 0.05, MOMENTUM: 0.05, ADAM: 0.003, ADADELTA: 1.0, ADAGRAD: 0.05, RMSPROP: 0.003, FTRL: 0.05}
FTRL_L1, FTRL_L2 = 0.5, 0.25
SENTINEL = 0x7FA0

_worst = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if _worst:
        print("\nworst error / bound: " + ", ".join("%s %.3g" % kv for kv in sorted(_worst.items())))


def _note(name, err, tol):
    if err.size:
        _worst[name] = max(_worst.get(name, 0.0), float(np.max(err / tol)))


def trains(L, fixed, fix_bias):
    """w_trains / b_trains of layers 0..L (sb_trainer_set_fixed_layers)"""
    w, b = [True] * (L + 1), [True] * (L + 1)
    for x in fixed:
        w[x - 1] = False
        if fix_bias:
            b[x - 1] = False
    return w, b


def build_work(F, hidden, prec, w_trains, b_trains):
    """Net::build_work -> (runs as debug_exchange_layout reports them, begin[l], end[l])"""
    L, tc, npart = len(hidden), prec != FP32, NPARTS[prec]
    work, begin, end = [], [], []
    off, prev, lays = 0, F, []
    for l in range(L + 1):
        o = hidden[l] if l < L else 1
        lays.append((prev, o, off, off + prev * o))
        off += prev * o + o
        prev = o

    def add(o, n, l):
        for s in range(0, n, 1024):
            w = dict(off=o + s, count=min(1024, n - s), out_dim=0, mat_off=0, ld_out=0, np=1, layer=-1, part_stride=0)
            if l is not None:
                i, out, w_off, _ = lays[l]
                ld = -(-out // 8) * 8
                w.update(out_dim=out, mat_off=w_off, ld_out=ld, np=npart, layer=l, part_stride=-(-(i * ld * 2) // 256) * 128)
            work.append(w)

    for l, (i, o, w_off, b_off) in enumerate(lays):
        begin.append(len(work))
        if tc and l < L:
            if w_trains[l]:
                add(w_off, i * o, l)
            if b_trains[l]:
                add(b_off, o, None)
        elif w_trains[l] and b_trains[l]:
            add(w_off, i * o + o, None)
        else:
            if w_trains[l]:
                add(w_off, i * o, None)
            if b_trains[l]:
                add(b_off, o, None)
        end.append(len(work))
    return work, begin, end


def table(net, prec, fixed):
    F, hidden = NETS[net]
    return build_work(F, hidden, prec, *trains(len(hidden), *FROZEN[fixed]))


def vec_path(w):
    """optimizer_kernel's condition for the 16-byte path of a run"""
    return (w["off"] % 4 == 0 and w["count"] % 4 == 0 and
            (w["layer"] < 0 or (w["out_dim"] % 4 == 0 and (w["off"] - w["mat_off"]) % 4 == 0)))


def predicted_route(kind, work, begin, end, tail):
    inst = "optimizer<%s>" % ("ext" if kind in EXT else "base")
    launches = [("main", 0, len(work))] if not tail else [("main", begin[0], end[0]), ("side", end[0], len(work))]
    return "+".join("%s@%s[%d,%d)" % (inst, st, a, b) for st, a, b in launches if b > a)


def make_trainer(sb, prec, net, kind, lr, fixed):
    F, hidden = NETS[net]
    fz, fix_bias = FROZEN[fixed]
    desc = sb.make_desc(F, hidden, [sb.ACT_RELU] * len(hidden), optimizer=kind, learning_rate=lr, rho=RHO, epsilon=EPS,
                        beta1=BETA1, beta2=BETA2, momentum=MOM, max_batch=8, precision=prec)
    kw = dict(initial_accumulator=0.25, l1=FTRL_L1 if kind == FTRL else 0.0, l2=FTRL_L2 if kind == FTRL else 0.0) \
        if kind in (ADAGRAD, FTRL) else {}
    return sb.Trainer(desc, device=0, fixed_layers=fz, fixed_bias=fix_bias, **kw)


def shadow_dims(net, prec):
    F, hidden = NETS[net]
    return [(hidden[l - 1] if l else F, hidden[l]) for l in range(len(hidden))] if prec != FP32 else []


def read_shadows(sb, t, prec, dims):
    n = NPARTS[prec]
    return [t.debug_buffer(sb.capi.DEBUG_BUF_SHADOW + l, n=n * i * (-(-o // 8) * 8)).reshape(n, i, -1) for l, (i, o) in
            enumerate(dims)]


def fill_shadows(sb, t, prec, dims):
    sh = [np.full((NPARTS[prec], i, -(-o // 8) * 8), SENTINEL, np.uint16) for (i, o) in dims]
    for l, s in enumerate(sh):
        t.debug_buffer(sb.capi.DEBUG_BUF_SHADOW + l, s)
    return sh


class OptPass:
    """a world-1 trainer, its raw buffers and the model of what they must hold"""

    def __init__(self, sb, prec, net, kind, fixed, seed, exact):
        self.sb, self.prec, self.kind, self.exact = sb, prec, kind, exact
        self.lr = 2.0 ** -4 if exact else LR[kind]
        self.l1, self.l2 = (FTRL_L1, FTRL_L2) if kind == FTRL else (0.0, 0.0)
        self.t = make_trainer(sb, prec, net, kind, self.lr, fixed)
        self.work, self.begin, self.end = table(net, prec, fixed)
        lay = self.t.debug_exchange_layout()
        assert lay["world"] == 1 and lay["np"] == NPARTS[prec]
        assert lay["work"] == self.work
        self.n = self.t.n_params
        self.dims = shadow_dims(net, prec)
        # the elements of the work table, and per hidden layer the (rows, cols) of its shadow-backed elements
        runs = [np.arange(w["off"], w["off"] + w["count"]) for w in self.work]
        self.idx = np.concatenate(runs) if runs else np.zeros(0, np.int64)
        self.sh_at = []
        for l in range(len(self.dims)):
            pos = [r for r, w in zip(runs, self.work) if w["layer"] == l]
            if not pos:
                self.sh_at.append(None)
                continue
            w = next(w for w in self.work if w["layer"] == l)
            m = np.concatenate(pos) - w["mat_off"]
            self.sh_at.append((np.concatenate(pos), m // w["out_dim"], m % w["out_dim"]))
        self.rng = rng = np.random.default_rng(seed)
        if exact:
            self.theta = (rng.integers(-512, 512, self.n) * 2.0 ** -8).astype(np.float32)
        else:
            self.theta = (rng.standard_normal(self.n) * 0.5).astype(np.float32)
        self.s1 = s1_start(kind, rng.standard_normal(self.n) * 0.1)
        sq = kind in (ADAM, ADADELTA)
        self.s2 = (np.abs(rng.standard_normal(self.n)) * 0.01 if sq else rng.standard_normal(self.n)).astype(np.float32)
        c = sb.capi
        self.t.debug_buffer(c.DEBUG_BUF_THETA, self.theta)
        self.t.debug_buffer(c.DEBUG_BUF_S1, self.s1)
        self.t.debug_buffer(c.DEBUG_BUF_S2, self.s2)
        self.shadow = fill_shadows(sb, self.t, prec, self.dims)
        self.step = 0

    def close(self):
        self.t.close()

    def draw_grad(self):
        rng, n = self.rng, self.n
        if self.exact:
            return (rng.integers(-4096, 4096, n) * 2.0 ** -12).astype(np.float32)
        g = rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 1, n)
        k = max(1, n // 32)
        sel = rng.choice(n, 2 * k, replace=False)
        g[sel[:k]] = 0.0                                                              # exact zeros
        g[sel[k:]] = rng.choice([-1.0, 1.0], k) * 10.0 ** rng.uniform(-30, -24, k)   # g * g underflows in float32
        return g.astype(np.float32)

    def run(self, gscale, tail):
        sb, c, t = self.sb, self.sb.capi, self.t
        grad = self.draw_grad()
        t.debug_buffer(c.DEBUG_BUF_GRAD, grad)
        lr_t, route = t.debug_optimizer(gscale, tail)
        t.sync()
        self.step += 1
        assert route == predicted_route(self.kind, self.work, self.begin, self.end, tail)
        lr = float(np.float32(self.lr))
        if self.kind == ADAM:
            assert abs(lr_t - lr_t_of(ADAM, lr, self.step)) <= 1e-6 * lr_t
        else:
            assert lr_t == lr
        gs = np.float32(gscale if gscale > 0 else 1.0)
        got_t, got_1, got_2, got_g = (t.debug_buffer(b) for b in (c.DEBUG_BUF_THETA, c.DEBUG_BUF_S1, c.DEBUG_BUF_S2,
                                                                  c.DEBUG_BUF_GRAD))
        got_sh = read_shadows(sb, t, self.prec, self.dims)
        _bits_equal(got_g, grad, "raw gradient")
        idx, name = self.idx, ONAME[self.kind]
        g = (grad[idx] * gs).astype(np.float32)
        rt, r1, r2, St, S1, S2 = reference(self.kind, lr_t, self.theta[idx], self.s1[idx], self.s2[idx], g, self.l1, self.l2)
        gt = got_t[idx]
        if self.exact:
            assert np.array_equal(rt.astype(np.float32).astype(np.float64), rt)
            _bits_equal(gt, rt.astype(np.float32), "exact theta")
        use1, use2 = uses_s1(self.kind), uses_s2(self.kind)
        for q, gv, rv, S, used in (("theta", gt, rt, St, True), ("s1", got_1[idx], r1, S1, use1),
                                   ("s2", got_2[idx], r2, S2, use2)):
            if not used:
                continue
            err = np.abs(gv.astype(np.float64) - rv)
            tol = C_BOUND * U * S + 1e-45
            _note("%s %s" % (name, q), err, tol)
            bad = np.flatnonzero(err > tol)
            assert bad.size == 0, "%s of %d elements: worst error / bound %.3g, first at parameter %s" % (
                q, bad.size, float(np.max(err / tol)), idx[bad[:8]])
        check_l1_branch(self.kind, gt, r2, S2, self.l1, "theta")
        exp_t, exp_1, exp_2 = self.theta.copy(), self.s1.copy(), self.s2.copy()
        exp_t[idx] = gt
        if use1:
            exp_1[idx] = got_1[idx]
        if use2:
            exp_2[idx] = got_2[idx]
        # everything outside the work table (frozen parameters) and the streams the optimizer does not have keep their bits
        _bits_equal(got_t, exp_t, "raw theta")
        _bits_equal(got_1, exp_1, "raw s1")
        _bits_equal(got_2, exp_2, "raw s2")
        exp_sh = [s.copy() for s in self.shadow]
        for l, at in enumerate(self.sh_at):
            if at is None:
                continue
            pos, rows, cols = at
            for part in range(NPARTS[self.prec]):
                exp_sh[l][part, rows, cols] = shadow_bits(got_t[pos], part)
        for l in range(len(got_sh)):
            _bits_equal(got_sh[l], exp_sh[l], "shadow of layer %d" % l)
        self.theta, self.s1, self.s2, self.shadow = got_t, got_1, got_2, exp_sh


# (precision, optimizer, net, frozen set, tail, gscale, exact)
def _cases():
    out = []
    for opt in ONAME:                                        # every optimizer and precision, both run layouts
        for prec in PNAME:
            for nb, net in enumerate(("m8", "odd")):
                out.append((prec, opt, net, "none", (opt + prec + nb) % 2, (1.0, 0.2)[(opt + prec // 2 + nb) % 2], False))
    for prec in PNAME:                                       # one hidden layer; a one-element run (b_out alone trains)
        out.append((prec, (SGD, ADAM, FTRL, RMSPROP)[prec], "tiny", "none", 0, 1.0, False))
        out.append((prec, (MOMENTUM, ADAGRAD, ADADELTA, FTRL)[prec], "tiny", "l2b", 0, 0.2, False))
    for prec, opt, tail, gscale in ((BF16, ADAM, 1, 1.0), (FP32_TC, ADAM, 0, 0.2), (BF16, FTRL, 0, 0.2),
                                    (FP32_TC, FTRL, 1, 1.0)):    # the benchmark's cfg2 shape
        out.append((prec, opt, "cfg2", "none", tail, gscale, False))
    k = 0
    for fixed in ("l1", "l2b"):                               # shrunk tables; l1: the split tail's layer-0 range is empty
        for prec in PNAME:
            for tail in (0, 1):
                out.append((prec, list(ONAME)[k % 7], ("m8", "odd")[k % 2], fixed, tail, (1.0, 0.2)[(k // 2) % 2], False))
                k += 1
    for prec, net, tail in ((FP32, "m8", 0), (BF16, "odd", 1), (FP32_TC, "m8", 1), (BF16X2, "odd", 0)):   # no rounding
        out.append((prec, SGD, net, "none", tail, 0.25, True))
    return list(dict.fromkeys(out))


CASES = _cases()


def _id(c):
    prec, opt, net, fixed, tail, gscale, exact = c
    return "%s-%s-%s-%s-%s-gs%g%s" % (PNAME[prec], ONAME[opt], net, fixed, ("pass", "tail")[tail], gscale,
                                      "-exact" if exact else "")


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_optimizer_pass_against_float64(sb, case):
    prec, opt, net, fixed, tail, gscale, exact = case
    p = OptPass(sb, prec, net, opt, fixed, seed=zlib.crc32(_id(case).encode()), exact=exact)
    try:
        for _ in range(3):
            p.run(gscale, tail)
    finally:
        p.close()


def test_case_matrix_reaches_every_kernel_path():
    seen = set()
    for prec, opt, net, fixed, tail, gscale, exact in CASES:
        work, begin, end = table(net, prec, fixed)
        seen.add(("instantiation", opt in EXT))
        for w in work:
            seen.add(("path", vec_path(w)))
            if w["layer"] >= 0:
                seen.add(("shadow np", w["np"], vec_path(w)))
            if w["count"] < 4:
                seen.add("run shorter than 4")
        if tail:
            assert len(NETS[net][1]) > 1
            if begin[0] == end[0]:
                seen.add("split tail without layer-0 runs")
        if exact:
            seen.add(("exact", "tail", tail))
            seen |= {("exact", "path", vec_path(w)) for w in work}
    want = {("instantiation", False), ("instantiation", True), ("path", True), ("path", False),
            "run shorter than 4", "split tail without layer-0 runs"}
    want |= {("shadow np", n, v) for n in (1, 2, 3) for v in (True, False)}
    want |= {("exact", "tail", 0), ("exact", "tail", 1), ("exact", "path", True), ("exact", "path", False)}
    assert want <= seen, want - seen
    # every optimizer in every precision, both ways of running the update and both gradient scales
    assert {(c[0], c[1]) for c in CASES} == {(p, o) for p in PNAME for o in ONAME}
    for opt in ONAME:
        assert {c[4] for c in CASES if c[1] == opt} == {0, 1}
        assert {c[5] for c in CASES if c[1] == opt and not c[6]} == {1.0, 0.2}
    assert {(c[2], c[3]) for c in CASES} >= {("cfg2", "none"), ("tiny", "l2b"), ("m8", "l1"), ("odd", "l1"), ("m8", "l2b"),
                                             ("odd", "l2b")}
    assert {(c[0], c[1]) for c in CASES if c[2] == "cfg2"} == {(p, o) for p in (BF16, FP32_TC) for o in (ADAM, FTRL)}


@pytest.mark.gpu
def test_restated_work_table_matches_the_trainer(sb):
    for net in NETS:
        for fixed in FROZEN:
            for prec in PNAME:
                t = make_trainer(sb, prec, net, SGD, 0.05, fixed)
                try:
                    assert t.debug_exchange_layout()["work"] == table(net, prec, fixed)[0], (net, fixed, PNAME[prec])
                finally:
                    t.close()


def test_optimizer_hook_rejects_bad_arguments_without_a_trainer(sb):
    lib, c = sb.capi.lib(), sb.capi
    assert lib.sb_debug_optimizer(None, 0.0, 0, None, None, 0) == c.SB_ERR_INVALID


@pytest.mark.gpu
def test_optimizer_hook_rejects_bad_arguments(sb):
    c = sb.capi
    F, hidden = NETS["tiny"]
    lone = sb.Trainer(sb.make_desc(F, hidden, [sb.ACT_RELU], precision=BF16, max_batch=8), device=0, nccl_id=None, rank=0,
                      world=2)
    try:
        with pytest.raises(sb.ShifuB200Error) as e:            # a peer or NCCL rank
            lone.debug_optimizer()
        assert e.value.code == c.SB_ERR_STATE
        for kw in (dict(gscale=-1.0), dict(gscale=float("nan")), dict(gscale=float("inf")), dict(tail=2), dict(tail=-1)):
            with pytest.raises(sb.ShifuB200Error) as e:
                lone.debug_optimizer(**kw)
            assert e.value.code == c.SB_ERR_INVALID
        assert lone.global_step == 0
    finally:
        lone.close()
    p = OptPass(sb, BF16, "tiny", MOMENTUM, "none", seed=2, exact=False)
    try:
        for kw in (dict(tail=1), dict(gscale=-0.5), dict(tail=3)):   # one hidden layer: no split tail
            with pytest.raises(sb.ShifuB200Error) as e:
                p.t.debug_optimizer(**kw)
            assert e.value.code == c.SB_ERR_INVALID
        # nothing was queued by the refused calls: the first pass is step 1 and matches the model
        assert p.t.global_step == 0
        p.run(0.0, 0)
    finally:
        p.close()


# ---- shadow refresh ----
def edge_theta(rng, n):
    """theta with the edges of bf16 rounding: round-to-nearest-even ties (both directions), values exact in bf16 (their
    residual parts are +0), -0.0, float32 subnormals and large magnitudes below the bf16 overflow threshold"""
    v = (rng.standard_normal(n) * 0.5).astype(np.float32)
    bits = v.view(np.uint32)
    kind = rng.integers(0, 6, n)
    hi = rng.integers(0, 0x7F7F, n).astype(np.uint32) | (rng.integers(0, 2, n).astype(np.uint32) << 31)
    bits[kind == 0] = (hi[kind == 0] << 16) | 0x8000                       # ties: upper half even or odd
    bits[kind == 1] = hi[kind == 1] << 16                                  # exact in bf16
    bits[kind == 2] = 0x80000000                                           # -0.0
    sub = rng.integers(1, 0x800000, n).astype(np.uint32) | (rng.integers(0, 2, n).astype(np.uint32) << 31)
    bits[kind == 3] = sub[kind == 3]                                       # subnormals
    big = rng.integers(0x7F000000, 0x7F7F8000, n).astype(np.uint32) | (rng.integers(0, 2, n).astype(np.uint32) << 31)
    bits[kind == 4] = big[kind == 4]                                       # large, rounds to a finite bf16
    return bits.view(np.float32)


def expected_shadows(theta, net, prec):
    F, hidden = NETS[net]
    out, off = [], 0
    for l, (i, o) in enumerate(shadow_dims(net, prec)):
        s = np.full((NPARTS[prec], i, -(-o // 8) * 8), SENTINEL, np.uint16)
        W = theta[off:off + i * o].reshape(i, o)
        for part in range(NPARTS[prec]):
            s[part, :, :o] = shadow_bits(W, part)
        out.append(s)
        off += i * o + o
    return out


def _check_shadows(sb, t, theta, net, prec, what):
    got = read_shadows(sb, t, prec, shadow_dims(net, prec))
    for l, (g, w) in enumerate(zip(got, expected_shadows(theta, net, prec))):
        _bits_equal(g, w, "%s: shadow of layer %d" % (what, l))


def test_edge_theta_reaches_every_rounding_edge():
    v = edge_theta(np.random.default_rng(5), 4096)
    b = v.view(np.uint32)
    low, up = b & 0xFFFF, (b >> 16) & 0x7FFF
    assert np.any((low == 0x8000) & (up % 2 == 0)) and np.any((low == 0x8000) & (up % 2 == 1))
    assert np.any((low == 0) & (up != 0)) and np.any(b == 0x80000000)
    assert np.any((up < 0x80) & (b & 0x7FFFFFFF != 0)) and np.any(np.abs(v) > 1e38)
    assert np.all(np.isfinite(v)) and np.all(np.isfinite((shadow_bits(v, 0).astype(np.uint32) << 16).view(np.float32)))
    assert np.all(shadow_bits(v[(low == 0)], 1) == 0)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [BF16, BF16X2, FP32_TC], ids=lambda p: PNAME[p])
@pytest.mark.parametrize("net,fixed", [("odd", "none"), ("m8", "none"), ("odd", "l2b"), ("m8", "l1")])
def test_shadow_refresh_writes_every_part(sb, tmp_path, prec, net, fixed):
    c = sb.capi
    rng = np.random.default_rng(zlib.crc32(("%s-%s-%d" % (net, fixed, prec)).encode()))
    t = make_trainer(sb, prec, net, MOMENTUM, 0.05, fixed)
    dims = shadow_dims(net, prec)
    try:
        n = t.n_params
        v = edge_theta(rng, n)
        fill_shadows(sb, t, prec, dims)
        t.debug_buffer(c.DEBUG_BUF_THETA, v, refresh_shadows=True)
        _check_shadows(sb, t, v, net, prec, "debug_buffer(refresh_shadows)")
        _bits_equal(t.debug_buffer(c.DEBUG_BUF_THETA), v, "theta after debug_buffer")
        v = edge_theta(rng, n)
        fill_shadows(sb, t, prec, dims)
        t.set_params(v)
        _check_shadows(sb, t, v, net, prec, "set_params")
        _bits_equal(t.get_params(), v, "get_params")
        path = str(tmp_path / "ckpt.bin")
        t.save_checkpoint(path)
        t.debug_buffer(c.DEBUG_BUF_THETA, edge_theta(rng, n), refresh_shadows=True)
        fill_shadows(sb, t, prec, dims)
        t.load_checkpoint(path)
        _check_shadows(sb, t, v, net, prec, "load_checkpoint")
        _bits_equal(t.debug_buffer(c.DEBUG_BUF_THETA), v, "theta after load_checkpoint")
    finally:
        t.close()
