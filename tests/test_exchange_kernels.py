"""Kernel-level checks of the peer-memory gradient exchange (csrc/xchg_p2p.cuh) through the trainer's own launch code.

W in-process replicas on one device are joined by their peer tables (sb_trainer_set_peer_pointers).  Each case writes
every rank's raw arena buffers (sb_debug_trainer_buffer): theta, s1 and s2 different on every rank, the bf16 shadows
filled with a per-rank sentinel, then, before each of three consecutive exchanges, fresh gradients.  sb_debug_exchange
queues one exchange on every rank as a step does (the descriptor of the next update, then enqueue_xchg: the trainer's
slot and work tables, grid rule and kernel choice), and the test waits for all ranks (Trainer.sync, which turns a lost
peer into an error after SB_XCHG_TIMEOUT_S).  After each exchange every raw buffer of every rank is compared with a
model built here from a Python restatement of xchg_share, not from anything the kernels report:

  reduced gradient   the owner's raw gradient of each run of the launch's slots is the float32 sum of the ranks'
                     gradients added left to right in rank order 0 .. W-1, bit for bit (both protocols, both paths)
  ownership          only the owner's raw theta / s1 / s2 change; every other rank's master, state and gradient (its
                     own contribution) are unchanged byte for byte, and runs outside the launch's slots are untouched
  master and state   the owner's theta, s1, s2 against a float64 evaluation of opt_update's algebra on the float32
                     inputs, with g = float32(sum * gscale) (one float32 product, as in the kernel)
  operands           shadow-backed runs: every part of every rank's shadow is the bf16 (round to nearest even) of
                     bf16_residual(owner's new theta, part), bit for bit, and the pad columns keep their sentinels;
                     runs without a shadow: every rank's raw theta equals the owner's, bit for bit
After the three exchanges get_params() (which gathers the stale masters from the owners) is the owners' theta on every
rank, and get_grads() the owners' raw gradients times gscale, bit-identical on all ranks.

Bounds for the master and state: tests/opt_ref.py derives them (|got - ref| <= C u S, S the sum of the magnitudes of an
expression's terms) for every optimizer; FTRL's l1 branch is also checked apart from the bound.  The exact case (SGD,
lr = 2^-4, gscale = 1/4, dyadic theta and gradients with few bits) has no rounding anywhere and must match the float64
result bit for bit.

Co-residency: every exchange block of every rank must be resident at once (they spin on each other), and nothing but
exchange kernels runs here, so W x grid <= SM count is asserted before each launch; W >= 5 runs at most 8 blocks per
rank.  The kernel each launch ran ("xchg_ll<4>", "xchg_update<16>", ...) is checked against the instantiation the world
size selects, and the case matrix reaches both kernels at W = 2, 4, 8 and 16 with the reference's four rules
(<W, OPT_BASE>) and at W = 2 and 3 (U = 2 and U = 1 update loops) with Adagrad, RMSProp and FTRL (<W, OPT_EXT>)."""
import ctypes as C
import zlib

import numpy as np
import pytest

from opt_ref import (ADADELTA, ADAGRAD, ADAM, BETA1, BETA2, BF16, BF16X2, C_BOUND, EPS, EXT, FP32, FP32_TC, FTRL, MOM,
                     MOMENTUM, NPARTS, ONAME, PNAME, RHO, RMSPROP, SGD, U, _bits_equal, check_l1_branch, lr_t_of, reference,
                     s1_start, shadow_bits, uses_s1, uses_s2)
TIMEOUT_S = "5"
FTRL_L1, FTRL_L2 = 0.5, 0.25

# nets (features, hidden widths): the layouts of the work runs
NETS = {
    "m8": (200, [64, 48]),           # widths % 8 == 0: every run on the 16-byte paths
    "odd": (150, [45, 30, 7]),       # widths = 1, 2, 3 mod 4: shadow-backed runs on the element paths; fp32: unaligned runs
    "chunk": (600, [24, 40]),        # tensor-core modes: layer 0 in two row-chunk slots (in >= 512, out % 8 == 0)
    "tiny": (8, [8]),                # slot 0 = 1 run, slot 1 = 2 runs: most ranks own nothing
}

LR = {SGD: 0.05, MOMENTUM: 0.05, ADAM: 0.003, ADADELTA: 1.0, ADAGRAD: 0.05, RMSPROP: 0.003, FTRL: 0.05}

_worst = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if _worst:
        print("\nworst error / bound: " + ", ".join("%s %.3g" % kv for kv in sorted(_worst.items())))


def _note(name, err, tol):
    if err.size:
        _worst[name] = max(_worst.get(name, 0.0), float(np.max(err / tol)))


def xchg_share(b, e, r, world):
    """first run of rank r's share of [b, e) (xchg_p2p.cuh)"""
    return b + ((e - b) * r) // world


def owners(b, e, world):
    own = np.empty(e - b, np.int64)
    for r in range(world):
        own[xchg_share(b, e, r, world) - b:xchg_share(b, e, r + 1, world) - b] = r
    return own


def kernel_name(W, prec):
    t = next(k for k in (2, 4, 8, 16) if W <= k)
    return ("xchg_ll<%d>" if prec == BF16 else "xchg_update<%d>") % t


def predicted_grid(lay, W, mask, alone):
    """the grid rule of enqueue_xchg (xchg_grid in capi.cu) for replicas that share a device"""
    runs = all_runs = 0
    for s in range(lay["slots"]):
        if (mask >> s) & 1:
            n = lay["end"][s] - lay["begin"][s]
            runs += -(-n // W)
            all_runs += n
    u = 2 if W <= 2 else 1
    want = max(-(-runs // u), -(-(all_runs - runs) // 4))
    grid = (2 if alone else 1) * lay["sms"]
    if lay["share_device"]:
        grid = min(grid, 32)
    return max(1, min(grid, want))


class Replicas:
    """W trainers on device 0 joined by their peer tables, their raw buffers and the model of what they must hold"""

    def __init__(self, sb, W, prec, net, kind, lr, seed, exact):
        F, hidden = NETS[net]
        acts = [sb.ACT_RELU] * len(hidden)
        desc = sb.make_desc(F, hidden, acts, optimizer=kind, learning_rate=lr, rho=RHO, epsilon=EPS, beta1=BETA1, beta2=BETA2,
                            momentum=MOM, max_batch=8, precision=prec)
        # FTRL runs with both penalties on (and Adagrad / FTRL with a non-default start accumulator, which the raw s1
        # written below replaces)
        self.l1, self.l2 = (FTRL_L1, FTRL_L2) if kind == FTRL else (0.0, 0.0)
        kw = dict(initial_accumulator=0.25, l1=self.l1, l2=self.l2) if kind in (ADAGRAD, FTRL) else {}
        self.ts = [sb.Trainer(desc, device=0, nccl_id=None, rank=r, world=W, **kw) for r in range(W)]
        bases = [t.exchange_base for t in self.ts]
        for t in self.ts:
            t.set_peer_pointers(bases)
        self.sb, self.W, self.prec, self.kind, self.exact = sb, W, prec, kind, exact
        self.lay = self.ts[0].debug_exchange_layout()
        for t in self.ts[1:]:
            other = t.debug_exchange_layout()
            assert (other["begin"], other["end"], other["work"]) == (self.lay["begin"], self.lay["end"], self.lay["work"])
        self.n = self.ts[0].n_params
        self.np = NPARTS[prec]
        self.dims = [(hidden[l - 1] if l else F, hidden[l]) for l in range(len(hidden))] if prec != FP32 else []
        self.rng = np.random.default_rng(seed)
        rng = self.rng
        if exact:
            self.theta = [(rng.integers(-512, 512, self.n) * 2.0 ** -8).astype(np.float32) for _ in range(W)]
        else:
            self.theta = [(rng.standard_normal(self.n) * 0.5).astype(np.float32) for _ in range(W)]
        sq = kind in (ADAM, ADADELTA)           # squared-gradient accumulators are >= 0
        self.s1 = [s1_start(kind, v) for v in (rng.standard_normal(self.n) * 0.1 for _ in range(W))]
        self.s2 = [(np.abs(rng.standard_normal(self.n)) * 0.01 if sq else rng.standard_normal(self.n)).astype(np.float32)
                   for _ in range(W)]
        self.shadow = [[np.full((self.np, i, -(-o // 8) * 8), 0x7FA0 + r, np.uint16) for (i, o) in self.dims] for r in range(W)]
        for r, t in enumerate(self.ts):
            t.debug_buffer(self.sb.capi.DEBUG_BUF_THETA, self.theta[r])
            t.debug_buffer(self.sb.capi.DEBUG_BUF_S1, self.s1[r])
            t.debug_buffer(self.sb.capi.DEBUG_BUF_S2, self.s2[r])
            for l, sh in enumerate(self.shadow[r]):
                t.debug_buffer(self.sb.capi.DEBUG_BUF_SHADOW + l, sh)
        self.grad = [np.zeros(self.n, np.float32) for _ in range(W)]
        self.step = 0

    def close(self):
        for t in self.ts:
            t.close()

    def read(self, r):
        c = self.sb.capi
        t = self.ts[r]
        return (t.debug_buffer(c.DEBUG_BUF_THETA), t.debug_buffer(c.DEBUG_BUF_S1), t.debug_buffer(c.DEBUG_BUF_S2),
                t.debug_buffer(c.DEBUG_BUF_GRAD),
                [t.debug_buffer(c.DEBUG_BUF_SHADOW + l, n=self.np * i * (-(-o // 8) * 8)).reshape(self.np, i, -1)
                 for l, (i, o) in enumerate(self.dims)])

    def exchange(self, mask, gscale, grid, alone):
        W, rng = self.W, self.rng
        if self.exact:
            self.grad = [(rng.integers(-4096, 4096, self.n) * 2.0 ** -12).astype(np.float32) for _ in range(W)]
        else:
            self.grad = [(rng.standard_normal(self.n) * 10.0 ** rng.uniform(-3, 1, self.n)).astype(np.float32) for _ in range(W)]
        for r, t in enumerate(self.ts):
            t.debug_buffer(self.sb.capi.DEBUG_BUF_GRAD, self.grad[r])
        g_used = grid if grid > 0 else predicted_grid(self.lay, W, mask, alone)
        assert W * g_used <= self.lay["sms"], "%d ranks x %d blocks do not fit on %d SMs at once" % (W, g_used, self.lay["sms"])
        res = [t.debug_exchange(mask, gscale, grid, alone) for t in self.ts]
        for t in self.ts:
            t.sync()
        self.step += 1
        lr_t = res[0][0]
        for (lr_r, g_r, route) in res:
            assert (lr_r, g_r, route) == (lr_t, g_used, kernel_name(W, self.prec))
        lr = float(np.float32(self.ts[0].desc.learning_rate))
        assert abs(lr_t - lr_t_of(self.kind, lr, self.step)) <= 1e-6 * lr_t
        gs = np.float32(gscale if gscale > 0 else np.float32(1.0) / np.float32(W))
        self._check(mask, gs, lr_t)
        return gs

    def _check(self, mask, gs, lr_t):
        W = self.W
        got = [self.read(r) for r in range(W)]
        exp_t = [v.copy() for v in self.theta]
        exp_1 = [v.copy() for v in self.s1]
        exp_2 = [v.copy() for v in self.s2]
        exp_g = [v.copy() for v in self.grad]
        exp_sh = [[v.copy() for v in sh] for sh in self.shadow]
        use1, use2 = uses_s1(self.kind), uses_s2(self.kind)
        for s in range(self.lay["slots"]):
            if not (mask >> s) & 1:
                continue
            b, e = self.lay["begin"][s], self.lay["end"][s]
            own = owners(b, e, W)
            for w in range(b, e):
                wk = self.lay["work"][w]
                o = int(own[w - b])
                idx = np.arange(wk["off"], wk["off"] + wk["count"])
                acc = self.grad[0][idx].copy()
                for q in range(1, W):
                    acc = (acc + self.grad[q][idx]).astype(np.float32)
                where = "run %d (owner %d of %d, slot %d)" % (w, o, W, s)
                _bits_equal(got[o][3][idx], acc, "reduced gradient of " + where)
                exp_g[o][idx] = acc
                g = (acc * gs).astype(np.float32)
                rt, r1, r2, St, S1, S2 = reference(self.kind, lr_t, self.theta[o][idx], self.s1[o][idx], self.s2[o][idx], g,
                                                   self.l1, self.l2)
                gt, g1, g2 = got[o][0][idx], got[o][1][idx], got[o][2][idx]
                if self.exact:
                    _bits_equal(gt, rt.astype(np.float32), "exact theta of " + where)
                    assert np.array_equal(rt.astype(np.float32).astype(np.float64), rt)
                for name, gv, rv, S, used in (("theta", gt, rt, St, True), ("s1", g1, r1, S1, use1), ("s2", g2, r2, S2, use2)):
                    if not used:
                        continue
                    err = np.abs(gv.astype(np.float64) - rv)
                    tol = C_BOUND * U * S + 1e-45
                    _note("%s %s" % (ONAME[self.kind], name), err, tol)
                    assert np.all(err <= tol), "%s of %s: worst error / bound %.3g" % (name, where, float(np.max(err / tol)))
                check_l1_branch(self.kind, gt, r2, S2, self.l1, "theta of " + where)
                exp_t[o][idx] = gt
                if use1:
                    exp_1[o][idx] = g1
                if use2:
                    exp_2[o][idx] = g2
                if wk["layer"] >= 0:
                    l = wk["layer"]
                    m = idx - wk["mat_off"]
                    rows, cols = m // wk["out_dim"], m % wk["out_dim"]
                    assert wk["np"] == self.np
                    for part in range(self.np):
                        bits = shadow_bits(gt, part)
                        for r in range(W):
                            exp_sh[r][l][part, rows, cols] = bits
                else:
                    for r in range(W):
                        exp_t[r][idx] = gt
        for r in range(W):
            th, a, b, gr, sh = got[r]
            _bits_equal(gr, exp_g[r], "raw gradient of rank %d" % r)
            _bits_equal(th, exp_t[r], "raw theta of rank %d" % r)
            _bits_equal(a, exp_1[r], "raw s1 of rank %d" % r)
            _bits_equal(b, exp_2[r], "raw s2 of rank %d" % r)
            for l in range(len(sh)):
                _bits_equal(sh[l], exp_sh[r][l], "shadow of layer %d on rank %d" % (l, r))
        self.theta, self.s1, self.s2, self.grad, self.shadow = exp_t, exp_1, exp_2, exp_g, exp_sh

    def check_host_view(self, gs):
        """get_params / get_grads: the owners' values on every rank, bit-identical"""
        W = self.W
        want_p = np.empty(self.n, np.float32)
        want_g = np.empty(self.n, np.float32)
        for s in range(self.lay["slots"]):
            b, e = self.lay["begin"][s], self.lay["end"][s]
            own = owners(b, e, W)
            for w in range(b, e):
                wk = self.lay["work"][w]
                idx = slice(wk["off"], wk["off"] + wk["count"])
                want_p[idx] = self.theta[own[w - b]][idx]
                want_g[idx] = self.grad[own[w - b]][idx] * gs
        for r, t in enumerate(self.ts):
            _bits_equal(t.get_params(), want_p, "get_params() of rank %d" % r)
        for r, t in enumerate(self.ts):
            _bits_equal(t.get_grads(), want_g, "get_grads() of rank %d" % r)
        for t in self.ts:
            t.sync()


def _plan(lay, plan):
    """slot masks of the three exchanges of a case"""
    s = lay["slots"]
    if plan == "each":
        return [1 << (k % s) for k in range(3)]
    if plan == "all":
        return [(1 << s) - 1] * 3
    if plan == "step":                       # the step's order: the row chunks of layer 0, then slot A
        order = [1 << c for c in range(1, s)] + [1]
        return (order * 3)[:3]
    raise ValueError(plan)


# (W, precision, optimizer, net, plan, grid, gscale, exact); grid: 0 = the trainer's rule, -1 = alone, -2 = the most
# blocks per rank that fit (<= 8), k > 0 = k blocks
def _cases():
    out = []
    opts = [ADAM, MOMENTUM, SGD, ADADELTA]
    k = 0
    for W in (2, 3, 4, 5, 8, 16):                               # every template, even and uneven shares
        for prec in (FP32, BF16):
            for net in ("m8", "odd"):
                out.append((W, prec, opts[k % 4], net, ("each", "all", "step")[k % 3], 0 if W <= 4 else -2, 0.0, False))
                k += 1
    for prec in (FP32_TC, BF16X2):                              # split modes: np = 3 / 2 shadow parts
        for W in (2, 3, 8):
            for net in ("m8", "odd"):
                out.append((W, prec, opts[k % 4], net, ("each", "all", "step")[k % 3], 0 if W <= 4 else -2, 0.0, False))
                k += 1
    for opt in opts:                                            # every optimizer through both protocols, uneven shares
        for prec in (FP32, BF16, FP32_TC):
            out.append((3, prec, opt, "odd", "all", 0, 0.0, False))
    for prec in (BF16, FP32_TC, BF16X2):                        # layer 0 in two chunk slots
        for W, plan in ((2, "step"), (3, "each"), (5, "all"), (4, "step")):
            out.append((W, prec, MOMENTUM, "chunk", plan, 0 if W <= 4 else -2, 0.0, False))
    for prec in (FP32, BF16, FP32_TC):                          # one block loops over every run (W = 2: the U = 2 tail)
        for W, net in ((2, "m8"), (2, "odd"), (3, "odd")):
            out.append((W, prec, ADAM, net, "all", 1, 0.0, False))
    for prec in (FP32, BF16):                                   # the last launch of a step: two blocks per SM
        out.append((2, prec, MOMENTUM, "m8", "all", -1, 0.0, False))
        out.append((4, prec, ADADELTA, "odd", "each", -1, 0.0, False))
    for prec in (FP32, BF16, BF16X2):                           # gscale of the epoch-sync schedule (1 / total pushes)
        out.append((2, prec, MOMENTUM, "odd", "all", 0, 0.2, False))
        out.append((3, prec, SGD, "m8", "all", 0, 0.2, False))
    for prec in (FP32, BF16, FP32_TC):                          # slots with fewer runs than ranks
        out.append((8, prec, ADAM, "tiny", "all", -2, 0.0, False))
        out.append((16, prec, MOMENTUM, "tiny", "each", -2, 0.0, False))
    for W, prec, net in ((3, FP32, "odd"), (5, BF16, "m8"), (2, FP32_TC, "odd"), (16, BF16, "odd")):   # no rounding anywhere
        out.append((W, prec, SGD, net, "all", 0 if W <= 4 else -2, 0.25, True))
    for opt in EXT:                                             # the <W, OPT_EXT> instantiations: U = 2 and U = 1, both protocols
        for W, prec, net, plan in ((2, BF16, "m8", "all"), (3, BF16, "odd", "each"), (2, FP32, "odd", "each"),
                                   (3, FP32, "m8", "all"), (3, FP32_TC, "odd", "all"), (2, BF16X2, "m8", "step")):
            out.append((W, prec, opt, net, plan, 0, 0.0, False))
    return list(dict.fromkeys(out))


CASES = _cases()


def _id(c):
    W, prec, opt, net, plan, grid, gscale, exact = c
    g = {0: "rule", -1: "alone", -2: "fit"}.get(grid, "g%d" % grid)
    return "W%d-%s-%s-%s-%s-%s%s%s" % (W, PNAME[prec], ONAME[opt], net, plan, g, "-gs%g" % gscale if gscale else "",
                                       "-exact" if exact else "")


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_exchange_against_float64(sb, monkeypatch, case):
    W, prec, opt, net, plan, grid, gscale, exact = case
    monkeypatch.setenv("SB_XCHG_TIMEOUT_S", TIMEOUT_S)
    monkeypatch.delenv("SB_XCHG_BLOCKS", raising=False)
    lr = 2.0 ** -4 if exact else LR[opt]
    reps = Replicas(sb, W, prec, net, opt, lr, seed=zlib.crc32(_id(case).encode()), exact=exact)
    try:
        lay = reps.lay
        assert lay["share_device"] and lay["world"] == W and lay["ll"] == (prec == BF16)
        if net == "chunk":
            assert lay["slots"] == 3
        if grid == -2:
            grid = min(8, lay["sms"] // W)
        gs = None
        for mask in _plan(lay, plan):
            gs = reps.exchange(mask, gscale, max(grid, 0), grid == -1)
        reps.check_host_view(gs)
    finally:
        reps.close()


def test_case_matrix_reaches_every_instantiation():
    # kernel_name names both optimizer groups alike: <W, OPT_BASE> for the reference's four rules, <W, OPT_EXT> for the others
    routes = {(kernel_name(c[0], c[1]), c[2] in EXT) for c in CASES}
    want = {("xchg_%s<%d>" % (k, w), False) for k in ("ll", "update") for w in (2, 4, 8, 16)}
    want |= {("xchg_%s<%d>" % (k, w), True) for k in ("ll", "update") for w in (2, 4)}
    assert want <= routes, want - routes
    assert {c[2] for c in CASES} == set(ONAME)
    # every kernel also meets uneven shares, and every split mode a W = 8 exchange
    assert {(c[0], c[1]) for c in CASES} >= {(3, FP32), (3, BF16), (5, FP32), (5, BF16), (8, FP32_TC), (8, BF16X2)}


def test_exchange_hooks_reject_bad_arguments_without_a_trainer(sb):
    lib, c = sb.capi.lib(), sb.capi
    buf = np.zeros(4, np.float32)
    assert lib.sb_debug_trainer_buffer(None, 0, buf.ctypes.data_as(C.c_void_p), 4, 0) == c.SB_ERR_INVALID
    assert lib.sb_debug_exchange(None, 1, 0.0, 0, 0, None, None, None, 0) == c.SB_ERR_INVALID
    info = (C.c_int32 * c.DEBUG_XINFO_WORDS)()
    n = C.c_int32()
    assert lib.sb_debug_exchange_layout(None, info, c.DEBUG_XINFO_WORDS, None, 0, C.byref(n)) == c.SB_ERR_INVALID


@pytest.mark.gpu
def test_exchange_hooks_reject_bad_arguments(sb, monkeypatch):
    monkeypatch.setenv("SB_XCHG_TIMEOUT_S", TIMEOUT_S)
    F, hidden = NETS["m8"]
    c = sb.capi
    lone = sb.Trainer(sb.make_desc(F, hidden, [sb.ACT_RELU] * 2, precision=FP32, max_batch=8), device=0, nccl_id=None, rank=0,
                      world=2)
    try:
        with pytest.raises(sb.ShifuB200Error) as e:              # no peer table
            lone.debug_exchange(1)
        assert e.value.code == c.SB_ERR_STATE
        with pytest.raises(sb.ShifuB200Error) as e:              # fp32 mode keeps no shadow
            lone.debug_buffer(c.DEBUG_BUF_SHADOW, n=8)
        assert e.value.code == c.SB_ERR_STATE
    finally:
        lone.close()
    reps = Replicas(sb, 2, BF16, "m8", MOMENTUM, 0.05, seed=1, exact=False)
    try:
        t = reps.ts[0]
        slots = reps.lay["slots"]
        for bad in (0, 1 << slots, -1):                           # empty mask, a slot the trainer does not have
            with pytest.raises(sb.ShifuB200Error) as e:
                t.debug_exchange(bad)
            assert e.value.code == c.SB_ERR_INVALID
        for kw in (dict(gscale=-1.0), dict(gscale=float("nan")), dict(grid=-3), dict(grid=70000)):
            with pytest.raises(sb.ShifuB200Error) as e:
                t.debug_exchange(1, **kw)
            assert e.value.code == c.SB_ERR_INVALID
        with pytest.raises(sb.ShifuB200Error) as e:               # wrong lengths
            t.debug_buffer(c.DEBUG_BUF_THETA, np.zeros(t.n_params - 1, np.float32))
        assert e.value.code == c.SB_ERR_INVALID
        with pytest.raises(sb.ShifuB200Error) as e:               # layer 0's shadow is F x 64 (np = 1)
            t.debug_buffer(c.DEBUG_BUF_SHADOW, n=F * 64 + 1)
        assert e.value.code == c.SB_ERR_INVALID
        for which in (-1, c.DEBUG_BUF_SHADOW + len(hidden)):      # no such buffer
            with pytest.raises(sb.ShifuB200Error) as e:
                t.debug_buffer(which, n=8)
            assert e.value.code == c.SB_ERR_INVALID
        # nothing was queued by the refused calls: the replicas still exchange and agree
        gs = reps.exchange(1, 0.0, 0, False)
        reps.check_host_view(gs)
    finally:
        reps.close()
