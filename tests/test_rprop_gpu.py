"""RPROP (SB_OPT_RPROP, iRPROP-) on the H100, held bit for bit to the float32 restatement in tests/rprop_ref.py:

  state start      s1 (prev) = 0 and s2 (step) = float32(learning_rate) after creation, init_xavier and set_params, on
                   every rank; sb_trainer_set_optimizer_params is refused
  optimizer pass   sb_debug_optimizer through apply_accumulated (one launch over the work table) and through the step's
                   split tail, in every precision: after each of four updates with chosen gradient words, theta, s1 and s2
                   of every run equal the rule bit for bit; every part of every shadow is bf16_residual of the new theta
                   and the pad columns keep their sentinel; frozen parameters, their state and shadows keep their bits
  peer exchange    W = 2 and 4 in-process replicas, fp32 and bf16 (both exchange protocols): each owner's theta, s1, s2
                   are the rule applied to the copies summed in rank order; get_params is bit-identical on every rank
  checkpoint       a round trip keeps the state bits; Adadelta's checkpoint is refused by an RPROP trainer and the reverse
  worker           Optimizer: rprop with Schedule: sync_replicas (fp32, fp32_tc) against the oracle's SyncReplicasTrainer:
                   every epoch's losses within 1e-4, the exported weights by relative L2 norm (the sign rule turns rounding
                   noise in a gradient near 0 into a whole step, as Adam's division does, DESIGN section 2);
                   Deterministic: true gives two bit-identical runs"""
import zlib

import numpy as np
import pytest

import rprop_ref as rr
from opt_ref import BF16, BF16X2, FP32, FP32_TC, NPARTS, PNAME, _bits_equal, shadow_bits
from oracle import shifu_oracle as so
from test_exchange_kernels import NETS as XNETS, kernel_name, owners
from test_optimizer_pass import FROZEN, fill_shadows, make_trainer, read_shadows, shadow_dims, table

pytestmark = pytest.mark.gpu

PRECS = [FP32, BF16, FP32_TC, BF16X2]
LR = 0.0125


def _draw_state(rng, n):
    """theta, prev (signed, with zeros, -0 and magnitudes whose products underflow) and step sizes, some outside
    [1e-6, 50] so that the first update clamps them"""
    theta = (rng.standard_normal(n) * 0.5).astype(np.float32)
    prev = _draw_grad(rng, n)
    step = (10.0 ** rng.uniform(-7, 2.2, n)).astype(np.float32)
    return theta, prev, step


def _draw_grad(rng, n, neg_zero=True):
    """neg_zero=False: +0 in place of -0 (the exchange's element path sums the copies from +0, so a -0 sum is +0 there)"""
    g = rng.choice([-1.0, 1.0], n) * 10.0 ** rng.uniform(-3, 1, n)
    k = rng.integers(0, 16, n)
    g[k == 0] = 0.0
    g[k == 1] = -0.0 if neg_zero else 0.0
    g[k == 2] *= 10.0 ** rng.uniform(-24, -22, int(np.sum(k == 2)))     # products of two of these underflow
    return g.astype(np.float32)


def _state(sb, t):
    return t.debug_buffer(sb.capi.DEBUG_BUF_S1), t.debug_buffer(sb.capi.DEBUG_BUF_S2)


@pytest.mark.parametrize("prec", PRECS, ids=lambda p: PNAME[p])
def test_state_starts_at_zero_and_the_learning_rate(sb, prec):
    F, hidden = 40, [24, 16]
    net = so.NetDesc(F, hidden, [so.ACT_RELU] * 2)
    desc = sb.make_desc(F, hidden, [sb.ACT_RELU] * 2, optimizer=sb.OPT_RPROP, learning_rate=LR, max_batch=32, precision=prec)
    with sb.Trainer(desc) as t:
        for what in ("create", "init_xavier", "set_params"):
            if what == "init_xavier":
                t.init_xavier(3)
            elif what == "set_params":
                t.set_params(so.flatten_params(so.xavier_init(net, 4)))
            s1, s2 = _state(sb, t)
            assert np.all(s1.view(np.uint32) == 0) and np.all(s2 == np.float32(LR)), what
        with pytest.raises(sb.ShifuB200Error) as e:
            t.set_optimizer_params(0.1, 0.0, 0.0)
        assert e.value.code == sb.capi.SB_ERR_INVALID
    ts = [sb.Trainer(desc, device=0, nccl_id=None, rank=r, world=2) for r in range(2)]
    try:
        for t in ts:
            s1, s2 = _state(sb, t)
            assert np.all(s1.view(np.uint32) == 0) and np.all(s2 == np.float32(LR))
    finally:
        for t in ts:
            t.close()


# ---- the single-GPU pass (optimizer_kernel<OPT_RPROP>) ----
def _pass_cases():
    out = []
    for prec in PRECS:
        for nb, net in enumerate(("m8", "odd")):
            for tail in (0, 1):
                out.append((prec, net, "none", tail, (1.0, 0.2)[(nb + tail) % 2]))
        out.append((prec, "m8", "l1", 1, 1.0))       # layer 0 frozen: the split tail's layer-0 range is empty
        out.append((prec, "odd", "l2b", 0, 0.2))
    return out


PASS_CASES = _pass_cases()


def _pass_id(c):
    prec, net, fixed, tail, gscale = c
    return "%s-%s-%s-%s-gs%g" % (PNAME[prec], net, fixed, ("pass", "tail")[tail], gscale)


@pytest.mark.parametrize("case", PASS_CASES, ids=[_pass_id(c) for c in PASS_CASES])
def test_optimizer_pass_is_the_rule_bit_for_bit(sb, case):
    prec, net, fixed, tail, gscale = case
    c = sb.capi
    rng = np.random.default_rng(zlib.crc32(_pass_id(case).encode()))
    t = make_trainer(sb, prec, net, sb.OPT_RPROP, LR, fixed)
    try:
        work, begin, end = table(net, prec, fixed)
        assert t.debug_exchange_layout()["work"] == work
        n = t.n_params
        idx = np.concatenate([np.arange(w["off"], w["off"] + w["count"]) for w in work])
        dims = shadow_dims(net, prec)
        theta, s1, s2 = _draw_state(rng, n)
        t.debug_buffer(c.DEBUG_BUF_THETA, theta)
        t.debug_buffer(c.DEBUG_BUF_S1, s1)
        t.debug_buffer(c.DEBUG_BUF_S2, s2)
        shadow = fill_shadows(sb, t, prec, dims)
        launches = [("main", 0, len(work))] if not tail else [("main", begin[0], end[0]), ("side", end[0], len(work))]
        route_want = "+".join("optimizer<rprop>@%s[%d,%d)" % l for l in launches if l[2] > l[1])
        gs = np.float32(gscale)
        for step in range(4):
            grad = _draw_grad(rng, n)
            t.debug_buffer(c.DEBUG_BUF_GRAD, grad)
            lr_t, route = t.debug_optimizer(gscale, tail)
            t.sync()
            assert route == route_want and lr_t == np.float32(LR)
            exp_t, exp_1, exp_2 = theta.copy(), s1.copy(), s2.copy()
            exp_t[idx], exp_1[idx], exp_2[idx] = rr.rprop_update(theta[idx], (grad[idx] * gs).astype(np.float32), s1[idx],
                                                                 s2[idx])
            got_t, got_1, got_2 = t.debug_buffer(c.DEBUG_BUF_THETA), *_state(sb, t)
            what = "update %d" % (step + 1)
            _bits_equal(got_t, exp_t, what + ": theta")
            _bits_equal(got_1, exp_1, what + ": s1 (prev)")
            _bits_equal(got_2, exp_2, what + ": s2 (step)")
            _bits_equal(t.debug_buffer(c.DEBUG_BUF_GRAD), grad, what + ": raw gradient")
            for l, w in enumerate(dims):
                runs = [x for x in work if x["layer"] == l]
                if runs:
                    pos = np.concatenate([np.arange(x["off"], x["off"] + x["count"]) for x in runs])
                    m = pos - runs[0]["mat_off"]
                    for part in range(NPARTS[prec]):
                        shadow[l][part, m // runs[0]["out_dim"], m % runs[0]["out_dim"]] = shadow_bits(exp_t[pos], part)
            for l, g in enumerate(read_shadows(sb, t, prec, dims)):
                _bits_equal(g, shadow[l], what + ": shadow of layer %d" % l)
            theta, s1, s2 = exp_t, exp_1, exp_2
        assert np.any(s2[idx] == rr.STEP_MIN) and np.any(s2[idx] == rr.STEP_MAX)
    finally:
        t.close()


# ---- the peer exchange (xchg_update_kernel<W, OPT_RPROP>, xchg_ll_kernel<W, OPT_RPROP>) ----
@pytest.mark.parametrize("plan", ["all", "each"])
@pytest.mark.parametrize("net", ["m8", "odd"])
@pytest.mark.parametrize("prec", [FP32, BF16], ids=lambda p: PNAME[p])
@pytest.mark.parametrize("W", [2, 4])
def test_exchange_owner_update_is_the_rule_bit_for_bit(sb, monkeypatch, W, prec, net, plan):
    monkeypatch.setenv("SB_XCHG_TIMEOUT_S", "5")
    monkeypatch.delenv("SB_XCHG_BLOCKS", raising=False)
    c = sb.capi
    F, hidden = XNETS[net]
    rng = np.random.default_rng(zlib.crc32(("%d-%d-%s-%s" % (W, prec, net, plan)).encode()))
    desc = sb.make_desc(F, hidden, [sb.ACT_RELU] * len(hidden), optimizer=sb.OPT_RPROP, learning_rate=LR, max_batch=8,
                        precision=prec)
    ts = [sb.Trainer(desc, device=0, nccl_id=None, rank=r, world=W) for r in range(W)]
    try:
        bases = [t.exchange_base for t in ts]
        for t in ts:
            t.set_peer_pointers(bases)
        lay = ts[0].debug_exchange_layout()
        n, npart = ts[0].n_params, NPARTS[prec]
        dims = [(hidden[l - 1] if l else F, hidden[l]) for l in range(len(hidden))] if prec != FP32 else []
        theta, s1, s2, shadow = [], [], [], []
        for r, t in enumerate(ts):
            th, a, b = _draw_state(rng, n)
            sh = [np.full((npart, i, -(-o // 8) * 8), 0x7FA0 + r, np.uint16) for (i, o) in dims]
            t.debug_buffer(c.DEBUG_BUF_THETA, th)
            t.debug_buffer(c.DEBUG_BUF_S1, a)
            t.debug_buffer(c.DEBUG_BUF_S2, b)
            for l, s in enumerate(sh):
                t.debug_buffer(c.DEBUG_BUF_SHADOW + l, s)
            theta.append(th); s1.append(a); s2.append(b); shadow.append(sh)
        slots = lay["slots"]
        masks = [(1 << slots) - 1] * 3 if plan == "all" else [1 << (k % slots) for k in range(3)]
        gs = np.float32(1.0) / np.float32(W)
        for k, mask in enumerate(masks):
            grad = [_draw_grad(rng, n, neg_zero=False) for _ in range(W)]
            for t, g in zip(ts, grad):
                t.debug_buffer(c.DEBUG_BUF_GRAD, g)
            res = [t.debug_exchange(mask, 0.0, 0, False) for t in ts]
            for t in ts:
                t.sync()
            assert all(route == kernel_name(W, prec) for (_, _, route) in res)
            exp_t, exp_1, exp_2 = [v.copy() for v in theta], [v.copy() for v in s1], [v.copy() for v in s2]
            exp_g, exp_sh = [v.copy() for v in grad], [[v.copy() for v in sh] for sh in shadow]
            for s in range(slots):
                if not (mask >> s) & 1:
                    continue
                b, e = lay["begin"][s], lay["end"][s]
                own = owners(b, e, W)
                for w in range(b, e):
                    wk, o = lay["work"][w], int(own[w - b])
                    idx = np.arange(wk["off"], wk["off"] + wk["count"])
                    acc = grad[0][idx].copy()
                    for q in range(1, W):
                        acc = (acc + grad[q][idx]).astype(np.float32)
                    exp_g[o][idx] = acc
                    rt, exp_1[o][idx], exp_2[o][idx] = rr.rprop_update(theta[o][idx], (acc * gs).astype(np.float32),
                                                                       s1[o][idx], s2[o][idx])
                    exp_t[o][idx] = rt
                    if wk["layer"] >= 0:
                        m = idx - wk["mat_off"]
                        for part in range(npart):
                            bits = shadow_bits(rt, part)
                            for r in range(W):
                                exp_sh[r][wk["layer"]][part, m // wk["out_dim"], m % wk["out_dim"]] = bits
                    else:
                        for r in range(W):
                            exp_t[r][idx] = rt
            for r, t in enumerate(ts):
                what = "exchange %d, rank %d" % (k + 1, r)
                _bits_equal(t.debug_buffer(c.DEBUG_BUF_GRAD), exp_g[r], what + ": raw gradient")
                _bits_equal(t.debug_buffer(c.DEBUG_BUF_THETA), exp_t[r], what + ": raw theta")
                got_1, got_2 = _state(sb, t)
                _bits_equal(got_1, exp_1[r], what + ": s1 (prev)")
                _bits_equal(got_2, exp_2[r], what + ": s2 (step)")
                for l, (i, o) in enumerate(dims):
                    got = t.debug_buffer(c.DEBUG_BUF_SHADOW + l, n=npart * i * (-(-o // 8) * 8)).reshape(npart, i, -1)
                    _bits_equal(got, exp_sh[r][l], what + ": shadow of layer %d" % l)
            theta, s1, s2, shadow = exp_t, exp_1, exp_2, exp_sh
        params = [t.get_params() for t in ts]
        for r in range(1, W):
            _bits_equal(params[r], params[0], "get_params of rank %d" % r)
        for t in ts:
            t.sync()
    finally:
        for t in ts:
            t.close()


# ---- checkpoint ----
@pytest.mark.parametrize("prec", [FP32, BF16], ids=lambda p: PNAME[p])
def test_checkpoint_round_trip_keeps_the_state_bits(sb, tmp_path, prec):
    F, hidden, B = 96, [64, 32], 128
    net = so.NetDesc(F, hidden, [so.ACT_RELU] * 2)
    theta0 = so.flatten_params(so.xavier_init(net, 9))
    X, y, w = so.synth_batch(4 * B, F, 5, weights="mixed")
    mk = lambda kind: sb.Trainer(sb.make_desc(F, hidden, [sb.ACT_RELU] * 2, optimizer=kind, learning_rate=LR, max_batch=B,
                                              precision=prec), deterministic=True)
    ck, ck_ada = str(tmp_path / "rprop.ckpt"), str(tmp_path / "adadelta.ckpt")
    with mk(sb.OPT_RPROP) as t:
        t.set_params(theta0); t.load_dataset(X, y, w)
        for i in range(4):
            t.step_resident((i % 4) * B, B)
        t.save_checkpoint(ck)
        saved = (t.get_params(), *_state(sb, t))
        assert np.any(saved[2] != np.float32(LR)) and np.any(saved[1] != 0)
        for i in range(4):
            t.step_resident((i % 4) * B, B)
        cont = (t.get_params(), *_state(sb, t))
    with mk(sb.OPT_RPROP) as t:
        t.load_checkpoint(ck)
        assert t.global_step == 4
        for a, b, what in zip((t.get_params(), *_state(sb, t)), saved, ("theta", "s1", "s2")):
            _bits_equal(a, b, "loaded " + what)
        t.load_dataset(X, y, w)
        for i in range(4):
            t.step_resident((i % 4) * B, B)
        for a, b, what in zip((t.get_params(), *_state(sb, t)), cont, ("theta", "s1", "s2")):
            _bits_equal(a, b, "resumed " + what)
    with mk(sb.OPT_ADADELTA) as t:
        t.set_params(theta0)
        t.save_checkpoint(ck_ada)
        with pytest.raises(sb.ShifuB200Error) as e:
            t.load_checkpoint(ck)
        assert e.value.code == sb.capi.SB_ERR_FORMAT
    with mk(sb.OPT_RPROP) as t:
        with pytest.raises(sb.ShifuB200Error) as e:
            t.load_checkpoint(ck_ada)
        assert e.value.code == sb.capi.SB_ERR_FORMAT
        s1, s2 = _state(sb, t)
        assert np.all(s1 == 0) and np.all(s2 == np.float32(LR))


# ---- the worker ----
def _worker_epochs(lines):
    return [(int(l.split("current_epoch:")[1].split(",")[0]), float(l.split("training_loss:")[1].split(",")[0]),
             float(l.split("valid_loss:")[1])) for l in lines]


def _exported(sb, final):
    return sb.capi.savedmodel_read(final, "shifu_input_0", "shifu_output_0")[4]


@pytest.mark.parametrize("precision", ["fp32", "fp32_tc"])
def test_worker_sync_replicas_matches_the_oracle(sb, tmp_path, precision):
    from test_host_mirrors import _Seq, _run_worker
    from shifu_tensorflow_b200 import trainer as tr
    lr, epochs = 0.01, 6
    rc, lines, env, (X, y, w, F, conf) = _run_worker(sb, tmp_path, 1000, epochs, {
        "Optimizer": "rprop", "LearningRate": lr, "Schedule": "sync_replicas", "Precision": precision})
    assert rc == 0
    ctx = tr.load_data(env["TRAINING_DATA_PATH"], list(range(1, F + 1)), 0, -1, 0.2, rng=_Seq(5))
    tx, ty, tw, vx, vy, vw = (np.asarray(ctx[k], np.float32) for k in (
        "train_data", "train_target", "train_data_sample_weight", "valid_data", "valid_target", "valid_data_sample_weight"))
    net = so.NetDesc(F, [8, 4], [so.ACT_TANH, so.ACT_RELU])
    with sb.Trainer(tr.model(F, conf, 128)) as t0:
        assert t0.desc.optimizer == sb.OPT_RPROP
        t0.init_xavier(11)
        theta = t0.get_params()
    ref = rr.SyncReplicasTrainer(net, so.unflatten_params(net, theta), so.OptConfig(kind=rr.RPROP, lr=lr),
                                 so.replicas_to_aggregate(1000, 0.2, 100))
    batches = so.split_batches(len(tx), 100)
    want = []
    while ref.global_step < epochs:
        for bi in batches:
            L, gs = ref.run(tx[bi], ty[bi], tw[bi])
            if gs >= epochs:
                break
        A, z, yh = so.forward(net, so.unflatten_params(net, ref.theta), vx)
        want.append((gs, float(L), float(so.loss_value(z, yh, vy, vw, so.LOSS_MSE)[0])))
    got = _worker_epochs(lines)
    assert [g[0] for g in got] == [x[0] for x in want]
    assert np.abs(np.array(got)[:, 1:] - np.array(want)[:, 1:]).max() <= 1e-4
    assert want[-1][2] < want[0][2], "the loss must move"
    flat = _exported(sb, env["FINAL_MODEL_PATH"])
    assert np.linalg.norm(flat - ref.theta) <= 1e-3 * np.linalg.norm(ref.theta)


def test_worker_deterministic_runs_are_bit_identical(sb, tmp_path):
    from test_host_mirrors import _run_worker
    runs = []
    for k in range(2):
        d = tmp_path / ("run%d" % k)
        d.mkdir()
        rc, lines, env, _ = _run_worker(sb, d, 1000, 4, {"Optimizer": "rprop", "LearningRate": 0.01, "Precision": "bf16",
                                                         "Deterministic": True})
        assert rc == 0
        runs.append(([e[1:] for e in _worker_epochs(lines)], _exported(sb, env["FINAL_MODEL_PATH"])))
    assert runs[0][0] == runs[1][0] and len(runs[0][0]) >= 4
    _bits_equal(runs[0][1], runs[1][1], "exported weights")
