"""The scorer's per-row boundary: compute() (sb_model_score_row_f64) latency and rate from many threads, and
sb_model_score time by row count on both sides of SMALL_ROWS.

Two nets, seeded weights: cfg2's eval net (2000 -> 1024 -> 512 -> 256 -> 1, relu) and a dummydl-shaped one
(1522 -> 100 x 20 -> 1, relu), each in fp32 and fp32_tc.

    python scripts/bench_score_rows.py [--trees DIR ...] [--rounds N] [--out FILE]

Every tree is a checkout with its library built (default: this one).  Each (tree, net, precision) is measured in a
subprocess of its own, the trees alternating within every round, so that two builds compare in one session.  compute()
is timed through the C-ABI (ctypes, the GIL released during the call) with a host clock around each call; a call ends
when its score is on the host.  sb_model_score is timed the same way (host rows in, scores out), and
sb_model_score_device by CUDA events on the model's stream (the forward alone).  Prints the card, its power limit and max SM clock, one JSON line per measurement and a
table of the medians over rounds."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NETS = {"cfg2": (2000, [1024, 512, 256]), "dummydl": (1522, [100] * 20)}
PRECS = {"fp32": 0, "fp32_tc": 2}
THREADS = [1, 2, 4, 8, 16, 32, 64]
SCORE_ROWS = [1, 2, 4, 8, 16, 32, 64, 96, 128, 129, 192, 256]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"card": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:      # noqa: BLE001 - reported, not fatal
        return {"card": "not measured (%s)" % e, "power_limit": "not measured", "max_sm_clock": "not measured"}


def worker(tree, net, prec):
    sys.path.insert(0, tree)
    import shifu_tensorflow_b200 as sb
    F, hidden = NETS[net]
    rng = np.random.default_rng(1)
    parts, prev = [], F
    for h in hidden + [1]:
        parts += [rng.standard_normal((prev, h)).astype(np.float32) * np.float32(np.sqrt(2.0 / prev)),
                  np.zeros(h, np.float32)]
        prev = h
    flat = np.concatenate([p.ravel() for p in parts])
    m = sb.Model.create(sb.make_desc(F, hidden, [sb.ACT_RELU] * len(hidden), precision=PRECS[prec]), flat)
    lib = sb.capi.lib()
    fn, h = lib.sb_model_score_row_f64, m._h
    X = rng.standard_normal((4096, F))
    ptrs = [X[i].ctypes.data_as(C.POINTER(C.c_double)) for i in range(len(X))]
    res = {"net": net, "precision": prec, "compute": {}, "score_ms": {}}

    def calls(tid, n, lat):
        out = C.c_double()
        for i in range(n):
            p = ptrs[(tid * 997 + i) % len(ptrs)]
            t0 = time.perf_counter()
            s = fn(h, p, F, C.byref(out))
            lat.append(time.perf_counter() - t0)
            if s != 0:
                raise RuntimeError(lib.sb_last_error().decode())

    calls(0, 100, [])                                   # warm-up (modules, graphs)
    for T in THREADS:
        per = max(40, 3000 // T)
        lats = [[] for _ in range(T)]
        th = [threading.Thread(target=calls, args=(t, per, lats[t])) for t in range(T)]
        t0 = time.perf_counter()
        [t.start() for t in th]; [t.join() for t in th]
        wall = time.perf_counter() - t0
        lat = np.concatenate([np.asarray(l) for l in lats]) * 1e6
        res["compute"][T] = {"p50_us": float(np.percentile(lat, 50)), "p99_us": float(np.percentile(lat, 99)),
                             "rows_per_s": T * per / wall}
    Xf = rng.standard_normal((max(SCORE_ROWS), F)).astype(np.float32)
    for r in SCORE_ROWS:
        for _ in range(3):
            m.score(Xf[:r])
        ts = []
        for _ in range(50):
            t0 = time.perf_counter(); m.score(Xf[:r]); ts.append(time.perf_counter() - t0)
        res["score_ms"][r] = statistics.median(ts) * 1e3
    # device time of the forward alone: sb_model_score_device between CUDA events on the model's stream
    import torch
    dX = torch.from_numpy(Xf).cuda()
    dOut = torch.empty(len(Xf), device="cuda")
    st = torch.cuda.ExternalStream(m.stream)
    torch.cuda.synchronize()
    res["device_us"] = {}
    for r in SCORE_ROWS:
        for _ in range(3):
            m.score_device(dX.data_ptr(), r, dOut.data_ptr())
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for _ in range(50):
            m.score_device(dX.data_ptr(), r, dOut.data_ptr())
        e1.record(st)
        m.sync()
        res["device_us"][r] = e0.elapsed_time(e1) * 1e3 / 50
    m.close()
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trees", nargs="+", default=[ROOT])
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", nargs=3, metavar=("TREE", "NET", "PREC"), help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(*a.worker)
    info = card()
    print(json.dumps(info))
    rows = []
    for rnd in range(a.rounds):
        for net in NETS:
            for prec in PRECS:
                for tree in (a.trees if rnd % 2 == 0 else a.trees[::-1]):
                    p = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", tree, net, prec],
                                       capture_output=True, text=True)
                    if p.returncode != 0:
                        raise SystemExit("worker %s %s %s failed:\n%s" % (tree, net, prec, p.stderr[-3000:]))
                    r = json.loads(p.stdout.strip().splitlines()[-1])
                    r.update(tree=tree, round=rnd, **info)
                    print(json.dumps(r), flush=True)
                    rows.append(r)
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(json.dumps(r) for r in rows) + "\n")
    # medians over rounds
    print("\n%s, power limit %s, max SM clock %s" % (info["card"], info["power_limit"], info["max_sm_clock"]))
    for net in NETS:
        for prec in PRECS:
            print("\n== %s %s ==" % (net, prec))
            for tree in a.trees:
                rs = [r for r in rows if r["tree"] == tree and r["net"] == net and r["precision"] == prec]
                med = lambda f: statistics.median(f(r) for r in rs)
                print("  %s" % tree)
                print("    compute(): " + "  ".join("T=%s p50 %.0fus p99 %.0fus %.0f rows/s" % (
                    T, med(lambda r: r["compute"][str(T)]["p50_us"]), med(lambda r: r["compute"][str(T)]["p99_us"]),
                    med(lambda r: r["compute"][str(T)]["rows_per_s"])) for T in THREADS))
                print("    score(): " + "  ".join("%d rows %.3f ms" % (n, med(lambda r: r["score_ms"][str(n)]))
                                                  for n in SCORE_ROWS))
                print("    score_device() device time: " + "  ".join("%d rows %.1f us" % (
                    n, med(lambda r: r["device_us"][str(n)])) for n in SCORE_ROWS))


if __name__ == "__main__":
    main()
