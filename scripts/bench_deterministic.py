#!/usr/bin/env python
"""Cost of deterministic training (sb_trainer_set_deterministic): resident rows/s of the cfg2 and cfg1 steps with the
flag off and on, alternated, several rounds (medians and ranges), and the in-graph spans (SB_STEP_TRACE) of the kernels
whose epilogues or plans change (the fused output layer, the dA GEMMs, the dW GEMMs).  bf16 mode, synthetic data.

    python scripts/bench_deterministic.py [--rounds 3] [--steps 200] [--warmup 20]

Prints the card name and power limit, then one JSON object."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import shifu_tensorflow_b200 as sb  # noqa: E402

CONFIGS = {
    "cfg2": dict(F=2000, hidden=[1024, 512, 256], batch=8192, optimizer=sb.OPT_MOMENTUM, lr=0.01),
    "cfg1": dict(F=1000, hidden=[512, 256, 128], batch=4096, optimizer=sb.OPT_ADAM, lr=0.001),
}
N_BATCHES = 8


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def trainer(c, det, trace=False):
    desc = sb.make_desc(c["F"], c["hidden"], [sb.ACT_RELU] * len(c["hidden"]), loss=sb.LOSS_MSE, optimizer=c["optimizer"],
                        learning_rate=c["lr"], max_batch=c["batch"], precision=sb.PREC_BF16)
    if trace:
        os.environ["SB_STEP_TRACE"] = "1"
    try:
        t = sb.Trainer(desc, deterministic=det)
    finally:
        os.environ.pop("SB_STEP_TRACE", None)
    t.init_xavier(1234)
    return t


def rate(c, data, det, steps, warmup):
    B = c["batch"]
    with trainer(c, det) as t:
        t.load_dataset(*data)
        offs = [(i % N_BATCHES) * B for i in range(max(steps, warmup))]
        t.run_resident(offs[:warmup], B)
        t.sync()
        t0 = time.perf_counter()
        t.run_resident(offs[:steps], B)
        t.sync()
        return steps * B / (time.perf_counter() - t0)


def spans(c, data, det):
    B = c["batch"]
    with trainer(c, det, trace=True) as t:
        t.load_dataset(*data)
        t.run_resident([(i % N_BATCHES) * B for i in range(16)], B)
        t.sync()
        names, st = t.debug_step_trace()
    return {n: round((int(s[10]) - int(s[2])) * 1e-3, 2) for n, s in zip(names, st) if s[10] > s[2] > 0}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    a = ap.parse_args()
    print("card (name, power limit):", card(), flush=True)
    out = {}
    for name, c in CONFIGS.items():
        X = np.random.RandomState(1).rand(N_BATCHES * c["batch"], c["F"]).astype(np.float32)
        y = (np.random.RandomState(2).rand(N_BATCHES * c["batch"]) > 0.5).astype(np.float32)
        w = np.ones_like(y)
        data = (X, y, w)
        r = {False: [], True: []}
        for _ in range(a.rounds):
            for det in (False, True):
                r[det].append(rate(c, data, det, a.steps, a.warmup))
        res = {}
        for det in (False, True):
            v = np.asarray(r[det]) / 1e6
            res["det" if det else "default"] = {"M_rows_s_median": round(float(np.median(v)), 3),
                                                "range": [round(float(v.min()), 3), round(float(v.max()), 3)]}
        res["cost_pct"] = round(100.0 * (1 - res["det"]["M_rows_s_median"] / res["default"]["M_rows_s_median"]), 2)
        res["spans_us"] = {"default": spans(c, data, False), "det": spans(c, data, True)}
        out[name] = res
        print(name, json.dumps(res), flush=True)
    print(json.dumps({"card": card(), "rounds": a.rounds, "steps": a.steps, "results": out}))


if __name__ == "__main__":
    main()
