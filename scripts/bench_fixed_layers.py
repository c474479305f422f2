#!/usr/bin/env python
"""Gain of fine-tuning with frozen layers (sb_trainer_set_fixed_layers, ModelConfig FixedLayers): resident rows/s and
kernels per step of the cfg2 and cfg1 steps with nothing frozen, layer 1 frozen and layers 1 and 2 frozen (FixedBias
true), alternated within one process, several rounds (medians and ranges).  bf16 mode, run_resident, synthetic data.
With two GPUs it also times a two-rank peer-exchange run (Schedule = batch: one update per mini-batch) of the same
settings; with one it says so and skips it.

    python scripts/bench_fixed_layers.py [--rounds 3] [--steps 200] [--warmup 20]

Prints the card name and power limit, one line per configuration, then one JSON object."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import shifu_tensorflow_b200 as sb  # noqa: E402

CONFIGS = {
    "cfg2": dict(F=2000, hidden=[1024, 512, 256], batch=8192, optimizer=sb.OPT_MOMENTUM, lr=0.01),
    "cfg1": dict(F=1000, hidden=[512, 256, 128], batch=4096, optimizer=sb.OPT_ADAM, lr=0.001),
}
SETTINGS = {"none": (), "[1]": (1,), "[1,2]": (1, 2)}
N_BATCHES = 8


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def trainer(c, fixed, device=0, rank=0, world=1):
    desc = sb.make_desc(c["F"], c["hidden"], [sb.ACT_RELU] * len(c["hidden"]), loss=sb.LOSS_MSE, optimizer=c["optimizer"],
                        learning_rate=c["lr"], max_batch=c["batch"], precision=sb.PREC_BF16)
    t = sb.Trainer(desc, device=device, rank=rank, world=world, fixed_layers=fixed)
    t.init_xavier(1234)
    return t


def rate(c, data, fixed, steps, warmup):
    """-> (rows/s, kernels per step) of one trainer"""
    B = c["batch"]
    with trainer(c, fixed) as t:
        t.load_dataset(*data)
        offs = [(i % N_BATCHES) * B for i in range(max(steps, warmup))]
        t.run_resident(offs[:warmup], B)
        t.sync()
        t0 = time.perf_counter()
        t.run_resident(offs[:steps], B)
        t.sync()
        dt = time.perf_counter() - t0
        t.step_resident(0, B)           # a single captured step: what kernels_per_step reports
        return steps * B / dt, t.kernels_per_step(B)


def rate_two_ranks(c, data, fixed, steps, warmup):
    """two ranks on devices 0 and 1 with the peer-memory exchange, one host thread each; -> rows/s over both ranks"""
    B = c["batch"]
    ts = [trainer(c, fixed, device=r, rank=r, world=2) for r in range(2)]
    try:
        bases = [t.exchange_base for t in ts]
        for t in ts:
            t.set_peer_pointers(bases)
            t.load_dataset(*data)
        offs = [(i % N_BATCHES) * B for i in range(max(steps, warmup))]

        def run(t, n):
            t.run_resident(offs[:n], B)
            t.sync()

        def both(n):
            th = [threading.Thread(target=run, args=(t, n)) for t in ts]
            for x in th:
                x.start()
            for x in th:
                x.join()

        both(warmup)
        t0 = time.perf_counter()
        both(steps)
        return 2 * steps * B / (time.perf_counter() - t0)
    finally:
        for t in ts:
            t.close()


def summary(v):
    v = np.asarray(v) / 1e6
    return {"M_rows_s_median": round(float(np.median(v)), 3), "range": [round(float(v.min()), 3), round(float(v.max()), 3)]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    a = ap.parse_args()
    print("card (name, power limit):", card(), flush=True)
    two = sb.capi.device_count() >= 2
    if not two:
        print("one GPU: the two-rank peer-exchange run is skipped", flush=True)
    out = {}
    for name, c in CONFIGS.items():
        X = np.random.RandomState(1).rand(N_BATCHES * c["batch"], c["F"]).astype(np.float32)
        y = (np.random.RandomState(2).rand(N_BATCHES * c["batch"]) > 0.5).astype(np.float32)
        w = np.ones_like(y)
        data = (X, y, w)
        r = {k: [] for k in SETTINGS}
        r2 = {k: [] for k in SETTINGS}
        kps = {}
        for _ in range(a.rounds):
            for k, fixed in SETTINGS.items():      # alternated within a round
                v, kps[k] = rate(c, data, fixed, a.steps, a.warmup)
                r[k].append(v)
                if two:
                    r2[k].append(rate_two_ranks(c, data, fixed, a.steps, a.warmup))
        res = {}
        for k in SETTINGS:
            res[k] = dict(summary(r[k]), kernels_per_step=kps[k])
            res[k]["gain_pct"] = round(100.0 * (res[k]["M_rows_s_median"] / res["none"]["M_rows_s_median"] - 1), 1)
            if two:
                res[k]["two_ranks_p2p"] = summary(r2[k])
        out[name] = res
        print(name, json.dumps(res), flush=True)
    print(json.dumps({"card": card(), "rounds": a.rounds, "steps": a.steps, "results": out}))


if __name__ == "__main__":
    main()
