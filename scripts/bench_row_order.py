#!/usr/bin/env python
"""Cost of reading the resident set through a row order (sb_trainer_set_row_order): resident rows/s of the cfg2 and cfg1
steps (bf16, run_resident) in the physical order and through a random permutation, alternated, several rounds (medians
and ranges); the in-graph span of gather_batch_kernel (SB_STEP_TRACE) and its bytes over that span against the H100
SXM's 3.35 TB/s.  Synthetic data.

    python scripts/bench_row_order.py [--rounds 3] [--steps 200] [--warmup 20]

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
HBM_BYTES_S = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def trainer(c, trace=False):
    desc = sb.make_desc(c["F"], c["hidden"], [sb.ACT_RELU] * len(c["hidden"]), loss=sb.LOSS_MSE, optimizer=c["optimizer"],
                        learning_rate=c["lr"], max_batch=c["batch"], precision=sb.PREC_BF16)
    if trace:
        os.environ["SB_STEP_TRACE"] = "1"
    try:
        t = sb.Trainer(desc)
    finally:
        os.environ.pop("SB_STEP_TRACE", None)
    t.init_xavier(1234)
    return t


def rate(c, data, ordered, steps, warmup):
    B = c["batch"]
    with trainer(c) as t:
        t.load_dataset(*data)
        if ordered:
            t.set_row_order(np.random.default_rng(5).permutation(len(data[0])))
        offs = [(i % N_BATCHES) * B for i in range(max(steps, warmup))]
        t.run_resident(offs[:warmup], B)
        t.sync()
        t0 = time.perf_counter()
        t.run_resident(offs[:steps], B)
        t.sync()
        return steps * B / (time.perf_counter() - t0)


def spans(c, data, ordered):
    B = c["batch"]
    with trainer(c, trace=True) as t:
        t.load_dataset(*data)
        if ordered:
            t.set_row_order(np.random.default_rng(5).permutation(len(data[0])))
        t.run_resident([(i % N_BATCHES) * B for i in range(16)], B)
        t.sync()
        names, st = t.debug_step_trace()
    return {n: round((int(s[10]) - int(s[2])) * 1e-3, 2) for n, s in zip(names, st) if s[10] > s[2] > 0}


def gather_bytes(c):
    """bytes gather_batch_kernel must move for one bf16 batch: each row's ldF bf16 read and written, its order entry, y and
    w read and written"""
    ldF = (c["F"] + 7) // 8 * 8
    return c["batch"] * (2 * 2 * ldF + 4 + 2 * 2 * 4)


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
            for ordered in (False, True):
                r[ordered].append(rate(c, data, ordered, a.steps, a.warmup))
        res = {}
        for ordered in (False, True):
            v = np.asarray(r[ordered]) / 1e6
            res["ordered" if ordered else "physical"] = {"M_rows_s_median": round(float(np.median(v)), 3),
                                                         "range": [round(float(v.min()), 3), round(float(v.max()), 3)]}
        res["cost_pct"] = round(100.0 * (1 - res["ordered"]["M_rows_s_median"] / res["physical"]["M_rows_s_median"]), 2)
        res["spans_us"] = {"physical": spans(c, data, False), "ordered": spans(c, data, True)}
        g_us = res["spans_us"]["ordered"].get("gather_batch")
        res["gather_bytes"] = gather_bytes(c)
        if g_us:
            bw = gather_bytes(c) / (g_us * 1e-6)
            res["gather_TB_s"] = round(bw / 1e12, 3)
            res["gather_share_of_3.35TB_s"] = round(bw / HBM_BYTES_S, 3)
        out[name] = res
        print(name, json.dumps(res), flush=True)
    print(json.dumps({"card": card(), "rounds": a.rounds, "steps": a.steps, "results": out}))


if __name__ == "__main__":
    main()
