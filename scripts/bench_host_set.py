#!/usr/bin/env python
"""Training from a set in pinned host memory against the same set in HBM: resident rows/s of run_resident at cfg1 and
cfg2 (bf16), with the set in HBM and in host memory (sb_debug_force_host_set), in the physical order and through a random
row order, alternated within one process, several rounds (medians and ranges).  A host-set step reads its batch's rows
over PCIe (ldF x 2 bytes per row and bf16 part); inside a run_resident graph the next step's rows are fetched on k CTAs
while the current step's GEMMs run on the other SMs.  The host runs sweep k (SB_FETCH_CTAS) in the physical order.  The
achieved PCIe rate is rows/s times the bytes per row, set beside a plain pinned host-to-device copy measured in the same
run.

    python scripts/bench_host_set.py [--rounds 3] [--steps 200] [--warmup 20] [--out DIR]

Prints the card name, power limit and host RAM, one line per measurement, then one JSON object (also written to
DIR/bench_host_set.json when --out is given)."""
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
FETCH_CTAS = (4, 8, 16, 32)
DEFAULT_CTAS = 16
VARIANTS = ([("hbm", "physical", 0)] + [("host", "physical", k) for k in FETCH_CTAS] +
            [("hbm", "shuffled", 0), ("host", "shuffled", DEFAULT_CTAS)])


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def host_ram_gb():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemTotal:"):
                return int(line.split()[1]) / 1e6
    return float("nan")


def pinned_h2d_gbs(nbytes=1 << 30, reps=10):
    """plain cudaMemcpy from pinned host memory to the device (torch's copy), GB/s"""
    import torch
    src = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    dst = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    dst.copy_(src, non_blocking=True)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        dst.copy_(src, non_blocking=True)
    b.record()
    torch.cuda.synchronize()
    return nbytes * reps / (a.elapsed_time(b) * 1e-3) / 1e9


def trainer(c, host, ctas):
    os.environ["SB_FETCH_CTAS"] = str(ctas or DEFAULT_CTAS)      # read when the trainer is created
    desc = sb.make_desc(c["F"], c["hidden"], [sb.ACT_RELU] * len(c["hidden"]), loss=sb.LOSS_MSE, optimizer=c["optimizer"],
                        learning_rate=c["lr"], max_batch=c["batch"], precision=sb.PREC_BF16)
    t = sb.Trainer(desc)
    t.init_xavier(1234)
    t.debug_force_host_set(host)
    return t


def rate(c, data, host, order, ctas, steps, warmup):
    B = c["batch"]
    with trainer(c, host == "host", ctas) as t:
        t.load_dataset(*data)
        assert t.dataset_on_host == (host == "host")
        if order == "shuffled":
            t.set_row_order(np.random.default_rng(5).permutation(len(data[1])))
        offs = [(i % N_BATCHES) * B for i in range(max(steps, warmup))]
        t.run_resident(offs[:warmup], B)
        t.sync()
        t0 = time.perf_counter()
        t.run_resident(offs[:steps], B)
        t.sync()
        return steps * B / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert sb.capi.device_count() > 0, "needs an H100"
    info = {"card": card(), "host_ram_gb": round(host_ram_gb(), 1)}
    print("card: %s, host RAM %.0f GB" % (info["card"], info["host_ram_gb"]), flush=True)
    h2d = [pinned_h2d_gbs() for _ in range(3)]
    info["pinned_h2d_gbs"] = sorted(h2d)
    print("pinned H2D copy: %s GB/s" % ", ".join("%.1f" % v for v in sorted(h2d)), flush=True)
    res = {}
    for name, c in CONFIGS.items():
        rng = np.random.default_rng(1)
        n = N_BATCHES * c["batch"]
        data = (rng.standard_normal((n, c["F"]), dtype=np.float32), (rng.random(n) < 0.3).astype(np.float32),
                np.ones(n, np.float32))
        got = {v: [] for v in VARIANTS}
        for _ in range(a.rounds):
            for v in VARIANTS:
                got[v].append(rate(c, data, v[0], v[1], v[2], a.steps, a.warmup))
        row_bytes = (c["F"] + 7) // 8 * 8 * 2
        for (host, order, ctas), r in got.items():
            med = float(np.median(r))
            key = "%s/%s/%s" % (name, host, order) + ("/k=%d" % ctas if ctas else "")
            res[key] = {"rows_per_s": sorted(r), "median": med,
                        "pcie_gbs": med * row_bytes / 1e9 if host == "host" else None}
            print("%-22s %6.2f M rows/s (%s)%s" % (key, med / 1e6, ", ".join("%.2f" % (x / 1e6) for x in sorted(r)),
                                                  "  PCIe %.1f GB/s" % (med * row_bytes / 1e9) if host == "host" else ""),
                  flush=True)
    out = {"info": info, "results": res, "steps": a.steps, "rounds": a.rounds}
    print(json.dumps(out))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_host_set.json"), "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
