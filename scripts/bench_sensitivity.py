"""Column sensitivity on the eval net (2000 -> 1024 -> 512 -> 256 -> 1, relu, seeded weights): sb_model_sensitivity over
every column of a device-resident set, against re-scoring materialised modified rows with sb_model_score_device over a
column subset, in the same run.

    python scripts/bench_sensitivity.py [--rows 16384] [--iters 3] [--base-cols 32] [--precs bf16,fp32_tc]

Prints one JSON line per precision: pairs/s of both paths, their ratio, and the achieved TFLOP/s of the sensitivity call
from the shapes (rows 2 W0 + pairs 2 (sum W - W0)), with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

F, HIDDEN = 2000, [1024, 512, 256]
PRECS = {"fp32": 0, "bf16": 1, "fp32_tc": 2, "bf16x2": 3}


def seeded(seed=7, gains=(1.4, 1.4, 1.4, 4.0)):
    rng = np.random.default_rng(seed)
    parts, prev = [], F
    for h, g in zip(HIDDEN + [1], gains):
        parts.append(rng.standard_normal((prev, h)).astype(np.float32) * np.float32(g / np.sqrt(prev)))
        parts.append((rng.standard_normal(h) * 0.1).astype(np.float32))
        prev = h
    return np.concatenate([p.ravel() for p in parts])


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def flops(rows, pairs):
    sizes = [F] + HIDDEN + [1]
    w = [a * b for a, b in zip(sizes[:-1], sizes[1:])]
    return rows * 2.0 * w[0] + pairs * 2.0 * (sum(w) - w[0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=16384)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--base-cols", type=int, default=32)
    ap.add_argument("--precs", default="bf16,fp32_tc")
    a = ap.parse_args()
    import torch
    import shifu_tensorflow_b200 as sb
    name = card()
    flat = seeded()
    X = torch.from_numpy(np.clip(np.random.default_rng(1).standard_normal((a.rows, F), dtype=np.float32), -4, 4)).cuda()
    for pn in a.precs.split(","):
        prec = PRECS[pn]
        m = sb.Model.create(sb.make_desc(F, HIDDEN, [sb.capi.ACT_RELU] * 3, precision=prec), flat)
        m.sensitivity(X)                                  # warm-up: buffers, module loads
        t0 = time.perf_counter()
        for _ in range(a.iters):
            m.sensitivity(X)
        dt = (time.perf_counter() - t0) / a.iters
        routes = m.routes()
        pairs = a.rows * F
        # re-scoring baseline: for each of base_cols columns, the set with that column zeroed, scored in full
        out = torch.empty(a.rows, dtype=torch.float32, device="cuda")
        Xm = X.clone()
        cols = list(range(0, F, F // a.base_cols))[:a.base_cols]

        def rescore():
            for c in cols:
                Xm.copy_(X)
                Xm[:, c] = 0.0
                torch.cuda.synchronize()
                m.score_device(Xm.data_ptr(), a.rows, out.data_ptr())
                m.sync()

        rescore()
        t0 = time.perf_counter()
        rescore()
        db = time.perf_counter() - t0
        # the copy of the set per column is the materialisation a caller pays; report the scoring share apart
        t0 = time.perf_counter()
        for c in cols:
            m.score_device(Xm.data_ptr(), a.rows, out.data_ptr())
        m.sync()
        ds = time.perf_counter() - t0
        base_rate = a.rows * len(cols) / db
        score_rate = a.rows * len(cols) / ds
        rate = pairs / dt
        print(json.dumps({"precision": pn, "card": name, "rows": a.rows, "cols": F, "sec_per_call": round(dt, 4),
                          "pairs_per_s": round(rate / 1e6, 2), "tflops": round(flops(a.rows, pairs) / dt / 1e12, 1),
                          "rescore_rows_per_s": round(base_rate / 1e6, 2), "score_only_rows_per_s": round(score_rate / 1e6, 2),
                          "speedup_vs_rescore": round(rate / base_rate, 2),
                          "speedup_vs_score_only": round(rate / score_rate, 2), "routes": routes}), flush=True)
        m.close()


if __name__ == "__main__":
    main()
