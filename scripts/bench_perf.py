"""Evaluate 100 M device-resident scores (sb_perf_*): add, summary, and the gains / ROC / PR points at 10 levels, each
weighted and unweighted.  Alternated with a torch arm on the same card (torch.sort(stable=True), fp64 cumsum,
unique_consecutive, the same formulas); the two arms' results are checked against each other.  Kernel times come from a
separate torch.profiler run; achieved bytes/s are the bytes the passes move (counted here from the row and run counts and
the sort passes that run) over the summed kernel time, against the data sheet's 3.35 TB/s.

    python scripts/bench_perf.py [--rows 100000000] [--reps 5] [--out /tmp/bench_perf.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import shifu_tensorflow_b200 as sb  # noqa: E402

HBM_BPS = 3.35e12
LEVELS = np.arange(1, 11) / 10.0
AXES = ("action_rate", "recall", "fpr")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def ours(p, s, y, w, n):
    p.reset()
    p.add_device(s.data_ptr(), y.data_ptr(), w.data_ptr(), n)
    summ = p.summary()
    pts = {(a, wt): p.points(a, LEVELS, weighted=wt) for a in AXES for wt in (False, True)}
    return summ, pts


def torch_arm(s, y, w):
    order = torch.sort(s, descending=True, stable=True).indices
    ss, yy, ww = s[order], y[order], w[order].double()
    pos = yy == 1
    tp = torch.cumsum(pos.long(), 0)
    fp = torch.cumsum((~pos).long(), 0)
    wtp = torch.cumsum(torch.where(pos, ww, 0.0), 0)
    wfp = torch.cumsum(torch.where(pos, 0.0, ww), 0)
    t, counts = torch.unique_consecutive(ss, return_counts=True)
    last = torch.cumsum(counts, 0) - 1
    tp, fp, wtp, wfp = tp[last], fp[last], wtp[last], wfp[last]
    P, N, Wp, Wn = int(tp[-1]), int(fp[-1]), float(wtp[-1]), float(wfp[-1])
    z = torch.zeros(1, dtype=torch.long, device=s.device)
    tp0, fp0 = torch.cat([z, tp[:-1]]), torch.cat([z, fp[:-1]])
    wtp0, wfp0 = torch.cat([z.double(), wtp[:-1]]), torch.cat([z.double(), wfp[:-1]])
    a2 = int(((fp - fp0) * (2 * tp0 + tp - tp0)).sum())
    d = (tp * N - fp * P).abs()
    j = int(torch.argmax(d))          # torch returns the first maximum
    wd = (wtp * Wn - wfp * Wp).abs()
    summ = {"n_distinct": len(t), "auc": a2 / (2 * P * N), "ks": int(d[j]) / (P * N), "ks_score": float(t[j]),
            "w_auc": float(((wfp - wfp0) * (wtp0 + wtp) * 0.5).sum()) / (Wp * Wn), "w_ks": float(wd.max()) / (Wp * Wn),
            "ap": float(((tp - tp0).double() * (tp.double() / (tp + fp).double())).sum()) / P}
    lv = torch.tensor(LEVELS, device=s.device)
    pts = {}
    for a in AXES:
        for wt in (False, True):
            num = {"action_rate": (wtp + wfp) if wt else (tp + fp).double(), "recall": wtp if wt else tp.double(),
                   "fpr": wfp if wt else fp.double()}[a]
            idx = torch.searchsorted(num / num[-1], lv)
            pts[(a, wt)] = {"tp": tp[idx].cpu().numpy(), "fp": fp[idx].cpu().numpy()}
    return summ, pts


def agree(a, b):
    sa, pa = a
    sb_, pb = b
    assert sa["n_distinct"] == sb_["n_distinct"], (sa["n_distinct"], sb_["n_distinct"])
    assert sa["auc"] == sb_["auc"] and sa["ks"] == sb_["ks"] and sa["ks_score"] == sb_["ks_score"]
    for k in ("w_auc", "w_ks", "ap"):
        assert abs(sa[k] - sb_[k]) < 1e-9, (k, sa[k], sb_[k])
    for key in pa:
        assert np.array_equal(pa[key]["tp"], pb[key]["tp"]) and np.array_equal(pa[key]["fp"], pb[key]["fp"]), key


def sort_passes(s):
    u = s.view(torch.int32).long() & 0xFFFFFFFF
    u = torch.where(u == 0x80000000, torch.zeros_like(u), u)
    key = torch.where(u >= 0x80000000, u, (~u) & 0x7FFFFFFF)
    n = s.numel()
    return sum(1 for d in range(4) if int(torch.bincount((key >> (8 * d)) & 255, minlength=256).max()) != n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    n = a.rows
    g = torch.Generator("cuda").manual_seed(1)
    y = (torch.rand(n, device="cuda", generator=g) < 0.2).float()
    s = torch.sigmoid(torch.randn(n, device="cuda", generator=g) + 1.5 * y - 1.0)
    w = torch.randint(1, 4, (n,), device="cuda", generator=g).float() * 0.5
    torch.cuda.synchronize()
    info = {"card": card(), "rows": n}
    with sb.Performance(reserve_rows=n) as p:
        r_ours, r_torch = ours(p, s, y, w, n), torch_arm(s, y, w)   # warm-up, and the agreement check
        agree(r_ours, r_torch)
        t_ours, t_torch = [], []
        for _ in range(a.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ours(p, s, y, w, n)
            t_ours.append(time.perf_counter() - t0)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            torch_arm(s, y, w)
            torch.cuda.synchronize()
            t_torch.append(time.perf_counter() - t0)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            ours(p, s, y, w, n)
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            if "perf_" in e.key:
                kern[e.key.split("(")[0].replace("void sb::", "")] = (e.device_time_total / 1e3, e.count)
        m = r_ours[0]["n_distinct"]
    passes = sort_passes(s)
    bytes_moved = 20 * n + 16 * n * passes + 16 * n + 36 * m + 32 * m
    k_ms = sum(v[0] for v in kern.values())
    med = lambda v: float(np.median(v)) * 1e3
    info.update({
        "n_distinct": m, "sort_passes": passes, "summary": {k: float(v) for k, v in r_ours[0].items()},
        "ours_ms": {"median": med(t_ours), "min": min(t_ours) * 1e3, "max": max(t_ours) * 1e3},
        "torch_ms": {"median": med(t_torch), "min": min(t_torch) * 1e3, "max": max(t_torch) * 1e3},
        "kernels_ms": {k: {"total_ms": v[0], "launches": v[1]} for k, v in sorted(kern.items())},
        "kernel_ms_total": k_ms, "bytes": bytes_moved, "achieved_TBps": bytes_moved / (k_ms / 1e3) / 1e12,
        "share_of_3.35TBps": bytes_moved / (k_ms / 1e3) / HBM_BPS,
    })
    print(json.dumps(info, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
