"""Bagged-model scoring on the eval net (2000 -> 1024 -> 512 -> 256 -> 1, relu): one sb_ensemble_t of K members against K
sb_model_t called one after the other plus the statistics formed by the caller, with the two arms alternated in one run.
The members have distinct seeded weights (bench_sensitivity.seeded with seeds 7, 8, ...).

    (a) device   1 Mi device-resident rows per call (bench.py's eval chunk): sb_ensemble_score_device against K
                 sb_model_score_device calls + torch mean / max / min / median
    (b) host     131 072 pinned host rows (bench.py's eval e2e): sb_ensemble_score against K sb_model_score calls + numpy
                 statistics
    (c) compute  rows/s of compute() from 1 and 64 Python threads: sb_ensemble_score_row_f64 against the K models'
                 sb_model_score_row_f64 in turn

    python scripts/bench_ensemble.py [--k 5] [--iters 5] [--precs bf16,fp32_tc] [--out DIR]

Prints one JSON line per precision with the median and range of each arm, whether the outputs of the two arms agree
bit for bit at the timed sizes, and ensemble_stats_kernel's share of the device leg's kernel time from a torch.profiler
run of its own; the card's name and power limit are read in the same run."""
import argparse
import json
import os
import sys
import threading
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_sensitivity import F, HIDDEN, PRECS, ROOT, card, seeded  # noqa: E402

sys.path.insert(0, ROOT)

DEVICE_ROWS = 1 << 20      # bench.py EVAL_CHUNK
HOST_ROWS = 131072


def spread(ts):
    return {"median": round(float(np.median(ts)), 5), "min": round(float(np.min(ts)), 5), "max": round(float(np.max(ts)), 5)}


def rate(rows, ts):
    return {"median": round(rows / float(np.median(ts)) / 1e6, 3), "min": round(rows / float(np.max(ts)) / 1e6, 3),
            "max": round(rows / float(np.min(ts)) / 1e6, 3)}


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def stats_np(S):
    return np.stack([S.mean(axis=1, dtype=np.float32), S.max(axis=1), S.min(axis=1), np.median(S, axis=1)], axis=1)


def compute_rate(fn, X, threads):
    """rows/s of fn(row) over the rows of X split among `threads` Python threads"""
    per = len(X) // threads
    go = threading.Barrier(threads + 1)
    errs = []

    def run(t):
        go.wait()
        try:
            for i in range(t * per, (t + 1) * per):
                fn(X[i])
        except Exception as e:     # noqa: BLE001 - surfaced below
            errs.append(e)

    th = [threading.Thread(target=run, args=(t,)) for t in range(threads)]
    [t.start() for t in th]
    go.wait()
    t0 = time.perf_counter()
    [t.join() for t in th]
    dt = time.perf_counter() - t0
    if errs:
        raise errs[0]
    return per * threads / dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--k", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--precs", default="bf16,fp32_tc")
    ap.add_argument("--compute-rows", type=int, default=3200, help="rows per compute() measurement")
    ap.add_argument("--out", default=None, help="directory for the profiler's kernel table (not written when unset)")
    a = ap.parse_args()
    import torch
    import shifu_tensorflow_b200 as sb
    name = card()
    flats = [seeded(7 + g) for g in range(a.k)]
    g = torch.Generator(device="cuda"); g.manual_seed(1)
    Xd = torch.empty((DEVICE_ROWS, F), dtype=torch.float32, device="cuda").normal_(generator=g).clamp_(-4, 4)
    px = torch.empty((HOST_ROWS, F), dtype=torch.float32).pin_memory()
    px.numpy()[:] = np.clip(np.random.default_rng(2).standard_normal((HOST_ROWS, F), dtype=np.float32), -4, 4)
    Xc = np.clip(np.random.default_rng(3).standard_normal((a.compute_rows, F)), -4, 4)
    for pn in a.precs.split(","):
        descs = [sb.make_desc(F, HIDDEN, [sb.capi.ACT_RELU] * 3, precision=PRECS[pn]) for _ in range(a.k)]
        e = sb.Ensemble.create(descs, flats)
        models = [sb.Model.create(d, f) for d, f in zip(descs, flats)]
        dS = torch.empty((DEVICE_ROWS, a.k), dtype=torch.float32, device="cuda")
        dT = torch.empty((DEVICE_ROWS, 4), dtype=torch.float32, device="cuda")
        outs = [torch.empty(DEVICE_ROWS, dtype=torch.float32, device="cuda") for _ in models]
        torch.cuda.synchronize()

        def dev_ensemble():
            e.score_device(Xd.data_ptr(), DEVICE_ROWS, dS.data_ptr(), dT.data_ptr())
            e.sync()

        def dev_models():
            for m, o in zip(models, outs):
                m.score_device(Xd.data_ptr(), DEVICE_ROWS, o.data_ptr())
            for m in models:
                m.sync()
            S = torch.stack(outs, dim=1)
            st = torch.stack([S.mean(1), S.max(1).values, S.min(1).values, S.median(1).values], dim=1)
            torch.cuda.synchronize()
            return S, st

        host = {}

        def host_ensemble():
            host["e"] = e.score(px.numpy())

        def host_models():
            S = np.stack([m.score(px.numpy()) for m in models], axis=1)
            host["m"] = (S, stats_np(S))

        arms = {"device_ensemble": dev_ensemble, "device_models": dev_models, "host_ensemble": host_ensemble,
                "host_models": host_models}
        for f in arms.values():                          # warm-up: module loads, plans
            f()
        times = {k: [] for k in arms}
        for _ in range(a.iters):
            for k, f in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                f()
                times[k].append(time.perf_counter() - t0)
        # the outputs of the two arms at the timed sizes
        S_m, st_m = dev_models()
        dev_same = bool(torch.equal(dS.view(torch.int32), S_m.view(torch.int32)))
        dev_stats_same = {c: bool(torch.equal(dT[:, i].view(torch.int32), st_m[:, i].view(torch.int32)))
                          for i, c in enumerate(("mean", "max", "min", "median"))}
        dev_mean_diff = float((dT[:, 0] - st_m[:, 0]).abs().max().item())
        (hs, ht), (ms, mt) = host["e"], host["m"]
        host_same = bool((bits(hs) == bits(ms)).all())
        host_stats_same = {c: bool((bits(ht[:, i]) == bits(mt[:, i])).all()) for i, c in enumerate(("mean", "max", "min", "median"))}
        host_mean_diff = float(np.abs(ht[:, 0] - mt[:, 0]).max())
        # (c) compute() rows/s, the two arms alternated per thread count
        comp = {}
        for threads in (1, 64):
            ens_r, mod_r = [], []
            for _ in range(3):
                ens_r.append(compute_rate(e.score_row_f64, Xc, threads))
                mod_r.append(compute_rate(lambda row: [m.score_row_f64(row) for m in models], Xc, threads))
            comp[threads] = {"ensemble_rows_per_s": [round(v, 1) for v in sorted(ens_r)],
                             "models_rows_per_s": [round(v, 1) for v in sorted(mod_r)]}
        # ensemble_stats_kernel's share of the device call, profiled apart
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
            dev_ensemble()
        ev = [x for x in prof.key_averages() if x.device_type.name == "CUDA"]
        total_us = sum(x.self_device_time_total for x in ev)
        stats_us = sum(x.self_device_time_total for x in ev if "ensemble_stats_kernel" in x.key)
        load_us = sum(x.self_device_time_total for x in ev if "load_batch_kernel" in x.key)
        if a.out:
            os.makedirs(a.out, exist_ok=True)
            with open(os.path.join(a.out, "ensemble_%s_kernels.txt" % pn), "w") as fh:
                fh.write(prof.key_averages().table(sort_by="self_device_time_total", row_limit=25))
        dev_speed = float(np.median(times["device_models"]) / np.median(times["device_ensemble"]))
        host_speed = float(np.median(times["host_models"]) / np.median(times["host_ensemble"]))
        print(json.dumps({
            "precision": pn, "card": name, "k": a.k, "iters": a.iters,
            "device": {"rows": DEVICE_ROWS, "sec_ensemble": spread(times["device_ensemble"]),
                       "sec_models": spread(times["device_models"]),
                       "M_rows_per_s_ensemble": rate(DEVICE_ROWS, times["device_ensemble"]),
                       "M_rows_per_s_models": rate(DEVICE_ROWS, times["device_models"]), "speedup": round(dev_speed, 4),
                       "scores_bit_identical": dev_same, "stats_bit_identical": dev_stats_same,
                       "mean_max_abs_diff": dev_mean_diff},
            "host": {"rows": HOST_ROWS, "sec_ensemble": spread(times["host_ensemble"]), "sec_models": spread(times["host_models"]),
                     "M_rows_per_s_ensemble": rate(HOST_ROWS, times["host_ensemble"]),
                     "M_rows_per_s_models": rate(HOST_ROWS, times["host_models"]), "speedup": round(host_speed, 4),
                     "scores_bit_identical": host_same, "stats_bit_identical": host_stats_same,
                     "mean_max_abs_diff": host_mean_diff},
            "compute": comp,
            "device_kernels_ms": round(total_us / 1e3, 3), "ensemble_stats_ms": round(stats_us / 1e3, 3),
            "ensemble_stats_share_of_kernels": round(stats_us / max(total_us, 1e-9), 5),
            "load_batch_share_of_kernels": round(load_us / max(total_us, 1e-9), 5),
            "device_bytes": {"ensemble": e.device_bytes(), "models": sum(m.device_bytes() for m in models)},
        }), flush=True)
        for m in models:
            m.close()
        e.close()
        del dS, dT, outs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
