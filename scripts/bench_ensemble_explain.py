"""Explaining a bagged model's score on the eval net (K members of 2000 -> 1024 -> 512 -> 256 -> 1, relu, each with its own
seeded weights as in bench_sensitivity.py) over every column of a device-resident set, with three arms alternated in one
process:

    (a) sb_ensemble_sensitivity (mean)
    (b) sb_ensemble_reason_codes (mean, top k)
    (c) what a caller can do without them, and only for the mean: K sb_model_sensitivity calls with the [rows, 2000]
        deltas into K device buffers, then the torch mean of the deltas and its weighted sums

    python scripts/bench_ensemble_explain.py [--rows 16384] [--members 5] [--k 5] [--iters 3] [--precs bf16,fp32_tc] [--out DIR]

Prints one JSON line per precision: pairs/s and member-pairs/s of each arm, the device bytes (a) allocates for its
explanation buffers (measured as the free-memory drop of its first call) against the bytes of (c)'s deltas, the share of
(a)'s time in ensemble_stat_kernel from a torch.profiler run of its own, and the card's name and power limit.
(a) and (c) start from the same member pair scores (each member's are bit-identical to its model's), so their mean
deltas differ only by the fp32 rounding of the two means and the subtractions: with scores in [0, 1], at most
(3K + 5) u per delta, u = 2^-24.  The script checks (a)'s sums against (c)'s within that bound summed over rows."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_sensitivity import F, HIDDEN, PRECS, ROOT, card, seeded  # noqa: E402

sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=16384)
    ap.add_argument("--members", type=int, default=5)
    ap.add_argument("--k", type=int, default=5)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--precs", default="bf16,fp32_tc")
    ap.add_argument("--out", default=None, help="directory for the profiler's kernel table (not written when unset)")
    a = ap.parse_args()
    import torch
    import shifu_tensorflow_b200 as sb
    name = card()
    K, rows = a.members, a.rows
    flats = [seeded(7 + g) for g in range(K)]
    X = torch.from_numpy(np.clip(np.random.default_rng(1).standard_normal((rows, F), dtype=np.float32), -4, 4)).cuda()
    w = torch.from_numpy(np.random.default_rng(2).uniform(0.0, 2.0, rows).astype(np.float32)).cuda()
    pos = torch.empty((rows, a.k), dtype=torch.int32, device="cuda")
    d = torch.empty((rows, a.k), dtype=torch.float32, device="cuda")
    pairs = rows * F
    u = 2.0 ** -24
    for pn in a.precs.split(","):
        descs = [sb.make_desc(F, HIDDEN, [sb.capi.ACT_RELU] * 3, precision=PRECS[pn]) for _ in range(K)]
        e = sb.Ensemble.create(descs, flats)
        models = [sb.Model.create(descs[g], flats[g]) for g in range(K)]
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        res = {"a": e.sensitivity(X, w=w)}
        torch.cuda.synchronize()
        a_bytes = free0 - torch.cuda.mem_get_info()[0]
        bufs = [torch.empty((rows, F), dtype=torch.float32, device="cuda") for _ in range(K)]
        c_bytes = sum(b.numel() * 4 for b in bufs)

        def ens_sens():
            res["a"] = e.sensitivity(X, w=w)

        def ens_reason():
            e.reason_codes(X, a.k, pos=pos, d=d)

        def per_member():
            for m, b in zip(models, bufs):
                m.sensitivity(X, w=w, deltas=b)
            D = torch.stack(bufs).mean(0)
            wd = w.double()[:, None] * D.double()
            res["c"] = {"sum": wd.sum(0).cpu().numpy(), "sum_sq": (wd * D.double()).sum(0).cpu().numpy(), "D": D}

        paths = {"ensemble_sensitivity": ens_sens, "ensemble_reason_codes": ens_reason, "member_deltas_torch_mean": per_member}
        for f in paths.values():                       # warm-up: buffers, module loads
            f()
        times = {p: [] for p in paths}
        for _ in range(a.iters):
            for p, f in paths.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                f()
                torch.cuda.synchronize()
                times[p].append(time.perf_counter() - t0)
        # (a) against (c): the mean's rounding only
        wa = np.abs(w.double().cpu().numpy())
        Dc = res["c"]["D"].double().cpu().numpy()
        tol = (3 * K + 5) * u
        b1 = wa.sum() * tol
        b2 = (wa[:, None] * tol * (2 * np.abs(Dc) + tol)).sum(0)
        err1 = np.abs(res["a"]["sum"] - res["c"]["sum"])
        err2 = np.abs(res["a"]["sum_sq"] - res["c"]["sum_sq"])
        agree = bool(np.all(err1 <= b1) and np.all(err2 <= b2))
        # the statistic launch's share of (a), profiled apart
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
            t0 = time.perf_counter()
            ens_sens()
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
        ev = [x for x in prof.key_averages() if x.device_type.name == "CUDA"]
        total_us = sum(x.self_device_time_total for x in ev)
        stat_us = sum(x.self_device_time_total for x in ev if "ensemble_stat_kernel" in x.key)
        if a.out:
            os.makedirs(a.out, exist_ok=True)
            with open(os.path.join(a.out, "ensemble_explain_%s_kernels.txt" % pn), "w") as fh:
                fh.write(prof.key_averages().table(sort_by="self_device_time_total", row_limit=30))
        med = {p: float(np.median(t)) for p, t in times.items()}
        print(json.dumps({"precision": pn, "card": name, "rows": rows, "cols": F, "members": K, "k": a.k, "iters": a.iters,
                          "sec_per_call": {p: round(v, 4) for p, v in med.items()},
                          "pairs_per_s_M": {p: round(pairs / v / 1e6, 2) for p, v in med.items()},
                          "member_pairs_per_s_M": {p: round(K * pairs / v / 1e6, 2) for p, v in med.items()},
                          "ensemble_vs_member_deltas": round(med["member_deltas_torch_mean"] / med["ensemble_sensitivity"], 3),
                          "explain_buffer_bytes": int(a_bytes), "member_deltas_bytes": int(c_bytes),
                          "stat_kernel_ms": round(stat_us / 1e3, 3), "stat_share_of_call": round(stat_us / 1e6 / wall, 4),
                          "stat_share_of_kernels": round(stat_us / max(total_us, 1e-9), 4),
                          "mean_sums_agree": agree, "max_sum_err_over_bound": float(np.max(err1 / b1)),
                          "routes": e.routes()}), flush=True)
        del bufs, res
        for m in models:
            m.close()
        e.close()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
