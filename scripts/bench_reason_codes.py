"""Per-row reason codes on the eval net (2000 -> 1024 -> 512 -> 256 -> 1, relu, seeded weights as in
bench_sensitivity.py): sb_model_reason_codes over every column of a device-resident set, against what a caller does
without it, in one run with the three alternated:

    (a) reason_codes: the top k per row on the device, rows * k (position, delta) pairs out
    (b) sensitivity without deltas: the same pair forwards with only the per-column sums
    (c) sensitivity with the [rows, 2000] deltas into a device buffer, then torch.topk on it

    python scripts/bench_reason_codes.py [--rows 16384] [--k 5] [--iters 5] [--precs bf16,fp32_tc] [--out DIR]

Prints one JSON line per precision: pairs/s of (a), (b) and (c), and the share of (a)'s time spent in sens_topk_kernel
from a torch.profiler run of its own (its kernel time over the call's time, and over all the call's kernel time), with
the card's name and power limit."""
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
    ap.add_argument("--k", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--precs", default="bf16,fp32_tc")
    ap.add_argument("--out", default=None, help="directory for the profiler's kernel table (not written when unset)")
    a = ap.parse_args()
    import torch
    import shifu_tensorflow_b200 as sb
    name = card()
    flat = seeded()
    X = torch.from_numpy(np.clip(np.random.default_rng(1).standard_normal((a.rows, F), dtype=np.float32), -4, 4)).cuda()
    pos = torch.empty((a.rows, a.k), dtype=torch.int32, device="cuda")
    d = torch.empty((a.rows, a.k), dtype=torch.float32, device="cuda")
    deltas = torch.empty((a.rows, F), dtype=torch.float32, device="cuda")
    pairs = a.rows * F
    for pn in a.precs.split(","):
        m = sb.Model.create(sb.make_desc(F, HIDDEN, [sb.capi.ACT_RELU] * 3, precision=PRECS[pn]), flat)

        def reason():
            m.reason_codes(X, a.k, pos=pos, d=d)

        def sens():
            m.sensitivity(X)

        def sens_topk():
            m.sensitivity(X, deltas=deltas)
            torch.topk(deltas, a.k, dim=1)
            torch.cuda.synchronize()

        paths = {"reason_codes": reason, "sensitivity": sens, "sensitivity_deltas_topk": sens_topk}
        for f in paths.values():                       # warm-up: buffers, module loads
            f()
        times = {p: [] for p in paths}
        for _ in range(a.iters):
            for p, f in paths.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                f()
                times[p].append(time.perf_counter() - t0)
        # the same bits as the deltas (c) ranks: reason_codes' deltas at its positions
        got = torch.gather(deltas, 1, pos.long())
        same = bool(torch.equal(got.view(torch.int32), d.view(torch.int32)))
        # the topk kernel's share of (a), profiled apart
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
            t0 = time.perf_counter()
            reason()
            wall = time.perf_counter() - t0
        ev = [e for e in prof.key_averages() if e.device_type.name == "CUDA"]        # kernels and copies
        total_us = sum(e.self_device_time_total for e in ev)
        topk_us = sum(e.self_device_time_total for e in ev if "sens_topk_kernel" in e.key)
        if a.out:
            os.makedirs(a.out, exist_ok=True)
            with open(os.path.join(a.out, "reason_codes_%s_kernels.txt" % pn), "w") as fh:
                fh.write(prof.key_averages().table(sort_by="self_device_time_total", row_limit=25))
        med = {p: float(np.median(t)) for p, t in times.items()}
        print(json.dumps({"precision": pn, "card": name, "rows": a.rows, "cols": F, "k": a.k, "iters": a.iters,
                          "sec_per_call": {p: round(v, 4) for p, v in med.items()},
                          "pairs_per_s_M": {p: round(pairs / v / 1e6, 2) for p, v in med.items()},
                          "reason_vs_sensitivity": round(med["sensitivity"] / med["reason_codes"], 4),
                          "reason_vs_deltas_topk": round(med["sensitivity_deltas_topk"] / med["reason_codes"], 4),
                          "topk_kernel_ms": round(topk_us / 1e3, 3),
                          "topk_share_of_call": round(topk_us / 1e6 / wall, 4),
                          "topk_share_of_kernels": round(topk_us / max(total_us, 1e-9), 4),
                          "bit_identical_to_deltas": same, "routes": m.routes()}), flush=True)
        m.close()


if __name__ == "__main__":
    main()
