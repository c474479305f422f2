#!/usr/bin/env python
"""Print the headline numbers of bench.py JSON lines:  python scripts/summarize_bench.py <json> [...]"""
import json
import sys

for f in sys.argv[1:]:
    for line in open(f):
        line = line.strip()
        if not line.startswith("{"):
            continue
        d = json.loads(line)
        if d.get("impl") == "reference":
            print("%s: reference arm %.0f %s (%s cores, %s)" % (f, d["value"], d["unit"], d["cpu_baseline"].get("cores"), d["cpu_baseline"].get("sample")))
            continue
        r = d["roofline"]
        print("%s: N=%d %s  %.2f M rows/s  %.1f us/step  span %.1f us  longest GEMM %s %.1f us %.0f TF/s (frac %.3f)  step frac of peak %.3f" % (
            f, d["n_gpus"], d["config"]["workload"].split(":")[0], d["value"] / 1e6, d["ms_per_step"] * 1e3, r.get("step_span_us", 0),
            r.get("kernel", "").split()[1] if r.get("kernel") else "", r.get("kernel_us", 0), r["achieved"], r["frac"], r.get("step_fraction_of_peak", 0)))
        for k in r.get("kernels", []):
            c = k.get("cta0")
            print("    %-10s %7.2f us  [%7.2f .. %7.2f]  %s%s" % (k["kernel"], k["us"], k["begin_us"], k["end_us"],
                                                             ("%.0f TF/s" % k["tflops"]) if k.get("tflops") else "", ("  " + json.dumps(c)) if c and k["kernel"].startswith("xchg") else ""))
        for key in ("sustained", "e2e", "eval", "ingest", "cpu_baseline", "clocks"):
            if d.get(key):
                print("   ", key, json.dumps(d[key])[:400])
        a = d.get("also")
        if a:
            print("    also %s: %.2f M rows/s %.1f us/step" % (a["config"]["workload"].split(":")[0], a["value"] / 1e6, a["ms_per_step"] * 1e3))
