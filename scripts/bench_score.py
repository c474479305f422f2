"""Batch-scoring throughput of the trained cfg2 net (BASELINE.json configs[4]: eval path, 2000-col MLP [1024,512,256]).
device-resident: rows generated on the GPU (torch) and scored through sb_model_score_device in 1M-row slabs;
host: sb_model_score on pinned host rows (H2D + D2H inside).  Prints one JSON line."""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import shifu_tensorflow_b200 as sb
from oracle import shifu_oracle as so

F, hidden = 2000, [1024, 512, 256]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
try:      # the same peak source as bench.py: measured peaks, else the H100 SXM data-sheet dense bf16 rate
    PEAK = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))).get("bf16_tflops", 989.0)) * 1e12
except Exception:
    PEAK = 989e12
net = so.NetDesc(F, hidden, [so.ACT_RELU] * 3)
flat = so.flatten_params(so.xavier_init(net, 1))
out = {}
for prec, name in ((sb.PREC_BF16, "bf16"), (sb.PREC_FP32, "fp32")):
    m = sb.Model.create(sb.make_desc(F, hidden, net.acts, precision=prec), flat)
    slab = 1 << 20 if prec == sb.PREC_BF16 else 1 << 18
    X = torch.randn(slab, F, device="cuda").clamp_(-4, 4)
    Y = torch.empty(slab, device="cuda")
    st = torch.cuda.ExternalStream(m.stream)
    torch.cuda.synchronize()
    m.score_device(X.data_ptr(), slab, Y.data_ptr()); m.sync()
    n_slabs = 10 if prec == sb.PREC_BF16 else 3
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(n_slabs):
        m.score_device(X.data_ptr(), slab, Y.data_ptr())
    e1.record(st); m.sync()
    ms = e0.elapsed_time(e1)
    rows = slab * n_slabs
    rps = rows / (ms / 1e3)
    # parity spot check of the slab against the oracle
    idx = np.arange(0, slab, slab // 64)[:64]
    want = so.score_rows(net, so.unflatten_params(net, flat), X[idx].cpu().numpy().astype(np.float64))
    err = float(np.abs(Y[idx].cpu().numpy() - want).max())
    # host leg
    hrows = 1 << 18
    Xh = torch.randn(hrows, F).clamp_(-4, 4).pin_memory().numpy()
    m.score(Xh[:1024])
    t0 = time.perf_counter(); m.score(Xh); th = time.perf_counter() - t0
    out[name] = {"device_resident_rows_per_s": rps, "tflops": rps * 5407232 / 1e12, "frac_of_peak": rps * 5407232 / PEAK,
                 "seconds_per_100M_rows": 1e8 / rps, "max_abs_err_vs_oracle": err, "host_rows_per_s": hrows / th}
    m.close()
print(json.dumps({"metric": "rows/sec batch scoring, cfg2 net (2000 -> 1024 -> 512 -> 256 -> 1)", "n_gpus": 1, **out}))
