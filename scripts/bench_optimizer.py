"""In-graph span and bandwidth of layer 0's optimizer pass (`opt`) and of the other layers' (`opt_side`) on cfg2's shapes,
for each of the eight optimizers (run on the GPU box).  The span is read from the step trace (SB_STEP_TRACE: %globaltimer
of the kernel's dependency wait to the last block's exit) of several resident steps; bandwidth = the bytes the update
needs over that span.

    python scripts/bench_optimizer.py [out.json]

Bytes per parameter: theta read + write 8, gradient read 4, each state stream read + write 8 (Momentum and Adagrad 1,
Adam, Adadelta, RMSProp, FTRL and RPROP 2), bf16 shadow write 2 for the hidden-layer weights."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ["SB_STEP_TRACE"] = "1"
import numpy as np
import shifu_tensorflow_b200 as sb
from oracle import shifu_oracle as so
from oracle import tf_optimizers as tfo

B, F, HIDDEN = 8192, 2000, [1024, 512, 256]   # cfg2
OPTS = {"adadelta": so.OPT_ADADELTA, "adam": so.OPT_ADAM, "sgd": so.OPT_SGD, "momentum": so.OPT_MOMENTUM,
        "adagrad": tfo.OPT_ADAGRAD, "rmsprop": tfo.OPT_RMSPROP, "ftrl": tfo.OPT_FTRL, "rprop": sb.OPT_RPROP}
STATE_STREAMS = {"adadelta": 2, "adam": 2, "sgd": 0, "momentum": 1, "adagrad": 1, "rmsprop": 2, "ftrl": 2, "rprop": 2}


def op_bytes(name, n_weights, n_other):
    per = 12 + 8 * STATE_STREAMS[name]
    return n_weights * (per + 2) + n_other * per


dims = [F] + HIDDEN
w0, b0 = dims[0] * dims[1], dims[1]
w_rest = sum(dims[l] * dims[l + 1] for l in range(1, len(HIDDEN)))
b_rest = sum(HIDDEN[1:]) + HIDDEN[-1] + 1          # hidden biases, output layer weights and bias
rng = np.random.default_rng(0)
X = rng.standard_normal((4 * B, F), dtype=np.float32)
y = (rng.random(4 * B, dtype=np.float32) < 0.2).astype(np.float32)
w = np.ones(4 * B, np.float32)
res = {}
for name, kind in OPTS.items():
    desc = sb.make_desc(F, HIDDEN, [so.ACT_RELU] * len(HIDDEN), optimizer=kind, learning_rate=0.001, max_batch=B, precision=1)
    spans = {"opt": [], "opt_side": []}
    with sb.Trainer(desc) as t:
        t.init_xavier(1)
        t.load_dataset(X, y, w)
        t.run_resident([(i % 4) * B for i in range(8)], B)
        for rep in range(20):
            t.run_resident([(i % 4) * B for i in range(4)], B)
            names, stamps = t.debug_step_trace()
            for nm, st in zip(names, stamps):
                if nm in spans and st[2] and st[10]:
                    spans[nm].append((int(st[10]) - int(st[2])) / 1e3)
    out = {}
    for nm, nbytes in (("opt", op_bytes(name, w0, b0)), ("opt_side", op_bytes(name, w_rest, b_rest))):
        us = float(np.median(spans[nm]))
        out[nm] = {"us_median": us, "us_min": float(np.min(spans[nm])), "MB": nbytes / 1e6, "GB_per_s": nbytes / (us * 1e-6) / 1e9}
    res[name] = out
    print(name, json.dumps(out), flush=True)
if len(sys.argv) > 1:
    json.dump(res, open(sys.argv[1], "w"))
