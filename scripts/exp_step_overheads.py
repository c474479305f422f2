"""Where do the microseconds of a cfg1 step go?  Runs K resident steps per SB_EXP setting (separate processes, the
flag is read once) and prints ms/step.  Measurement aid only (SB_EXP variants compute wrong results)."""
import json, os, subprocess, sys, time

CHILD = r'''
import os, sys, time, numpy as np
sys.path.insert(0, os.getcwd())
import shifu_tensorflow_b200 as sb
cfg = dict(cfg1=(1000, [512, 256, 128], 4096, 1), cfg2=(2000, [1024, 512, 256], 8192, 3))[sys.argv[1]]
F, hidden, B, opt = cfg
desc = sb.make_desc(F, hidden, [2] * len(hidden), loss=0, optimizer=opt, learning_rate=0.01, max_batch=B, precision=1)
nb = 16
rng = np.random.RandomState(0)
X = rng.standard_normal((nb * B, F)).astype(np.float32); y = (rng.uniform(size=(nb * B, 1)) < 0.2).astype(np.float32)
with sb.Trainer(desc) as t:
    t.init_xavier(1); t.load_dataset(X, y, None)
    for i in range(30): t.step_resident_async((i % nb) * B, B)
    t.sync()
    best = 1e9
    for rep in range(5):
        t0 = time.perf_counter()
        for i in range(400): t.step_resident_async((i % nb) * B, B)
        t.sync()
        best = min(best, (time.perf_counter() - t0) / 400 * 1e3)
    print("%.5f" % best)
'''

def main():
    out = {}
    for cfg in ("cfg1", "cfg2"):
        for name, env in [("base", {}), ("no_dw_budget", {"SB_NO_DW_BUDGET": "1"}), ("old_tail_schedule", {"SB_OLD_SCHED": "1"}), ("no_desc_prefetch", {"SB_PREP": "0"})]:
            e = dict(os.environ); e.update(env)
            r = subprocess.run([sys.executable, "-c", CHILD, cfg], env=e, capture_output=True, text=True, timeout=300)
            out["%s/%s" % (cfg, name)] = r.stdout.strip().splitlines()[-1] if r.returncode == 0 and r.stdout.strip() else "ERR " + r.stderr[-300:]
            print(cfg, name, out["%s/%s" % (cfg, name)], flush=True)
    print(json.dumps(out, indent=1))

if __name__ == "__main__":
    main()
