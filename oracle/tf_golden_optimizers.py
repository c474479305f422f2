#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY - generator of TF-written golden vectors for the optimizers of oracle/tf_optimizers.py
(Adagrad, RMSProp, FTRL), the companion of oracle/tf_golden.py.  No TensorFlow exists where this project is built and
tested, so it has not been run; on any machine with tensorflow 1.x or 2.x

    python oracle/tf_golden_optimizers.py --out tests/golden/tf_golden_optimizers.npz

writes three updates of each case below on fixed gradients, and
tests/test_optimizers_oracle.py::test_tf_golden_optimizers_when_present checks the oracle's rules against them (it is
skipped while the file is absent).  What it pins: the update forms, RMSProp's `rms` slot starting at 1 (the oracle switch
OptConfig.rmsprop_ms_starts_at_one), and FTRL's exact zeros (one gradient coordinate is 0 in every step, with l1 = 0)."""
import argparse

import numpy as np

from oracle import tf_optimizers as tfo

# (name, kind, oracle keyword arguments); the TF optimizer of each is built from the same values below
CASES = [
    ("adagrad", tfo.OPT_ADAGRAD, {}),
    ("adagrad_acc05", tfo.OPT_ADAGRAD, dict(initial_accumulator=0.5)),
    ("rmsprop", tfo.OPT_RMSPROP, {}),
    ("rmsprop_mom", tfo.OPT_RMSPROP, dict(momentum=0.7, rho=0.8, eps=1e-6)),
    ("ftrl", tfo.OPT_FTRL, {}),
    ("ftrl_l1l2", tfo.OPT_FTRL, dict(l1=0.01, l2=0.2)),
]
N, LR = 64, 0.05


def inputs():
    rng = np.random.default_rng(11)
    theta0 = rng.standard_normal(N).astype(np.float32)
    grads = [(rng.standard_normal(N) * 10.0 ** rng.uniform(-3, 1, N)).astype(np.float32) for _ in range(3)]
    for g in grads:
        g[0] = 0.0
    return theta0, grads


def build_and_run(out_path):
    import tensorflow as tf
    tf1 = tf.compat.v1 if hasattr(tf, "compat") and hasattr(tf.compat, "v1") else tf
    if hasattr(tf1, "disable_eager_execution"):
        tf1.disable_eager_execution()
    theta0, grads = inputs()
    out = {"theta0": theta0, "lr": np.float32(LR), "tf_version": tf.__version__}
    for i, g in enumerate(grads):
        out["grad%d" % i] = g
    for name, kind, kw in CASES:
        cfg = tfo.tf_config(kind, LR, **kw)
        if kind == tfo.OPT_ADAGRAD:
            make = lambda: tf1.train.AdagradOptimizer(LR, initial_accumulator_value=cfg.initial_accumulator)
        elif kind == tfo.OPT_RMSPROP:
            make = lambda: tf1.train.RMSPropOptimizer(LR, decay=cfg.rho, momentum=cfg.momentum, epsilon=cfg.eps)
        else:
            make = lambda: tf1.train.FtrlOptimizer(LR, learning_rate_power=-0.5,
                                                   initial_accumulator_value=cfg.initial_accumulator,
                                                   l1_regularization_strength=cfg.l1, l2_regularization_strength=cfg.l2)
        g = tf1.Graph()
        with g.as_default():
            v = tf1.Variable(theta0, name="theta")
            gp = tf1.placeholder(tf.float32, [N])
            train = make().apply_gradients([(gp, v)])
            with tf1.Session() as sess:
                sess.run(tf1.global_variables_initializer())
                for step in range(3):
                    sess.run(train, {gp: grads[step]})
                    out["%s_step%d" % (name, step + 1)] = sess.run(v)
    np.savez_compressed(out_path, **out)
    print("wrote", out_path, "with TF", tf.__version__)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="tests/golden/tf_golden_optimizers.npz")
    build_and_run(ap.parse_args().out)
