"""CPU oracle for the shifu-tensorflow tabular-DNN hot path.

TEST INFRASTRUCTURE ONLY.  Nothing in the shipped product (the package
``shifu-tensorflow_b200/`` or its CUDA library) imports this module; only
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline /
``--impl reference`` legs do, and only as the checker / the CPU arm.

PARITY UNPINNED (training): the reference pins no numeric result for training
anywhere (its only test asserts 0 <= score <= 1 on unseeded random input,
shifu-tensorflow-eval/src/test/java/ml/shifu/shifu/tensorflow/TensorflowModelTest.java:50-59)
and its arithmetic lives in un-vendored TensorFlow 1.x binaries (python
``tensorflow`` unpinned; ``org.tensorflow:*:1.4.0`` for scoring,
shifu-tensorflow-eval/pom.xml:45,59-73).  This file therefore restates the TF
ops the reference's script instantiates, each function citing the script line
that selects it.  The scorer half IS anchored: the forward pass is checked
against the reference's own SavedModel fixture (``dummydl``) through
``oracle/tf_formats.py`` (see tests/test_oracle_fixture.py and
tests/golden/make_golden.py).

All citations ``res/`` = shifu-tensorflow-on-yarn/src/main/resources/.
"""
from __future__ import annotations

import gzip
import io
import math
import random as _pyrandom
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

# --------------------------------------------------------------------------
# activation table          res/ssgd_monitor.py:74-88 (get_activation_fun)
# --------------------------------------------------------------------------
ACT_SIGMOID, ACT_TANH, ACT_RELU, ACT_LEAKYRELU = 0, 1, 2, 3
LEAKY_ALPHA = 0.2  # tf.nn.leaky_relu default alpha (TF library constant)


def get_activation_fun(name: Optional[str]) -> int:
    """name -> activation id; None / unknown -> leaky_relu (res/ssgd_monitor.py:74-88)."""
    if name is None:
        return ACT_LEAKYRELU
    name = name.lower()
    if name == "sigmoid":
        return ACT_SIGMOID
    if name == "tanh":
        return ACT_TANH
    if name == "relu":
        return ACT_RELU
    if name == "leakyrelu":
        return ACT_LEAKYRELU
    return ACT_LEAKYRELU


def _sigmoid(z):
    # numerically-stable logistic, same dtype as z
    out = np.empty_like(z)
    pos = z >= 0
    out[pos] = 1.0 / (1.0 + np.exp(-z[pos]))
    ez = np.exp(z[~pos])
    out[~pos] = ez / (1.0 + ez)
    return out


def act_forward(z: np.ndarray, act: int) -> np.ndarray:
    if act == ACT_SIGMOID:
        return _sigmoid(z)
    if act == ACT_TANH:
        return np.tanh(z)
    if act == ACT_RELU:
        return np.maximum(z, 0)
    if act == ACT_LEAKYRELU:
        return np.where(z > 0, z, z * z.dtype.type(LEAKY_ALPHA))
    raise ValueError(act)


def act_grad_from_output(a: np.ndarray, act: int) -> np.ndarray:
    """d act / dz expressed in the *output* a (what TF's SigmoidGrad/TanhGrad/ReluGrad use).

    leaky_relu with alpha>0 is sign preserving so a>0 <=> z>0.
    """
    one = a.dtype.type(1)
    if act == ACT_SIGMOID:
        return a * (one - a)
    if act == ACT_TANH:
        return one - a * a
    if act == ACT_RELU:
        return (a > 0).astype(a.dtype)
    if act == ACT_LEAKYRELU:
        return np.where(a > 0, one, a.dtype.type(LEAKY_ALPHA))
    raise ValueError(act)


# --------------------------------------------------------------------------
# network description / parameters
# --------------------------------------------------------------------------
@dataclass
class NetDesc:
    """Topology as read from ModelConfig.json (res/ssgd_monitor.py:91-107, 121)."""
    n_features: int
    hidden: List[int]
    acts: List[int]

    @property
    def dims(self) -> List[Tuple[int, int]]:
        d, prev = [], self.n_features
        for h in self.hidden:
            d.append((prev, h))
            prev = h
        d.append((prev, 1))  # output layer "shifu_output_0", sigmoid (res/ssgd_monitor.py:121)
        return d

    @property
    def n_params(self) -> int:
        return sum(i * o + o for i, o in self.dims)


def net_from_modelconf(model_conf: dict, n_features: int) -> NetDesc:
    """generate_from_modelconf (res/ssgd_monitor.py:91-107)."""
    tp = model_conf["train"]["params"]
    n = int(tp["NumHiddenLayers"])
    nodes = [int(s) for s in tp["NumHiddenNodes"]][:n]
    acts = [get_activation_fun(s) for s in tp["ActivationFunc"]][:n]
    return NetDesc(n_features, nodes, acts)


def xavier_init(net: NetDesc, seed: int, dtype=np.float32) -> List[np.ndarray]:
    """tf.contrib.layers.xavier_initializer() (uniform) on weights AND biases
    (res/ssgd_monitor.py:59-68).  limit = sqrt(6/(fan_in+fan_out)); for the 1-D
    bias TF takes fan_in = fan_out = out, i.e. limit = sqrt(3/out).
    Returns [W0, b0, W1, b1, ..., Wout, bout]; W is [in, out] row-major.
    The reference is unseeded; a seed is injected here so both sides agree.
    """
    rng = np.random.RandomState(seed)
    params = []
    for (i, o) in net.dims:
        lim_w = math.sqrt(6.0 / (i + o))
        lim_b = math.sqrt(3.0 / o)
        params.append(rng.uniform(-lim_w, lim_w, size=(i, o)).astype(dtype))
        params.append(rng.uniform(-lim_b, lim_b, size=(o,)).astype(dtype))
    return params


def flatten_params(params: Sequence[np.ndarray]) -> np.ndarray:
    """Flat layer-major order [W0, b0, W1, b1, ..., Wout, bout] - the C-ABI's order
    (variable names weight_hidden_layer{l} / biases_hidden_layer{l} /
    weight_shifu_output_0 / biases_shifu_output_0, res/ssgd_monitor.py:59,64,99-104,121)."""
    return np.concatenate([p.reshape(-1) for p in params])


def unflatten_params(net: NetDesc, flat: np.ndarray) -> List[np.ndarray]:
    out, off = [], 0
    for (i, o) in net.dims:
        out.append(flat[off:off + i * o].reshape(i, o)); off += i * o
        out.append(flat[off:off + o]); off += o
    assert off == flat.size
    return out


# --------------------------------------------------------------------------
# forward / loss / backward       res/ssgd_monitor.py:57-71, 110-129, 142
# --------------------------------------------------------------------------
LOSS_MSE, LOSS_SIGMOID_CE = 0, 1


def forward(net: NetDesc, params: Sequence[np.ndarray], X: np.ndarray):
    """A_l = act_l(A_{l-1} W_l + b_l) (nn_layer, res/ssgd_monitor.py:70); output
    y = sigmoid(A_L w + b) (res/ssgd_monitor.py:121).  Returns (acts list incl. A_0=X, z_out, yhat)."""
    A = [X]
    for l, act in enumerate(net.acts):
        W, b = params[2 * l], params[2 * l + 1]
        A.append(act_forward(A[-1] @ W + b, act))
    Wo, bo = params[-2], params[-1]
    z = A[-1] @ Wo + bo  # [B,1]
    return A, z, _sigmoid(z)


def loss_value(z: np.ndarray, yhat: np.ndarray, y: np.ndarray, w: np.ndarray, loss: int):
    """tf.losses.mean_squared_error(predictions=y, labels=y_, weights=sample_weight)
    (res/ssgd_monitor.py:129) with TF's default reduction SUM_BY_NONZERO_WEIGHTS:
    sum_i w_i (yhat_i - y_i)^2 / #{w_i != 0}, 0 when no weight is non-zero.
    LOSS_SIGMOID_CE is the north-star variant (sigmoid_cross_entropy_with_logits under
    the same reduction); the reference itself never uses it.
    Returns (loss, n_nz)."""
    dt = z.dtype.type
    n_nz = int(np.count_nonzero(w))
    if n_nz == 0:
        return dt(0), 0
    if loss == LOSS_MSE:
        per = (yhat - y) ** 2
    else:
        per = np.maximum(z, 0) - z * y + np.log1p(np.exp(-np.abs(z)))
    return dt(np.sum(per * w, dtype=z.dtype) / dt(n_nz)), n_nz


def backward(net: NetDesc, params, A, z, yhat, y, w, loss: int):
    """Gradients of loss_value wrt every W, b (what opt.minimize builds,
    res/ssgd_monitor.py:142).  Returns list in param order."""
    dt = z.dtype.type
    n_nz = int(np.count_nonzero(w))
    grads = [np.zeros_like(p) for p in params]
    if n_nz == 0:
        return grads
    if loss == LOSS_MSE:
        dz = dt(2) * w * (yhat - y) * yhat * (dt(1) - yhat) / dt(n_nz)
    else:
        dz = w * (yhat - y) / dt(n_nz)
    # output layer
    grads[-2] = A[-1].T @ dz
    grads[-1] = dz.sum(axis=0)
    dA = dz @ params[-2].T
    for l in range(len(net.acts) - 1, -1, -1):
        dZ = dA * act_grad_from_output(A[l + 1], net.acts[l])
        grads[2 * l] = A[l].T @ dZ
        grads[2 * l + 1] = dZ.sum(axis=0)
        if l > 0:
            dA = dZ @ params[2 * l].T
    return grads


def loss_and_grads(net, params, X, y, w, loss=LOSS_MSE):
    A, z, yhat = forward(net, params, X)
    L, _ = loss_value(z, yhat, y, w, loss)
    return L, backward(net, params, A, z, yhat, y, w, loss), yhat


# --------------------------------------------------------------------------
# optimizers (TF 1.x kernel forms)
# --------------------------------------------------------------------------
OPT_ADADELTA, OPT_ADAM, OPT_SGD, OPT_MOMENTUM = 0, 1, 2, 3


@dataclass
class OptConfig:
    kind: int = OPT_ADADELTA       # reference default, res/ssgd_monitor.py:138
    lr: float = 0.001              # ModelConfig train.params.LearningRate (res/ssgd_monitor.py:133)
    rho: float = 0.95              # tf.train.AdadeltaOptimizer defaults
    eps: float = 1e-8              # Adadelta epsilon / Adam epsilon (both 1e-8 in TF 1.x)
    beta1: float = 0.9             # tf.train.AdamOptimizer defaults (res/ssgd.py:57)
    beta2: float = 0.999
    momentum: float = 0.9          # north-star "SGD+momentum"; TF MomentumOptimizer form
    # TF ApplyAdadelta evaluation order: whether `var` is updated with the pre- (False, the
    # textbook form and TF >= 1.9) or post-update accum_update expression.  Unpinned
    # (SURVEY 7.2); default False, the C-ABI implements exactly this default.
    adadelta_var_uses_new_accum_update: bool = False


class Optimizer:
    """State + update on a flat fp32 vector.  Forms restated from TF 1.x
    core/kernels/training_ops.cc (library code, not in the reference tree)."""

    def __init__(self, cfg: OptConfig, n: int, dtype=np.float32):
        self.cfg, self.t = cfg, 0
        self.s1 = np.zeros(n, dtype)  # adadelta accum | adam m | momentum accum
        self.s2 = np.zeros(n, dtype)  # adadelta accum_update | adam v

    def apply(self, theta: np.ndarray, g: np.ndarray) -> np.ndarray:
        c, dt = self.cfg, theta.dtype.type
        self.t += 1
        if c.kind == OPT_SGD:            # ApplyGradientDescent (res/ssgd_monitor_bk.py:81)
            return theta - dt(c.lr) * g
        if c.kind == OPT_MOMENTUM:       # ApplyMomentum, use_nesterov=False
            self.s1 = self.s1 * dt(c.momentum) + g
            return theta - dt(c.lr) * self.s1
        if c.kind == OPT_ADAM:           # ApplyAdam (res/ssgd.py:57)
            lr_t = dt(c.lr * math.sqrt(1 - c.beta2 ** self.t) / (1 - c.beta1 ** self.t))
            self.s1 = self.s1 + (g - self.s1) * dt(1 - c.beta1)
            self.s2 = self.s2 + (g * g - self.s2) * dt(1 - c.beta2)
            return theta - lr_t * self.s1 / (np.sqrt(self.s2) + dt(c.eps))
        if c.kind == OPT_ADADELTA:       # ApplyAdadelta (res/ssgd_monitor.py:138)
            rho, eps = dt(c.rho), dt(c.eps)
            self.s1 = self.s1 * rho + g * g * (dt(1) - rho)
            upd = np.sqrt(self.s2 + eps) / np.sqrt(self.s1 + eps) * g
            self.s2 = self.s2 * rho + upd * upd * (dt(1) - rho)
            if c.adadelta_var_uses_new_accum_update:
                upd = np.sqrt(self.s2 + eps) / np.sqrt(self.s1 + eps) * g
            return theta - upd * dt(c.lr)
        raise ValueError(c.kind)


# --------------------------------------------------------------------------
# trainers
# --------------------------------------------------------------------------
class CleanTrainer:
    """'Clean' variant: one optimizer update per mini-batch (what BASELINE.json's
    cfg1/cfg2 describe).  With world>1 it restates synchronous data-parallel:
    every rank computes the gradient of *its own* mini-batch loss (own n_nz) and
    the update uses the mean over ranks (ConditionalAccumulator mean,
    res/ssgd_monitor.py:136-141)."""

    def __init__(self, net: NetDesc, params, opt: OptConfig, loss=LOSS_MSE, dtype=np.float32):
        self.net, self.loss, self.dtype = net, loss, dtype
        self.theta = flatten_params(params).astype(dtype)
        self.opt = Optimizer(opt, self.theta.size, dtype)
        self.last_grads = None

    def params(self):
        return unflatten_params(self.net, self.theta)

    def step(self, shards):
        """shards: list over ranks of (X, y, w).  Returns list of per-rank losses."""
        gsum, losses = None, []
        P = self.params()
        for (X, y, w) in shards:
            L, g, _ = loss_and_grads(self.net, P, X.astype(self.dtype), y.astype(self.dtype),
                                     w.astype(self.dtype), self.loss)
            g = flatten_params(g)
            gsum = g if gsum is None else gsum + g
            losses.append(L)
        g = gsum / self.dtype(len(shards))
        self.last_grads = g
        self.theta = self.opt.apply(self.theta, g)
        return losses

    def eval_loss(self, X, y, w):
        A, z, yhat = forward(self.net, self.params(), X.astype(self.dtype))
        return loss_value(z, yhat, y.astype(self.dtype), w.astype(self.dtype), self.loss)[0]


def replicas_to_aggregate(total_training_data_number: int, valid_rate: float, batch_size: int = 100,
                          ratio: float = 1) -> int:
    """int(total*(1-validRate)/BATCH_SIZE*ratio) (res/ssgd_monitor.py:139)."""
    return int(total_training_data_number * (1 - valid_rate) / batch_size * ratio)


def split_batches(n_rows: int, batch_size: int = 100) -> List[np.ndarray]:
    """total_batch=int(N/BATCH_SIZE); np.array_split -> sizes differ by <= 1
    (res/ssgd_monitor.py:189-192).  Returns index arrays."""
    total_batch = int(n_rows / batch_size)
    return np.array_split(np.arange(n_rows), total_batch)


class SyncReplicasTrainer:
    """Single-worker restatement of SyncReplicasOptimizer + ConditionalAccumulator as the
    reference drives it (res/ssgd_monitor.py:136-142, 218, 259-260, 268-276; TF library
    semantics restated, SURVEY 3.2): every run pushes its gradient tagged with the worker's
    local_step and then dequeues a token (local_step := token).  A push whose tag is older
    than the accumulator's step is dropped.  After R accepted pushes the accumulator MEAN is
    applied once, global_step += 1 and R tokens valued global_step are enqueued.  The chief
    seeds R tokens valued 0.  Arrival order = batch order."""

    def __init__(self, net, params, opt: OptConfig, R: int, loss=LOSS_MSE, dtype=np.float32):
        self.net, self.loss, self.dtype, self.R = net, loss, dtype, max(1, R)
        self.theta = flatten_params(params).astype(dtype)
        self.opt = Optimizer(opt, self.theta.size, dtype)
        self.global_step = 0
        self.local_step = 0
        self.tokens = [0] * self.R          # chief_init_op / get_init_tokens_op
        self.acc_sum, self.acc_n = np.zeros_like(self.theta), 0

    def run(self, X, y, w):
        """One sess.run([train_step, loss, global_step]).  Returns (loss, global_step)."""
        P = unflatten_params(self.net, self.theta)
        L, g, _ = loss_and_grads(self.net, P, X.astype(self.dtype), y.astype(self.dtype),
                                 w.astype(self.dtype), self.loss)
        if self.local_step >= self.global_step:       # fresh -> accepted
            self.acc_sum += flatten_params(g); self.acc_n += 1
        if self.acc_n >= self.R:                      # take_grad(R): mean, apply, new tokens
            self.theta = self.opt.apply(self.theta, self.acc_sum / self.dtype(self.acc_n))
            self.acc_sum[:] = 0; self.acc_n = 0
            self.global_step += 1
            self.tokens.extend([self.global_step] * self.R)
        if not self.tokens:
            raise RuntimeError("token queue empty: single worker would block")
        self.local_step = self.tokens.pop(0)
        return L, self.global_step


# --------------------------------------------------------------------------
# data loader                                   res/ssgd_monitor.py:348-454
# --------------------------------------------------------------------------
def load_data(paths: Sequence[str], feature_column_nums: Optional[Sequence[int]], target_column_num: int,
              sample_weight_column_num: int, valid_rate: float, rng=None, delimiter: str = "|"):
    """Restatement of load_data: gunzip each file (:376-377), split on '|' (:387), pick the selected
    columns -> float (:404-410), target float(columns[target]) (:398), weight: absent -> 1.0,
    negative -> 1.0 (:412-419), Bernoulli split: `random.random() >= validRate` -> train (:396).
    `rng` is an object with .random() (python's `random` module in the reference, unseeded there)."""
    rng = rng or _pyrandom
    out = {k: [] for k in ("train_data", "train_target", "valid_data", "valid_target",
                           "train_data_sample_weight", "valid_data_sample_weight")}
    for path in paths:
        with open(path, "rb") as f:
            gf = gzip.GzipFile(fileobj=io.BytesIO(f.read()))
            for raw in gf:
                line = raw.decode("utf-8")
                if len(line) == 0:
                    break
                columns = line.split(delimiter)
                if feature_column_nums is None:
                    feature_column_nums = [c for c in range(len(columns))
                                           if c != target_column_num and
                                           not (sample_weight_column_num >= 0 and c == sample_weight_column_num)]
                pre = "train" if rng.random() >= valid_rate else "valid"
                out[pre + "_target"].append([float(columns[target_column_num])])
                row = []
                for c in feature_column_nums:
                    try:
                        row.append(float(columns[c].strip("\n")))
                    except Exception:      # the reference logs and silently skips the cell (:409-411)
                        pass
                out[pre + "_data"].append(row)
                if 0 <= sample_weight_column_num < len(columns):
                    wt = float(columns[sample_weight_column_num].strip("\n"))
                    if wt < 0.0:
                        wt = 1.0
                    out[pre + "_data_sample_weight"].append([wt])
                else:
                    out[pre + "_data_sample_weight"].append([1.0])
    out["feature_count"] = len(feature_column_nums) if feature_column_nums is not None else 0
    return out


# --------------------------------------------------------------------------
# scorer            shifu-tensorflow-eval/.../TensorflowModel.java:53-94
# --------------------------------------------------------------------------
def score_rows(net: NetDesc, params, rows_f64: np.ndarray) -> np.ndarray:
    """compute(): double[] -> float[] cast (:64-68), [1,F] forward in fp32 (:70-86), float -> double (:87-88)."""
    X = np.asarray(rows_f64, dtype=np.float64).astype(np.float32)
    _, _, yhat = forward(net, [p.astype(np.float32) for p in params], X)
    return yhat[:, 0].astype(np.float64)


# --------------------------------------------------------------------------
# synthetic data (BASELINE.md section 4)
# --------------------------------------------------------------------------
def synth_batch(rows: int, n_features: int, seed: int, weights: str = "ones"):
    """X~N(0,1) clipped to +-4 fp32 row-major; y~Bernoulli(0.2) as f32 {0,1}; w=1 or U{0,1,2.5}."""
    rng = np.random.RandomState(seed)
    X = np.clip(rng.standard_normal((rows, n_features)), -4, 4).astype(np.float32)
    y = (rng.uniform(size=(rows, 1)) < 0.2).astype(np.float32)
    if weights == "ones":
        w = np.ones((rows, 1), np.float32)
    else:
        w = rng.choice(np.array([0.0, 1.0, 2.5], np.float32), size=(rows, 1)).astype(np.float32)
    return X, y, w


# --------------------------------------------------------------------------
# bf16 performance-mode emulation (checker for SB_PREC_BF16)
# --------------------------------------------------------------------------
def bf16_round(a: np.ndarray) -> np.ndarray:
    """fp32 -> nearest-even bf16 -> fp32 (what __float2bfloat16_rn does)."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    u = a.view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32).reshape(a.shape)


def loss_and_grads_bf16(net: NetDesc, params, X, y, w, loss=LOSS_MSE, fused_out=True):
    """The SAME math as loss_and_grads, with a bf16 rounding wherever the CUDA performance mode stores an
    operand as bf16 (DESIGN.md 'precision modes'): X, hidden-layer W, every activation A_l and every dZ_l that is
    fed to a tensor-core GEMM.  Accumulation stays in higher precision (fp64 here vs fp32 in the GEMM), the output
    layer uses fp32 w_o, and bias gradients / dw_o are summed from the un-rounded values exactly like the kernels
    do.  Lets the tests check the tensor-core path to ~1e-5 instead of the loose bf16-vs-fp32 bound.
    fused_out=True (training steps with h_L <= 256): the last hidden activation A_L never leaves the GEMM epilogue, so
    it is NOT rounded to bf16 before the output layer; fused_out=False is the forward-only / scoring path."""
    q = bf16_round
    f64 = np.float64
    L_hidden = len(net.acts)
    A = [q(X).astype(f64)]
    for l, act in enumerate(net.acts):
        W, b = q(params[2 * l]).astype(f64), params[2 * l + 1].astype(f64)
        a = act_forward((A[-1] @ W + b).astype(np.float32), act)
        A.append((a if (fused_out and l == L_hidden - 1) else q(a)).astype(f64))
    Wo, bo = params[-2].astype(f64), params[-1].astype(f64)
    z = (A[-1] @ Wo + bo).astype(np.float32)
    yhat = _sigmoid(z)
    Lv, n_nz = loss_value(z, yhat, y.astype(np.float32), w.astype(np.float32), loss)
    grads = [np.zeros_like(p, dtype=np.float32) for p in params]
    if n_nz == 0:
        return Lv, grads, yhat
    y64, w64, yh = y.astype(f64), w.astype(f64), yhat.astype(f64)
    dz = (2 * w64 * (yh - y64) * yh * (1 - yh) / n_nz) if loss == LOSS_MSE else (w64 * (yh - y64) / n_nz)
    dz = dz.astype(np.float32).astype(f64)
    grads[-2] = (A[-1].T @ dz).astype(np.float32)
    grads[-1] = dz.sum(axis=0).astype(np.float32)
    g_un = (dz @ Wo.T) * act_grad_from_output(A[-1].astype(np.float32), net.acts[-1]).astype(f64)  # un-rounded dZ_L
    for l in range(L_hidden - 1, -1, -1):
        grads[2 * l + 1] = g_un.sum(axis=0).astype(np.float32)          # bias grad from un-rounded values
        dZ = q(g_un.astype(np.float32)).astype(f64)                     # stored bf16 -> GEMM operand
        grads[2 * l] = (A[l].T @ dZ).astype(np.float32)
        if l > 0:
            Wl = q(params[2 * l]).astype(f64)
            g_un = (dZ @ Wl.T) * act_grad_from_output(A[l].astype(np.float32), net.acts[l - 1]).astype(f64)
    return Lv, grads, yhat


class Bf16Trainer:
    """Multi-step companion of loss_and_grads_bf16: fp32 master weights + fp32 optimizer state, every step's loss and
    gradient computed with the bf16 roundings of the CUDA performance mode (the bf16 weight shadows are re-rounded from
    the fp32 master after every update, exactly like optimizer_kernel refreshes them).  Checker for loss CURVES of
    SB_PREC_BF16 (tests/test_benchmarked_paths.py); same interface as CleanTrainer."""

    def __init__(self, net: NetDesc, params, opt: OptConfig, loss=LOSS_MSE, fused_out=True):
        self.net, self.loss, self.fused_out = net, loss, fused_out
        self.theta = flatten_params(params).astype(np.float32)
        self.opt = Optimizer(opt, self.theta.size, np.float32)
        self.last_grads = None

    def step(self, shards):
        P = unflatten_params(self.net, self.theta)
        gsum, losses = None, []
        for (X, y, w) in shards:
            L, g, _ = loss_and_grads_bf16(self.net, P, X, y, w, self.loss, fused_out=self.fused_out)
            g = flatten_params(g)
            gsum = g if gsum is None else gsum + g
            losses.append(L)
        g = gsum / np.float32(len(shards))
        self.last_grads = g
        self.theta = self.opt.apply(self.theta, g)
        return losses
