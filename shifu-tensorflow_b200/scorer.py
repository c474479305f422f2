"""Host-side mirror of the reference Java scorer `ml.shifu.shifu.tensorflow.TensorflowModel`
(shifu-tensorflow-eval/src/main/java/ml/shifu/shifu/tensorflow/TensorflowModel.java), an implementation of Shifu's
`Computable` (init / compute / releaseResource), with the same error behaviour, plus the batched entry point the
per-row Session.run of the reference never had.  The Java class of the same shape that binds the same C-ABI through
JNI is java/ml/shifu/shifu/tensorflow/B200Model.java (INTEGRATION.md).

    config = {"inputnames": ["shifu_input_0"],
              "properties": {"modelpath": "/path/to/saved_model_dir", "outputnames": "shifu_output_0",
                             "tags": ["serve"], "algorithm": "tensorflow", "normtype": "ZSCALE"}}
    m = TensorflowModel(); m.init(config); score = m.compute(row_of_doubles)
    e = TensorflowEnsemble(); e.init([config_of_model0, ..., config_of_model4]); r = e.compute(row_of_doubles)
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Sequence

import numpy as np

from . import _capi as capi


class IllegalStateException(RuntimeError):
    """TensorflowModel.compute before init (TensorflowModel.java:55-57)."""


class IllegalArgumentException(ValueError):
    """more than one output name (TensorflowModel.java:137-139)."""


def check_phase_switch(name: str, value: Any) -> None:
    """rule for GenericModelConfig inputnames[1:] (see TensorflowModel.init below and java/.../B200Model.java)"""
    if value is None:
        return
    if isinstance(value, (bool, int, float, np.bool_, np.integer, np.floating)):
        if bool(value):
            raise IllegalArgumentException("Input %s = %r selects the training branch of the graph; only inference "
                                           "(false / 0) is supported." % (name, value))
        return
    raise IllegalArgumentException("Input %s has unsupported type %s: only boolean / numeric inference-phase switches can be "
                                   "honoured." % (name, type(value).__name__))


# computePerformance's tables: Shifu's gains, ROC and PR lists, each the operating points at fixed levels of one axis
PERF_TABLES = (("gains", "action_rate"), ("roc", "fpr"), ("pr", "recall"))


def _perf_table(pts: dict, pos: float, neg: float, weighted: bool) -> dict:
    """operating points -> the table entries with their ratios formed from the counts (NaN where a ratio's denominator is 0)"""
    tp, fp = (pts["w_tp"], pts["w_fp"]) if weighted else (pts["tp"].astype(np.float64), pts["fp"].astype(np.float64))
    with np.errstate(invalid="ignore", divide="ignore"):
        precision = tp / (tp + fp)
        out = dict(pts, recall=tp / pos, precision=precision, fpr=fp / neg, lift=precision / (pos / (pos + neg)))
    return out


def _performance(perf: capi.Performance, buckets: int, weighted: bool) -> dict:
    """summary and tables of the rows added to `perf`: {"summary", "gains", "roc", "pr"} and, when weighted,
    "weighted_gains" / "weighted_roc" / "weighted_pr"; a table whose axis is undefined (its total is 0) is None"""
    if buckets < 1:
        raise ValueError("buckets must be >= 1")
    summ = perf.summary()
    levels = np.arange(1, buckets + 1, dtype=np.float64) / buckets
    out = {"summary": summ}
    for w in ((False, True) if weighted else (False,)):
        pos, neg = (summ["w_pos"], summ["w_neg"]) if w else (float(summ["pos"]), float(summ["neg"]))
        for name, axis in PERF_TABLES:
            den = {"action_rate": pos + neg, "recall": pos, "fpr": neg}[axis]
            key = ("weighted_" if w else "") + name
            out[key] = _perf_table(perf.points(axis, levels, weighted=w), pos, neg, w) if den > 0 else None
    return out


def _targets(targets, weights, rows: int):
    y = np.asarray(targets, dtype=np.float64).astype(np.float32).reshape(-1)
    w = None if weights is None else np.asarray(weights, dtype=np.float64).astype(np.float32).reshape(-1)
    if y.size != rows or (w is not None and w.size != rows):
        raise ValueError("one target (and weight) per row")
    return y, w


def _sensitivity(fn, rows, weights, columns, values, **kw) -> dict:
    """computeSensitivity through fn (Model.sensitivity or Ensemble.sensitivity; kw: its further arguments)"""
    X = np.asarray(rows, dtype=np.float64).astype(np.float32)     # the same double -> float cast as computeBatch
    w = None if weights is None else np.asarray(weights, dtype=np.float64).astype(np.float32)
    vals = None if values is None else np.asarray(values, dtype=np.float64).astype(np.float32)
    r = fn(X, w=w, cols=columns, values=vals, **kw)
    ws = r["w_sum"]
    with np.errstate(invalid="ignore", divide="ignore"):
        mse, mean = r["sum_sq"] / ws, r["sum"] / ws
    return {"sum_sq": r["sum_sq"], "sum": r["sum"], "w_sum": ws, "mse": mse, "mean": mean}


def _reason_codes(fn, rows, k, columns, values, order, **kw) -> dict:
    """computeReasonCodes through fn (Model.reason_codes or Ensemble.reason_codes; kw: its further arguments)"""
    X = np.asarray(rows, dtype=np.float64).astype(np.float32)     # the same double -> float cast as computeBatch
    vals = None if values is None else np.asarray(values, dtype=np.float64).astype(np.float32)
    cl = np.arange(X.shape[1], dtype=np.int32) if columns is None else np.asarray(columns, dtype=np.int32).reshape(-1)
    r = fn(X, k, cols=columns, values=vals, order=order, scores=True, **kw)
    return {"columns": cl[r["pos"]], "deltas": r["d"], "scores": r["scores"]}


class TensorflowModel:
    def __init__(self, device: int = 0, precision: int = capi.PREC_FP32):
        self.properties: Dict[str, Any] = {}
        self.initiate = False
        self.modelPath: Optional[str] = None
        self._model: Optional[capi.Model] = None
        self.config = None
        self.tags: Optional[List[str]] = None
        self.inputNames: Optional[List[str]] = None
        self.outputNames: Optional[str] = None
        self._device, self._precision = device, precision

    # -- Computable.init (TensorflowModel.java:112-172) --
    def init(self, config) -> None:
        if self.initiate:                                   # idempotent (:114-116)
            return
        self.init_config(config)
        self._model = capi.Model.load(self.modelPath, self.inputNames[0], self.outputNames, tag=self.tags[0],
                                      device=self._device, precision=self._precision)
        self.initiate = True

    def init_config(self, config) -> None:
        """init's reading and checking of the GenericModelConfig, without loading the model (TensorflowEnsemble checks
        each member's config this way)"""
        if config is None:
            raise RuntimeError("Config is null")
        self.config = config
        get = (lambda k: config.get(k)) if isinstance(config, dict) else (lambda k: getattr(config, k, None))
        self.properties = get("properties")
        if self.properties is None or len(self.properties) == 0:
            raise RuntimeError("Properties is null")
        self.modelPath = self.properties.get("modelpath")
        names = get("inputnames")
        self.inputNames = list(names) if names is not None else None
        output_names = self.properties.get("outputnames")
        if isinstance(output_names, str):
            self.outputNames = output_names
        elif isinstance(output_names, (list, tuple)):
            if len(output_names) == 1:
                self.outputNames = output_names[0]
            else:
                raise IllegalArgumentException("Output now only support single output in inference.")
        tag_list = self.properties.get("tags")
        self.tags = list(tag_list) if tag_list is not None else None
        if not self.modelPath:
            raise RuntimeError("Model path is null")
        if not self.inputNames:
            raise RuntimeError("Input names is null")
        if not self.outputNames:
            raise RuntimeError("Output names is null")
        if not self.tags:
            raise RuntimeError("Tags is null")
        # SavedModelBundle.load(modelPath, tags) + feed inputNames[0] / fetch outputNames by op name (:71,85,169).
        # Extra named inputs (inputNames[1:], fed from `properties` as constants, :73-83 - in the reference's test a Keras
        # learning-phase bool): the loader walks the INFERENCE branch of the graph, so such an input is honoured only when it
        # selects that branch.  False / 0 -> accepted (not fed); missing -> skipped like the reference's catch block (:78-80);
        # True / non-zero (training branch: dropout active) or any other type -> rejected here, at init.
        for name in self.inputNames[1:]:
            check_phase_switch(name, self.properties.get(name))

    # -- Computable.compute (TensorflowModel.java:53-94): double[] -> float[] -> [1,n] forward -> double --
    def compute(self, input) -> float:
        if not self.initiate or self._model is None:
            raise IllegalStateException("TF model not initialized.")
        data = input.getData() if hasattr(input, "getData") else input
        return self._model.score_row_f64(np.asarray(data, dtype=np.float64))

    # -- new: the whole table in one call (rows are scored in parallel on the GPU) --
    def computeBatch(self, rows) -> np.ndarray:
        if not self.initiate or self._model is None:
            raise IllegalStateException("TF model not initialized.")
        X = np.asarray(rows, dtype=np.float64).astype(np.float32)     # the same double -> float cast, vectorised
        return self._model.score(X).astype(np.float64)

    # -- new: column sensitivity (varsel filterBy SE / ST): each column replaced by a value, over the whole table --
    def computeSensitivity(self, rows, weights=None, columns=None, values=None) -> dict:
        """-> {"sum_sq", "sum": per-column sums of w d^2 and w d, "w_sum", "mse" = sum_sq / w_sum, "mean" = sum / w_sum},
        with d = compute(row) - compute(row with the column set to its value); columns None: every column; values None:
        0 per column (the mean of a ZSCALE-normalised column)"""
        if not self.initiate or self._model is None:
            raise IllegalStateException("TF model not initialized.")
        return _sensitivity(self._model.sensitivity, rows, weights, columns, values)

    # -- new: per-row reason codes: the columns whose replacement moves each row's score the most --
    def computeReasonCodes(self, rows, k, columns=None, values=None, order="raise") -> dict:
        """-> {"columns": int32 [rows, k] the k columns that rank first per row, "deltas": their d = compute(row) -
        compute(row with the column set to its value), "scores": compute(row) as the call computes it}; order "raise"
        (largest d first: the values that push the score up the most), "lower" or "magnitude"; columns None: every
        column; values None: 0 per column (the mean of a ZSCALE-normalised column)"""
        if not self.initiate or self._model is None:
            raise IllegalStateException("TF model not initialized.")
        return _reason_codes(self._model.reason_codes, rows, k, columns, values, order)

    # -- new: how good the model is on a scored set (what `shifu eval` reports), computed on the GPU --
    def computePerformance(self, rows, targets, weights=None, buckets=10) -> dict:
        """Scores the rows as computeBatch does and evaluates them against targets (0 / 1) and weights (None: 1):
        -> {"summary": AUC, average precision, KS, ... (include/shifu_b200.h, sb_perf_summary), "gains" / "roc" / "pr":
        the operating points at action rate / FPR / recall (1 .. buckets) / buckets, each entry with its threshold,
        counts, recall, precision, fpr and lift; with weights also "weighted_gains" / "weighted_roc" / "weighted_pr"}"""
        scores = self.computeBatch(rows).astype(np.float32)
        y, w = _targets(targets, weights, scores.size)
        with capi.Performance(self._device, scores.size) as perf:
            perf.add(scores, y, w)
            return _performance(perf, buckets, w is not None)

    def releaseResource(self) -> None:
        """The reference never closes its bundle (TensorflowModel.java:175-176); here device memory is returned."""
        if self._model is not None:
            self._model.close()
            self._model = None
        self.initiate = False


class TensorflowEnsemble:
    """The bagged form of TensorflowModel: `shifu eval` over a run's models/model0 .. model{K-1} (train.baggingNum
    members), each row scored by every member, with the members' mean, max, min and median.  init takes one
    GenericModelConfig per member, checked as TensorflowModel.init checks one; the members are scored together on one
    device from one staged copy of the rows (sb_ensemble_*)."""

    def __init__(self, device: int = 0, precision: int = capi.PREC_FP32):
        self.initiate = False
        self.members: List[TensorflowModel] = []
        self._ensemble: Optional[capi.Ensemble] = None
        self._device, self._precision = device, precision

    def init(self, configs: Sequence[Any]) -> None:
        if self.initiate:
            return
        if configs is None or len(configs) == 0:
            raise RuntimeError("Configs is null")
        members = []
        for config in configs:
            m = TensorflowModel(self._device, self._precision)
            m.init_config(config)
            members.append(m)
        names = {(m.inputNames[0], m.outputNames, m.tags[0]) for m in members}
        if len(names) != 1:
            raise IllegalArgumentException("Every member must have the same input name, output name and tag.")
        inp, outp, tag = names.pop()
        self._ensemble = capi.Ensemble.load([m.modelPath for m in members], inp, outp, tag=tag, device=self._device,
                                            precision=self._precision)
        self.members = members
        self.initiate = True

    def _check(self) -> capi.Ensemble:
        if not self.initiate or self._ensemble is None:
            raise IllegalStateException("TF ensemble not initialized.")
        return self._ensemble

    # -- compute() of every member: double[] -> {"scores": [K] in member order, "mean", "max", "min", "median"} --
    def compute(self, input) -> dict:
        e = self._check()
        data = input.getData() if hasattr(input, "getData") else input
        r = e.score_row_f64(np.asarray(data, dtype=np.float64))
        out = {"scores": r[:e.k]}
        out.update({name: float(r[e.k + i]) for i, name in enumerate(capi.ENSEMBLE_STATS)})
        return out

    # -- the whole table in one call: {"scores": [rows, K], "mean" .. "median": [rows]} as float64 --
    def computeBatch(self, rows) -> dict:
        e = self._check()
        X = np.asarray(rows, dtype=np.float64).astype(np.float32)     # the same double -> float cast as compute()
        s, t = e.score(X)
        out = {"scores": s.astype(np.float64)}
        out.update({name: t[:, i].astype(np.float64) for i, name in enumerate(capi.ENSEMBLE_STATS)})
        return out

    def _stat(self, score) -> str:
        if not isinstance(score, str) or score not in capi.ENSEMBLE_STATS:
            raise ValueError("score must be one of %s" % (capi.ENSEMBLE_STATS,))
        return score

    # -- column sensitivity of the shipped score: score = "mean" | "max" | "min" | "median" of the member scores --
    def computeSensitivity(self, rows, weights=None, columns=None, values=None, score="mean") -> dict:
        """TensorflowModel.computeSensitivity with d = S(row) - S(row with the column set to its value), S the
        statistic `score` of the members' scores"""
        e = self._check()
        return _sensitivity(e.sensitivity, rows, weights, columns, values, stat=self._stat(score))

    # -- per-row reason codes of the shipped score --
    def computeReasonCodes(self, rows, k, columns=None, values=None, order="raise", score="mean") -> dict:
        """TensorflowModel.computeReasonCodes with d = S(row) - S(row with the column set to its value) and "scores" =
        S(row), S the statistic `score` of the members' scores"""
        e = self._check()
        return _reason_codes(e.reason_codes, rows, k, columns, values, order, stat=self._stat(score))

    # -- how good one column is on a scored set: score = "mean" | "max" | "min" | "median" or a member index --
    def computePerformance(self, rows, targets, weights=None, buckets=10, score="mean") -> dict:
        """TensorflowModel.computePerformance for one column of the ensemble's output.  The rows are scored in chunks
        into device memory and the column is read there in place (sb_perf_add's score_stride): the scores never come
        back to the host."""
        e = self._check()
        X = np.asarray(rows, dtype=np.float64).astype(np.float32)
        if X.ndim != 2 or X.shape[1] != e.n_features:
            raise ValueError("rows must be [rows, %d]" % e.n_features)
        n = X.shape[0]
        y, w = _targets(targets, weights, n)
        if isinstance(score, str):
            if score not in capi.ENSEMBLE_STATS:
                raise ValueError("score must be one of %s or a member index" % (capi.ENSEMBLE_STATS,))
            col, stride = capi.ENSEMBLE_STATS.index(score), 4
        else:
            col, stride = int(score), e.k
            if not 0 <= col < e.k:
                raise ValueError("member index %d outside [0, %d)" % (col, e.k))
        chunk = min(max(n, 1), 1 << 20)
        buf = capi.DeviceArray.empty((chunk, stride), self._device)
        try:
            base = capi.C.cast(buf.ptr, capi.C.c_void_p).value
            with capi.Performance(self._device, n) as perf:
                for r0 in range(0, n, chunk):
                    c = min(chunk, n - r0)
                    xc = np.ascontiguousarray(X[r0:r0 + c])
                    out = capi.C.c_void_p(base)
                    capi.check(capi.lib().sb_ensemble_score(e._h, xc.ctypes.data_as(capi.C.c_void_p), c,
                                                            None if isinstance(score, str) else out,
                                                            out if isinstance(score, str) else None))
                    perf.add_device(base + 4 * col, y[r0:r0 + c].ctypes.data, None if w is None else w[r0:r0 + c].ctypes.data,
                                    c, stride=stride)
                return _performance(perf, buckets, w is not None)
        finally:
            buf.free()

    def releaseResource(self) -> None:
        if self._ensemble is not None:
            self._ensemble.close()
            self._ensemble = None
        self.members = []
        self.initiate = False
