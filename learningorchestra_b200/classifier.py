"""The builder's five classifiers on the GPU: Spark 2.4's multinomial ``NaiveBayes`` ("NB"), ``LogisticRegression``
("LR"), ``DecisionTreeClassifier`` ("DT"), ``GBTClassifier`` ("GB") and ``RandomForestClassifier`` ("RF")
(``builder_image/builder.py:55-61``) fitted on, applied to and evaluated over the feature matrix in HBM
(:meth:`DeviceFrame.features`), on one GPU or on every shard of a local :class:`~sharding.ShardedEngine`.  DESIGN.md
§3.6.2 to §3.6.6 state the semantics.

NaiveBayes: the device computes the class counts and per-class feature sums (``lo_nb_fit``); LogisticRegression: the
column statistics and label counts (``lo_lr_stats``) and one pass of loss and gradient sums per function evaluation of
the host's L-BFGS (``lo_lr_loss_grad``, :mod:`lbfgs`).  Both compute every row's raw values, probabilities and prediction
(``lo_nb_predict`` / ``lo_lr_predict``) and the confusion counts of an evaluation on the device; the models' arrays and
the evaluator's metrics are computed here, on the host, from those.  DecisionTreeClassifier: the device sorts the
columns, answers rank queries, bins the values and counts every tree level (``lo_dt_*``); :mod:`tree` chooses the
thresholds and splits from those counts.  GBTClassifier grows its regression trees on the same codes from exact
fixed-point residual sums (``lo_gb_level``) and keeps every row's margin and residual on the device (``lo_gb_update``).
RandomForestClassifier grows batches of trees together on the same codes, one pass per level of the whole batch
(``lo_rf_level``), each row weighted by its counter-based bagging draw and each node over its own feature subset; the
forest's votes are summed per row on the device (``lo_rf_predict``)."""
from __future__ import annotations

import contextlib
import math

import numpy as np

from . import _native as N


_NB_REASONS = ("is negative or NaN", "is not a class of the model")
_LR_REASONS = ("is NaN or infinite", "is not an integer label >= 0")


def _on_device(features, call, per_part: bool = False, name: str = "NaiveBayes",
               reasons: tuple[str, str] = _NB_REASONS):
    """``call(engine, rows)`` on the features' engine: a ShardedEngine takes every shard's rows and gives one result per
    shard where it gives one per row (``per_part``); an Engine takes its one part, and its result is made a list of one
    where ``per_part``.  A refused cell (its row a row of the features, shards concatenated) is raised as the ``_id``
    and field it holds: "<name>: field F of the row with _id I <reason>", ``reasons`` (a feature's, the label's)."""
    from .builder_frontend import named_cell
    from .engine import InvalidCellError
    from .sharding import ShardedEngine
    engine = features._frame._cache.engine
    sharded = isinstance(engine, ShardedEngine)
    try:
        out = call(engine, features._parts if sharded else features._parts[0])
    except InvalidCellError as e:
        raise named_cell(e, features.fields, features.label, features.row_ids, name, reasons) from None
    return [out] if per_part and not sharded else out


def _usable(features) -> None:
    """Refuses features that have been released (their tables freed) before anything reads them."""
    if not features._parts:
        raise ValueError("the features have been released")


def _labelled(features, name: str) -> None:
    """The fits' preamble: refuses released features, and features without a label."""
    _usable(features)
    if features.label is None:
        raise ValueError(f"{name} needs features with a label")


def _some_rows(n: int, name: str) -> None:
    """Refuses a call ``name`` over no row."""
    if n == 0:
        raise N.LoexecError(N.LO_ERR_INVALID, f"{name} needs at least one row")


def _free(held) -> None:
    """Frees device results: a list of them (one per shard), one, or None."""
    for h in held if isinstance(held, list) else [] if held is None else [held]:
        h.free()


def _labels(features, name: str = "NaiveBayes", reasons: tuple[str, str] = _NB_REASONS) -> np.ndarray:
    """The distinct label values of the features' rows, ascending (every shard's union)."""
    _labelled(features, name)
    return _on_device(features, lambda engine, rows: engine.nb_labels(rows), name=name, reasons=reasons)


def model_arrays(sums: np.ndarray, counts: np.ndarray, smoothing: float) -> tuple[np.ndarray, np.ndarray]:
    """(pi, theta) of Spark's multinomial NaiveBayes from the class counts and per-class feature sums:
    pi_c = log(n_c + λ) - log(N + C λ), theta_cj = log(s_cj + λ) - log(S_c + k λ) with S_c summed over j ascending."""
    nclasses, k = sums.shape
    lam = float(smoothing)
    n_docs = float(np.cumsum(counts.astype(np.float64))[-1])
    with np.errstate(divide="ignore"):
        pi = np.log(counts.astype(np.float64) + lam) - np.log(n_docs + nclasses * lam)
    totals = np.cumsum(sums, axis=1)[:, -1]
    with np.errstate(invalid="ignore", divide="ignore"):     # +inf sums or λ = 0 give Spark's inf / NaN logs
        theta = np.log(sums + lam) - np.log(totals + k * lam)[:, None]
    return pi, theta


class NaiveBayes:
    """``pyspark.ml.classification.NaiveBayes(smoothing=smoothing)`` with its defaults (``modelType="multinomial"``, no
    ``weightCol``, no ``thresholds``) on the GPU."""

    def __init__(self, smoothing: float = 1.0):
        s = float(smoothing)
        if not np.isfinite(s) or s < 0.0:
            raise ValueError(f"smoothing must be finite and >= 0, not {smoothing!r}")
        self.smoothing = s

    def fit(self, features) -> "NaiveBayesModel":
        """The model of ``features`` (:class:`~builder_frontend.Features` with a label, on one GPU or sharded).  The
        classes are the distinct label values, ascending; a NaN label, more than LO_NB_MAX_CLASSES of them, C x k above
        LO_NB_MAX_THETA or no row at all are refused, and so is a negative or NaN feature (InvalidCellError naming the
        ``_id`` and field of the lowest such row)."""
        classes = _labels(features)
        _some_rows(len(features.row_ids), "NaiveBayes")
        k = len(features.fields)
        if len(classes) * k > N.LO_NB_MAX_THETA:
            raise N.LoexecError(N.LO_ERR_INVALID, f"{len(classes)} classes x {k} features exceed LO_NB_MAX_THETA = "
                                f"{N.LO_NB_MAX_THETA}")
        sums, counts = _on_device(features, lambda engine, rows: engine.nb_fit(rows, classes))
        pi, theta = model_arrays(sums, counts, self.smoothing)
        return NaiveBayesModel(classes, pi, theta, features.fields, sums, counts)


class _Model:
    """What every fitted classifier shares: the ``fields`` it was fitted on, ``transform`` and ``evaluate``.  A model
    states ``_name`` and ``_reasons`` (the words of a refused cell, see :func:`_on_device`) and supplies
    ``_predict(engine, rows, raw, labels)``, its engine's ``*_predict`` call."""
    _name, _reasons = "NaiveBayes", _NB_REASONS

    def _check(self, features) -> None:
        if list(features.fields) != self.fields:
            raise ValueError(f"the model was fitted on fields {self.fields}, not {list(features.fields)}")

    def transform(self, features, raw: bool = False) -> "Predictions":
        """Spark's ``model.transform``: every row's ``probability`` and ``prediction`` (a class INDEX as float64), and
        with ``raw`` its ``rawPrediction``, written in HBM on the rows' own devices."""
        _usable(features)
        self._check(features)
        parts = _on_device(features, lambda engine, rows: self._predict(engine, rows, raw=raw), per_part=True,
                           name=self._name, reasons=self._reasons)
        return Predictions(features, parts)

    def evaluate(self, features) -> dict:
        """``MulticlassClassificationEvaluator`` f1 and accuracy over ``transform(features)`` (builder.py:124-142), as one
        fused pass per device that writes nothing per row: ``{"f1", "accuracy", "labels", "confusion"}`` where
        ``confusion[a, p]`` counts the rows labelled ``labels[a]`` predicted as class index p."""
        _usable(features)
        self._check(features)
        labels = _labels(features, self._name, self._reasons)
        _some_rows(len(features.row_ids), "evaluate")
        confusion = _on_device(features, lambda engine, rows: self._predict(engine, rows, labels=labels),
                               name=self._name, reasons=self._reasons)
        f1, accuracy = metrics(labels, confusion)
        return {"f1": f1, "accuracy": accuracy, "labels": labels, "confusion": confusion}


class NaiveBayesModel(_Model):
    """A fitted multinomial NaiveBayes model, host data: ``labels`` (float64[C], the class values ascending), ``pi``
    (float64[C]), ``theta`` (float64[C, k]) and the ``fields`` it was fitted on; ``sums`` / ``counts`` are the device's
    per-class feature sums and row counts it was made from."""

    def __init__(self, labels, pi, theta, fields, sums=None, counts=None):
        self.labels, self.pi, self.theta = np.asarray(labels, np.float64), np.asarray(pi, np.float64), np.asarray(theta, np.float64)
        self.fields, self.sums, self.counts = list(fields), sums, counts

    def _predict(self, engine, rows, raw=False, labels=None):
        return engine.nb_predict(rows, self.pi, self.theta, raw=raw, labels=labels)


def metrics(labels: np.ndarray, confusion: np.ndarray) -> tuple[float, float]:
    """(weighted F1, accuracy) of Spark 2.4's MulticlassMetrics from the confusion counts: a prediction is a class index
    and counts as a true positive of label L when it EQUALS L.  Per label L (ascending): precision tp / (tp + fp) (0 when
    nothing is predicted as L), recall tp / count(L), f = 2 p r / (p + r) (0 when p + r == 0); f1 = sum of f(L) count(L) /
    N; accuracy = sum tp / N."""
    confusion = np.asarray(confusion, np.int64)
    nclasses = confusion.shape[1]
    n = int(confusion.sum())
    f1, tp_total = 0.0, 0
    for a, lab in enumerate(labels):
        count = int(confusion[a].sum())
        p_idx = int(lab) if float(lab).is_integer() and 0 <= lab < nclasses else None
        tp = int(confusion[a, p_idx]) if p_idx is not None else 0
        fp = int(confusion[:, p_idx].sum()) - tp if p_idx is not None else 0
        precision = 0.0 if tp + fp == 0 else tp / (tp + fp)
        recall = tp / count
        f = 0.0 if precision + recall == 0 else 2.0 * precision * recall / (precision + recall)
        f1 += f * count / n
        tp_total += tp
    return f1, tp_total / n


FAMILIES = ("auto", "binomial", "multinomial")


def standardization(n: int, total, m2) -> np.ndarray:
    """The unbiased std of every column from its sum and squared deviations over n rows (0 when n == 1)."""
    return np.sqrt(m2 / (n - 1)) if n > 1 else np.zeros_like(np.asarray(total, np.float64))


def scaled_objective(loss_grad, n: int, std, nc: int, reg_param: float):
    """Spark's objective in the scaled space x_j / std_j as ``fun(v) -> (value, gradient)`` for :func:`lbfgs.minimize`;
    v = [w (nc x k, row-major), b (nc)].  ``loss_grad(beta, b)`` gives LogisticAggregator's sums (loss, gradient sums
    nc x k of multiplier * x_j in the original space, intercept sums) at the effective coefficients beta = w / std (0
    where std == 0).  value = loss / n + reg/2 * sum(w^2), gradient = (sums_j / std_j) / n + reg * w and b's sums / n."""
    std = np.asarray(std, np.float64)
    k, live = len(std), std != 0
    div = np.where(live, std, 1.0)

    def fun(v):
        w, b = v[:nc * k].reshape(nc, k), v[nc * k:]
        loss, g, gb = loss_grad(np.where(live, w / div, 0.0), b)
        gw = np.where(live, g / div, 0.0) / n + reg_param * w
        return loss / n + 0.5 * reg_param * float((w * w).sum()), np.concatenate([gw.ravel(), np.asarray(gb) / n])

    return fun


def start_point(label_counts, num_classes: int, k: int, multinomial: bool) -> np.ndarray:
    """Spark's initial point: coefficients 0; binomial intercept log(n_1 / n_0); multinomial intercepts
    log(n_c + 1) - mean_c log(n_c + 1)."""
    hist = np.asarray(label_counts[:num_classes], np.float64)
    nc = num_classes if multinomial else 1
    v = np.zeros(nc * (k + 1))
    if multinomial:
        raw = np.log1p(hist)
        v[nc * k:] = raw - raw.sum() / len(raw)
    else:
        v[k] = math.log(hist[1] / hist[0])
    return v


def unscale(v, std, nc: int, reg_param: float, multinomial: bool) -> tuple[np.ndarray, np.ndarray]:
    """(coefficient matrix nc x k, intercepts nc) of the scaled-space point v, as Spark leaves them: coef_j / std_j (0
    where the std is 0); multinomial with reg_param == 0 centres each feature's coefficients across classes; multinomial
    always centres the intercepts."""
    std = np.asarray(std, np.float64)
    k = len(std)
    w, b = np.array(v[:nc * k]).reshape(nc, k), np.array(v[nc * k:])
    coef = np.where(std != 0, w / np.where(std != 0, std, 1.0), 0.0)
    if multinomial and reg_param == 0.0:
        coef = coef - coef.sum(axis=0) / nc
    if multinomial:
        b = b - b.sum() / nc
    return coef, b


class LogisticRegression:
    """``pyspark.ml.classification.LogisticRegression(maxIter, regParam, tol, family, threshold)`` with its other
    defaults (``elasticNetParam=0``, ``fitIntercept``, ``standardization``, no ``weightCol``, no bounds) on the GPU."""

    def __init__(self, max_iter: int = 100, reg_param: float = 0.0, tol: float = 1e-6, family: str = "auto",
                 threshold: float = 0.5):
        if isinstance(max_iter, bool) or int(max_iter) != max_iter or max_iter < 0:
            raise ValueError(f"max_iter must be an integer >= 0, not {max_iter!r}")
        reg, t, th = float(reg_param), float(tol), float(threshold)
        if not np.isfinite(reg) or reg < 0.0:
            raise ValueError(f"reg_param must be finite and >= 0, not {reg_param!r}")
        if not np.isfinite(t) or t <= 0.0:
            raise ValueError(f"tol must be finite and > 0, not {tol!r}")
        if family not in FAMILIES:
            raise ValueError(f"family must be one of {list(FAMILIES)}, not {family!r}")
        if not 0.0 <= th <= 1.0:
            raise ValueError(f"threshold must lie in [0, 1], not {threshold!r}")
        self.max_iter, self.reg_param, self.tol, self.family, self.threshold = int(max_iter), reg, t, family, th

    def fit(self, features) -> "LogisticRegressionModel":
        """The model of ``features`` (:class:`~builder_frontend.Features` with a label, on one GPU or sharded).  Every
        label must be an integer >= 0 and every feature finite (InvalidCellError naming the ``_id`` and field of the
        lowest refused row); numClasses = max label + 1.  No row, a label >= LO_NB_MAX_CLASSES or (binomial ? 2 : C) x k
        above LO_NB_MAX_THETA are refused, and so is ``family="binomial"`` with more than 2 classes."""
        from . import lbfgs
        _labelled(features, "LogisticRegression")
        k = len(features.fields)
        least = 2 if self.family == "binomial" else 1        # classes the model has at least: refused before any pass
        if least * k > N.LO_NB_MAX_THETA:
            raise N.LoexecError(N.LO_ERR_INVALID, f"{least} classes x {k} features exceed LO_NB_MAX_THETA = "
                                f"{N.LO_NB_MAX_THETA}")
        n, total, m2, counts = _on_device(features, lambda engine, rows: engine.lr_stats(rows), name="LogisticRegression",
                                          reasons=_LR_REASONS)
        _some_rows(n, "LogisticRegression")
        num_classes = int(np.flatnonzero(counts)[-1]) + 1
        if self.family == "binomial" and num_classes > 2:
            raise ValueError(f"family='binomial' needs at most 2 classes, the labels give {num_classes}")
        multinomial = self.family == "multinomial" or (self.family == "auto" and num_classes > 2)
        if (num_classes if multinomial else 2) * k > N.LO_NB_MAX_THETA:
            raise N.LoexecError(N.LO_ERR_INVALID, f"{num_classes if multinomial else 2} classes x {k} features exceed "
                                f"LO_NB_MAX_THETA = {N.LO_NB_MAX_THETA}")
        nc = num_classes if multinomial else 1
        std = standardization(n, total, m2)
        if np.count_nonzero(counts) == 1:                  # constant label: Spark trains nothing
            intercept = np.zeros(nc)
            if multinomial:
                intercept[num_classes - 1] = np.inf
            else:
                intercept[0] = np.inf if num_classes == 2 else -np.inf
            return LogisticRegressionModel(np.zeros((nc, k)), intercept, num_classes, multinomial, features.fields,
                                           [], 0, self.threshold)

        def loss_grad(beta, b):
            return _on_device(features, lambda engine, rows: engine.lr_loss_grad(rows, beta, b, multinomial),
                              name="LogisticRegression", reasons=_LR_REASONS)

        res = lbfgs.minimize(scaled_objective(loss_grad, n, std, nc, self.reg_param),
                             start_point(counts, num_classes, k, multinomial), self.max_iter, self.tol)
        coef, intercept = unscale(res.x, std, nc, self.reg_param, multinomial)
        return LogisticRegressionModel(coef, intercept, num_classes, multinomial, features.fields, res.history,
                                       res.iterations, self.threshold)


class LogisticRegressionModel(_Model):
    """A fitted LogisticRegression model, host data: ``coefficient_matrix`` (float64[C', k]) and ``intercept_vector``
    (float64[C']) with C' = ``num_classes`` when ``is_multinomial`` else 1; binomial also ``coefficients`` (float64[k])
    and ``intercept``; ``fields`` it was fitted on; ``objective_history`` (the objective at every optimizer state, the
    start included; empty for a constant label) and ``iterations``; ``threshold`` of the binomial prediction."""
    _name, _reasons = "LogisticRegression", _LR_REASONS

    def __init__(self, coefficient_matrix, intercept_vector, num_classes, is_multinomial, fields, objective_history=(),
                 iterations=0, threshold=0.5):
        self.coefficient_matrix = np.asarray(coefficient_matrix, np.float64)
        self.intercept_vector = np.asarray(intercept_vector, np.float64)
        self.num_classes, self.is_multinomial, self.fields = int(num_classes), bool(is_multinomial), list(fields)
        self.objective_history, self.iterations = list(objective_history), int(iterations)
        self.threshold = float(threshold)
        if not self.is_multinomial:
            self.coefficients, self.intercept = self.coefficient_matrix[0], float(self.intercept_vector[0])

    def _predict(self, engine, rows, raw=False, labels=None):
        return engine.lr_predict(rows, self.coefficient_matrix, self.intercept_vector, self.is_multinomial,
                                 self.threshold, raw=raw, labels=labels)

    def transform(self, features, raw: bool = False) -> "Predictions":
        """Spark's ``model.transform``: every row's ``probability`` and ``prediction`` (a class index as float64), and
        with ``raw`` its ``rawPrediction`` ([-m, m] when binomial), written in HBM on the rows' own devices."""
        return super().transform(features, raw)


class Predictions:
    """What :meth:`NaiveBayesModel.transform` wrote: per shard i (one on a single GPU), on ``devices[i]``, zero-copy
    ``__cuda_array_interface__`` views ``prediction[i]`` (n_i f64 class indices), ``probability[i]`` (n_i x C f64) and,
    with ``raw``, ``raw[i]`` (n_i x C f64, Spark's rawPrediction; else ``raw`` is None); ``row_ids`` the ``_id`` of every
    row, shards concatenated in order.  Owns its tables and frees them in :meth:`release` (or with ``with``)."""

    def __init__(self, features, parts):
        self._features, self._parts = features, list(parts)
        self.devices = list(features.devices)
        self.row_ids = features.row_ids
        self.prediction = [p.prediction(keepalive=self) for p in self._parts]
        self.probability = [p.probability(keepalive=self) for p in self._parts]
        self.raw = [p.raw_view(keepalive=self) for p in self._parts] if self._parts and self._parts[0].raw is not None else None

    def release(self):
        parts, self._parts = self._parts, []
        for p in parts:
            p.free()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.release()


_DT_SORT_BUDGET = 2 << 30      # bytes of sorted codes and sort scratch per column batch of lo_dt_sort


def split_thresholds(features, n: int, k: int, max_bins: int, name: str) -> tuple[list, int]:
    """Every column's split thresholds (DecisionTreeClassifier and GBTClassifier): the columns sorted on the device in
    batches within _DT_SORT_BUDGET, each batch's distinct values merged or its order statistics found by rank rounds
    (:func:`tree.column_thresholds`), and its sorted copies freed before the next.  Returns (thresholds, rank rounds)."""
    from . import tree as T
    f32 = features._parts[0].x.dtype_code == N.LO_F32
    per_col = 2 * (4 if f32 else 8) * max(n, 1)
    kc = max(1, min(k, _DT_SORT_BUDGET // per_col))
    cap = T.num_splits(max_bins, n) + 1
    out, rounds = [], 0
    for j0 in range(0, k, kc):
        w = min(kc, k - j0)
        got = _on_device(features, lambda engine, rows: engine.dt_sort(rows, j0, w, cap), name=name)
        members = got if isinstance(got, list) else [got]
        try:
            distinct = [T.merge_distinct([m.distinct[c] for m in members]) for c in range(w)]

            def rank(cols, codes):
                return _on_device(features, lambda engine, rows: engine.dt_rank(got, cols, codes), name=name)

            thr, r = T.column_thresholds(n, max_bins, distinct, rank, f32, w)
        finally:
            _free(got)
        out += thr
        rounds += r
    return out, rounds


def _integer(v, name, lo, hi=None):
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < lo or (hi is not None and v > hi):
        span = f"in [{lo}, {hi}]" if hi is not None else f">= {lo}"
        raise ValueError(f"{name} must be an integer {span}, not {v!r}")
    return int(v)


def _tree_params(est, max_depth, max_bins, min_instances_per_node, min_info_gain) -> None:
    """Checks and sets the tree parameters DecisionTreeClassifier and GBTClassifier share, with Spark's bounds."""
    from . import tree as T
    est.max_depth = _integer(max_depth, "max_depth", 0, T.MAX_DEPTH)
    est.max_bins = _integer(max_bins, "max_bins", 2, T.MAX_BINS)
    est.min_instances_per_node = _integer(min_instances_per_node, "min_instances_per_node", 1)
    g = float(min_info_gain)
    if not np.isfinite(g) or g < 0.0:
        raise ValueError(f"min_info_gain must be finite and >= 0, not {min_info_gain!r}")
    est.min_info_gain = g


def _impurity(impurity) -> str:
    """DecisionTreeClassifier's and RandomForestClassifier's ``impurity``, one of tree.IMPURITIES in any case."""
    from . import tree as T
    if not isinstance(impurity, str) or impurity.lower() not in T.IMPURITIES:
        raise ValueError(f"impurity must be one of {list(T.IMPURITIES)}, not {impurity!r}")
    return impurity.lower()


def _rate(v, name: str) -> float:
    """A real in (0, 1]: GBTClassifier's ``step_size``, RandomForestClassifier's ``subsampling_rate``."""
    r = float(v) if isinstance(v, (int, float, np.floating)) and not isinstance(v, bool) else float("nan")
    if not 0.0 < r <= 1.0:
        raise ValueError(f"{name} must lie in (0, 1], not {v!r}")
    return r


def _classes(features, name: str) -> tuple[int, int]:
    """(n, numClasses = max label + 1) of DecisionTreeClassifier's and RandomForestClassifier's features (lo_lr_stats:
    every label an integer >= 0 and every feature finite).  No row and more than LO_DT_MAX_CLASSES classes are refused."""
    _labelled(features, name)
    n, _total, _m2, counts = _on_device(features, lambda engine, rows: engine.lr_stats(rows), name=name,
                                        reasons=_LR_REASONS)
    _some_rows(n, name)
    num_classes = int(np.flatnonzero(counts)[-1]) + 1
    if num_classes > N.LO_DT_MAX_CLASSES:
        raise N.LoexecError(N.LO_ERR_INVALID, f"{num_classes} classes exceed LO_DT_MAX_CLASSES = "
                            f"{N.LO_DT_MAX_CLASSES}")
    return n, num_classes


@contextlib.contextmanager
def _binned(features, n: int, max_bins: int, name: str, kf: int, per_bin: int, unit: str):
    """The tree fits' codes, after refusing a one-node histogram (kf features x min(max_bins, n) bins x per_bin u64
    ``unit``) above LO_DT_PASS_HIST: yields (:func:`split_thresholds`' thresholds and rank rounds, nbins, the rows binned
    on the device by ``dt_bin``) and frees the codes when the block ends."""
    k = len(features.fields)
    if kf * min(max_bins, n) * per_bin * 8 > N.LO_DT_PASS_HIST:
        raise N.LoexecError(N.LO_ERR_INVALID, f"{kf} features x {min(max_bins, n)} bins x {per_bin} {unit}: one node's "
                            f"histogram exceeds LO_DT_PASS_HIST = {N.LO_DT_PASS_HIST} bytes")
    thresholds, rounds = split_thresholds(features, n, k, max_bins, name)
    nbins = max(len(t) for t in thresholds) + 1
    binned = _on_device(features, lambda engine, rows: engine.dt_bin(rows, thresholds), name=name)
    try:
        yield thresholds, rounds, nbins, binned
    finally:
        _free(binned)


class DecisionTreeClassifier:
    """``pyspark.ml.classification.DecisionTreeClassifier(maxDepth, maxBins, minInstancesPerNode, minInfoGain,
    impurity)`` with its other defaults (every feature continuous, no ``weightCol``, no ``thresholds``) on the GPU.
    max_bins above LO_DT_MAX_BINS (256) is refused: a bin index is a byte on the device."""

    def __init__(self, max_depth: int = 5, max_bins: int = 32, min_instances_per_node: int = 1,
                 min_info_gain: float = 0.0, impurity: str = "gini"):
        _tree_params(self, max_depth, max_bins, min_instances_per_node, min_info_gain)
        self.impurity = _impurity(impurity)

    def fit(self, features) -> "DecisionTreeClassificationModel":
        """The tree of ``features`` (:class:`~builder_frontend.Features` with a label, on one GPU or sharded).  Every
        label must be an integer >= 0 and every feature finite (InvalidCellError naming the ``_id`` and field of the
        lowest refused row); numClasses = max label + 1.  No row, more than LO_DT_MAX_CLASSES classes or a one-node
        histogram (k x min(max_bins, n) x C x 8 bytes) above LO_DT_PASS_HIST are refused."""
        from . import tree as T
        name, k = "DecisionTreeClassifier", len(features.fields)
        n, num_classes = _classes(features, name)
        with _binned(features, n, self.max_bins, name, k, num_classes, "classes") as (thresholds, rounds, nbins, binned):
            def level(splits, nnodes):
                return _on_device(features, lambda engine, rows: engine.dt_level(rows, binned, nbins, num_classes,
                                                                                splits, nnodes), name=name)

            tree, _shapes = T.grow(level, thresholds, num_classes, self.max_depth, self.impurity,
                                   self.min_instances_per_node, self.min_info_gain)
        model = DecisionTreeClassificationModel(tree, features.fields, thresholds)
        model.rank_rounds = rounds
        return model


class DecisionTreeClassificationModel(_Model):
    """A fitted decision tree, host data: ``tree`` (:class:`~tree.Tree`: the node arrays feature, threshold, left, right,
    counts, prediction, impurity and gain), ``depth``, ``num_nodes``, ``num_classes``, the ``fields`` it was fitted on
    and every column's split ``thresholds``."""
    _name, _reasons = "DecisionTreeClassifier", _LR_REASONS

    def __init__(self, tree, fields, thresholds=None):
        self.tree, self.fields, self.thresholds = tree, list(fields), thresholds
        self.depth, self.num_nodes, self.num_classes = tree.depth, tree.num_nodes, tree.num_classes

    def _predict(self, engine, rows, raw=False, labels=None):
        return engine.dt_predict(rows, self.tree, raw=raw, labels=labels)

    def transform(self, features, raw: bool = False) -> "Predictions":
        """Spark's ``model.transform``: every row's ``probability`` (the leaf's class counts over their sum) and
        ``prediction`` (a class index as float64), and with ``raw`` its ``rawPrediction`` (the leaf's counts), written in
        HBM on the rows' own devices."""
        return super().transform(features, raw)


_GB_REASONS = ("is NaN or infinite", "is not a label 0 or 1")


class GBTClassifier:
    """``pyspark.ml.classification.GBTClassifier(maxIter, stepSize, maxDepth, maxBins, minInstancesPerNode,
    minInfoGain)`` with its other defaults (``lossType="logistic"``, ``subsamplingRate=1``, every feature and every row
    in every tree, no validation, no ``weightCol``, no ``thresholds``) on the GPU (DESIGN.md §3.6.5).  max_iter 0 is
    refused, and so is max_bins above LO_DT_MAX_BINS (256): a bin index is a byte on the device."""

    def __init__(self, max_iter: int = 20, step_size: float = 0.1, max_depth: int = 5, max_bins: int = 32,
                 min_instances_per_node: int = 1, min_info_gain: float = 0.0):
        self.max_iter = _integer(max_iter, "max_iter", 1)
        self.step_size = _rate(step_size, "step_size")
        _tree_params(self, max_depth, max_bins, min_instances_per_node, min_info_gain)

    def fit(self, features) -> "GBTClassificationModel":
        """The boosted trees of ``features`` (:class:`~builder_frontend.Features` with a label, on one GPU or sharded).
        Every label must be 0 or 1 and every feature finite (InvalidCellError naming the ``_id`` and field of the lowest
        refused cell over both checks).  No row, or a one-node level (k x min(max_bins, n) x 40 bytes) above LO_DT_PASS_HIST, is
        refused.  The margins and residuals stay on the device, the trees are chosen here from each level's sums."""
        from . import tree as T
        name, k = "GBTClassifier", len(features.fields)
        _labelled(features, name)
        from .engine import InvalidCellError
        # the labels (lo_gb_update's first call) and the features (lo_lr_stats_range) are both checked, and the lowest
        # refused cell of the two is raised, as one pass over both would find it
        refused, rows = [], None
        try:
            rows = _on_device(features, lambda engine, part: engine.gb_update(part), name=name, reasons=_GB_REASONS)
        except InvalidCellError as e:
            refused.append(e)
        try:
            try:
                n = _on_device(features, lambda engine, part: engine.lr_stats(part), name=name, reasons=_GB_REASONS)[0]
            except InvalidCellError as e:
                refused.append(e)
            except N.LoexecError:                    # a label >= LO_NB_MAX_CLASSES: already a refused label cell
                if not refused:
                    raise
            if refused:
                raise min(refused, key=lambda e: (e.row, e.position))
            _some_rows(n, name)
            trees, weights = [], []
            with _binned(features, n, self.max_bins, name, k, N.LO_GB_WORDS, "words") as (thresholds, _, nbins, binned):
                for m in range(self.max_iter):
                    def level(splits, nnodes):
                        return _on_device(features, lambda engine, part: engine.gb_level(part, binned, rows, nbins,
                                                                                        splits, nnodes), name=name)

                    tree, _shapes = T.grow(level, thresholds, 0, self.max_depth, T.VARIANCE,
                                           self.min_instances_per_node, self.min_info_gain)
                    weight = 1.0 if m == 0 else self.step_size
                    trees.append(tree)
                    weights.append(weight)
                    if m + 1 < self.max_iter:
                        _on_device(features, lambda engine, part: engine.gb_update(part, rows, tree, weight), name=name,
                                   reasons=_GB_REASONS)
        finally:
            _free(rows)
        return GBTClassificationModel(trees, weights, features.fields, thresholds)


class GBTClassificationModel(_Model):
    """A fitted GBT model, host data: ``trees`` (regression :class:`~tree.Tree` s in breadth-first arrays: feature,
    threshold, left, right, prediction, impurity, gain and ``counts`` the node's (count, sum, sumSq)), ``tree_weights``
    ([1.0, step_size, ...]), ``num_classes`` (2), ``total_num_nodes``, the ``fields`` it was fitted on and every column's
    split ``thresholds``."""
    _name, _reasons = "GBTClassifier", _GB_REASONS

    def __init__(self, trees, tree_weights, fields, thresholds=None):
        self.trees, self.tree_weights = list(trees), np.asarray(tree_weights, np.float64)
        self.fields, self.thresholds = list(fields), thresholds
        self.num_classes = 2
        self.total_num_nodes = sum(t.num_nodes for t in self.trees)

    def _predict(self, engine, rows, raw=False, labels=None):
        return engine.gb_predict(rows, self.trees, self.tree_weights, raw=raw, labels=labels)

    def transform(self, features, raw: bool = False) -> "Predictions":
        """Spark's ``model.transform``: every row's ``probability`` ([1 / (1 + exp(2m)), the rest] of the margin m) and
        ``prediction`` (m > 0), and with ``raw`` its ``rawPrediction`` ([-m, m]), written in HBM on the rows' own
        devices."""
        return super().transform(features, raw)


_RF_SLOT_BUDGET = 2 << 30      # bytes of the two int32 slot tables of one batch of trees (ntrees * n rows each)


class RandomForestClassifier:
    """``pyspark.ml.classification.RandomForestClassifier(numTrees, maxDepth, maxBins, minInstancesPerNode,
    minInfoGain, impurity, featureSubsetStrategy, subsamplingRate, seed)`` with its other defaults (every feature
    continuous, no ``weightCol``, no ``thresholds``) on the GPU (DESIGN.md §3.6.6).  Bagging and the feature subsets
    are counter-based hashes of ``seed``, so a forest is the same on one GPU and on any shard cut.  max_bins above
    LO_DT_MAX_BINS (256) is refused: a bin index is a byte on the device."""

    def __init__(self, num_trees: int = 20, max_depth: int = 5, max_bins: int = 32, min_instances_per_node: int = 1,
                 min_info_gain: float = 0.0, impurity: str = "gini", feature_subset_strategy: str = "auto",
                 subsampling_rate: float = 1.0, seed: int | None = None):
        from . import tree as T
        self.num_trees = _integer(num_trees, "num_trees", 1)
        _tree_params(self, max_depth, max_bins, min_instances_per_node, min_info_gain)
        self.impurity = _impurity(impurity)
        T.subset_size(feature_subset_strategy, 1, self.num_trees)          # refuses an unknown strategy now
        self.feature_subset_strategy = feature_subset_strategy
        self.subsampling_rate = _rate(subsampling_rate, "subsampling_rate")
        self.seed = T.DEFAULT_SEED if seed is None else _integer(seed, "seed", -(1 << 63), (1 << 63) - 1)

    def fit(self, features) -> "RandomForestClassificationModel":
        """The forest of ``features`` (:class:`~builder_frontend.Features` with a label, on one GPU or sharded).  Every
        label must be an integer >= 0 and every feature finite (InvalidCellError naming the ``_id`` and field of the
        lowest refused row); numClasses = max label + 1.  No row, more than LO_DT_MAX_CLASSES classes or a one-node
        histogram (m x min(max_bins, n) x C x 8 bytes, m the features a node searches) above LO_DT_PASS_HIST are
        refused.  The trees grow in batches whose slot tables fit _RF_SLOT_BUDGET, one level pass per batch level."""
        from . import tree as T
        name, k = "RandomForestClassifier", len(features.fields)
        n, num_classes = _classes(features, name)
        m = T.subset_size(self.feature_subset_strategy, k, self.num_trees)
        draw = T.draw_table(self.num_trees, self.subsampling_rate)
        batch = max(1, min(self.num_trees, _RF_SLOT_BUDGET // (8 * n)))
        trees = []
        with _binned(features, n, self.max_bins, name, m, num_classes, "classes") as (thresholds, _, nbins, binned):
            for tree0 in range(0, self.num_trees, batch):
                ntrees = min(batch, self.num_trees - tree0)

                def level(splits, nnodes, feats):
                    return _on_device(features, lambda engine, rows: engine.rf_level(
                        rows, binned, nbins, num_classes, self.seed, draw, tree0, ntrees, splits, feats), name=name)

                grown, _shapes = T.grow(level, thresholds, num_classes, self.max_depth, self.impurity,
                                        self.min_instances_per_node, self.min_info_gain, trees=ntrees,
                                        subsets=lambda t, node: T.feature_subset(self.seed, tree0 + t, node, k, m))
                trees += grown
        model = RandomForestClassificationModel(trees, features.fields, thresholds, m)
        model.tree_batch = batch
        return model


class RandomForestClassificationModel(_Model):
    """A fitted random forest, host data: ``trees`` (classification :class:`~tree.Tree` s: the node arrays feature,
    threshold, left, right, counts (bagging-weighted class counts), prediction, impurity and gain), ``tree_weights``
    (all 1.0), ``num_classes``, ``total_num_nodes``, the ``fields`` it was fitted on, every column's split
    ``thresholds``, ``feature_subset`` (the features each node searched) and, after a fit, ``tree_batch`` (the trees
    grown together per level pass)."""
    _name, _reasons = "RandomForestClassifier", _LR_REASONS

    def __init__(self, trees, fields, thresholds=None, feature_subset=None):
        self.trees, self.fields, self.thresholds = list(trees), list(fields), thresholds
        self.tree_weights = np.ones(len(self.trees))
        self.num_classes = self.trees[0].num_classes
        self.total_num_nodes = sum(t.num_nodes for t in self.trees)
        self.feature_subset = feature_subset

    def _predict(self, engine, rows, raw=False, labels=None):
        return engine.rf_predict(rows, self.trees, raw=raw, labels=labels)

    def transform(self, features, raw: bool = False) -> "Predictions":
        """Spark's ``model.transform``: every row's ``rawPrediction`` (with ``raw``; the sum over trees of the leaf's
        class counts over their total), ``probability`` (raw over its sum) and ``prediction`` (the first argmax of
        raw, a class index as float64), written in HBM on the rows' own devices."""
        return super().transform(features, raw)
