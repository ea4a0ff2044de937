"""The builder's "NB" classifier on the GPU: Spark 2.4's multinomial ``NaiveBayes`` (``builder_image/builder.py:55-61``)
fitted on, applied to and evaluated over the feature matrix in HBM (:meth:`DeviceFrame.features`), on one GPU or on
every shard of a local :class:`~sharding.ShardedEngine`.  DESIGN.md §3.6.2 states the semantics.

The device computes the class counts and per-class feature sums (``lo_nb_fit``), every row's raw values, probabilities
and prediction (``lo_nb_predict``) and the confusion counts of an evaluation; the model's logs (C x k values) and the
evaluator's metrics are computed here, on the host, from those."""
from __future__ import annotations

import numpy as np

from . import _native as N


def _on_device(features, call, per_part: bool = False):
    """``call(engine, rows)`` on the features' engine: a ShardedEngine takes every shard's rows and gives one result per
    shard where it gives one per row (``per_part``); an Engine takes its one part, and its result is made a list of one
    where ``per_part``.  A refused cell (its row a row of the features, shards concatenated) is raised as the ``_id``
    and field it holds."""
    from .builder_frontend import named_cell
    from .engine import InvalidCellError
    from .sharding import ShardedEngine
    engine = features._frame._cache.engine
    sharded = isinstance(engine, ShardedEngine)
    try:
        out = call(engine, features._parts if sharded else features._parts[0])
    except InvalidCellError as e:
        raise named_cell(e, features.fields, features.label, features.row_ids, "NaiveBayes",
                         ("is negative or NaN", "is not a class of the model")) from None
    return [out] if per_part and not sharded else out


def _usable(features) -> None:
    """Refuses features that have been released (their tables freed) before anything reads them."""
    if not features._parts:
        raise ValueError("the features have been released")


def _labels(features) -> np.ndarray:
    """The distinct label values of the features' rows, ascending (every shard's union)."""
    _usable(features)
    if features.label is None:
        raise ValueError("NaiveBayes needs features with a label")
    return _on_device(features, lambda engine, rows: engine.nb_labels(rows))


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
        if len(features.row_ids) == 0:
            raise N.LoexecError(N.LO_ERR_INVALID, "NaiveBayes needs at least one row")
        k = len(features.fields)
        if len(classes) * k > N.LO_NB_MAX_THETA:
            raise N.LoexecError(N.LO_ERR_INVALID, f"{len(classes)} classes x {k} features exceed LO_NB_MAX_THETA = "
                                f"{N.LO_NB_MAX_THETA}")
        sums, counts = _on_device(features, lambda engine, rows: engine.nb_fit(rows, classes))
        pi, theta = model_arrays(sums, counts, self.smoothing)
        return NaiveBayesModel(classes, pi, theta, features.fields, sums, counts)


class NaiveBayesModel:
    """A fitted multinomial NaiveBayes model, host data: ``labels`` (float64[C], the class values ascending), ``pi``
    (float64[C]), ``theta`` (float64[C, k]) and the ``fields`` it was fitted on; ``sums`` / ``counts`` are the device's
    per-class feature sums and row counts it was made from."""

    def __init__(self, labels, pi, theta, fields, sums=None, counts=None):
        self.labels, self.pi, self.theta = np.asarray(labels, np.float64), np.asarray(pi, np.float64), np.asarray(theta, np.float64)
        self.fields, self.sums, self.counts = list(fields), sums, counts

    def _check(self, features) -> None:
        if list(features.fields) != self.fields:
            raise ValueError(f"the model was fitted on fields {self.fields}, not {list(features.fields)}")

    def transform(self, features, raw: bool = False) -> "Predictions":
        """Spark's ``model.transform``: every row's ``probability`` and ``prediction`` (a class INDEX as float64), and
        with ``raw`` its ``rawPrediction``, written in HBM on the rows' own devices."""
        _usable(features)
        self._check(features)
        parts = _on_device(features, lambda engine, rows: engine.nb_predict(rows, self.pi, self.theta, raw=raw),
                           per_part=True)
        return Predictions(features, parts)

    def evaluate(self, features) -> dict:
        """``MulticlassClassificationEvaluator`` f1 and accuracy over ``transform(features)`` (builder.py:124-142), as one
        fused pass per device that writes nothing per row: ``{"f1", "accuracy", "labels", "confusion"}`` where
        ``confusion[a, p]`` counts the rows labelled ``labels[a]`` predicted as class index p."""
        _usable(features)
        self._check(features)
        labels = _labels(features)
        if len(features.row_ids) == 0:
            raise N.LoexecError(N.LO_ERR_INVALID, "evaluate needs at least one row")
        confusion = _on_device(features, lambda engine, rows: engine.nb_predict(rows, self.pi, self.theta, labels=labels))
        f1, accuracy = metrics(labels, confusion)
        return {"f1": f1, "accuracy": accuracy, "labels": labels, "confusion": confusion}


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
