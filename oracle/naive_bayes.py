"""numpy restatement of Spark 2.4's multinomial NaiveBayes and its evaluator (test infrastructure only; the library
never imports it).  DESIGN.md §3.6.2 lists the rules and where they come from.

* fit: classes = the distinct label values ascending (-0.0 as 0.0); n_c the class's rows; s_cj = math.fsum of feature j
  over them (the exact sum, correctly rounded); pi / theta as Spark computes them from those.
* raw: (sum_j theta_cj * x_j from 0.0, j ascending, every product and add rounded on its own) + pi_c.
* probability: m = left-fold max, e = exp(raw - m) summed in c order, p = e / sum; prediction: the first index of the
  strictly greatest probability.
* metrics: MulticlassMetrics' weighted F1 and accuracy, a prediction (a class index) matching a label by equality."""
from __future__ import annotations

import math

import numpy as np


def classes_of(y) -> np.ndarray:
    y = np.asarray(y, np.float64)
    if np.isnan(y).any():
        raise ValueError("NaN label")
    return np.unique(y + 0.0)          # -0.0 + 0.0 == +0.0


def fit_sums(x, y) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(classes, counts int64[C], sums float64[C, k]) with every sum exact (math.fsum)."""
    x = np.asarray(x, np.float64)
    y = np.asarray(y, np.float64) + 0.0
    classes = classes_of(y)
    counts = np.array([(y == c).sum() for c in classes], np.int64)
    sums = np.array([[math.fsum(x[y == c, j]) for j in range(x.shape[1])] for c in classes], np.float64)
    return classes, counts, sums.reshape(len(classes), x.shape[1])


def model(counts, sums, smoothing: float = 1.0) -> tuple[np.ndarray, np.ndarray]:
    """(pi, theta) as NaiveBayes.trainWithLabelCheck: log(n_c + λ) - log(N + C λ) and log(s_cj + λ) - log(S_c + k λ),
    N and S_c summed in order."""
    counts = np.asarray(counts, np.float64)
    sums = np.asarray(sums, np.float64)
    nclasses, k = sums.shape
    n_docs = 0.0
    for c in counts:
        n_docs += float(c)
    pi = np.log(counts + smoothing) - np.log(n_docs + nclasses * smoothing)
    totals = np.zeros(nclasses)
    for j in range(k):
        totals = totals + sums[:, j]
    theta = np.log(sums + smoothing) - np.log(totals + k * smoothing)[:, None]
    return pi, theta


def raw(x, pi, theta) -> np.ndarray:
    """n x C raw values: F2J dgemv's separately rounded loop, then + pi."""
    x = np.asarray(x, np.float64)
    out = np.zeros((x.shape[0], len(pi)))
    for j in range(x.shape[1]):
        out = out + x[:, j:j + 1] * theta[:, j][None, :]
    return out + pi[None, :]


def probability(r) -> np.ndarray:
    m = r[:, 0].copy()
    for c in range(1, r.shape[1]):
        m = np.where(m >= r[:, c], m, r[:, c])
    e = np.exp(r - m[:, None])
    s = np.zeros(r.shape[0])
    for c in range(r.shape[1]):
        s = s + e[:, c]
    return e / s[:, None]


def prediction(p) -> np.ndarray:
    best = np.zeros(p.shape[0], np.int64)
    top = p[:, 0].copy()
    for c in range(1, p.shape[1]):
        up = p[:, c] > top
        best = np.where(up, c, best)
        top = np.where(up, p[:, c], top)
    return best.astype(np.float64)


def confusion(y, pred, labels, nclasses: int) -> np.ndarray:
    y = np.asarray(y, np.float64) + 0.0
    out = np.zeros((len(labels), nclasses), np.int64)
    slot = np.searchsorted(labels, y)
    np.add.at(out, (slot, pred.astype(np.int64)), 1)
    return out


def metrics(y, pred) -> tuple[float, float]:
    """(weighted F1, accuracy) straight from the (label, prediction) pairs, as MulticlassMetrics does."""
    y = np.asarray(y, np.float64) + 0.0
    pred = np.asarray(pred, np.float64)
    n = len(y)
    f1, tp_all = 0.0, 0
    for lab in np.unique(y):
        count = int((y == lab).sum())
        tp = int(((y == lab) & (pred == lab)).sum())
        fp = int(((pred == lab) & (y != lab)).sum())
        precision = 0.0 if tp + fp == 0 else tp / (tp + fp)
        recall = tp / count
        f = 0.0 if precision + recall == 0 else 2.0 * precision * recall / (precision + recall)
        f1 += f * count / n
        tp_all += tp
    return f1, tp_all / n
