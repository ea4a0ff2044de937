"""numpy restatement of Spark 2.4's LogisticRegression pieces that run on the device or beside it (test infrastructure;
the library never imports it).  DESIGN.md §3.6.3 lists the rules.

* stats: n, the exact column sums (math.fsum), the sums of (x - sum / n)^2 (fsum of the rounded squares) and the label
  counts; refuses non-finite features and labels that are not integers >= 0 (the lowest row, then column).
* loss_grad: LogisticAggregator's per-row loss and multipliers at the effective coefficients, every slot summed with
  math.fsum, and the sums of |term| the device's error is bounded by.
* objective: Spark's value and gradient in the scaled space, from loss_grad.
* unscale: coef / std, centring as Spark does.
* binomial transform: m = (sum_j w_j x_j from 0.0, every product and add rounded) + b, raw [-m, m], p1 = 1 / (1 +
  exp(-m)), p0 = 1 - p1, prediction p1 > threshold.  Multinomial transform: raw as oracle/naive_bayes.py's (coefficients
  for theta, intercepts for pi), then LogisticRegressionModel's raw2probabilityInPlace: m the first greatest raw value;
  m == +inf gives a one-hot probability at its index; else e = exp(raw - m) when m > 0, exp(raw) otherwise, summed in
  class order, p = e * (1 / sum); prediction the first index of the strictly greatest probability."""
from __future__ import annotations

import math

import numpy as np


def stats(x, y):
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    n, k = x.shape
    bad_x = ~np.isfinite(x)
    bad_y = ~(np.isfinite(y) & (y >= 0) & (np.floor(y) == y))
    bad = np.concatenate([bad_x, bad_y[:, None]], 1)
    if bad.any():
        r, c = np.argwhere(bad)[0]
        raise ValueError((int(r), int(c)))
    total = np.array([math.fsum(x[:, j]) for j in range(k)])
    mean = total / n if n else total
    m2 = np.array([math.fsum((x[:, j] - mean[j]) ** 2) for j in range(k)])
    counts = np.bincount(y.astype(np.int64), minlength=1) if n else np.zeros(1, np.int64)
    return n, total, m2, counts


def _log1p_exp(v):
    return np.where(v > 0, v + np.log1p(np.exp(-np.abs(v))), np.log1p(np.exp(np.minimum(v, 0))))


def row_terms(x, y, beta, b, multinomial: bool):
    """(loss per row, multipliers n x C') of LogisticAggregator at effective coefficients beta (C' x k), intercepts b."""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    margins = x @ np.asarray(beta, np.float64).T + np.asarray(b, np.float64)[None, :]
    if not multinomial:
        margin = -margins[:, 0]
        mult = 1.0 / (1.0 + np.exp(margin)) - y
        loss = np.where(y > 0, _log1p_exp(margin), _log1p_exp(margin) - margin)
        return loss, mult[:, None]
    nc = margins.shape[1]
    lab = y.astype(np.int64)
    of_label = margins[np.arange(len(y)), lab]
    top = margins.max(axis=1)
    shift = np.where(top > 0, top, 0.0)
    e = np.exp(margins - shift[:, None])
    s = e.sum(axis=1)
    mult = e / s[:, None] - (lab[:, None] == np.arange(nc)[None, :])
    loss = np.log(s) - of_label + shift
    return loss, mult


def loss_grad(x, y, beta, b, multinomial: bool):
    """((loss, grad C' x k, intercept sums C'), (the same of |term|)): every sum exact-rounded (math.fsum)."""
    x = np.asarray(x, np.float64)
    loss, mult = row_terms(x, y, beta, b, multinomial)
    nc, k = mult.shape[1], x.shape[1]
    grad = np.array([[math.fsum(mult[:, c] * x[:, j]) for j in range(k)] for c in range(nc)]).reshape(nc, k)
    agrad = np.array([[math.fsum(np.abs(mult[:, c] * x[:, j])) for j in range(k)] for c in range(nc)]).reshape(nc, k)
    icpt = np.array([math.fsum(mult[:, c]) for c in range(nc)])
    aicpt = np.array([math.fsum(np.abs(mult[:, c])) for c in range(nc)])
    return (math.fsum(loss), grad, icpt), (math.fsum(np.abs(loss)), agrad, aicpt)


def objective(x, y, std, v, nc: int, reg: float, multinomial: bool):
    """Spark's (value, gradient) at the scaled-space point v = [w (nc x k), b (nc)]."""
    std = np.asarray(std, np.float64)
    k, n = len(std), len(y)
    w, b = v[:nc * k].reshape(nc, k), v[nc * k:]
    beta = np.zeros_like(w)
    beta[:, std != 0] = w[:, std != 0] / std[std != 0]
    (loss, g, gb), _ = loss_grad(x, y, beta, b, multinomial)
    gw = np.zeros_like(w)
    gw[:, std != 0] = g[:, std != 0] / std[std != 0]
    value = loss / n + 0.5 * reg * float((w * w).sum())
    return value, np.concatenate([(gw / n + reg * w).ravel(), gb / n])


def unscale(v, std, nc: int, reg: float, multinomial: bool):
    std = np.asarray(std, np.float64)
    k = len(std)
    w, b = v[:nc * k].reshape(nc, k).copy(), v[nc * k:].copy()
    coef = np.zeros_like(w)
    coef[:, std != 0] = w[:, std != 0] / std[std != 0]
    if multinomial and reg == 0.0:
        coef -= coef.sum(axis=0) / nc
    if multinomial:
        b -= b.sum() / nc
    return coef, b


def binomial_raw(x, w, b):
    x = np.asarray(x, np.float64)
    m = np.zeros(x.shape[0])
    for j in range(x.shape[1]):
        m = m + x[:, j] * w[j]
    m = m + b
    return np.stack([-m, m], 1)


def binomial_probability(raw):
    p1 = 1.0 / (1.0 + np.exp(-raw[:, 1]))
    return np.stack([1.0 - p1, p1], 1)


def binomial_prediction(prob, threshold: float = 0.5):
    return (prob[:, 1] > threshold).astype(np.float64)


def multinomial_probability(raw):
    raw = np.asarray(raw, np.float64)
    at = np.zeros(raw.shape[0], np.int64)
    m = raw[:, 0].copy()
    for c in range(1, raw.shape[1]):
        up = raw[:, c] > m
        at = np.where(up, c, at)
        m = np.where(up, raw[:, c], m)
    with np.errstate(invalid="ignore", over="ignore"):
        e = np.exp(np.where((m > 0)[:, None], raw - m[:, None], raw))
    s = np.zeros(raw.shape[0])
    for c in range(raw.shape[1]):
        s = s + e[:, c]
    with np.errstate(divide="ignore", invalid="ignore"):
        p = e * (1.0 / s)[:, None]
    hot = np.isposinf(m)
    p[hot] = 0.0
    p[hot, at[hot]] = 1.0
    return p
