"""breeze 0.13's ``LBFGS`` with its ``StrongWolfeLineSearch``, as Spark 2.4's LogisticRegression drives it (m = 10, a
``CachedDiffFunction``, breeze's default convergence check), in host numpy.  It knows nothing of the device: ``fun(x)``
returns (value, gradient) and :class:`~classifier.LogisticRegression` makes each call one device pass.  DESIGN.md §3.6.3
lists the rules; they are recalled from breeze's source, not checked against it."""
from __future__ import annotations

import math

import numpy as np

M = 10                    # L-BFGS history pairs
C1, C2 = 1e-4, 0.9        # strong-Wolfe constants
MAX_ZOOM = 10
MAX_BRACKET = 10
FVAL_MEMORY = 20


class LineSearchFailed(Exception):
    """breeze's FirstOrderException: the line search, or the two-loop recursion, gave up."""


class _Cached:
    """breeze's CachedDiffFunction: the last point's (value, gradient) is not evaluated again."""

    def __init__(self, fun):
        self.fun, self.calls, self._x, self._out = fun, 0, None, None

    def __call__(self, x):
        if self._x is None or not np.array_equal(self._x, x):
            value, grad = self.fun(x)
            self.calls += 1
            self._x, self._out = x.copy(), (float(value), np.asarray(grad, np.float64))
        return self._out


def _direction(grad, steps, deltas):
    """ApproximateInverseHessian * grad, negated: the two-loop recursion over the newest-first pairs, H0 = s.y / y.y of
    the newest pair (1 with none)."""
    diag = 1.0
    if steps:
        sy, yy = float(steps[0] @ deltas[0]), float(deltas[0] @ deltas[0])
        if sy < 0 or math.isnan(sy):
            raise LineSearchFailed("NaN history")
        diag = sy / yy
    d = grad.copy()
    alphas, rhos = [], []
    for s, y in zip(steps, deltas):
        rho = float(s @ y)
        a = float(s @ d) / rho
        if math.isnan(a):
            raise LineSearchFailed("NaN history")
        d -= a * y
        alphas.append(a)
        rhos.append(rho)
    d *= diag
    for i in range(len(steps) - 1, -1, -1):
        beta = float(deltas[i] @ d) / rhos[i]
        d += (alphas[i] - beta) * steps[i]
    return -d


def _interp(l, r):
    """Safeguarded cubic interpolation between brackets (t, value, slope), clamped to [10 %, 90 %] of [l.t, r.t]."""
    (lt, lf, ld), (rt, rf, rd) = l, r
    d1 = ld + rd - 3 * (lf - rf) / (lt - rt)
    d2 = math.sqrt(d1 * d1 - ld * rd) if d1 * d1 - ld * rd >= 0 else math.nan
    t = rt - (rt - lt) * (rd + d2 - d1) / (rd - ld + 2 * d2)
    lo, hi = lt + 0.1 * (rt - lt), lt + 0.9 * (rt - lt)
    if t < lo:
        return lo
    if t > hi:
        return hi
    return t            # NaN falls through, as in breeze


def _line_search(phi, f0, d0, init):
    """StrongWolfeLineSearch.minimize: the step t >= 0 along the direction, phi(t) = (value, slope)."""
    if d0 > 0:
        raise LineSearchFailed(f"not a descent direction: {d0}")

    def zoom(low, hi):
        for _ in range(MAX_ZOOM):
            t = _interp(hi, low) if low[0] > hi[0] else _interp(low, hi)
            f, d = phi(t)
            c = (t, f, d)
            if f > f0 + C1 * t * d0 or f >= low[1]:
                hi = c
            else:
                if abs(d) <= C2 * abs(d0):
                    return t
                if d * (hi[0] - low[0]) >= 0:
                    hi = low
                low = c
        raise LineSearchFailed("zoom failed")

    low, t = (0.0, f0, d0), init
    for i in range(MAX_BRACKET):
        f, d = phi(t)
        if math.isinf(f) or math.isnan(f):
            t /= 2.0
            continue
        c = (t, f, d)
        if f > f0 + C1 * t * d0 or (f >= low[1] and i > 0):
            return zoom(low, c)
        if abs(d) <= C2 * abs(d0):
            return t
        if d >= 0:
            return zoom(c, low)
        low = c
        t *= 1.5
    raise LineSearchFailed("line search failed")


class Result:
    """What :func:`minimize` found: ``x``; ``history``, the value of every state it went through, the start included
    (a failed line search repeats the value it stayed at); ``iterations``, the steps taken; ``evaluations``, the calls of
    ``fun``; ``reason``, why it stopped."""

    def __init__(self, x, history, iterations, evaluations, reason):
        self.x, self.history, self.iterations, self.evaluations, self.reason = x, history, iterations, evaluations, reason


def minimize(fun, x0, max_iter: int = 100, tol: float = 1e-6) -> Result:
    """L-BFGS from ``x0``: ``fun(x)`` -> (value, gradient).  Stops when ``iter >= max_iter``; when at least 2 values are
    recorded and |f - max(last 20)| <= tol |f0|; when ||g||_2 <= max(tol |f|, 1e-8); or when the line search fails twice
    in a row (the first failure drops the history and tries again)."""
    f = _Cached(fun)
    x = np.array(x0, np.float64)
    value, grad = f(x)
    f0 = value
    steps, deltas, recorded = [], [], []
    history, it, failed_once = [value], 0, False

    def converged():
        if it >= max_iter:
            return "max_iter"
        if len(recorded) >= 2 and abs(value - max(recorded[-FVAL_MEMORY:])) <= tol * abs(f0):
            return "function values"
        if float(np.linalg.norm(grad)) <= max(tol * abs(value), 1e-8):
            return "gradient"
        return None

    reason = converged()
    while reason is None:
        try:
            d = _direction(grad, steps, deltas)
            init = 1.0 / float(np.linalg.norm(d)) if it == 0 else 1.0

            def phi(t, d=d):
                v, g = f(x + d * t)
                return v, float(g @ d)

            t = _line_search(phi, value, float(grad @ d), init)
            if t * float(np.linalg.norm(grad)) < 1e-10:
                raise LineSearchFailed("step size underflow")
            nx = x + d * t
            nvalue, ngrad = f(nx)
        except LineSearchFailed:
            if failed_once:
                history.append(value)
                reason = "line search failed"
                break
            failed_once = True
            steps, deltas = [], []
            history.append(value)
            reason = converged()
            continue
        steps, deltas = ([nx - x] + steps)[:M], ([ngrad - grad] + deltas)[:M]
        recorded.append(nvalue)
        x, value, grad, it, failed_once = nx, nvalue, ngrad, it + 1, False
        history.append(value)
        reason = converged()
    return Result(x, history, it, f.calls, reason)
