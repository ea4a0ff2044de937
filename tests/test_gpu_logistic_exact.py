"""GPU: LogisticRegression's device passes (lo_lr_stats, lo_lr_loss_grad, lo_lr_predict) against references that do not
restate the device's formulas — exact rationals for the column statistics, mpmath at 60 digits for log1pExp, the sigmoid
and the softmax — on parameter sets picked from a restatement of the launch shapes so that every route runs, with the
row padding filled with NaN, at the margins where exp overflows or underflows, and with a constant column's std exactly
0 on one GPU and over shard cuts."""
import ctypes as C
import math
from fractions import Fraction

import mpmath
import numpy as np
import pytest

import logistic_oracle as lo
from learningorchestra_b200 import _native as N
from learningorchestra_b200.classifier import LogisticRegression, standardization
from test_gpu_logistic import _cut, _sharded, _sk_objective
from test_gpu_naive_bayes import _features, _free, _part, _ulps

pytestmark = pytest.mark.gpu
mpmath.mp.dps = 60

# ---- the launch shapes of lo_lr_stats / lo_lr_loss_grad, restated (tests/test_logistic_cpu.py pins these constants) ----
CONSTANTS = {"kLrThreads": 256, "kLrCtaRows": 2048, "kLrTileMax": 128, "kLrStatCols": 512, "kLrHist": 1024,
             "kLrSmemMax": 227 * 1024, "kLrMarginBlock": 4, "kLrBlockC": 2, "kLrBlockJ": 4, "kLrUnroll": 4}
K = CONSTANTS


def lr_rows(fixed, per_row):
    r = K["kLrTileMax"]
    while r > 0 and fixed + r * per_row > K["kLrSmemMax"]:
        r >>= 1
    return r


def lr_vw(esz, ld):
    """Values per load; device tables start 16-byte aligned, so the row stride decides."""
    return 16 // esz if ld * esz % 16 == 0 else 1


def lr_stats_shape(k, esz, ld):
    """The kLrSum pass (the larger of the two: its min / max and label bins sit beside the sums)."""
    kc = min(k, K["kLrStatCols"])
    g = 1 if kc >= K["kLrThreads"] else K["kLrThreads"] // kc
    fixed = g * kc * 8 * 3 + (K["kLrHist"] + 1) * 4
    chunks = -(-k // kc)
    return {"R": lr_rows(fixed, ((kc | 1) + 1) * 8), "G": g, "chunks": chunks, "last": k - (chunks - 1) * kc,
            "vw": lr_vw(esz, ld)}


def lr_model_shape(k, nc, esz, ld):
    s = 1 + nc * (k + 1)
    nbj = -(-(k + 1) // K["kLrBlockJ"])
    nb = -(-nc // K["kLrBlockC"]) * nbj + 1
    g = 1 if nb >= K["kLrThreads"] else K["kLrThreads"] // nb
    fixed, per_row, coef = g * s * 8, (((k + 1) | 1) + 1 + nc + 1) * 8, nc * k * 8
    bare, staged = lr_rows(fixed, per_row), lr_rows(fixed + coef, per_row)
    cs = int(staged > 0 and staged >= min(32, bare))
    return {"R": staged if cs else bare, "G": g, "cs": cs, "vw": lr_vw(esz, ld)}


F32, F64 = np.float32, np.float64
# (dtype, k, n)
STATS_CASES = [(F32, 3, 1), (F64, 8, 100), (F32, 16, 4099), (F64, 33, 20_011), (F64, 256, 4173), (F64, 513, 3001),
               (F32, 1025, 2100), (F32, 8192, 300)]
# (dtype, k, nc, multinomial, n)
MODEL_CASES = [(F32, 4, 1, False, 1), (F64, 6, 3, True, 100), (F32, 12, 5, True, 5003), (F64, 9, 7, True, 4097),
               (F32, 301, 1, False, 3001), (F64, 1024, 8, True, 700), (F64, 8192, 2, True, 37), (F32, 2, 2, True, 2048)]


def _esz(dtype):
    return np.dtype(dtype).itemsize


def shape_coverage():
    """What the parameter sets reach, by the restated shapes."""
    st = [lr_stats_shape(k, _esz(d), k) | {"n": n} for d, k, n in STATS_CASES]
    md = [lr_model_shape(k, nc, _esz(d), k) | {"n": n, "k": k, "nc": nc} for d, k, nc, _m, n in MODEL_CASES]
    every = st + md
    return {
        "stats G > 1": any(s["G"] > 1 for s in st), "stats G = 1": any(s["G"] == 1 for s in st),
        "1 chunk": any(s["chunks"] == 1 for s in st),
        "2 chunks, last 1": any(s["chunks"] == 2 and s["last"] == 1 for s in st),
        "3 chunks, last 1": any(s["chunks"] == 3 and s["last"] == 1 for s in st),
        "16 chunks": any(s["chunks"] == 16 for s in st),
        "vw 1, 2, 4": {s["vw"] for s in every} >= {1, 2, 4},
        "cs 1": any(m["cs"] == 1 for m in md), "cs 0": any(m["cs"] == 0 for m in md),
        "R 128": any(m["R"] == 128 for m in md), "1 < R < 32": any(1 < m["R"] < 32 for m in md),
        "R 1": any(m["R"] == 1 for m in md), "model G = 1": any(m["G"] == 1 for m in md),
        "nc 3, 5, 7": {m["nc"] for m in md} >= {3, 5, 7},
        "(k + 1) % 4 != 0": any((m["k"] + 1) % 4 for m in md),
        "n < R": any(s["n"] < s["R"] for s in every),
        "n % R != 0": any(s["n"] % s["R"] for s in every),
        "n % 2048 != 0, n > 2048": any(s["n"] % 2048 and s["n"] > 2048 for s in every),
        "n % 2048 == 0": any(s["n"] % 2048 == 0 for s in every),
        "n = 1": any(s["n"] == 1 for s in st) and any(m["n"] == 1 for m in md),
    }


def test_the_parameter_sets_reach_every_launch_shape():
    missed = [name for name, hit in shape_coverage().items() if not hit]
    assert not missed, missed


# ---- exact references --------------------------------------------------------------------------------------------------
def _exact_stats(col):
    """(sum, mean, M2) of a column as Fractions: M2 = sum x^2 - (sum x)^2 / n, exact."""
    q = [Fraction(float(v)) for v in col]
    s = sum(q)
    return s, s / len(q), sum(v * v for v in q) - s * s / len(q)


def _m2_error_bound(n, total, mu, m2_exact):
    """The device's m2 is sum (x - m)^2 about its mean m = fl(total / n).  Exactly, sum (x - m)^2 = M2 + n (m - mu)^2
    (the cross term 2 (mu - m) sum (x - mu) vanishes), and its rounded squares are added, all >= 0, in runs of at most
    2048 then a tree, within 1e-12 of their sum.  So |m2 - M2| <= n e^2 + 1e-12 (M2 + n e^2) with e = |m - mu|; where
    the sum is exact, e <= ulp(mu) / 2 and this is the 1e-12 M2 + n ulp(mean)^2 of DESIGN §3.6.3."""
    e = abs(Fraction(float(total) / n) - mu)
    shift = n * e * e
    return float(shift + Fraction(1, 10 ** 12) * (m2_exact + shift)) * (1 + 1e-15) + 1e-300


def _check_stats(x, n, total, m2, label):
    for j in range(x.shape[1]):
        col = x[:, j].astype(np.float64)
        s, mu, m2_exact = _exact_stats(col)
        where = f"{label}, column {j}"
        assert abs(Fraction(float(total[j])) - s) <= Fraction(1, 10 ** 12) * math.fsum(np.abs(col)), where
        if col.min() == col.max():
            assert m2[j] == 0.0, (where, m2[j])
        else:
            assert abs(Fraction(float(m2[j])) - m2_exact) <= _m2_error_bound(n, total[j], mu, m2_exact), (where, m2[j])


@pytest.mark.parametrize("dtype,k,n", STATS_CASES)
def test_stats_at_every_launch_shape(engine, dtype, k, n):
    """Integer-valued features, so every sum is exact: a row read twice, skipped or taken from the wrong chunk shows."""
    rng = np.random.default_rng(k + n)
    x = rng.integers(-8, 9, (n, k)).astype(dtype)
    y = rng.integers(0, 3, n).astype(np.float64)
    part = _part(engine, x, y)
    try:
        got_n, total, m2, counts = engine.lr_stats(part)
    finally:
        part.free()
    xi = x.astype(np.int64)
    s1, s2 = xi.sum(0), (xi * xi).sum(0)
    assert got_n == n
    np.testing.assert_array_equal(total, s1.astype(np.float64))
    np.testing.assert_array_equal(counts[:3], np.bincount(y.astype(np.int64), minlength=3))
    for j in range(k):
        exact = Fraction(int(s2[j])) - Fraction(int(s1[j]) ** 2, n)
        if s2[j] * n == s1[j] ** 2:
            assert m2[j] == 0.0
        else:
            assert abs(Fraction(float(m2[j])) - exact) <= _m2_error_bound(n, total[j], Fraction(int(s1[j]), n), exact)


def _adversarial(n, dtype, seed):
    """Columns where a two-pass M2 about a rounded mean goes wrong: constants that are not dyadic, ±0, a tiny spread on
    a large offset, one outlier in a constant column (first row, last row, first row of the second CTA) and mixed
    magnitudes."""
    rng = np.random.default_rng(seed)
    cols = [np.full(n, v) for v in (0.1, 1 / 3, 123.456, -7.3, 1e-300)]
    zeros = np.where(rng.random(n) < 0.5, -0.0, 0.0)
    cols.append(zeros)
    cols.append(1e8 + np.arange(n) * 2.0 ** -26)
    for at in (0, n - 1, min(2048, n - 1)):
        c = np.full(n, 0.1)
        c[at] = 5.0
        cols.append(c)
    cols.append(rng.normal(size=n) * rng.choice([1e-8, 1.0, 1e8], n))
    x = np.stack(cols, 1).astype(dtype)
    y = rng.integers(0, 2, n).astype(np.float64)
    return x, y


@pytest.mark.parametrize("dtype", [F32, F64])
@pytest.mark.parametrize("n", [1, 5_000, 20_011])
def test_constant_columns_have_m2_exactly_zero_and_the_rest_match_exact_rationals(engine, dtype, n):
    x, y = _adversarial(n, dtype, seed=n)
    part = _part(engine, x, y)
    try:
        stats = engine.lr_stats(part)
    finally:
        part.free()
    got_n, total, m2, _counts = stats
    assert got_n == n
    xd = x.astype(np.float64)
    assert np.all(stats.min == xd.min(0)) and np.all(stats.max == xd.max(0))
    _check_stats(x, n, total, m2, f"{dtype.__name__}, n = {n}")
    std = standardization(n, total, m2)
    constant = xd.min(0) == xd.max(0)
    assert constant[:6].all() and np.all(std[constant] == 0.0)


@pytest.mark.parametrize("cuts", [2, 3, 8])
def test_constant_columns_have_m2_exactly_zero_over_shards(engine, cuts):
    """Chan's combine of the shards: the shards' rounded means of one constant differ, so only the merged min / max can
    give 0.  The other columns: each shard's q_i within the single-GPU bound (m_i e_i^2 + 1e-12), and each merge adds
    delta^2 n m / (n + m) with delta = the difference of two means, at most the column's range D, off by at most E =
    2 (max e_i + cuts ulp(mu)) (the shards' and the running mean's errors), so by at most n (2 D E + E^2) per merge."""
    n = 20_011
    x, y = _adversarial(n, F64, seed=cuts)
    parts = _cut(engine, x, y, cuts)
    try:
        got_n, total, m2, _counts = _sharded(engine, cuts).lr_stats(parts)
        shard_err = []
        for p, (a, b) in zip(parts, zip(np.linspace(0, n, cuts + 1).astype(int)[:-1],
                                        np.linspace(0, n, cuts + 1).astype(int)[1:])):
            _m, s, _q, _c = engine.lr_stats(p)
            shard_err.append([abs(Fraction(float(s[j] / (b - a))) - _exact_stats(x[a:b, j])[1]) for j in range(x.shape[1])])
    finally:
        _free(parts)
    assert got_n == n
    for j in range(x.shape[1]):
        col = x[:, j]
        s, mu, m2_exact = _exact_stats(col)
        assert abs(Fraction(float(total[j])) - s) <= Fraction(1, 10 ** 12) * math.fsum(np.abs(col))
        if col.min() == col.max():
            assert m2[j] == 0.0, (cuts, j, m2[j])
            continue
        e = max(err[j] for err in shard_err)
        big_e = 2 * (e + cuts * Fraction(math.ulp(float(mu))))
        span = Fraction(float(col.max())) - Fraction(float(col.min()))
        bound = n * e * e + Fraction(1, 10 ** 12) * m2_exact + (cuts - 1) * n * (2 * span * big_e + big_e * big_e)
        assert abs(Fraction(float(m2[j])) - m2_exact) <= float(bound) * (1 + 1e-15), (cuts, j, m2[j])


# ---- loss / gradient at every launch shape -------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,k,nc,multinomial,n", MODEL_CASES)
def test_loss_grad_at_every_launch_shape(engine, dtype, k, nc, multinomial, n):
    rng = np.random.default_rng(k * 31 + nc)
    x = rng.normal(size=(n, k)).astype(dtype)
    y = rng.integers(0, nc if multinomial else 2, n).astype(np.float64)
    beta, b = rng.normal(size=(nc, k)) / math.sqrt(k), rng.normal(size=nc)
    part = _part(engine, x, y)
    try:
        loss, g, gb = engine.lr_loss_grad(part, beta, b, multinomial)
    finally:
        part.free()
    (oloss, og, ogb), (aloss, ag, agb) = lo.loss_grad(x.astype(np.float64), y, beta, b, multinomial)
    assert abs(loss - oloss) <= 1e-12 * aloss
    assert np.all(np.abs(g - og) <= 1e-12 * ag)
    assert np.all(np.abs(gb - ogb) <= 1e-12 * agb)


# ---- the row padding is never read ------------------------------------------------------------------------------------
def _stats_call(engine, part, ld, k, n):
    """lo_lr_stats_range's (rc, [sum, m2, min, max], label counts); lo_lr_stats must give the same sums, m2 and counts."""
    out = [np.zeros(k) for _ in range(4)]
    counts = np.zeros(N.LO_NB_MAX_CLASSES, np.int64)
    info, t = N.NbInfo(), N.HostTiming()
    rc = engine._lib.lo_lr_stats_range(engine._ctx, part.x._h, ld, k, part.y._h, n,
                                       *(o.ctypes.data_as(C.c_void_p) for o in out), counts.ctypes.data_as(C.c_void_p),
                                       C.byref(info), C.byref(t))
    plain, plain_counts = [np.zeros(k) for _ in range(2)], np.zeros(N.LO_NB_MAX_CLASSES, np.int64)
    assert engine._lib.lo_lr_stats(engine._ctx, part.x._h, ld, k, part.y._h, n,
                                   *(o.ctypes.data_as(C.c_void_p) for o in plain),
                                   plain_counts.ctypes.data_as(C.c_void_p), C.byref(info), C.byref(t)) == rc
    for a, b in zip(out, plain):
        np.testing.assert_array_equal(a.view(np.int64), b.view(np.int64))
    np.testing.assert_array_equal(counts, plain_counts)
    return rc, out, counts


@pytest.mark.parametrize("dtype,k", [(F64, 6), (F32, 8), (F64, 513)])
@pytest.mark.parametrize("pad", [1, 3])
def test_padding_is_never_read(engine, dtype, k, pad):
    """ld = k + pad with NaN in the padding: no refused cell, and stats, loss / gradient and the transform's raw values
    bit for bit those of the unpadded matrix (the load width changes, the order of the sums does not)."""
    n, ld = 4_099, k + pad
    rng = np.random.default_rng(k + pad)
    x = rng.normal(size=(n, k)).astype(dtype)
    y = rng.integers(0, 3, n).astype(np.float64)
    xp = np.full((n, ld), np.nan, dtype)
    xp[:, :k] = x
    flat, padded = _part(engine, x, y), _part(engine, xp, y)
    coef, icpt = rng.normal(size=(3, k)) / math.sqrt(k), rng.normal(size=3)
    try:
        rc_f, flat_stats, flat_counts = _stats_call(engine, flat, k, k, n)
        rc_p, pad_stats, pad_counts = _stats_call(engine, padded, ld, k, n)
        assert rc_f == rc_p == N.LO_OK
        for a, b in zip(flat_stats, pad_stats):
            np.testing.assert_array_equal(a.view(np.int64), b.view(np.int64))
        np.testing.assert_array_equal(flat_counts, pad_counts)
        for multinomial, nc in ((False, 1), (True, 3)):
            yy = y if multinomial else (y > 0).astype(np.float64)
            want = engine.lr_loss_grad(_part_y(engine, flat, yy), coef[:nc], icpt[:nc], multinomial)
            out = np.zeros(1 + nc * (k + 1))
            t = N.HostTiming()
            yt = _part_y(engine, padded, yy)
            assert engine._lib.lo_lr_loss_grad(engine._ctx, padded.x._h, ld, k, yt.y._h, n,
                                               np.ascontiguousarray(coef[:nc]).ctypes.data_as(C.c_void_p),
                                               icpt[:nc].ctypes.data_as(C.c_void_p), nc, int(multinomial),
                                               out.ctypes.data_as(C.c_void_p), C.byref(t)) == N.LO_OK
            np.testing.assert_array_equal(out.view(np.int64), np.concatenate([[want[0]], want[1].ravel(),
                                                                               want[2]]).view(np.int64))
            got = engine.lr_predict(flat, coef[:nc], icpt[:nc], multinomial, raw=True)
            try:
                nout = got.nclasses
                raw_flat = got.raw.to_numpy(0)[:n * nout]
                prob_flat = got.prob.to_numpy(0)[:n * nout]
            finally:
                got.free()
            prob, raw, pred = (engine.table("f64", n * nout, 1), engine.table("f64", n * nout, 1),
                               engine.table("f64", n, 1))
            try:
                info, t = N.NbInfo(), N.HostTiming()
                rc = engine._lib.lo_lr_predict(engine._ctx, padded.x._h, ld, k, n,
                                               np.ascontiguousarray(coef[:nc]).ctypes.data_as(C.c_void_p),
                                               icpt[:nc].ctypes.data_as(C.c_void_p), nc, int(multinomial), 0.5,
                                               prob._h, raw._h, pred._h, None, None, 0, None, C.byref(info), C.byref(t))
                assert rc == N.LO_OK
                np.testing.assert_array_equal(raw.to_numpy(0).view(np.int64), raw_flat.view(np.int64))
                np.testing.assert_array_equal(prob.to_numpy(0).view(np.int64), prob_flat.view(np.int64))
            finally:
                _free([prob, raw, pred])
    finally:
        _free([flat, padded])


def _part_y(engine, part, y):
    """part's labels replaced by y (in place; the x table is shared)."""
    part.y.upload(0, np.asarray(y, part.y.np_dtype))
    return part


# ---- loss and gradient at the numeric edges, against mpmath --------------------------------------------------------------
def _mp_sums(margins, x, y, multinomial):
    """LogisticAggregator's sums from exact per-row terms: (loss, grad nc x k, icpt nc) and their sums of |term|."""
    nc, k = len(margins[0]), x.shape[1]
    loss, grad, icpt = mpmath.mpf(0), [[mpmath.mpf(0)] * k for _ in range(nc)], [mpmath.mpf(0)] * nc
    aloss, agrad, aicpt = mpmath.mpf(0), [[mpmath.mpf(0)] * k for _ in range(nc)], [mpmath.mpf(0)] * nc
    for m, xr, lab in zip(margins, x, y):
        m = [mpmath.mpf(float(v)) for v in m]
        if not multinomial:
            p1 = 1 / (1 + mpmath.exp(-m[0]))
            mult = [p1 - lab]
            term = mpmath.log1p(mpmath.exp(-m[0])) if lab > 0 else mpmath.log1p(mpmath.exp(m[0]))
        else:
            top = max(m)
            z = mpmath.fsum(mpmath.exp(v - top) for v in m)
            mult = [mpmath.exp(v - top) / z - (1 if c == lab else 0) for c, v in enumerate(m)]
            term = top + mpmath.log(z) - m[int(lab)]
        loss, aloss = loss + term, aloss + abs(term)
        for c in range(nc):
            icpt[c], aicpt[c] = icpt[c] + mult[c], aicpt[c] + abs(mult[c])
            for j in range(k):
                grad[c][j] += mult[c] * float(xr[j])
                agrad[c][j] += abs(mult[c] * float(xr[j]))
    f = lambda a: np.array([[float(v) for v in r] for r in a])
    return (float(loss), f(grad), np.array([float(v) for v in icpt])), (float(aloss), f(agrad),
                                                                        np.array([float(v) for v in aicpt]))


def _check_against_mp(engine, x, y, coef, icpt, multinomial, margins):
    part = _part(engine, x, y)
    try:
        loss, g, gb = engine.lr_loss_grad(part, coef, icpt, multinomial)
    finally:
        part.free()
    (el, eg, eb), (al, ag, ab) = _mp_sums(margins, x, y, multinomial)
    assert np.isfinite(loss) and np.isfinite(g).all() and np.isfinite(gb).all()
    # The sums' own error (1e-12 of the sum of |terms|) plus each term's rounding in Spark's double formulas: a
    # multiplier p - [y == c] with p in [0, 1] is off by at most an ulp of 1 (p rounds to 1, or exp flushes to 0), a
    # loss by a few ulps of its margin (log1pExp(m) - m cancels).
    eps = 2.0 ** -52
    ax = np.abs(x).sum(0)
    assert abs(loss - el) <= 1e-12 * al + 4 * eps * (np.abs(margins).max(1).sum() + len(y)), (loss, el)
    assert np.all(np.abs(g - eg) <= 1e-12 * ag + eps * ax[None, :]), (g, eg)
    assert np.all(np.abs(gb - eb) <= 1e-12 * ab + eps * len(y)), (gb, eb)
    return loss


BINOMIAL_MARGINS = [0.0, 1e-300, -1e-300, 36.8, -36.8, 709.8, -709.8, 745.2, -745.2, 1e4, -1e4, 2.5, -0.75]


def test_binomial_loss_grad_edges_against_mpmath(engine):
    """k = 1, coefficient 1, intercept 0: each row's margin is its feature, exactly.  Both labels at every margin, then
    only the rows whose loss is tiny (label 1, margin >= 36.8), where a cancellation or a flushed term would show."""
    m = np.array(BINOMIAL_MARGINS * 2)
    y = np.repeat([0.0, 1.0], len(BINOMIAL_MARGINS))
    x = m[:, None]
    _check_against_mp(engine, x, y, np.ones((1, 1)), np.zeros(1), False, m[:, None])
    small = np.array([36.8, 709.8, 745.2, 1e4, 40.0])
    loss = _check_against_mp(engine, small[:, None], np.ones(len(small)), np.ones((1, 1)), np.zeros(1), False,
                             small[:, None])
    assert 0.0 < loss < 1e-15


def _identity_model(nc):
    return np.eye(nc), np.zeros(nc)


def test_multinomial_loss_grad_edges_against_mpmath(engine):
    """k = C, coefficients the identity, intercepts 0: each row's margins are its features, exactly.  A max > 0 and
    large (shifted), a max <= 0 (not shifted), empty classes (labels {0, 5} of 6), label -0.0 as class 0."""
    rows = [[1000.0, 999.0, -5.0, 0.0, 3.0, 1000.0], [-1.0, -2.0, -3.0, -0.5, -7.0, -1.0],
            [-700.0, -701.0, -702.0, -703.0, -704.0, -700.5], [0.0, 0.0, 0.0, 0.0, 0.0, 0.0],
            [2.0, -2.0, 40.0, -40.0, 1e-300, 0.5], [-0.0, 1.0, 2.0, 3.0, 4.0, 5.0]]
    x = np.array(rows * 2)
    y = np.array([0.0] * len(rows) + [5.0] * len(rows))
    y[0] = -0.0
    coef, icpt = _identity_model(6)
    _check_against_mp(engine, x, y, coef, icpt, True, x)


def test_multinomial_loss_grad_label_1023(engine):
    """1024 classes over one column of ones: the margins are the coefficients, the labels 0, 1023 and one between."""
    rng = np.random.default_rng(5)
    margins = rng.normal(size=1024) * 30.0
    margins[1023] = 800.0
    y = np.array([0.0, 1023.0, 512.0, 1023.0])
    x = np.ones((4, 1))
    _check_against_mp(engine, x, y, margins[:, None], np.zeros(1024), True, np.tile(margins, (4, 1)))


# ---- predict epilogues against mpmath --------------------------------------------------------------------------------
def _predict(engine, x, coef, icpt, multinomial, threshold=0.5):
    part = _part(engine, x, np.zeros(len(x)))
    try:
        got = engine.lr_predict(part, coef, icpt, multinomial, threshold)
        try:
            n, nout = len(x), got.nclasses
            return got.prob.to_numpy(0)[:n * nout].reshape(n, nout), got.pred.to_numpy(0)[:n]
        finally:
            got.free()
    finally:
        part.free()


def test_binomial_predict_edges_against_mpmath(engine):
    """p1 within 4 ulp of the exact sigmoid where that is a normal double (below, within the least normal: Spark's
    1 / (1 + exp(-m)) flushes once exp overflows), p0 = 1 - p1 exactly; thresholds 0 and 1 compare exactly."""
    m = np.array(BINOMIAL_MARGINS)
    exact = np.array([float(1 / (1 + mpmath.exp(-mpmath.mpf(v)))) for v in m])
    for threshold in (0.5, 0.0, 1.0):
        prob, pred = _predict(engine, m[:, None], np.ones((1, 1)), np.zeros(1), False, threshold)
        normal = exact >= np.finfo(np.float64).tiny
        assert np.all(_ulps(prob[normal, 1], exact[normal]) <= 4), (prob[:, 1], exact)
        assert np.all(np.abs(prob[~normal, 1] - exact[~normal]) <= np.finfo(np.float64).tiny)
        np.testing.assert_array_equal(prob[:, 0], 1.0 - prob[:, 1])
        np.testing.assert_array_equal(pred, (prob[:, 1] > threshold).astype(np.float64))
    _prob, pred = _predict(engine, m[:, None], np.ones((1, 1)), np.zeros(1), False, 1.0)
    assert not pred.any()                                   # p1 never exceeds 1
    prob, pred = _predict(engine, m[:, None], np.ones((1, 1)), np.zeros(1), False, 0.0)
    np.testing.assert_array_equal(pred, (prob[:, 1] > 0.0).astype(np.float64))
    assert pred[m == -1e4].tolist() == [0.0] and pred[m == 1e4].tolist() == [1.0]


def test_multinomial_predict_edges_against_mpmath(engine):
    """Softmax within 4 ulp of mpmath; a row whose max is <= 0 and every value below -745 has sum 0: NaN probabilities
    and prediction 0, as the restated rule gives; ties go to the first index."""
    rows = np.array([[1000.0, 999.0, -5.0], [-1.0, -2.0, -3.0], [-800.0, -900.0, -1000.0], [2.0, 2.0, 1.0],
                     [1.0, 3.0, 3.0], [0.0, -0.0, 0.0], [40.0, -40.0, 1e-300]])
    coef, icpt = _identity_model(3)
    prob, pred = _predict(engine, rows, coef, icpt, True)
    for r, row in enumerate(rows):
        if r == 2:
            assert np.isnan(prob[r]).all() and pred[r] == 0.0
            continue
        mp = [mpmath.mpf(float(v)) for v in row]
        z = mpmath.fsum(mpmath.exp(v - max(mp)) for v in mp)
        exact = np.array([float(mpmath.exp(v - max(mp)) / z) for v in mp])
        assert np.all(_ulps(prob[r], exact) <= 4), (r, prob[r], exact)
    assert pred.tolist() == [0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0]


# ---- end to end: a constant 0.1 column in float64 features ---------------------------------------------------------------
@pytest.mark.parametrize("cuts", [1, 2, 3])
def test_fit_with_a_constant_column_is_the_fit_without_it(engine, cuts):
    lm = pytest.importorskip("sklearn.linear_model")
    rng = np.random.default_rng(17)
    n = 5_000
    x2 = rng.normal(size=(n, 2)) * [1.5, 0.7] + [0.3, -1.0]
    y = (x2 @ [1.0, 0.5] + rng.logistic(size=n) > 0).astype(np.float64)
    x3 = np.stack([x2[:, 0], np.full(n, 0.1), x2[:, 1]], 1)
    with_c, without = _cut(engine, x3, y, cuts), _cut(engine, x2, y, cuts)
    try:
        eng = engine if cuts == 1 else _sharded(engine, cuts)
        m3 = LogisticRegression(tol=1e-10).fit(_features(eng, with_c, 3))
        m2 = LogisticRegression(tol=1e-10).fit(_features(eng, without, 2))
    finally:
        _free(with_c + without)
    assert m3.coefficients[1] == 0.0 and m3.iterations > 0
    np.testing.assert_allclose(m3.objective_history, m2.objective_history, rtol=1e-12)
    np.testing.assert_allclose(m3.coefficients[[0, 2]], m2.coefficients, rtol=1e-9)
    sk = lm.LogisticRegression(C=np.inf, tol=1e-12, max_iter=10000).fit(x2, y)
    n_, total, m2s, _c = lo.stats(x2, y)
    best = _sk_objective(x2, y, standardization(n_, total, m2s), sk.coef_, sk.intercept_, 1, 0.0, False)
    assert abs(m3.objective_history[-1] - best) <= 1e-7 * abs(best)
