"""CPU: the host side of the "LR" classifier — the header <-> ctypes mirror of lo_lr_*, the kernels in the SASS, the numpy
oracle against finite differences and scikit-learn, the host L-BFGS on test functions, and the classifier / the shards'
merge with test doubles standing in for the devices."""
import ctypes as C
import math
import re
from types import SimpleNamespace

import numpy as np
import pytest

import logistic_oracle as lo
from learningorchestra_b200 import _native, lbfgs
from learningorchestra_b200.classifier import (LogisticRegression, LogisticRegressionModel, NaiveBayes, scaled_objective,
                                               standardization, start_point, unscale)
from learningorchestra_b200.engine import ColumnStats, InvalidCellError
from learningorchestra_b200.sharding import ShardedEngine

from test_naive_bayes_cpu import _sass_with_offsets
from test_text_shards_cpu import HEADER


def test_ctypes_mirror_of_the_logistic_entry_points_matches_the_header():
    text = re.sub(r"/\*.*?\*/", "", HEADER.read_text(), flags=re.S)
    assert int(re.search(r"#define LO_ABI_VERSION (\d+)", text).group(1)) == _native.LO_ABI_VERSION == 7

    def params(name):
        return [p.strip() for p in re.search(r"\b%s\s*\(([^)]*)\)" % name, text).group(1).split(",")]

    assert params("lo_lr_stats") == ["lo_ctx *ctx", "const lo_table *x", "int64_t ld", "int32_t k", "const lo_table *y",
                                     "int64_t n", "double *sum_out", "double *m2_out", "int64_t *label_counts_out",
                                     "lo_nb_info *info", "lo_host_timing *timing"]
    assert params("lo_lr_loss_grad") == ["lo_ctx *ctx", "const lo_table *x", "int64_t ld", "int32_t k",
                                         "const lo_table *y", "int64_t n", "const double *coef", "const double *intercept",
                                         "int32_t nclasses", "int32_t multinomial", "double *out", "lo_host_timing *timing"]
    assert params("lo_lr_predict") == ["lo_ctx *ctx", "const lo_table *x", "int64_t ld", "int32_t k", "int64_t n",
                                       "const double *coef", "const double *intercept", "int32_t nclasses",
                                       "int32_t multinomial", "double threshold", "lo_table *prob", "lo_table *raw",
                                       "lo_table *pred", "const lo_table *y", "const double *eval_labels", "int32_t neval",
                                       "int64_t *confusion_out", "lo_nb_info *info", "lo_host_timing *timing"]
    P, T, I = C.c_void_p, C.POINTER(_native.HostTiming), C.POINTER(_native.NbInfo)
    assert _native.SIGNATURES["lo_lr_stats"] == (C.c_int, [P, P, C.c_int64, C.c_int32, P, C.c_int64, P, P, P, I, T])
    assert _native.SIGNATURES["lo_lr_loss_grad"] == (C.c_int, [P, P, C.c_int64, C.c_int32, P, C.c_int64, P, P, C.c_int32,
                                                               C.c_int32, P, T])
    assert _native.SIGNATURES["lo_lr_predict"] == (C.c_int, [P, P, C.c_int64, C.c_int32, C.c_int64, P, P, C.c_int32,
                                                             C.c_int32, C.c_double, P, P, P, P, P, C.c_int32, P, I, T])


def test_ctypes_mirror_of_lo_lr_stats_range_matches_the_header():
    text = re.sub(r"/\*.*?\*/", "", HEADER.read_text(), flags=re.S)
    params = [p.strip() for p in re.search(r"\blo_lr_stats_range\s*\(([^)]*)\)", text).group(1).split(",")]
    assert params == ["lo_ctx *ctx", "const lo_table *x", "int64_t ld", "int32_t k", "const lo_table *y", "int64_t n",
                      "double *sum_out", "double *m2_out", "double *min_out", "double *max_out",
                      "int64_t *label_counts_out", "lo_nb_info *info", "lo_host_timing *timing"]
    P, T, I = C.c_void_p, C.POINTER(_native.HostTiming), C.POINTER(_native.NbInfo)
    assert _native.SIGNATURES["lo_lr_stats_range"] == (C.c_int, [P, P, C.c_int64, C.c_int32, P, C.c_int64, P, P, P, P, P,
                                                                 I, T])


def test_launch_shape_mirror_matches_logistic_cuh():
    """tests/test_gpu_logistic_exact.py picks its parameter sets from a restatement of lr_stats_shape / lr_model_shape:
    its constants are csrc/logistic.cuh's, its formulas loexec.cu's, and its sets still reach every launch shape."""
    import test_gpu_logistic_exact as ex
    csrc = HEADER.parent.parent / "learningorchestra_b200" / "csrc"
    found = {name: eval(value) for name, value in
             re.findall(r"constexpr int (kLr\w+) = ([0-9 *]+);", (csrc / "logistic.cuh").read_text())}
    assert found == ex.CONSTANTS
    assert all(ex.shape_coverage().values()), ex.shape_coverage()
    cu = (csrc / "loexec.cu").read_text()
    assert "(int64_t)sh.G * kc * 8 * (bins ? 3 : 1) + (bins ? (lo::kLrHist + 1) * 4 : 0)" in cu
    assert "fixed = (int64_t)sh->G * sh->S * 8, per_row = ((int64_t)sh->ks + 1 + nc + 1) * 8" in cu
    assert "sh->cs = staged > 0 && staged >= std::min(32, bare) ? 1 : 0;" in cu


def test_logistic_kernels_in_the_sass(built):
    fns = _sass_with_offsets()
    stats = [f for f in fns if "k_lr_stats" in f]
    grad = [f for f in fns if "k_lr_loss_grad" in f]
    assert len(stats) == 4 and len(grad) == 4
    for f in stats + grad:
        assert not any(re.search(r"\b(LDL|STL)\b", t) for _o, t in fns[f]), f
    for f in grad:
        assert any(re.search(r"\bLDG\.E\.[A-Z0-9.]*128\b", t) for _o, t in fns[f]), f       # 16-byte loads
    for f in [f for f in fns if "k_nb_predict" in f]:
        # both epilogues (softmax, and the binomial [-m, m] / sigmoid) keep the raw rule out of DFMA in the kernel's
        # own code; the library's exp and division live in the out-of-line subroutines after it
        calls = [int(m.group(1), 16) for _o, t in fns[f] for m in [re.search(r"\bCALL\.REL\S*\s+(0x[0-9a-f]+)", t)] if m]
        assert len(set(calls)) >= 2, f                                 # nb_softmax, lr_sigmoid (and their callees)
        body = [t for o, t in fns[f] if o < min(calls)]
        assert not any(re.search(r"\bDFMA\b", t) for t in body), f


# ---- the oracle ------------------------------------------------------------------------------------------------------
def _data(n, k, nc, seed):
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(n, k)) * rng.uniform(0.5, 3.0, k) + rng.normal(size=k)
    w = rng.normal(size=(nc, k))
    z = x @ w.T + rng.gumbel(size=(n, nc)) * 2.0
    y = (z.argmax(1) if nc > 1 else (z[:, 0] > 0)).astype(np.float64)
    return x, y


@pytest.mark.parametrize("multinomial,nc", [(False, 1), (True, 3), (True, 2)])
def test_oracle_objective_gradient_matches_finite_differences(multinomial, nc):
    x, y = _data(300, 4, nc if multinomial else 2, seed=nc)
    n, total, m2, counts = lo.stats(x, y)
    std = standardization(n, total, m2)
    rng = np.random.default_rng(1)
    v = rng.normal(size=nc * 5) * 0.3
    for reg in (0.0, 0.1):
        f, g = lo.objective(x, y, std, v, nc, reg, multinomial)
        for i in range(len(v)):
            h = 1e-6
            e = np.zeros_like(v)
            e[i] = h
            fd = (lo.objective(x, y, std, v + e, nc, reg, multinomial)[0]
                  - lo.objective(x, y, std, v - e, nc, reg, multinomial)[0]) / (2 * h)
            assert abs(fd - g[i]) <= 1e-6 * max(1.0, abs(g[i])), (i, fd, g[i])


def test_oracle_loss_is_sklearns_log_loss():
    sk = pytest.importorskip("sklearn.metrics")
    for nc, multinomial in ((1, False), (4, True)):
        x, y = _data(500, 3, nc if multinomial else 2, seed=7)
        rng = np.random.default_rng(3)
        beta, b = rng.normal(size=(nc, 3)) * 0.3, rng.normal(size=nc) * 0.3     # no probability near sklearn's clip
        (loss, _g, _b), _abs = lo.loss_grad(x, y, beta, b, multinomial)
        m = x @ beta.T + b
        if multinomial:
            p = np.exp(m - m.max(1, keepdims=True))
            p /= p.sum(1, keepdims=True)
        else:
            p1 = 1 / (1 + np.exp(-m[:, 0]))
            p = np.stack([1 - p1, p1], 1)
        ref = sk.log_loss(y, p, labels=np.arange(p.shape[1]))
        assert abs(loss / len(y) - ref) <= 1e-12 * ref


def test_library_host_formulas_are_the_oracles():
    x, y = _data(400, 5, 3, seed=11)
    n, total, m2, counts = lo.stats(x, y)
    std = standardization(n, total, m2)
    np.testing.assert_allclose(std, x.std(0, ddof=1), rtol=1e-12)
    v = np.random.default_rng(2).normal(size=3 * 6)
    for reg in (0.0, 0.3):
        fun = scaled_objective(lambda beta, b: lo.loss_grad(x, y, beta, b, True)[0], n, std, 3, reg)
        f, g = fun(v)
        of, og = lo.objective(x, y, std, v, 3, reg, True)
        assert f == of
        np.testing.assert_array_equal(g, og)
        for multinomial in (True, False):
            nc = 3 if multinomial else 1
            c1, b1 = unscale(v[:nc * 6], std, nc, reg, multinomial)
            c2, b2 = lo.unscale(v[:nc * 6], std, nc, reg, multinomial)
            np.testing.assert_array_equal(c1, c2)
            np.testing.assert_array_equal(b1, b2)
    sp = start_point(np.array([10, 30, 0, 5]), 4, 2, True)
    raw = np.log1p([10.0, 30.0, 0.0, 5.0])
    np.testing.assert_array_equal(sp[8:], raw - raw.sum() / 4)
    assert start_point(np.array([10, 30]), 2, 2, False)[2] == math.log(3.0)


# ---- the host L-BFGS -------------------------------------------------------------------------------------------------
def _quadratic(a, c):
    return lambda v: (0.5 * float((v - c) @ a @ (v - c)), a @ (v - c))


def _rosenbrock(v):
    x, y = v
    return (1 - x) ** 2 + 100 * (y - x * x) ** 2, np.array([-2 * (1 - x) - 400 * x * (y - x * x), 200 * (y - x * x)])


def test_lbfgs_converges_on_a_quadratic_and_rosenbrock():
    rng = np.random.default_rng(0)
    q = rng.normal(size=(6, 6))
    a, c = q @ q.T + 6 * np.eye(6), rng.normal(size=6)
    res = lbfgs.minimize(_quadratic(a, c), np.zeros(6), max_iter=100, tol=1e-12)
    np.testing.assert_allclose(res.x, c, atol=1e-6)
    assert len(res.history) == res.iterations + 1 and res.history == sorted(res.history, reverse=True)
    res = lbfgs.minimize(_rosenbrock, np.array([-1.2, 1.0]), max_iter=500, tol=1e-14)
    np.testing.assert_allclose(res.x, [1.0, 1.0], atol=1e-5)


def test_lbfgs_stopping_rules():
    fun = _quadratic(np.diag([1.0, 10.0, 100.0]), np.array([1.0, -2.0, 3.0]))
    res = lbfgs.minimize(fun, np.zeros(3), max_iter=0)
    assert (res.iterations, res.reason, res.evaluations) == (0, "max_iter", 1) and len(res.history) == 1
    res = lbfgs.minimize(fun, np.zeros(3), max_iter=2, tol=1e-30)
    assert (res.iterations, res.reason) == (2, "max_iter") and len(res.history) == 3
    res = lbfgs.minimize(fun, np.array([1.0, -2.0, 3.0]), max_iter=10)         # at the optimum: gradient 0
    assert (res.iterations, res.reason) == (0, "gradient")
    # Rosenbrock's valley: two recorded values within tol |f0| of each other while the gradient is still large
    res = lbfgs.minimize(_rosenbrock, np.array([-1.2, 1.0]), max_iter=500, tol=1e-2)
    assert (res.reason, res.iterations) == ("function values", 2)
    assert abs(res.history[-1] - max(res.history[1:])) <= 1e-2 * res.history[0]


def test_lbfgs_survives_one_line_search_failure_and_stops_at_the_second():
    calls = {"n": 0}
    base = _quadratic(np.diag([1.0, 4.0]), np.array([2.0, -1.0]))

    def once(v):                  # the first trial step returns NaN slope: the search gives up, the history resets
        calls["n"] += 1
        f, g = base(v)
        return (math.nan, g) if calls["n"] in range(2, 13) else (f, g)

    res = lbfgs.minimize(once, np.zeros(2), max_iter=100, tol=1e-12)
    assert res.reason != "line search failed"
    np.testing.assert_allclose(res.x, [2.0, -1.0], atol=1e-6)
    assert res.history[1] == res.history[0]                   # the failed state repeats its value
    res = lbfgs.minimize(lambda v: (float(v @ v), -v), np.ones(2), max_iter=100)   # never a descent direction
    assert res.reason == "line search failed" and res.iterations == 0 and len(res.history) == 3


# ---- the classifier with test doubles for the devices ------------------------------------------------------------------
class _Part:
    def __init__(self, x, y):
        self.x, self.y, self.k, self.nkept = SimpleNamespace(engine=SimpleNamespace(device=0)), y, x.shape[1], len(x)
        self.hx = x

    def free(self):
        pass


class _Engine:
    """Stands in for Engine: runs the oracle on the part's host arrays."""

    def lr_stats(self, part):
        try:
            n, total, m2, counts = lo.stats(part.hx, part.y)
        except ValueError as e:
            r, c = e.args[0]
            raise InvalidCellError(r, c, "bad") from None
        out = np.zeros(_native.LO_NB_MAX_CLASSES, np.int64)
        out[:len(counts)] = counts
        return n, total, m2, out

    def lr_loss_grad(self, part, beta, b, multinomial):
        return lo.loss_grad(part.hx, part.y, beta, b, multinomial)[0]


def _feats(engine, parts, label="y"):
    n = sum(p.nkept for p in parts)
    return SimpleNamespace(_frame=SimpleNamespace(_cache=SimpleNamespace(engine=engine)), _parts=parts,
                           fields=[f"f{j}" for j in range(parts[0].k)], label=label, row_ids=np.arange(10, 10 + n),
                           devices=[0] * len(parts))


def _sharded(world):
    sh = object.__new__(ShardedEngine)
    sh._N, sh.world, sh.nlocal = _native, world, world
    sh.engines = [_Engine() for _ in range(world)]
    return sh


@pytest.mark.parametrize("nc", [2, 3])
def test_fit_through_one_engine_and_shards_agree(nc):
    x, y = _data(600, 3, nc, seed=nc)
    one = LogisticRegression(tol=1e-10).fit(_feats(_Engine(), [_Part(x, y)]))
    parts = [_Part(x[a:b], y[a:b]) for a, b in ((0, 200), (200, 201), (201, 600))]
    many = LogisticRegression(tol=1e-10).fit(_feats(_sharded(3), parts))
    assert one.is_multinomial == (nc > 2) and one.num_classes == nc
    np.testing.assert_allclose(many.coefficient_matrix, one.coefficient_matrix, rtol=1e-6, atol=1e-9)
    assert one.objective_history[0] >= one.objective_history[-1] and len(one.objective_history) == one.iterations + 1
    if nc == 2:
        assert one.coefficients.shape == (3,) and one.intercept == one.intercept_vector[0]


class _RangeEngine(_Engine):
    """Stands in for Engine with its column range: m2 exactly 0 where a part's column holds one value."""

    def lr_stats(self, part):
        n, total, m2, out = super().lr_stats(part)
        least, most = (part.hx.min(0), part.hx.max(0)) if n else (np.zeros(part.k), np.zeros(part.k))
        return ColumnStats(n, total, np.where(least == most, 0.0, m2), out, least, most)


def test_shards_give_a_column_constant_over_all_of_them_m2_exactly_zero():
    """Chan's delta between two shards' rounded means of 123.456 (300 and 700 rows) is not 0; the merged min / max zero
    it.  A column constant in each shard but not over all (123.456 then 0.2) keeps its M2, and so does a plain one; a
    part without rows does not count."""
    rng = np.random.default_rng(0)
    n = 1000
    x = np.stack([np.full(n, 123.456), np.where(np.arange(n) < 300, 123.456, 0.2), rng.normal(size=n)], 1)
    y = (rng.random(n) < 0.5).astype(np.float64)
    cuts = ((0, 0), (0, 300), (300, 1000))
    parts = [_Part(x[a:b], y[a:b]) for a, b in cuts]
    got_n, total, m2, _c = _sharded_with(_RangeEngine, len(cuts)).lr_stats(parts)
    plain = _sharded(len(cuts)).lr_stats(parts)[2]
    assert got_n == n and plain[0] != 0.0                           # the bug the merged range fixes
    assert m2[0] == 0.0
    np.testing.assert_array_equal(m2[1:], plain[1:])
    assert abs(m2[1] - 300 * 700 / 1000 * (123.456 - 0.2) ** 2) <= 1e-12 * m2[1]


def _sharded_with(engine_cls, world):
    sh = _sharded(world)
    sh.engines = [engine_cls() for _ in range(world)]
    return sh


def test_edges_constant_label_zero_std_and_max_iter_zero():
    x, y = _data(200, 3, 2, seed=4)
    m = LogisticRegression().fit(_feats(_Engine(), [_Part(x, np.ones(200))]))
    assert m.intercept == np.inf and not m.coefficients.any() and m.objective_history == []
    m = LogisticRegression().fit(_feats(_Engine(), [_Part(x, np.zeros(200))]))
    assert m.intercept == -np.inf and m.num_classes == 1
    m = LogisticRegression(family="multinomial").fit(_feats(_Engine(), [_Part(x, np.full(200, 2.0))]))
    np.testing.assert_array_equal(m.intercept_vector, [0.0, 0.0, np.inf])
    x0 = x.copy()
    x0[:, 1] = 7.0
    m = LogisticRegression().fit(_feats(_Engine(), [_Part(x0, y)]))
    assert m.coefficients[1] == 0.0 and m.iterations > 0
    m = LogisticRegression(max_iter=0).fit(_feats(_Engine(), [_Part(x, y)]))
    assert m.iterations == 0 and len(m.objective_history) == 1 and not m.coefficients.any()
    assert m.intercept == math.log((y == 1).sum() / (y == 0).sum())


def test_refused_cells_name_the_global_row_id_and_field():
    x, y = np.ones((30, 3)), np.zeros(30)
    y[::2] = 1.0
    x[25, 2] = np.inf
    x[12, 1] = np.nan
    with pytest.raises(InvalidCellError) as e:
        LogisticRegression().fit(_feats(_sharded(2), [_Part(x[:20], y[:20]), _Part(x[20:], y[20:])]))
    assert e.value.message == "LogisticRegression: field 'f1' of the row with _id 22 is NaN or infinite"
    x[12, 1] = 1.0
    y[21] = 0.5
    with pytest.raises(InvalidCellError) as e:
        LogisticRegression().fit(_feats(_sharded(2), [_Part(x[:20], y[:20]), _Part(x[20:], y[20:])]))
    assert e.value.message == "LogisticRegression: field 'y' of the row with _id 31 is not an integer label >= 0"


def test_refusals_and_naive_bayes_messages_unchanged():
    for kw in ({"max_iter": -1}, {"max_iter": 1.5}, {"reg_param": -0.1}, {"reg_param": math.inf}, {"tol": 0.0},
               {"tol": math.nan}, {"family": "poisson"}, {"threshold": 1.5}):
        with pytest.raises(ValueError):
            LogisticRegression(**kw)
    LogisticRegression(max_iter=0, reg_param=0.0, family="multinomial", threshold=1.0)
    x, y = np.ones((6, 2)), np.array([0.0, 1.0, 2.0, 0.0, 1.0, 2.0])
    x[:, 0] = np.arange(6)
    with pytest.raises(ValueError, match="binomial"):
        LogisticRegression(family="binomial").fit(_feats(_Engine(), [_Part(x, y)]))
    with pytest.raises(ValueError):
        LogisticRegression().fit(_feats(_Engine(), [_Part(x, y)], label=None))
    with pytest.raises(_native.LoexecError):
        LogisticRegression().fit(_feats(_Engine(), [_Part(x[:0], y[:0])]))
    with pytest.raises(_native.LoexecError) as e:                                   # 2 x 8193 above the cap
        LogisticRegression().fit(_feats(_Engine(), [_Part(np.ones((2, 8193)), np.array([0.0, 1.0]))]))
    assert "LO_NB_MAX_THETA" in e.value.message

    class _NoPass(_Engine):
        def lr_stats(self, part):
            raise AssertionError("a pass ran")

    with pytest.raises(_native.LoexecError) as e:                                   # binomial: refused before a pass
        LogisticRegression(family="binomial").fit(_feats(_NoPass(), [_Part(np.ones((2, 8193)), np.array([0.0, 1.0]))]))
    assert "2 classes x 8193 features" in e.value.message
    rank = _sharded(2)
    rank.nlocal = 1
    for call in (lambda: rank.lr_stats([]), lambda: rank.lr_loss_grad([], [[0.0]], [0.0], False),
                 lambda: rank.lr_predict([], [[0.0]], [0.0], False)):
        with pytest.raises(_native.LoexecError) as e:
            call()
        assert "every row" in e.value.message
    released = _feats(_Engine(), [_Part(x, y)])
    released._parts = []
    m = LogisticRegressionModel([[0.0, 0.0]], [0.0], 2, False, ["f0", "f1"])
    for call in (lambda: LogisticRegression().fit(released), lambda: m.transform(released), lambda: m.evaluate(released)):
        with pytest.raises(ValueError, match="released"):
            call()

    class _NbEngine:                                                                # NaiveBayes' words stay
        def nb_labels(self, part):
            return np.array([0.0])

        def nb_fit(self, part, classes):
            raise InvalidCellError(1, 0, "bad")

    with pytest.raises(InvalidCellError) as e:
        NaiveBayes().fit(_feats(_NbEngine(), [_Part(x, y)]))
    assert e.value.message == "NaiveBayes: field 'f0' of the row with _id 11 is negative or NaN"
    with pytest.raises(ValueError, match="^NaiveBayes needs features with a label$"):
        NaiveBayes().fit(_feats(_NbEngine(), [_Part(x, y)], label=None))
