"""GPU: the builder's "LR" classifier (Spark 2.4's LogisticRegression) over the feature matrix in HBM against the numpy
restatement in tests/logistic_oracle.py and scikit-learn — the statistics and one loss / gradient pass within 1e-12 of
the sum of |terms| (exact where the sums are), the same bits on every run, fits at scikit-learn's optimum and along the
host optimizer fed by the oracle, the edges, transform and evaluate, refused cells on one GPU and on shards, the caps,
sharded fits, and a Titanic CSV end to end."""
import csv
import json
import math
from pathlib import Path

import numpy as np
import pytest
from werkzeug.test import Client

import logistic_oracle as lo
from learningorchestra_b200 import _native as N
from learningorchestra_b200 import builder_frontend, lbfgs, server
from learningorchestra_b200.classifier import (LogisticRegression, LogisticRegressionModel, metrics, standardization,
                                               start_point)
from learningorchestra_b200.column_store import ColumnarDatabase
from learningorchestra_b200.engine import InvalidCellError
from learningorchestra_b200.sharding import ShardedEngine
from oracle import naive_bayes as nb
from test_gpu_naive_bayes import _features, _free, _host, _part, _ulps

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).resolve().parent / "golden"


def _data(n, k, nc, seed, dtype=np.float64, integer=False):
    """Well-conditioned, non-separable rows: labels drawn from a softmax of a random linear model."""
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(n, k)) * rng.uniform(0.5, 2.0, k) + rng.normal(size=k)
    if integer:
        x = np.round(x * 4)
    x = x.astype(dtype).astype(np.float64)
    w = rng.normal(size=(max(nc, 2), k)) * 0.5
    z = x @ w.T + rng.gumbel(size=(n, max(nc, 2)))
    return x.astype(dtype), z.argmax(1).astype(np.float64)


def _sharded(engine, cuts):
    sh = object.__new__(ShardedEngine)                 # every cut on this device, one host thread each
    sh._N, sh.world, sh.nlocal, sh.engines = N, cuts, cuts, [engine] * cuts
    return sh


def _cut(engine, x, y, cuts):
    bounds = np.linspace(0, len(y), cuts + 1).astype(int)
    return [_part(engine, x[a:b], y[a:b]) for a, b in zip(bounds[:-1], bounds[1:])]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("multinomial", [False, True])
@pytest.mark.parametrize("k", [1, 33, 512])
def test_stats_and_one_pass_match_the_oracle(engine, dtype, multinomial, k):
    n = 20_011 if k < 512 else 5_003                    # no multiple of a tile, a CTA's rows or a window
    nc = 3 if multinomial else 1
    for integer in (True, False):
        x, y = _data(n, k, 3 if multinomial else 2, seed=k + integer, dtype=dtype, integer=integer)
        part = _part(engine, x, y)
        try:
            xn, total, m2, counts = engine.lr_stats(part)
            on, ototal, om2, ocounts = lo.stats(x, y)
            assert xn == on
            np.testing.assert_array_equal(counts[:len(ocounts)], ocounts)
            assert not counts[len(ocounts):].any()
            if integer:
                np.testing.assert_array_equal(total, ototal)
            else:
                assert np.all(np.abs(total - ototal) <= 1e-12 * np.abs(x).sum(0))
            assert np.all(np.abs(m2 - om2) <= 1e-12 * om2 + 1e-300)
            rng = np.random.default_rng(k)
            beta, b = rng.normal(size=(nc, k)) / math.sqrt(k), rng.normal(size=nc)
            loss, g, gb = engine.lr_loss_grad(part, beta, b, multinomial)
            (oloss, og, ogb), (aloss, ag, agb) = lo.loss_grad(x, y, beta, b, multinomial)
            assert abs(loss - oloss) <= 1e-12 * aloss
            assert np.all(np.abs(g - og) <= 1e-12 * ag)
            assert np.all(np.abs(gb - ogb) <= 1e-12 * agb)
            again = engine.lr_loss_grad(part, beta, b, multinomial)
            assert again[0] == loss
            np.testing.assert_array_equal(again[1].view(np.int64), g.view(np.int64))
            np.testing.assert_array_equal(again[2].view(np.int64), gb.view(np.int64))
            assert engine.lr_stats(part)[2].tobytes() == m2.tobytes()
        finally:
            part.free()


def _sk_objective(x, y, std, coef, icpt, nc, reg, multinomial):
    """Spark's objective at an unscaled model (coef nc x k, icpt nc), through the oracle."""
    v = np.concatenate([(coef * std).ravel(), icpt])
    return lo.objective(x, y, std, v, nc, reg, multinomial)[0]


@pytest.mark.parametrize("nclasses", [2, 3])
@pytest.mark.parametrize("reg", [0.0, 0.01])
def test_fit_reaches_sklearns_optimum(engine, nclasses, reg):
    lm = pytest.importorskip("sklearn.linear_model")
    x, y = _data(20_000, 5, nclasses, seed=nclasses + int(reg * 100))
    part = _part(engine, x, y)
    try:
        feats = _features(engine, [part], 5)
        n, total, m2, _c = lo.stats(x, y)
        std = standardization(n, total, m2)
        multinomial = nclasses > 2
        nc = nclasses if multinomial else 1
        if reg == 0.0:
            sk = lm.LogisticRegression(C=np.inf, tol=1e-12, max_iter=10000).fit(x, y)
            coef, icpt = sk.coef_, sk.intercept_
        else:
            sk = lm.LogisticRegression(C=1.0 / (len(y) * reg), l1_ratio=0, tol=1e-12, max_iter=10000).fit(x / std, y)
            coef, icpt = sk.coef_ / std, sk.intercept_
        best = _sk_objective(x, y, std, coef, icpt, nc, reg, multinomial)
        m = LogisticRegression(reg_param=reg).fit(feats)
        assert m.is_multinomial == multinomial and m.num_classes == nclasses
        assert abs(m.objective_history[-1] - best) <= 1e-7 * abs(best)
        tight = LogisticRegression(reg_param=reg, tol=1e-10, max_iter=1000).fit(feats)
        np.testing.assert_allclose(tight.coefficient_matrix, coef, rtol=1e-4, atol=1e-4 * np.abs(coef).max())
        np.testing.assert_allclose(tight.intercept_vector, icpt - (icpt.mean() if multinomial else 0.0), rtol=1e-4,
                                   atol=1e-4 * np.abs(icpt).max())
    finally:
        part.free()


@pytest.mark.parametrize("nclasses,dtype", [(2, np.float32), (4, np.float64)])
def test_fit_follows_the_host_optimizer_fed_by_the_oracle(engine, nclasses, dtype):
    x, y = _data(8_000, 6, nclasses, seed=21, dtype=dtype)
    part = _part(engine, x, y)
    try:
        m = LogisticRegression(max_iter=10).fit(_features(engine, [part], 6))
        n, total, m2, counts = lo.stats(x, y)
        std = standardization(n, total, m2)
        multinomial = nclasses > 2
        nc = nclasses if multinomial else 1
        ref = lbfgs.minimize(lambda v: lo.objective(x.astype(np.float64), y, std, v, nc, 0.0, multinomial),
                             start_point(np.bincount(y.astype(int)), nclasses, 6, multinomial), 10, 1e-6)
        assert len(m.objective_history) == len(ref.history)
        np.testing.assert_allclose(m.objective_history, ref.history, rtol=1e-10)
    finally:
        part.free()


def test_edges_constant_label_zero_std_and_max_iter_zero(engine):
    x, y = _data(5_000, 4, 2, seed=5)
    for label, want in ((1.0, np.inf), (0.0, -np.inf)):
        part = _part(engine, x, np.full(len(y), label))
        try:
            m = LogisticRegression().fit(_features(engine, [part], 4))
            assert m.intercept == want and not m.coefficients.any() and m.objective_history == []
        finally:
            part.free()
    x0 = x.copy()
    x0[:, 2] = 3.25
    part = _part(engine, x0, y)
    try:
        m = LogisticRegression().fit(_features(engine, [part], 4))
        assert m.coefficients[2] == 0.0 and m.coefficients[[0, 1, 3]].all()
        z = LogisticRegression(max_iter=0).fit(_features(engine, [part], 4))
        assert z.iterations == 0 and len(z.objective_history) == 1 and not z.coefficients.any()
        assert z.intercept == math.log((y == 1).sum() / (y == 0).sum())
        assert z.objective_history[0] == m.objective_history[0]
    finally:
        part.free()


@pytest.mark.parametrize("nclasses,dtype", [(2, np.float32), (2, np.float64), (5, np.float32), (5, np.float64)])
def test_transform_and_evaluate_match_the_oracle(engine, nclasses, dtype):
    x, y = _data(30_001, 7, nclasses, seed=nclasses, dtype=dtype)
    part = _part(engine, x, y)
    try:
        feats = _features(engine, [part], 7)
        m = LogisticRegression(threshold=0.4).fit(feats)
        xd = x.astype(np.float64)
        if nclasses == 2:
            r = lo.binomial_raw(xd, m.coefficients, m.intercept)
            p = lo.binomial_probability(r)
            pred = lo.binomial_prediction(p, 0.4)
            away = np.abs(p[:, 1] - 0.4) > 1e-12
        else:
            r = nb.raw(xd, m.intercept_vector, m.coefficient_matrix)
            p = lo.multinomial_probability(r)
            pred = nb.prediction(p)
            top2 = np.sort(p, axis=1)[:, -2:]
            away = _ulps(top2[:, 1], top2[:, 0]) > 4
        with m.transform(feats, raw=True) as out:
            np.testing.assert_array_equal(_host(out.raw[0], 0).view(np.int64), r.view(np.int64))
            prob = _host(out.probability[0], 0)
            if nclasses == 2:       # p1 within 4 ulp; p0 is 1 - p1 (its ulps scale with p1's, not its own)
                assert np.all(_ulps(prob[:, 1], p[:, 1]) <= 4)
                np.testing.assert_array_equal(prob[:, 0], 1.0 - prob[:, 1])
            else:
                assert np.all(_ulps(prob, p) <= 4)
            got = _host(out.prediction[0], 0)
            np.testing.assert_array_equal(got[away], pred[away])
        ev = m.evaluate(feats)
        labels = nb.classes_of(y)
        assert away.all()                                   # no tie in this data, so the counts are exact
        np.testing.assert_array_equal(ev["confusion"], nb.confusion(y, pred, labels, nclasses))
        f1, acc = metrics(labels, nb.confusion(y, pred, labels, nclasses))
        assert (ev["f1"], ev["accuracy"]) == (f1, acc)
    finally:
        part.free()


@pytest.mark.parametrize("family,label,nclasses", [("multinomial", 2.0, 3), ("multinomial", 1.0, 2),
                                                   ("multinomial", 0.0, 1), ("auto", 1.0, 2), ("auto", 0.0, 1)])
def test_constant_label_model_predicts_its_class(engine, family, label, nclasses):
    """Spark's constant-label model (an infinite intercept) applied: a one-hot probability on that class (multinomial),
    p1 = 1 or 0 (binomial), every row predicted as its label, accuracy 1."""
    x, _y = _data(3_001, 3, 2, seed=9, dtype=np.float32)
    y = np.full(len(x), label)
    part = _part(engine, x, y)
    try:
        feats = _features(engine, [part], 3)
        m = LogisticRegression(family=family).fit(feats)
        assert m.num_classes == nclasses
        want = np.zeros((len(y), 2 if not m.is_multinomial else nclasses))
        want[:, int(label) if m.is_multinomial else int(label == 1.0)] = 1.0
        with m.transform(feats, raw=True) as out:
            np.testing.assert_array_equal(_host(out.probability[0], 0), want)
            np.testing.assert_array_equal(_host(out.prediction[0], 0), y)
            if m.is_multinomial:
                np.testing.assert_array_equal(_host(out.raw[0], 0), nb.raw(x.astype(np.float64), m.intercept_vector,
                                                                            m.coefficient_matrix))
        ev = m.evaluate(feats)
        assert ev["accuracy"] == 1.0 and ev["f1"] == 1.0
        assert ev["confusion"][0, int(label) if m.is_multinomial else int(label == 1.0)] == len(y)
    finally:
        part.free()


def test_loss_grad_over_several_windows_is_the_windows_added(engine):
    """More rows than one window of partials (256 MiB of them at 1024 x 16: 1927 CTAs of 2048 rows): the pass over all
    rows equals, bit for bit, the two windows' sums (each a call of its own) added by the tree, and the oracle."""
    wrows = (256 << 20) // ((1 + 1024 * 17) * 8) * 2048
    n = wrows + 50_001
    rng = np.random.default_rng(3)
    x = rng.normal(size=(n, 16)).astype(np.float32)
    y = rng.integers(0, 1024, n).astype(np.float64)
    coef, icpt = rng.normal(size=(1024, 16)) * 0.1, rng.normal(size=1024) * 0.1
    parts = [_part(engine, x, y), _part(engine, x[:wrows], y[:wrows]), _part(engine, x[wrows:], y[wrows:])]
    try:
        whole, first, second = (engine.lr_loss_grad(p, coef, icpt, True) for p in parts)
        assert whole[0] == first[0] + second[0]
        np.testing.assert_array_equal(whole[1], first[1] + second[1])
        np.testing.assert_array_equal(whole[2], first[2] + second[2])
        g, ag, losses = np.zeros((1024, 16)), np.zeros((1024, 16)), []
        for a in range(0, n, 200_000):                      # the oracle's terms in chunks: n x 1024 at once is 32 GB
            loss, mult = lo.row_terms(x[a:a + 200_000], y[a:a + 200_000], coef, icpt, True)
            xd = x[a:a + 200_000].astype(np.float64)
            g, ag, losses = g + mult.T @ xd, ag + np.abs(mult).T @ np.abs(xd), losses + [loss]
        assert np.all(np.abs(whole[1] - g) <= 1e-10 * ag)  # BLAS's sum is the less exact one here
        loss = np.concatenate(losses)
        assert abs(whole[0] - math.fsum(loss)) <= 1e-12 * math.fsum(np.abs(loss))
    finally:
        _free(parts)


@pytest.mark.parametrize("cuts", [1, 2, 3, 8])
def test_refused_cells_on_one_gpu_and_shards(engine, cuts):
    x, y = _data(12_000, 4, 2, seed=cuts)
    cases = [("feature", 7001, 2, np.nan, "'f2' of the row with _id 7101 is NaN or infinite"),
             ("feature", 9000, 0, -np.inf, "'f0' of the row with _id 9100 is NaN or infinite"),
             ("label", 5000, 4, 0.5, "'y' of the row with _id 5100 is not an integer label >= 0"),
             ("label", 11000, 4, -1.0, "'y' of the row with _id 11100 is not an integer label >= 0"),
             ("label", 3, 4, np.nan, "'y' of the row with _id 103 is not an integer label >= 0")]
    for kind, row, col, value, words in cases:
        xb, yb = x.copy(), y.copy()
        if kind == "feature":
            xb[row, col] = value
            xb[row + 500, 1] = np.inf                       # a later row does not win
        else:
            yb[row] = value
        parts = _cut(engine, xb, yb, cuts)
        try:
            eng = engine if cuts == 1 else _sharded(engine, cuts)
            with pytest.raises(InvalidCellError) as e:
                LogisticRegression().fit(_features(eng, parts, 4))
            assert (e.value.row, e.value.position) == (row, col)
            assert e.value.message == f"LogisticRegression: field {words}"
        finally:
            _free(parts)


def test_caps_at_their_boundaries(engine):
    rng = np.random.default_rng(0)
    x = rng.normal(size=(300, 8192)).astype(np.float32)
    y = (rng.random(300) < 0.5).astype(np.float64)
    part = _part(engine, x, y)                              # binomial: 2 x 8192 = LO_NB_MAX_THETA
    try:
        m = LogisticRegression(max_iter=2).fit(_features(engine, [part], 8192))
        (loss, g, gb), (aloss, ag, agb) = lo.loss_grad(x.astype(np.float64), y, m.coefficient_matrix,
                                                        m.intercept_vector, False)
        got = engine.lr_loss_grad(part, m.coefficient_matrix, m.intercept_vector, False)
        assert abs(got[0] - loss) <= 1e-12 * aloss and np.all(np.abs(got[1] - g) <= 1e-12 * ag)
        with m.transform(_features(engine, [part], 8192)) as out:
            assert _host(out.probability[0], 0).shape == (300, 2)
    finally:
        part.free()
    part = _part(engine, np.ones((4, 8193), np.float32), [0.0, 1.0, 0.0, 1.0])
    try:
        with pytest.raises(N.LoexecError) as e:             # 2 x 8193
            LogisticRegression().fit(_features(engine, [part], 8193))
        assert e.value.code == N.LO_ERR_INVALID
    finally:
        part.free()
    n = 4096
    y = (np.arange(n) % 1024).astype(np.float64)
    x = rng.normal(size=(n, 16)).astype(np.float32)
    part = _part(engine, x, y)                              # multinomial: 1024 x 16
    try:
        m = LogisticRegression(max_iter=1).fit(_features(engine, [part], 16))
        assert m.coefficient_matrix.shape == (1024, 16) and np.isfinite(m.objective_history).all()
        (loss, g, gb), (aloss, ag, agb) = lo.loss_grad(x.astype(np.float64), y, m.coefficient_matrix,
                                                        m.intercept_vector, True)
        got = engine.lr_loss_grad(part, m.coefficient_matrix, m.intercept_vector, True)
        assert abs(got[0] - loss) <= 1e-12 * aloss and np.all(np.abs(got[1] - g) <= 1e-12 * ag)
    finally:
        part.free()
    part = _part(engine, np.ones((3, 2), np.float32), [0.0, 1024.0, 1.0])
    try:
        with pytest.raises(N.LoexecError) as e:             # label 1024: 1025 classes
            LogisticRegression().fit(_features(engine, [part], 2))
        assert e.value.code == N.LO_ERR_INVALID and not isinstance(e.value, InvalidCellError)
    finally:
        part.free()


@pytest.mark.parametrize("cuts", [1, 2, 3, 8])
@pytest.mark.parametrize("integer", [True, False])
def test_sharded_fits_agree_with_one_gpu(engine, cuts, integer):
    x, y = _data(40_003, 6, 3, seed=cuts, integer=integer)
    whole = _part(engine, x, y)
    pieces = _cut(engine, x, y, cuts)
    try:
        one = LogisticRegression(tol=1e-10).fit(_features(engine, [whole], 6))
        many = LogisticRegression(tol=1e-10).fit(_features(_sharded(engine, cuts), pieces, 6))
        if integer:
            np.testing.assert_allclose(many.objective_history[:5], one.objective_history[:5], rtol=1e-12)
        np.testing.assert_allclose(many.objective_history[-1], one.objective_history[-1], rtol=1e-9)
        np.testing.assert_allclose(many.coefficient_matrix, one.coefficient_matrix, rtol=1e-4,
                                   atol=1e-4 * np.abs(one.coefficient_matrix).max())
        ev1 = one.evaluate(_features(engine, [whole], 6))
        evn = many.evaluate(_features(_sharded(engine, cuts), pieces, 6))
        assert abs(ev1["accuracy"] - evn["accuracy"]) <= 2 / len(y)
    finally:
        _free([whole] + pieces)


NUMBER_FIELDS = ["PassengerId", "Survived", "Pclass", "Age", "SibSp", "Parch", "Fare"]


@pytest.mark.parametrize("sharded", [False, True])
def test_titanic_end_to_end(engine, tmp_path, sharded):
    g = json.loads((GOLD / "titanic_shaped_input.json").read_text())
    path = tmp_path / "t.csv"
    with open(path, "w", newline="") as f:
        csv.writer(f).writerows([g["headers"]] + g["rows"])
    eng = ShardedEngine.local() if sharded else engine
    try:
        eng.resident.clear()
        db = ColumnarDatabase()
        db.ingest_csv("t", str(path), engine=eng)
        c = Client(server.create_app(db, eng, synchronous=True))
        r = c.patch("/fieldTypes", json={"inputDatasetName": "t", "types": {f: "number" for f in NUMBER_FIELDS}})
        assert r.status_code == 200, r.get_data(as_text=True)
        host = builder_frontend.file_processor(db, "t")
        with builder_frontend.device_frame(db, "t", eng, text=True) as frame:
            fields = [f for f in frame.fields if f != "Survived"]
            with frame.features(fields, label="Survived", handle_invalid="skip") as feats:
                cols = {}
                for f in frame.fields:
                    if frame.kinds[f] == "text":
                        index = {s: i for i, s in enumerate(frame.dictionaries[f].to_pylist())}
                        cols[f] = np.array([-1 if v is None else index[v] for v in host.column(f).to_pylist()], np.float64)
                    else:
                        cols[f] = np.array([np.nan if v is None else v for v in host.column(f).to_pylist()], np.float64)
                stack = np.stack([cols[f] for f in fields + ["Survived"]])
                is_text = np.array([frame.kinds[f] == "text" for f in fields + ["Survived"]])[:, None]
                keep = ~np.any(np.isnan(stack) | ((stack == -1) & is_text), axis=0)       # handle_invalid="skip"
                x = np.stack([cols[f][keep] for f in feats.fields], 1).astype(np.float32).astype(np.float64)
                y = cols["Survived"][keep].astype(np.float32).astype(np.float64)
                assert x.shape[0] == len(feats.row_ids)
                m = LogisticRegression().fit(feats)
                assert not m.is_multinomial and m.num_classes == 2
                n, total, m2, counts = lo.stats(x, y)
                std = standardization(n, total, m2)
                best = _sk_objective(x, y, std, m.coefficient_matrix, m.intercept_vector, 1, 0.0, False)
                assert abs(best - m.objective_history[-1]) <= 1e-9 * best
                p = lo.binomial_probability(lo.binomial_raw(x, m.coefficients, m.intercept))
                pred = lo.binomial_prediction(p)
                with m.transform(feats) as out:
                    got = np.concatenate([_host(v, d) for v, d in zip(out.prediction, out.devices)])
                    np.testing.assert_array_equal(got, pred)
                    prob = np.concatenate([_host(v, d) for v, d in zip(out.probability, out.devices)])
                    assert np.all(_ulps(prob[:, 1], p[:, 1]) <= 4)
                    np.testing.assert_array_equal(prob[:, 0], 1.0 - prob[:, 1])
                ev = m.evaluate(feats)
                f1, acc = nb.metrics(y, pred)
                assert abs(ev["f1"] - f1) <= 1e-15 and ev["accuracy"] == acc
        eng.resident.clear()
    finally:
        if sharded:
            eng.close()


def test_the_c_abi_refuses_before_any_launch(engine):
    import ctypes as C
    lib = engine._lib
    small = _part(engine, np.ones((4, 2), np.float64), [0.0, 1.0, 0.0, 1.0])
    prob, pred = engine.table("f64", 8, 1), engine.table("f64", 4, 1)
    try:
        P = C.c_void_p
        out = np.zeros(64)
        info, t = N.NbInfo(), N.HostTiming()

        def arr(v):
            return np.ascontiguousarray(v, np.float64).ctypes.data_as(P)

        def lg(nc, multi, k=2):
            return lib.lo_lr_loss_grad(engine._ctx, small.x._h, k, k, small.y._h, 4, arr(np.zeros(nc * k)),
                                       arr(np.zeros(nc)), nc, multi, out.ctypes.data_as(P), C.byref(t))

        def pr(nc, multi, threshold=0.5):
            return lib.lo_lr_predict(engine._ctx, small.x._h, 2, 2, 4, arr(np.zeros(nc * 2)), arr(np.zeros(nc)), nc, multi,
                                     threshold, prob._h, None, pred._h, None, None, 0, None, C.byref(info), C.byref(t))

        before = engine.launch_count
        for name, call in {"binomial with 2 rows": lambda: lg(2, 0), "multinomial = 2": lambda: lg(2, 2),
                           "multinomial of one class": lambda: lg(1, 1),
                           "1025 classes": lambda: lg(1025, 1), "threshold 1.5": lambda: pr(1, 0, 1.5),
                           "threshold NaN": lambda: pr(1, 0, math.nan), "ld < k": lambda: lib.lo_lr_loss_grad(
                               engine._ctx, small.x._h, 1, 2, small.y._h, 4, arr(np.zeros(2)), arr(np.zeros(1)), 1, 0,
                               out.ctypes.data_as(P), C.byref(t))}.items():
            assert call() == N.LO_ERR_INVALID, name
        assert engine.launch_count == before
        assert lg(1, 0) == N.LO_OK and abs(out[0] - 4 * math.log(2.0)) <= 1e-15
        assert pr(1, 0) == N.LO_OK
        zero = LogisticRegressionModel([[0.0, 0.0]], [0.0], 2, False, ["f0", "f1"])
        with zero.transform(_features(engine, [small], 2)) as got:           # p1 = 0.5 is not > 0.5
            np.testing.assert_array_equal(_host(got.prediction[0], 0), np.zeros(4))
    finally:
        small.free()
        prob.free()
        pred.free()
