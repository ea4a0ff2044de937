"""GPU: the builder's "GB" classifier (Spark 2.4's GBTClassifier) over the feature matrix in HBM against the numpy
restatement in tests/gbt_oracle.py — every level's exact residual sums on every launch route, each tree node for node
from the device's own residuals, the residual and margin chain, transform and evaluate, bit-identical models over
shard cuts, the edges and the refused cells."""
import numpy as np
import pytest

import gbt_oracle as go
import tree_oracle as to
from learningorchestra_b200 import _native as N
from learningorchestra_b200 import tree as T
from learningorchestra_b200.classifier import GBTClassifier
from learningorchestra_b200.engine import InvalidCellError
from test_gpu_naive_bayes import _free, _host
from test_gpu_tree import _on

pytestmark = pytest.mark.gpu


def _data(n, k, seed, dtype=np.float64):
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(n, k)) * rng.uniform(0.5, 3.0, k)
    w = rng.normal(size=k)
    y = ((x.astype(dtype).astype(np.float64) @ w + rng.logistic(size=n)) > 0).astype(np.float64)
    return x.astype(dtype), y


def _arrays(tree):
    return dict(feature=tree.feature, threshold=tree.threshold, left=tree.left, right=tree.right, stats=tree.counts,
                prediction=tree.prediction, impurity=tree.impurity, gain=tree.gain)


def _same(tree, want):
    """Node for node and bit for bit."""
    got = _arrays(tree)
    for key in ("feature", "left", "right"):
        assert got[key].tolist() == want[key].tolist(), key
    for key in ("threshold", "stats", "prediction", "impurity", "gain"):
        np.testing.assert_array_equal(np.asarray(got[key], np.float64).view(np.int64),
                                      np.asarray(want[key], np.float64).reshape(np.shape(got[key])).view(np.int64), key)


def _words(codes, slot, r, nnodes, nbins):
    """lo_gb_level's words from the residuals, with Python ints."""
    q1, q2 = go.quantise(r)
    n, k = codes.shape
    out = np.zeros((nnodes, k, nbins, T.WORDS), np.uint64)
    live = slot >= 0
    for j in range(k):
        g = (slot[live] * nbins + codes[live, j])
        cnt = np.bincount(g, minlength=nnodes * nbins)
        s1 = go.exact_sum(q1[live] + (1 << 60), g, nnodes * nbins)
        s2 = go.exact_sum(q2[live], g, nnodes * nbins)
        for c in range(nnodes * nbins):
            a, b = divmod(c, nbins)
            out[a, j, b] = [cnt[c], s1[c] & (2 ** 64 - 1), s1[c] >> 64, s2[c] & (2 ** 64 - 1), s2[c] >> 64]
    return out


def _chain(engine, x, y, cuts, max_iter, max_depth=5, max_bins=32, level_check=None):
    """The fit step by step through the engine: after every tree the device's residuals and margins are read back, the
    next tree is compared with the oracle's tree on those residuals, and the residuals with numpy's formula."""
    feats, parts = _on(engine, x, y, cuts)
    eng = feats._frame._cache.engine
    rows_of = parts if cuts > 1 else parts[0]
    thr = [to.splits(x[:, j], max_bins) for j in range(x.shape[1])]
    codes = to.bins(x, thr)
    nbins = max(len(t) for t in thr) + 1
    shapes = []
    try:
        state = eng.gb_update(rows_of)
        binned = eng.dt_bin(rows_of, thr)
        try:
            members = state if cuts > 1 else [state]
            for m in range(max_iter):
                r = np.concatenate([s.residual.to_numpy(0)[:p.nkept] for s, p in zip(members, parts)])
                slot = {}

                def level(splits, nnodes):
                    sh = []
                    words = eng.gb_level(rows_of, binned, state, nbins, splits, nnodes, sh)
                    shapes.append(tuple(sh))
                    if level_check:
                        if splits is None:
                            s = np.zeros(len(y), np.int64)
                        else:
                            p = slot["s"]
                            sp = splits[np.maximum(p, 0)]
                            f = np.where(p >= 0, sp[:, 0], -1)
                            c = codes[np.arange(len(y)), np.maximum(f, 0)]
                            s = np.where(f >= 0, np.where(c <= sp[:, 1], sp[:, 2], sp[:, 3]), -1)
                        slot["s"] = s
                        np.testing.assert_array_equal(words, _words(codes, s, r, nnodes, nbins))
                    return words

                tree, _ = T.grow(level, thr, 0, max_depth, T.VARIANCE, 1, 0.0)
                _same(tree, go.arrays(go.regression_tree(codes, thr, r, max_depth)))
                w = 1.0 if m == 0 else 0.1
                F0 = np.concatenate([s.margin.to_numpy(0)[:p.nkept] for s, p in zip(members, parts)]) if m else 0.0
                eng.gb_update(rows_of, state, tree, w)
                F = np.concatenate([s.margin.to_numpy(0)[:p.nkept] for s, p in zip(members, parts)])
                np.testing.assert_array_equal(F, F0 + tree.prediction[_leaf(tree, x)] * w)
                r2 = np.concatenate([s.residual.to_numpy(0)[:p.nkept] for s, p in zip(members, parts)])
                want = go.residual(y, F)
                ulp = np.abs(np.spacing(want))
                assert np.all(np.abs(r2 - want) <= 2 * ulp)
        finally:
            for b in (binned if cuts > 1 else [binned]) + (state if cuts > 1 else [state]):
                b.free()
    finally:
        _free(parts)
    return shapes


def _leaf(tree, x):
    x = np.asarray(x).astype(np.float64)
    node = np.zeros(len(x), np.int64)
    for _ in range(tree.num_nodes):
        f = tree.feature[node]
        go_left = x[np.arange(len(x)), np.maximum(f, 0)] <= tree.threshold[node]
        node = np.where(f >= 0, np.where(go_left, tree.left[node], tree.right[node]), node)
    return node


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("cuts", [1, 2, 3, 8])
def test_each_tree_from_the_devices_residuals(engine, dtype, cuts):
    x, y = _data(4001, 4, seed=cuts, dtype=dtype)
    x[:, 2] = np.round(x[:, 2])
    _chain(engine, x, y, cuts, 4, level_check=True)


def test_level_words_on_every_route(engine):
    routes = set()
    cases = [(_data(20_000, 6, seed=1), 32, 1, 6),                    # 16-byte loads, node groups
             (_data(3_000, 300, seed=2, dtype=np.float32), 32, 2, 3),   # several feature chunks
             (_data(6_000, 3, seed=3), 256, 3, 4)]                      # 256 bins x 5 words: scalar loads, passes
    for (x, y), bins, cuts, depth in cases:
        for vec, fc, gn, passes in _chain(engine, x, y, cuts, 2, max_depth=depth, max_bins=bins, level_check=True):
            routes.add((vec, fc < ((x.shape[1] + 15) // 16 * 16 if vec else x.shape[1]), passes > 1))
    assert {r[0] for r in routes} == {0, 1}
    assert any(r[1] for r in routes)
    assert any(r[2] for r in routes)


def _fit_all(engine, x, y, cuts, **params):
    feats, parts = _on(engine, x, y, cuts)
    try:
        m = GBTClassifier(**params).fit(feats)
        with m.transform(feats, raw=True) as out:
            d = feats.devices[0]
            raw = np.concatenate([_host(v, d) for v in out.raw])
            prob = np.concatenate([_host(v, d) for v in out.probability])
            pred = np.concatenate([_host(v, d) for v in out.prediction])
        ev = m.evaluate(feats)
        return m, raw, prob, pred, ev
    finally:
        _free(parts)


def _model_margin(m, x):
    out = np.zeros(len(x))
    for t, w in zip(m.trees, m.tree_weights):
        out = out + t.prediction[_leaf(t, x)] * w
    return out


def _check_model(m, raw, prob, pred, ev, x, y):
    margin = _model_margin(m, x)
    np.testing.assert_array_equal(raw.view(np.int64), np.stack([-margin, margin], 1).view(np.int64))
    p0 = 1.0 / (1.0 + np.exp(2.0 * margin))
    want = np.stack([p0, 1.0 - p0], 1)
    # 2 ulp of the larger probability: exp may differ by an ulp, and 1 - p0 keeps p0's absolute error
    assert np.all(np.abs(prob - want) <= 2 * np.spacing(want.max(axis=1, keepdims=True)))
    np.testing.assert_array_equal(pred, (margin > 0).astype(np.float64))
    labels = np.unique(y)
    conf = np.zeros((len(labels), 2), np.int64)
    np.add.at(conf, (np.searchsorted(labels, y), pred.astype(np.int64)), 1)
    np.testing.assert_array_equal(ev["confusion"], conf)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_fit_matches_the_oracle_and_every_cut_gives_the_same_model(engine, dtype):
    x, y = _data(3001, 4, seed=11, dtype=dtype)
    trees, weights, thr, _chain_r = go.fit(x, y, max_iter=6)
    models = []
    for cuts in (1, 2, 3, 8):
        m, raw, prob, pred, ev = _fit_all(engine, x, y, cuts, max_iter=6)
        _check_model(m, raw, prob, pred, ev, x, y)
        models.append(m)
    m = models[0]
    for got, want in zip(m.thresholds, thr):
        np.testing.assert_array_equal(np.array(got, np.float64).view(np.int64), np.array(want, np.float64).view(np.int64))
    assert m.tree_weights.tolist() == weights and m.num_classes == 2
    _same(m.trees[0], go.arrays(trees[0]))
    for t, want in zip(m.trees[1:], trees[1:]):
        a = go.arrays(want)
        assert t.feature.tolist() == a["feature"].tolist() and t.left.tolist() == a["left"].tolist()
        assert t.right.tolist() == a["right"].tolist()
        np.testing.assert_array_equal(t.threshold.view(np.int64), a["threshold"].astype(np.float64).view(np.int64))
        np.testing.assert_allclose(t.prediction, a["prediction"], rtol=1e-12, atol=0)
    for other in models[1:]:
        for t, u in zip(m.trees, other.trees):
            _same(u, _arrays(t))
    _raw, _prob, want_pred = go.transform(trees, weights, x)
    assert (want_pred == (_model_margin(m, x) > 0)).mean() > 0.999


@pytest.mark.parametrize("case", ["all 0", "all 1", "constant columns", "n = 1", "n < max_bins", "max_depth 0",
                                  "max_iter 1", "step 1", "big forest"])
def test_edges(engine, case):
    x, y = _data(2000, 3, seed=5)
    params = dict(max_iter=3)
    if case == "all 0":
        y = np.zeros_like(y)
    elif case == "all 1":
        y = np.ones_like(y)
    elif case == "constant columns":
        x = np.full_like(x, 0.1)
    elif case == "n = 1":
        x, y = x[:1], y[:1]
    elif case == "n < max_bins":
        x, y = x[:20], y[:20]
    elif case == "max_depth 0":
        params["max_depth"] = 0
    elif case == "max_iter 1":
        params["max_iter"] = 1
    elif case == "step 1":
        params["step_size"] = 1.0
    elif case == "big forest":                          # depth 10 x 60 trees: the forest is read from global memory
        x, y = _data(6000, 3, seed=6)
        params = dict(max_iter=60, max_depth=10)
    m, raw, prob, pred, ev = _fit_all(engine, x, y, 1, **params)
    _check_model(m, raw, prob, pred, ev, x, y)
    trees, weights, _thr, _r = go.fit(x, y, max_iter=min(params["max_iter"], 3), step_size=params.get("step_size", 0.1),
                                      max_depth=params.get("max_depth", 5))
    _same(m.trees[0], go.arrays(trees[0]))
    if case == "big forest":
        assert (2 * m.total_num_nodes + 60) * 8 + (3 * m.total_num_nodes + 60) * 4 > 96 * 1024
    if case in ("constant columns", "max_depth 0"):
        assert all(t.num_nodes == 1 for t in m.trees)
    if case in ("all 0", "all 1"):                      # later trees fit one residual on every row: see DESIGN §3.6.5
        assert m.trees[0].num_nodes == 1 and m.trees[0].prediction[0] == (1.0 if case == "all 1" else -1.0)
        for t, want in zip(m.trees, trees):
            _same(t, go.arrays(want))


def test_refusals(engine):
    x, y = _data(3000, 3, seed=7)
    for bad_label, row in ((2.0, 77), (0.5, 1500)):
        y2 = y.copy()
        y2[row] = bad_label
        for cuts in (1, 3):
            feats, parts = _on(engine, x, y2, cuts)
            try:
                with pytest.raises(InvalidCellError,
                                   match=f"GBTClassifier: field 'y' of the row with _id {100 + row} is not a label 0 or 1"):
                    GBTClassifier(max_iter=2).fit(feats)
            finally:
                _free(parts)
    x2, y2 = x.copy(), y.copy()                        # the lowest refused cell over features and labels
    x2[1234, 1] = np.nan
    y2[2000] = 2.0
    for cuts in (1, 3):
        feats, parts = _on(engine, x2, y2, cuts)
        try:
            with pytest.raises(InvalidCellError, match="GBTClassifier: field 'f1' of the row with _id 1334 is NaN"):
                GBTClassifier(max_iter=2).fit(feats)
        finally:
            _free(parts)
    x2 = x.copy()
    x2[1234, 1] = np.nan
    feats, parts = _on(engine, x2, y, 2)
    try:
        with pytest.raises(InvalidCellError, match="GBTClassifier: field 'f1' of the row with _id 1334 is NaN"):
            GBTClassifier(max_iter=2).fit(feats)
    finally:
        _free(parts)
    feats, parts = _on(engine, x, y, 1)
    try:
        m = GBTClassifier(max_iter=2).fit(feats)
        feats.fields = ["a", "b", "c"]
        with pytest.raises(ValueError, match="fitted on fields"):
            m.transform(feats)
        feats.fields = ["f0", "f1", "f2"]
    finally:
        _free(parts)
    feats._parts = []
    with pytest.raises(ValueError, match="released"):
        m.transform(feats)
    with pytest.raises(ValueError, match="released"):
        GBTClassifier().fit(feats)


def test_the_c_abi_refuses_residuals_outside_the_fixed_point_range(engine):
    x, y = _data(500, 3, seed=8)
    feats, parts = _on(engine, x, y, 1)
    part = parts[0]
    try:
        thr = [to.splits(x[:, j], 8) for j in range(3)]
        state = engine.gb_update(part)
        binned = engine.dt_bin(part, thr)
        try:
            for bad in (np.nan, 4.000000000000001, -5.0):
                r = np.ones(500)
                r[321] = bad
                state.residual.upload(0, r)
                with pytest.raises(N.LoexecError, match="row 321: its residual is NaN or outside"):
                    engine.gb_level(part, binned, state, 8, None, 1)
            r[321] = -4.0
            state.residual.upload(0, r)
            engine.gb_level(part, binned, state, 8, None, 1)
        finally:
            state.free()
            binned.free()
    finally:
        _free(parts)
