"""GPU: the builder's "RF" classifier (Spark 2.4's RandomForestClassifier) over the feature matrix in HBM against the
restatement in tests/rf_oracle.py — every level's weighted histogram on every launch route and tree batch, whole
forests node for node on one GPU and shard cuts, one tree against DecisionTreeClassifier, transform and evaluate bit
for bit, the edges and the refused cells."""
import numpy as np
import pytest

import rf_oracle as ro
import tree_oracle as to
from learningorchestra_b200 import _native as N
from learningorchestra_b200 import classifier as CL
from learningorchestra_b200 import tree as T
from learningorchestra_b200.classifier import DecisionTreeClassifier, RandomForestClassifier
from learningorchestra_b200.engine import InvalidCellError
from test_gpu_naive_bayes import _free, _host
from test_gpu_tree import _data, _on, _part, _same_tree

pytestmark = pytest.mark.gpu


def _levels(engine, x, y, ntrees, batch, m, nbins_cap=32, shapes=None, cuts=1):
    """Grows `ntrees` trees in batches of `batch` through rf_level, each level's histogram checked against numpy's
    weighted bincount of the rows routed on the host; returns the trees."""
    feats, parts = _on(engine, x, y, cuts)
    eng = feats._frame._cache.engine
    rows_of = parts if cuts > 1 else parts[0]
    n, k = x.shape
    C = int(y.max()) + 1
    thr = [to.splits(x[:, j], nbins_cap) for j in range(k)]
    codes = to.bins(x, thr)
    nbins = max(len(t) for t in thr) + 1
    seed = T.DEFAULT_SEED
    tab = T.draw_table(ntrees, 1.0)
    out = []
    try:
        binned = eng.dt_bin(rows_of, thr)
        try:
            for tree0 in range(0, ntrees, batch):
                nt = min(batch, ntrees - tree0)
                w = np.array([ro.weights(seed, tree0 + t, range(n), tab) for t in range(nt)])
                state = {}

                def level(splits, nnodes, fl):
                    sh = []
                    hist = eng.rf_level(rows_of, binned, nbins, C, seed, tab, tree0, nt, splits, fl, shape=sh)
                    if shapes is not None:
                        shapes.append(tuple(sh))
                    if splits is None:
                        slot = np.repeat(np.arange(nt)[:, None], n, axis=1)
                    else:
                        p = state["slot"]
                        sp = splits[np.maximum(p, 0)]
                        f = np.where(p >= 0, sp[..., 0], -1)
                        c = codes[np.arange(n)[None, :], np.maximum(f, 0)]
                        slot = np.where(f >= 0, np.where(c <= sp[..., 1], sp[..., 2], sp[..., 3]), -1)
                    state["slot"] = slot
                    want = np.zeros(hist.shape, np.int64)
                    tt, rr = np.nonzero((slot >= 0) & (w > 0))
                    s = slot[tt, rr]
                    for q in range(fl.shape[1]):
                        np.add.at(want, (s, q, codes[rr, fl[s, q]], y[rr].astype(np.int64)), w[tt, rr])
                    np.testing.assert_array_equal(hist, want)
                    return hist

                grown, _ = T.grow(level, thr, C, 4, "gini", 1, 0.0, trees=nt,
                                  subsets=lambda t, node: T.feature_subset(seed, tree0 + t, node, k, m))
                out += grown
        finally:
            _free(binned if cuts > 1 else [binned])
    finally:
        _free(parts)
    return out


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_levels_are_weighted_bincounts_on_every_route(engine, dtype):
    x, y = _data(3001, 6, 3, seed=1, dtype=dtype)
    shapes = []
    small = _levels(engine, x, y, ntrees=5, batch=3, m=3, shapes=shapes)      # two tree batches, one node group
    assert all(s[0] == 0 and s[1] == 3 and s[3] == 1 for s in shapes)   # byte loads, all 3 features, one pass
    shapes = []
    x2, y2 = _data(2003, 5, 100, seed=2, dtype=dtype)
    y2[:100] = np.arange(100)
    _levels(engine, x2, y2, ntrees=3, batch=2, m=2, nbins_cap=256, shapes=shapes)
    assert all(s[1:3] == (1, 1) for s in shapes) and max(s[3] for s in shapes) > 1  # chunks and one node per pass
    assert len(small) == 5


def _check_forest(engine, x, y, cuts=1, **params):
    feats, parts = _on(engine, x, y, cuts)
    try:
        model = RandomForestClassifier(**params).fit(feats)
        o = dict(num_trees=params.get("num_trees", 20), max_depth=params.get("max_depth", 5),
                 max_bins=params.get("max_bins", 32), min_inst=params.get("min_instances_per_node", 1),
                 kind=params.get("impurity", "gini"), rate=params.get("subsampling_rate", 1.0))
        if params.get("feature_subset_strategy", "auto") != "auto":
            o["m"] = T.subset_size(params["feature_subset_strategy"], x.shape[1], o["num_trees"])
        trees, thr, m = ro.fit(x, y, **o)
        assert model.feature_subset == m and len(model.trees) == len(trees)
        for got, want in zip(model.thresholds, thr):
            np.testing.assert_array_equal(np.array(got, np.float64).view(np.int64), np.array(want, np.float64).view(np.int64))
        for t, want in zip(model.trees, trees):
            _same_tree(t, ro.arrays(want))
        raw, prob, pred = ro.transform(trees, x)
        with model.transform(feats, raw=True) as out:
            d = feats.devices[0]
            got_raw = np.concatenate([_host(r, d) for r in out.raw])
            got_prob = np.concatenate([_host(p, d) for p in out.probability])
            got_pred = np.concatenate([_host(p, d) for p in out.prediction])
        np.testing.assert_array_equal(got_raw.view(np.int64), raw.view(np.int64))
        nan = np.isnan(prob)                         # rows no tree votes for: 0 / 0 (its NaN's bits are the unit's)
        np.testing.assert_array_equal(np.isnan(got_prob), nan)
        np.testing.assert_array_equal(got_prob[~nan].view(np.int64), prob[~nan].view(np.int64))
        np.testing.assert_array_equal(got_pred, pred)
        ev = model.evaluate(feats)
        labels = np.unique(y)
        want_conf = np.zeros((len(labels), model.num_classes), np.int64)
        np.add.at(want_conf, (np.searchsorted(labels, y), pred.astype(np.int64)), 1)
        np.testing.assert_array_equal(ev["confusion"], want_conf)
        f1, acc = CL.metrics(labels, want_conf)
        assert (ev["f1"], ev["accuracy"]) == (f1, acc)
        return model
    finally:
        _free(parts)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_forest_is_the_oracles_on_every_cut(engine, dtype):
    x, y = _data(4001, 6, 3, seed=7, dtype=dtype)
    x[:, 2] = np.round(x[:, 2])
    models = [_check_forest(engine, x, y, cuts, num_trees=6, max_depth=4) for cuts in (1, 2, 3)]
    for other in models[1:]:
        for a, b in zip(models[0].trees, other.trees):
            _same_tree(b, dict(feature=a.feature, left=a.left, right=a.right, threshold=a.threshold, counts=a.counts,
                               impurity=a.impurity, gain=a.gain))


def test_forced_tree_batches_give_the_same_forest(engine, monkeypatch):
    x, y = _data(2000, 5, 2, seed=3)
    one = _check_forest(engine, x, y, num_trees=5, max_depth=3, subsampling_rate=0.7)
    monkeypatch.setattr(CL, "_RF_SLOT_BUDGET", 8 * 2000 * 2)
    many = _check_forest(engine, x, y, num_trees=5, max_depth=3, subsampling_rate=0.7)
    assert (one.tree_batch, many.tree_batch) == (5, 2)


def test_one_tree_is_the_decision_tree(engine):
    x, y = _data(3000, 5, 3, seed=5)
    feats, parts = _on(engine, x, y, 1)
    try:
        rf = RandomForestClassifier(num_trees=1).fit(feats)
        dt = DecisionTreeClassifier().fit(feats)
        a, b = rf.trees[0], dt.tree
        for key in ("feature", "threshold", "left", "right", "counts", "prediction", "impurity", "gain"):
            np.testing.assert_array_equal(getattr(a, key).view(np.int64) if getattr(a, key).dtype == np.float64
                                          else getattr(a, key), getattr(b, key).view(np.int64)
                                          if getattr(b, key).dtype == np.float64 else getattr(b, key), key)
    finally:
        _free(parts)


@pytest.mark.parametrize("case", ["n=1", "empty bag", "k=1", "depth 0", "one class", "100 classes", "constant column",
                                  "tiny rate", "forest in global memory"])
def test_edges(engine, case):
    x, y = _data(1500, 4, 3, seed=11)
    params = dict(num_trees=4, max_depth=3)
    if case == "n=1":
        x, y = x[:1], np.zeros(1)
    elif case == "empty bag":                       # one tree, Bernoulli at rate 1e-3 over 300 rows: no row in the bag
        x, y = x[:300], y[:300]
        params = dict(num_trees=1, subsampling_rate=1e-3)
        assert not ro.weights(T.DEFAULT_SEED, 0, range(300), ro.table(1, 1e-3)).any()
    elif case == "k=1":
        x = x[:, :1]
    elif case == "depth 0":
        params["max_depth"] = 0
    elif case == "one class":
        y = np.zeros_like(y)
    elif case == "100 classes":
        x, y = _data(3000, 4, 100, seed=12)
        y[:100] = np.arange(100)
    elif case == "constant column":
        x[:, 1] = 2.5
    elif case == "tiny rate":
        params["subsampling_rate"] = 0.01
    else:
        x, y = _data(3000, 4, 30, seed=13)
        y[:30] = np.arange(30)
        params = dict(num_trees=20, max_depth=5, feature_subset_strategy="all")
    model = _check_forest(engine, x, y, **params)
    if case == "empty bag":
        assert model.total_num_nodes == 1 and not model.trees[0].counts.any()
    if case == "forest in global memory":
        assert model.total_num_nodes * (8 + 8 * 30) > 96 * 1024


@pytest.mark.parametrize("what", ["nan", "label", "released"])
def test_refusals(engine, what):
    x, y = _data(500, 3, 2, seed=4)
    if what == "nan":
        x[[120, 300], 1] = np.nan
    if what == "label":
        y[[200, 400]] = 0.5
    feats, parts = _on(engine, x, y, 2)
    try:
        if what == "released":
            _free(parts)
            feats._parts = []
            with pytest.raises(ValueError, match="released"):
                RandomForestClassifier().fit(feats)
            return
        want = "field 'f1' of the row with _id 220" if what == "nan" else "field 'y' of the row with _id 300"
        with pytest.raises(InvalidCellError, match=f"RandomForestClassifier: {want}"):
            RandomForestClassifier(num_trees=3).fit(feats)
    finally:
        _free(parts)


def test_level_refusals_name_the_cell(engine):
    """lo_rf_level refuses a code >= nbins and a label that is not a class with lo_dt_level's messages, and leaves
    hist_out zeroed although the pass counted the other rows."""
    import ctypes as C
    x, y = _data(300, 3, 2, seed=13)
    part = _part(engine, x, y)
    try:
        binned = engine.dt_bin(part, [to.splits(x[:, j], 8) for j in range(3)])
        try:
            feats = np.array([[0, 1, 2], [2, 0, 1]], np.int32)
            tab = np.ascontiguousarray(T.draw_table(2, 1.0), np.uint64)
            assert engine.rf_level(part, binned, 8, 2, T.DEFAULT_SEED, tab, 0, 2, None, feats).sum() > 0
            for nbins, nclasses, want in ((2, 2, r"row \d+, feature \d: code >= nbins = 2"),
                                          (8, 1, r"row \d+: its label is not a class in \[0, 1\)")):
                hist = np.full((2, 3, nbins, nclasses), 7, np.int64)
                lead = (part.y._h, part.nkept, 0, nbins, nclasses, T.DEFAULT_SEED, 0, 2, tab.ctypes.data_as(C.c_void_p),
                        len(tab), feats.ctypes.data_as(C.c_void_p), 3)
                with pytest.raises(N.LoexecError, match=want):
                    engine._level(engine._lib.lo_rf_level, lead, part, binned, None, 2, hist, None, None)
                assert not hist.any()
        finally:
            binned.free()
    finally:
        part.free()
