"""CPU: the builder's "GB" classifier (Spark 2.4's GBTClassifier) without a GPU — the numpy oracle against a brute-force
regression split search, the 128-bit merge, prefix and rounding of lo_gb_stats against Python ints, the host's
variance growth against the oracle, the parameter refusals, the fit and predict merges through stand-in engines, the
header mirror and the SASS of the new kernels."""
import re
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest

import gbt_oracle as go
import tree_oracle as to
from learningorchestra_b200 import _native as N
from learningorchestra_b200 import tree as T
from learningorchestra_b200.classifier import GBTClassifier
from test_tree_cpu import _sass

ROOT = Path(__file__).resolve().parent.parent
M64 = 2 ** 64 - 1


def _data(n, k, seed):
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(n, k))
    y = ((x @ rng.normal(size=k) + rng.logistic(size=n)) > 0).astype(np.float64)
    return x, y


def _pack(values):
    """Python ints (count, s1 + 2^60 count, s2) -> the five words."""
    c, s1, s2 = values
    return [c, s1 & M64, s1 >> 64, s2 & M64, s2 >> 64]


def _words(codes, slot, r, nnodes, nbins):
    q1, q2 = go.quantise(r)
    n, k = codes.shape
    out = np.zeros((nnodes, k, nbins, T.WORDS), np.uint64)
    live = slot >= 0
    for j in range(k):
        g = slot[live] * nbins + codes[live, j]
        cnt = np.bincount(g, minlength=nnodes * nbins)
        s1 = go.exact_sum(q1[live] + (1 << 60), g, nnodes * nbins)
        s2 = go.exact_sum(q2[live], g, nnodes * nbins)
        for c in range(nnodes * nbins):
            out[c // nbins, j, c % nbins] = _pack((int(cnt[c]), s1[c], s2[c]))
    return out


def _numpy_level(x, r, thr, nbins=None):
    """A stand-in for lo_gb_level: the rows routed as lo_dt_level routes them, the words from Python ints."""
    codes = to.bins(x, thr)
    nbins = nbins or max(len(t) for t in thr) + 1
    state = {}

    def level(splits, nnodes):
        if splits is None:
            slot = np.zeros(len(r), np.int64)
        else:
            p = state["slot"]
            sp = splits[np.maximum(p, 0)]
            f = np.where(p >= 0, sp[:, 0], -1)
            c = codes[np.arange(len(r)), np.maximum(f, 0)]
            slot = np.where(f >= 0, np.where(c <= sp[:, 1], sp[:, 2], sp[:, 3]), -1)
        state["slot"] = slot
        return _words(codes, slot, r, nnodes, nbins)

    return level


def _same(tree, want):
    for key in ("feature", "left", "right"):
        assert getattr(tree, key).tolist() == want[key].tolist(), key
    for key, got in (("threshold", tree.threshold), ("stats", tree.counts), ("prediction", tree.prediction),
                     ("impurity", tree.impurity), ("gain", tree.gain)):
        np.testing.assert_array_equal(np.asarray(got, np.float64).view(np.int64),
                                      np.asarray(want[key], np.float64).reshape(got.shape).view(np.int64), key)


# ---- the oracle against a brute-force split search ----------------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_oracle_root_split_is_the_best_variance_reduction(seed):
    rng = np.random.default_rng(seed)
    x = np.round(rng.normal(size=(200, 3)) * 3) / 2
    r = rng.uniform(-4, 4, 200)
    thr = [to.splits(x[:, j], 32) for j in range(3)]
    root = go.regression_tree(to.bins(x, thr), thr, r, max_depth=1)
    gains = []
    for j in range(3):
        for t in thr[j]:
            left, right = r[x[:, j] <= t], r[x[:, j] > t]
            gains.append((np.var(r) - len(left) / 200 * np.var(left) - len(right) / 200 * np.var(right), j, t))
    gains.sort(key=lambda g: -g[0])
    assert gains[0][0] - gains[1][0] > 1e-9                      # certified: no near tie at the top
    assert not root["leaf"] and (root["feature"], root["threshold"]) == gains[0][1:]
    assert abs(root["gain"] - gains[0][0]) <= 1e-12 * max(1.0, abs(gains[0][0]))


# ---- 128-bit sums: lo_gb_stats and add_words against Python ints ---------------------------------------------------
def _stats_ints(cells, nsplits):
    """(left, right, total) of one node and feature from (count, s1 + 2^60 count, s2) Python ints per bin."""
    tot = [sum(c[i] for c in cells) for i in range(3)]
    left, right = [], []
    acc = [0, 0, 0]
    for i in range(nsplits):
        acc = [a + b for a, b in zip(acc, cells[i])]
        left.append(acc)
        right.append([t - a for t, a in zip(tot, acc)])
    fl = lambda v: (float(v[0]), float(v[1] - (v[0] << 60)) / 2 ** 58, float(v[2]) / 2 ** 58)
    return [fl(v) for v in left], [fl(v) for v in right], fl(tot)


@pytest.mark.parametrize("case", ["random", "carries", "negative", "extremes", "above 2^64"])
def test_word_stats_against_python_ints(built, case):
    rng = np.random.default_rng(1)
    nbins = 7
    cells = []
    for b in range(nbins):
        cnt = int(rng.integers(0, 50)) if case != "above 2^64" else int(rng.integers(2 ** 20, 2 ** 30))
        if case == "extremes":                       # every row at the bound |r| = 4: q1 = ±2^60, q2 = 2^62
            q1 = [(1 << 60) * (1 if rng.uniform() < 0.5 else -1) for _ in range(cnt)]
            s1 = sum(q1) + (cnt << 60)
            s2 = cnt * (1 << 62)
        elif case in ("carries", "above 2^64"):
            s1 = cnt * (1 << 61) - int(rng.integers(0, 1000))
            s1 = max(s1, 0)
            s2 = cnt * (1 << 62) - int(rng.integers(0, 1000))
            s2 = max(s2, 0)
        elif case == "negative":                     # every q1 = -2^60: the offset sums to 0
            s1, s2 = 0, cnt * (1 << 60)
        else:
            q = rng.integers(-(1 << 60), 1 << 60, cnt)
            s1 = sum(int(v) for v in q) + (cnt << 60)
            s2 = sum(int(v) for v in rng.integers(0, 1 << 62, cnt))
        cells.append((cnt, s1, s2))
    words = np.array([[[_pack(c) for c in cells]]], np.uint64)
    left, right, total = T.word_stats(words, nbins - 1)
    wl, wr, wt = _stats_ints(cells, nbins - 1)
    np.testing.assert_array_equal(total[0], wt)
    np.testing.assert_array_equal(left[0, 0], wl)
    np.testing.assert_array_equal(right[0, 0], wr)
    # shards: the words of two halves added with carries give the whole's words
    half = [(c // 2, s1 // 2, s2 // 3) for c, s1, s2 in cells]
    rest = [(c - a, s1 - b, s2 - d) for (c, s1, s2), (a, b, d) in zip(cells, half)]
    merged = T.add_words(np.array([[[_pack(c) for c in half]]], np.uint64), np.array([[[_pack(c) for c in rest]]], np.uint64))
    np.testing.assert_array_equal(merged, words)


def test_rounding_is_once_and_correct(built):
    """Sums that f64 cannot hold exactly, at and beside the ties of round-half-even: Python's int -> float rounding."""
    for s in (2 ** 60 + 1, 2 ** 60 + 2 ** 7, 2 ** 60 + 2 ** 7 + 1, 2 ** 60 + 3 * 2 ** 7, -(2 ** 61) - 3):
        words = np.array([[[_pack((4, s + (4 << 60), 5))]]], np.uint64)
        _l, _r, total = T.word_stats(words, 0)
        assert total[0, 1] == float(s) / 2 ** 58


# ---- growth: the host's variance levels against the oracle ------------------------------------------------------
@pytest.mark.parametrize("params", [dict(), dict(max_depth=0), dict(max_depth=2), dict(min_inst=30),
                                    dict(min_gain=0.01), dict(max_depth=7, max_bins=6)])
def test_variance_growth_matches_the_oracle(built, params):
    x, y = _data(800, 3, seed=len(params))
    x[:, 1] = np.round(x[:, 1] * 2)
    r = go.residual(y, np.random.default_rng(2).normal(size=800))
    thr = [to.splits(x[:, j], params.get("max_bins", 32)) for j in range(3)]
    depth = params.get("max_depth", 5)
    tree, _ = T.grow(_numpy_level(x, r, thr), thr, 0, depth, T.VARIANCE, params.get("min_inst", 1),
                     params.get("min_gain", 0.0))
    want = go.regression_tree(to.bins(x, thr), thr, r, depth, params.get("min_inst", 1), params.get("min_gain", 0.0))
    _same(tree, go.arrays(want))


def test_pure_leaves_of_tree_zero_are_pruned(built):
    x = np.linspace(0, 1, 400)[:, None]
    y = (x[:, 0] > 0.5).astype(np.float64)
    thr = [to.splits(x[:, 0], 32)]
    r = 2 * y - 1
    tree, shapes = T.grow(_numpy_level(x, r, thr), thr, 0, 5, T.VARIANCE, 1, 0.0)
    assert tree.num_nodes == 3 and tree.prediction[1:].tolist() == [-1.0, 1.0]


# ---- parameters and the classifier with stand-in engines ---------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(max_iter=0), dict(max_iter=2.0), dict(max_iter=True), dict(step_size=0.0),
                                dict(step_size=1.5), dict(step_size=float("nan")), dict(step_size=True),
                                dict(max_depth=31), dict(max_depth=-1), dict(max_bins=1), dict(max_bins=257),
                                dict(min_instances_per_node=0), dict(min_info_gain=-1.0),
                                dict(min_info_gain=float("inf"))])
def test_parameters_are_refused(kw):
    with pytest.raises(ValueError):
        GBTClassifier(**kw)


def test_parameter_bounds_are_accepted():
    GBTClassifier(max_iter=1, step_size=1.0, max_depth=0, max_bins=2)
    GBTClassifier(step_size=1e-300, max_depth=30, max_bins=256)


class StandInEngine:
    """An Engine's dt_sort / dt_rank / dt_bin, lr_stats and gb_* on numpy rows."""

    def __init__(self):
        from test_tree_cpu import StandInEngine as DtStandIn
        self._dt = DtStandIn()

    def __getattr__(self, name):
        return getattr(self._dt, name)

    def lr_stats(self, part):
        from learningorchestra_b200.engine import InvalidCellError
        x, y = part
        bad = np.argwhere(~np.isfinite(x))
        if len(bad):
            raise InvalidCellError(int(bad[0][0]), int(bad[0][1]), reason="row {row}, feature {position}: NaN")
        return self._dt.lr_stats(part)

    def dt_bin(self, part, thr):
        x, _y = part
        return SimpleNamespace(codes=to.bins(x, thr), slot=None, free=lambda: None)

    def gb_update(self, part, rows=None, tree=None, weight=1.0):
        from learningorchestra_b200.engine import InvalidCellError
        x, y = part
        bad = np.flatnonzero((y != 0) & (y != 1))
        if len(bad):
            raise InvalidCellError(bad[0], x.shape[1], reason="row {row}: its label is not 0 or 1")
        if rows is None:
            rows = SimpleNamespace(F=np.zeros(len(y)), r=2 * y - 1, free=lambda: None)
            return rows
        rows.F = rows.F + tree.prediction[_leaf(tree, x)] * weight
        rows.r = go.residual(y, rows.F)
        return rows

    def gb_level(self, part, binned, rows, nbins, splits, nnodes, shape=None):
        codes = binned.codes
        if splits is None:
            slot = np.zeros(len(rows.r), np.int64)
        else:
            p = binned.slot
            sp = splits[np.maximum(p, 0)]
            f = np.where(p >= 0, sp[:, 0], -1)
            c = codes[np.arange(len(p)), np.maximum(f, 0)]
            slot = np.where(f >= 0, np.where(c <= sp[:, 1], sp[:, 2], sp[:, 3]), -1)
        binned.slot = slot
        return _words(codes, slot, rows.r, nnodes, nbins)

    def gb_predict(self, part, trees, weights, raw=False, labels=None):
        x, y = part
        m = np.zeros(len(y))
        for t, w in zip(trees, weights):
            m = m + t.prediction[_leaf(t, x)] * w
        pred = (m > 0).astype(np.int64)
        conf = np.zeros((len(labels), 2), np.int64)
        np.add.at(conf, (np.searchsorted(labels, y), pred), 1)
        return conf


def _leaf(tree, x):
    node = np.zeros(len(x), np.int64)
    for _ in range(tree.num_nodes):
        f = tree.feature[node]
        go_left = x[np.arange(len(x)), np.maximum(f, 0)] <= tree.threshold[node]
        node = np.where(f >= 0, np.where(go_left, tree.left[node], tree.right[node]), node)
    return node


class _Part(tuple):
    x = SimpleNamespace(dtype_code=N.LO_F64)

    @property
    def nkept(self):
        return len(self[1])


def _features(engine, parts, n, k):
    return SimpleNamespace(_frame=SimpleNamespace(_cache=SimpleNamespace(engine=engine)), _parts=parts,
                           fields=[f"f{j}" for j in range(k)], label="y", row_ids=np.arange(100, 100 + n))


def _check_fit(feats, x, y):
    m = GBTClassifier(max_iter=4, max_depth=3).fit(feats)
    trees, weights, thr, _ = go.fit(x, y, max_iter=4, max_depth=3)
    assert m.thresholds == thr and m.tree_weights.tolist() == weights
    for t, want in zip(m.trees, trees):
        _same(t, go.arrays(want))
    return m


def test_fit_through_a_stand_in_engine(built):
    x, y = _data(500, 3, seed=3)
    _check_fit(_features(StandInEngine(), [_Part((x, y))], 500, 3), x, y)


def test_sharded_fit_and_predict_through_stand_in_engines(built):
    from learningorchestra_b200.engine import InvalidCellError
    from learningorchestra_b200.sharding import ShardedEngine
    x, y = _data(600, 3, seed=4)
    bounds = [0, 150, 151, 600]
    sh = object.__new__(ShardedEngine)
    sh._N, sh.world, sh.nlocal, sh.engines = N, 3, 3, [StandInEngine() for _ in range(3)]
    parts = [_Part((x[a:b], y[a:b])) for a, b in zip(bounds[:-1], bounds[1:])]
    m = _check_fit(_features(sh, parts, 600, 3), x, y)
    labels = np.array([0.0, 1.0])
    conf = sh.gb_predict(parts, m.trees, m.tree_weights, labels=labels)
    _raw, _prob, pred = go.transform(*go.fit(x, y, max_iter=4, max_depth=3)[:2], x)
    want = np.zeros((2, 2), np.int64)
    np.add.at(want, (y.astype(np.int64), pred.astype(np.int64)), 1)
    np.testing.assert_array_equal(conf, want)
    y2 = y.copy()
    y2[[300, 599]] = 2.0
    parts = [_Part((x[a:b], y2[a:b])) for a, b in zip(bounds[:-1], bounds[1:])]
    with pytest.raises(InvalidCellError, match="GBTClassifier: field 'y' of the row with _id 400 is not a label 0 or 1"):
        GBTClassifier().fit(_features(sh, parts, 600, 3))


def test_the_lowest_refused_cell_over_labels_and_features_is_raised():
    from learningorchestra_b200.engine import InvalidCellError
    x, y = _data(400, 3, seed=6)
    for nan_row, label_row, want in ((10, 300, "_id 110 is NaN"), (300, 10, "_id 110 is not a label 0 or 1")):
        xx, yy = x.copy(), y.copy()
        xx[nan_row, 2] = np.nan
        yy[label_row] = 0.5
        for feats in (_features(StandInEngine(), [_Part((xx, yy))], 400, 3),):
            with pytest.raises(InvalidCellError, match=want):
                GBTClassifier(max_iter=2).fit(feats)


# ---- header, SASS ---------------------------------------------------------------------------------------------------
def test_header_mirror_matches():
    text = (ROOT / "include" / "loexec.h").read_text()
    assert int(re.search(r"#define LO_GB_WORDS\s+(\d+)", text).group(1)) == N.LO_GB_WORDS == T.WORDS
    for fn in ("lo_gb_level", "lo_gb_stats", "lo_gb_update", "lo_gb_predict"):
        decl = re.search(rf"int {fn}\(([^;]*)\);", text, re.S).group(1)
        assert len(decl.split(",")) == len(N.SIGNATURES[fn][1]), fn
    assert N.LO_ABI_VERSION == 7


def test_sass_of_the_gbt_kernels(built):
    for prefix in ("_ZN2lo10k_gb_level", "_ZN2lo11k_gb_update", "_ZN2lo12k_gb_predict"):
        for f in _sass(built, prefix):
            assert "LDL" not in f and "STL" not in f, prefix          # no local memory
    vec = [f for f in _sass(built, "_ZN2lo10k_gb_level") if "Lb1EE" in f.split("\n")[0]]
    assert vec and all("LDG.E.NA.128" in f for f in vec)              # 16-byte read-once code loads
