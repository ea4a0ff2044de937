"""CPU: the builder's "RF" classifier (Spark 2.4's RandomForestClassifier) without a GPU — the bagging tables against
exact sums, the hash's known answers, the feature subset sizes, the default seed and the parameter refusals, the fit
through stand-in engines (one, and a 3-way shard cut) against the oracle node for node, a forced multi-batch fit, the
header mirror and the SASS of the new kernels."""
import re
from fractions import Fraction
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest

import rf_oracle as ro
import tree_oracle as to
from learningorchestra_b200 import _native as N
from learningorchestra_b200 import classifier as CL
from learningorchestra_b200 import tree as T
from learningorchestra_b200.classifier import RandomForestClassifier
from test_tree_cpu import StandInEngine as DtStandIn
from test_tree_cpu import _sass

ROOT = Path(__file__).resolve().parent.parent


def _data(n, k, C, seed):
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(n, k))
    y = np.clip(np.round(x[:, 0] + 0.5 * x[:, 1] + rng.normal(size=n) * 0.5 + C / 2), 0, C - 1).astype(np.float64)
    return x, y


# ---- bagging tables, hash, subsets, seed ----------------------------------------------------------------------------
@pytest.mark.parametrize("num_trees,rate", [(20, 1.0), (20, 0.5), (20, 1e-3), (2, 0.75), (1, 0.5), (1, 1e-3), (1, 1.0)])
def test_tables_match_exact_sums(num_trees, rate):
    got = T.draw_table(num_trees, rate)
    assert got == ro.table(num_trees, rate)
    assert got == sorted(got) and 1 <= len(got) <= N.LO_RF_MAX_DRAWS
    if num_trees == 1:
        assert got == ([0] if rate == 1.0 else [int((1 - Fraction(rate)) * 2 ** 64)])
    else:
        assert got[0] == int(ro.exp_neg(Fraction(rate)) * 2 ** 64)
    if (num_trees, rate) == (20, 1.0):
        assert len(got) == 20                      # Poisson(1)'s tail falls below 2^-64 after j = 19


def test_weights_follow_the_table():
    tab = T.draw_table(20, 1.0)
    assert [ro.weight(u, tab) for u in (0, tab[0] - 1, tab[0], tab[1] - 1, tab[1], ro.M64)] == [0, 0, 1, 1, 2, len(tab)]
    w = ro.weights(T.DEFAULT_SEED, 3, range(20000), tab)
    assert abs(w.mean() - 1.0) < 0.03 and abs(np.mean(w == 0) - np.exp(-1)) < 0.01


def test_splitmix_known_answers():
    # splitmix64 seeded with 0: its first three outputs
    want = [0xE220A8397B1DCDAF, 0x6E789E6AA1B965F4, 0x06C45D188009454F]
    states = [0x9E3779B97F4A7C15 * i % 2 ** 64 for i in range(3)]
    assert [ro.mix(s) for s in states] == want
    assert [int(v) for v in T.splitmix(np.array(states, np.uint64))] == want
    assert ro.bag_u(7, 2, 5) == ro.mix(ro.mix(ro.mix(7) ^ 2) ^ 5)


def test_subsets_match_the_oracle():
    for tree, node, k, m in ((0, 1, 20, 5), (3, 6, 20, 5), (1, 2 ** 30 + 1, 7, 3), (2, 5, 4, 4), (0, 1, 50, 1)):
        got = T.feature_subset(T.DEFAULT_SEED, tree, node, k, m)
        assert got.tolist() == ro.subset(T.DEFAULT_SEED, tree, node, k, m)
        assert got.tolist() == sorted(set(got.tolist())) and len(got) == m
    assert T.feature_subset(-5, 0, 1, 9, 3).tolist() == ro.subset(-5, 0, 1, 9, 3)


@pytest.mark.parametrize("strategy,k,trees,m", [("auto", 20, 1, 20), ("auto", 20, 2, 5), ("AUTO", 10, 5, 4),
                                                ("all", 20, 5, 20), ("sqrt", 1, 5, 1), ("sqrt", 17, 5, 5),
                                                ("log2", 1, 5, 1), ("log2", 2, 5, 1), ("log2", 9, 5, 4),
                                                ("onethird", 20, 5, 7), ("onethird", 1, 5, 1), ("3", 20, 5, 3),
                                                ("30", 20, 5, 20), ("0.5", 9, 5, 5), (".25", 20, 5, 5),
                                                ("1.0", 20, 5, 20), ("0.01", 20, 5, 1)])
def test_subset_sizes(strategy, k, trees, m):
    assert T.subset_size(strategy, k, trees) == m


@pytest.mark.parametrize("strategy", ["", "0", "-1", "1.5", "2.0", "0.0", "half", "sqrt ", 0.5, None, "01"])
def test_unknown_strategies_are_refused(strategy):
    with pytest.raises(ValueError, match="feature_subset_strategy"):
        RandomForestClassifier(feature_subset_strategy=strategy)


def test_default_seed_is_the_class_names_java_hash():
    assert ro.java_string_hash("hello") == 99162322                   # String.hashCode's known answer
    name = "org.apache.spark.ml.classification.RandomForestClassifier"
    assert T.java_hash(name) == ro.java_string_hash(name) == T.DEFAULT_SEED == 207336481
    assert RandomForestClassifier().seed == T.DEFAULT_SEED and RandomForestClassifier(seed=-3).seed == -3


@pytest.mark.parametrize("kw", [dict(num_trees=0), dict(num_trees=2.0), dict(num_trees=True), dict(max_depth=31),
                                dict(max_bins=1), dict(max_bins=257), dict(min_instances_per_node=0),
                                dict(min_info_gain=-1.0), dict(impurity="variance"), dict(subsampling_rate=0.0),
                                dict(subsampling_rate=1.5), dict(subsampling_rate=float("nan")),
                                dict(subsampling_rate=True), dict(seed=1.5), dict(seed=1 << 63)])
def test_parameters_are_refused(kw):
    with pytest.raises(ValueError):
        RandomForestClassifier(**kw)


def test_parameter_bounds_are_accepted():
    RandomForestClassifier(num_trees=1, max_depth=0, max_bins=2, subsampling_rate=1e-300, seed=-(1 << 63))
    RandomForestClassifier(max_depth=30, max_bins=256, impurity="Entropy", feature_subset_strategy="0.3",
                           seed=(1 << 63) - 1)


# ---- the classifier through stand-in engines --------------------------------------------------------------------
class StandInEngine(DtStandIn):
    """An Engine's dt_sort / dt_rank / lr_stats and rf_* on numpy rows, the bagging weights from the oracle's hash."""

    def dt_bin(self, part, thr):
        x, _y = part
        return SimpleNamespace(codes=to.bins(x, thr), slot=None, free=lambda: None)

    def rf_level(self, part, binned, nbins, C, seed, draw, tree0, ntrees, splits, feats, row0=0, shape=None):
        x, y = part
        n, codes = len(y), binned.codes
        self.calls.append(("level", tree0, ntrees, len(feats)))
        if splits is None:
            slot = np.repeat(np.arange(ntrees)[:, None], n, axis=1)
        else:
            p = binned.slot
            sp = splits[np.maximum(p, 0)]
            f = np.where(p >= 0, sp[..., 0], -1)
            c = codes[np.arange(n)[None, :], np.maximum(f, 0)]
            slot = np.where(f >= 0, np.where(c <= sp[..., 1], sp[..., 2], sp[..., 3]), -1)
        binned.slot = slot
        w = np.array([ro.weights(seed, tree0 + t, range(row0, row0 + n), draw) for t in range(ntrees)]).reshape(ntrees, n)
        nnodes, m = feats.shape
        hist = np.zeros((nnodes, m, nbins, C), np.int64)
        tt, rr = np.nonzero((slot >= 0) & (w > 0))
        s = slot[tt, rr]
        for q in range(m):
            np.add.at(hist, (s, q, codes[rr, feats[s, q]], y[rr].astype(np.int64)), w[tt, rr])
        return hist

    def rf_predict(self, part, trees, raw=False, labels=None):
        x, y = part
        votes = np.zeros((len(y), trees[0].num_classes))
        for t in trees:
            node = np.zeros(len(y), np.int64)
            for _ in range(t.num_nodes):
                f = t.feature[node]
                left = x[np.arange(len(y)), np.maximum(f, 0)] <= t.threshold[node]
                node = np.where(f >= 0, np.where(left, t.left[node], t.right[node]), node)
            votes = votes + T.votes(t)[node]
        pred = votes.argmax(1)
        conf = np.zeros((len(labels), votes.shape[1]), np.int64)
        np.add.at(conf, (np.searchsorted(labels, y), pred), 1)
        return conf


class _Part(tuple):
    x = SimpleNamespace(dtype_code=N.LO_F64)

    @property
    def nkept(self):
        return len(self[1])


def _features(engine, parts, n, k):
    return SimpleNamespace(_frame=SimpleNamespace(_cache=SimpleNamespace(engine=engine)), _parts=parts,
                           fields=[f"f{j}" for j in range(k)], label="y", row_ids=np.arange(100, 100 + n))


def _sharded(x, y, bounds):
    from learningorchestra_b200.sharding import ShardedEngine
    sh = object.__new__(ShardedEngine)
    sh._N, sh.world, sh.nlocal = N, len(bounds) - 1, len(bounds) - 1
    sh.engines = [StandInEngine() for _ in bounds[1:]]
    parts = [_Part((x[a:b], y[a:b])) for a, b in zip(bounds[:-1], bounds[1:])]
    return sh, parts


def _same(tree, want):
    for key in ("feature", "left", "right"):
        assert getattr(tree, key).tolist() == want[key].tolist(), key
    for key, got in (("threshold", tree.threshold), ("counts", tree.counts), ("impurity", tree.impurity),
                     ("gain", tree.gain)):
        np.testing.assert_array_equal(np.asarray(got, np.float64).view(np.int64),
                                      np.asarray(want[key], np.float64).reshape(got.shape).view(np.int64), key)


def _check_forest(model, x, y, **kw):
    trees, thr, m = ro.fit(x, y, **kw)
    assert model.thresholds == thr and model.feature_subset == m and len(model.trees) == len(trees)
    for t, want in zip(model.trees, trees):
        _same(t, ro.arrays(want))
    assert model.total_num_nodes == sum(t.num_nodes for t in model.trees)
    assert model.tree_weights.tolist() == [1.0] * len(trees)
    return trees


PARAMS = [dict(num_trees=6, max_depth=4), dict(num_trees=5, rate=0.6, kind="entropy", max_bins=8),
          dict(num_trees=4, m=2, min_inst=5, max_depth=6), dict(num_trees=1, rate=0.5), dict(num_trees=3, max_depth=0)]


def _estimator(kw):
    strategy = "auto" if kw.get("m") is None else str(kw["m"])
    return RandomForestClassifier(num_trees=kw["num_trees"], max_depth=kw.get("max_depth", 5),
                                  max_bins=kw.get("max_bins", 32), min_instances_per_node=kw.get("min_inst", 1),
                                  impurity=kw.get("kind", "gini"), feature_subset_strategy=strategy,
                                  subsampling_rate=kw.get("rate", 1.0))


@pytest.mark.parametrize("kw", PARAMS)
def test_fit_through_a_stand_in_engine(kw):
    x, y = _data(400, 5, 3, seed=len(kw))
    x[:, 2] = np.round(x[:, 2] * 2)
    model = _estimator(kw).fit(_features(StandInEngine(), [_Part((x, y))], 400, 5))
    _check_forest(model, x, y, **kw)


def test_sharded_fit_and_evaluate_match_the_oracle():
    x, y = _data(600, 4, 3, seed=9)
    bounds = [0, 150, 151, 600]
    sh, parts = _sharded(x, y, bounds)
    model = RandomForestClassifier(num_trees=5, max_depth=4).fit(_features(sh, parts, 600, 4))
    trees = _check_forest(model, x, y, num_trees=5, max_depth=4)
    labels = np.unique(y)
    conf = sh.rf_predict(parts, model.trees, labels=labels)
    _raw, _prob, pred = ro.transform(trees, x)
    want = np.zeros((len(labels), 3), np.int64)
    np.add.at(want, (np.searchsorted(labels, y), pred.astype(np.int64)), 1)
    np.testing.assert_array_equal(conf, want)


def test_forced_batches_give_the_same_forest(monkeypatch):
    x, y = _data(300, 4, 2, seed=4)
    engine = StandInEngine()
    one = RandomForestClassifier(num_trees=5).fit(_features(engine, [_Part((x, y))], 300, 4))
    assert one.tree_batch == 5 and {c[2] for c in engine.calls if c[0] == "level"} == {5}
    monkeypatch.setattr(CL, "_RF_SLOT_BUDGET", 8 * 300 * 2)            # two trees' slot tables per batch
    engine = StandInEngine()
    many = RandomForestClassifier(num_trees=5).fit(_features(engine, [_Part((x, y))], 300, 4))
    assert many.tree_batch == 2 and sorted({c[1:3] for c in engine.calls if c[0] == "level"}) == [(0, 2), (2, 2), (4, 1)]
    for a, b in zip(one.trees, many.trees):
        _same(a, {key: getattr(b, key) for key in ("feature", "left", "right", "threshold", "counts", "impurity", "gain")})


def test_one_tree_is_the_decision_tree():
    x, y = _data(500, 4, 3, seed=2)
    model = RandomForestClassifier(num_trees=1, max_depth=4).fit(_features(StandInEngine(), [_Part((x, y))], 500, 4))
    root, _thr = to.fit(x, y, max_depth=4)
    want = to.arrays(root)
    _same(model.trees[0], want)
    assert model.feature_subset == 4


def test_the_lowest_refused_cell_names_its_id():
    from learningorchestra_b200.engine import InvalidCellError
    x, y = _data(300, 3, 2, seed=6)
    bad_y = y.copy()
    bad_y[[150, 250]] = 0.5
    sh, parts = _sharded(x, bad_y, [0, 100, 300])
    for e in sh.engines:
        e.lr_stats = lambda part: _lr_stats(part)
    with pytest.raises(InvalidCellError, match="RandomForestClassifier: field 'y' of the row with _id 250"):
        RandomForestClassifier().fit(_features(sh, parts, 300, 3))


def _lr_stats(part):
    from learningorchestra_b200.engine import InvalidCellError
    x, y = part
    bad = np.flatnonzero(y != np.round(y))
    if len(bad):
        raise InvalidCellError(int(bad[0]), x.shape[1], reason="row {row}: its label is not an integer >= 0")
    return DtStandIn().lr_stats(part)


# ---- header, SASS ---------------------------------------------------------------------------------------------------
def test_header_mirror_matches():
    text = (ROOT / "include" / "loexec.h").read_text()
    assert int(re.search(r"#define LO_RF_MAX_DRAWS\s+(\d+)", text).group(1)) == N.LO_RF_MAX_DRAWS == T.MAX_DRAWS
    for fn in ("lo_rf_level", "lo_rf_predict"):
        decl = re.search(rf"int {fn}\(([^;]*)\);", text, re.S).group(1)
        assert len(decl.split(",")) == len(N.SIGNATURES[fn][1]), fn
    assert N.LO_ABI_VERSION == 7
    cuh = (ROOT / "learningorchestra_b200" / "csrc" / "tree.cuh").read_text()
    assert "constexpr int kRfMaxDraws = 32;" in cuh


def test_sass_of_the_rf_kernels(built):
    funcs = _sass(built, "_ZN2lo10k_rf_level") + _sass(built, "_ZN2lo12k_rf_predict")
    assert len(funcs) == 6                                            # level f32 / f64, predict f32 / f64 x EVAL
    for f in funcs:
        assert "LDL" not in f and "STL" not in f                      # no local memory: the votes stay in registers
