"""CPU: the builder's "DT" classifier (Spark 2.4's DecisionTreeClassifier) without a GPU — the numpy oracle against
scikit-learn, the host's rank-query replay of Spark's greedy split search against the literal loop on adversarial
columns with numpy stand-ins for the members, the level-wise growth against the oracle, the parameter refusals, the
launch-shape choice pinned to the sources, the header mirror and the SASS of the new kernels."""
import math
import re
import subprocess
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest

import tree_oracle as to
from learningorchestra_b200 import _native as N
from learningorchestra_b200 import tree as T
from learningorchestra_b200.classifier import DecisionTreeClassifier

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "learningorchestra_b200" / "csrc"


# ---- split candidates: the rank replay against the literal loop ------------------------------------------------
class Members:
    """numpy stand-ins for the members' sorted columns: each cut holds its rows' codes sorted; rank counts add up."""

    def __init__(self, col, cuts, f32):
        self.f32 = f32
        codes = np.array([T.encode(float(v), f32) for v in col], dtype=object)
        bounds = np.linspace(0, len(col), cuts + 1).astype(int)
        self.sorted = [np.sort(np.array(codes[a:b], dtype=np.uint64)) for a, b in zip(bounds[:-1], bounds[1:])]
        self.calls = 0

    def rank(self, cols, probes):
        self.calls += 1
        assert not np.any(cols)
        lt = sum(np.searchsorted(s, probes, side="left") for s in self.sorted)
        le = sum(np.searchsorted(s, probes, side="right") for s in self.sorted)
        return np.asarray(lt, np.int64), np.asarray(le, np.int64)


def _replayed(col, max_bins, cuts, f32):
    """The rank path, which the classifier takes only for a column with more distinct values than the midpoint rule
    takes (some member could not list its values); otherwise the listed values' greedy."""
    vals, cnts = to.value_counts(col)
    if len(vals) - 1 <= T.num_splits(max_bins, len(col)):
        return T.greedy(vals, cnts, T.num_splits(max_bins, len(col)), len(col)), 0
    m = Members(col, cuts, f32)
    thr, rounds = T.column_thresholds(len(col), max_bins, [None], m.rank, f32, 1)
    return thr[0], rounds


# three neighbouring doubles around one with an even mantissa: both midpoints round to 1.0, so Spark's split search
# returns two equal thresholds
EQUAL_MIDPOINTS = np.array([np.nextafter(1.0, 0.0), 1.0, np.nextafter(1.0, 2.0)])


def _adversarial():
    rng = np.random.default_rng(0)
    heavy = np.concatenate([np.full(500, 3.0), np.full(400, -1.0), rng.normal(size=100), np.full(300, 7.5)])
    gaps = np.repeat(np.arange(40, dtype=np.float64), 3)                 # equal counts: exact gap ties
    big = np.finfo(np.float64).max
    cols = {
        "heavy": heavy,
        "one heavy value over many targets": np.concatenate([np.zeros(900), np.arange(1, 101, dtype=np.float64)]),
        "gap ties": gaps,
        "31 values": np.arange(31, dtype=np.float64).repeat(2),
        "32 values": np.arange(32, dtype=np.float64).repeat(2),
        "33 values": np.arange(33, dtype=np.float64).repeat(2),
        "n = 1": np.array([4.0]),
        "n = 2": np.array([1.0, -2.0]),
        "signed zeros": np.concatenate([np.full(50, -0.0), np.full(50, 0.0), rng.normal(size=200)]),
        "near DBL_MAX": np.concatenate([np.full(40, big), np.full(40, big * (1 - 2 ** -52)), np.full(40, -big),
                                        rng.normal(size=100)]),
        "f32 widened": rng.normal(size=1000).astype(np.float32).astype(np.float64),
        "skewed": np.concatenate([np.full(5000, 1.0), rng.exponential(size=300)]),
        "equal midpoints": np.concatenate([np.repeat(EQUAL_MIDPOINTS, 40), rng.normal(size=200)]),
        "equal midpoints only": np.repeat(EQUAL_MIDPOINTS, 3),
    }
    return cols


@pytest.mark.parametrize("cuts", [1, 2, 3, 8])
@pytest.mark.parametrize("max_bins", [2, 5, 32])
def test_rank_replay_equals_the_literal_loop(cuts, max_bins):
    for name, col in _adversarial().items():
        f32 = name == "f32 widened"
        got, _rounds = _replayed(col, max_bins, cuts, f32)
        vals, cnts = to.value_counts(col)
        want = T.greedy(vals, cnts, T.num_splits(max_bins, len(col)), len(col))
        assert [float(v) for v in got] == [float(v) for v in want], name
        assert np.array_equal(np.array(want, np.float64).view(np.int64), np.array(got, np.float64).view(np.int64))
        if len(vals) - 1 > T.num_splits(max_bins, len(col)):       # the greedy itself, against the oracle's loop
            assert want == to.splits(col, max_bins), name


def test_greedy_matches_the_oracle_on_random_columns():
    rng = np.random.default_rng(3)
    for trial in range(200):
        n = int(rng.integers(1, 400))
        col = rng.integers(-5, int(rng.integers(1, 80)), n).astype(np.float64) * rng.choice([1.0, 0.5, 0.1])
        mb = int(rng.integers(2, 40))
        vals, cnts = to.value_counts(col)
        want = to.splits(col, mb)
        assert T.greedy(vals, cnts, T.num_splits(mb, n), n) == want
        got, _ = _replayed(col, mb, int(rng.integers(1, 5)), False)
        assert got == want, trial


def test_merged_member_lists_give_the_union_counts():
    a = (3, np.array([0.0, 1.0, 2.0]), np.array([2, 1, 1]))
    b = (2, np.array([1.0, 5.0]), np.array([4, 1]))
    vals, cnts = T.merge_distinct([a, b])
    assert vals.tolist() == [0.0, 1.0, 2.0, 5.0] and cnts.tolist() == [2, 5, 1, 1]
    assert T.merge_distinct([a, (300, None, None)]) is None


def test_codes_keep_the_order_of_values():
    for f32 in (False, True):
        big, tiny = (1e30, 1e-30) if f32 else (1e300, 1e-300)
        vals = [-np.inf, -big, -1.0, -tiny, -0.0, 0.0, tiny, 1.0, big, np.inf]
        codes = [T.encode(v, f32) for v in vals]
        assert codes == sorted(codes)
        assert T.encode(-0.0, f32) == T.encode(0.0, f32)
        assert all(T.decode(T.encode(v, f32), f32) == (np.float32(v) if f32 else v) for v in vals)


# ---- growth: the host's vectorised levels against the oracle ----------------------------------------------------
def _numpy_level(x, y, thr, C, nbins=None):
    """A stand-in for the device's levels: the codes by findBin, the rows' slots routed as lo_dt_level does."""
    codes = to.bins(x, thr)
    nbins = nbins or max(len(t) for t in thr) + 1
    state = {"slot": None}

    def level(splits, nnodes):
        if splits is None:
            slot = np.zeros(len(y), np.int64)
        else:
            p = state["slot"]
            slot = np.full(len(y), -1)
            live = p >= 0
            f = np.where(live, splits[np.maximum(p, 0), 0], -1)
            go = live & (f >= 0)
            c = codes[np.arange(len(y)), np.maximum(f, 0)]
            left = c <= splits[np.maximum(p, 0), 1]
            slot = np.where(go, np.where(left, splits[np.maximum(p, 0), 2], splits[np.maximum(p, 0), 3]), -1)
        state["slot"] = slot
        hist = np.zeros((nnodes, x.shape[1], nbins, C), np.int64)
        rows = slot >= 0
        for j in range(x.shape[1]):
            np.add.at(hist, (slot[rows], j, codes[rows, j], y[rows].astype(np.int64)), 1)
        return hist

    return level


def _host_tree(x, y, max_depth=5, max_bins=32, min_inst=1, min_gain=0.0, kind="gini"):
    thr = [to.splits(x[:, j], max_bins) for j in range(x.shape[1])]
    C = int(y.max()) + 1
    tree, _ = T.grow(_numpy_level(x, y, thr, C), thr, C, max_depth, kind, min_inst, min_gain)
    return tree


def _assert_same_tree(tree, want):
    assert tree.feature.tolist() == want["feature"].tolist()
    assert tree.left.tolist() == want["left"].tolist() and tree.right.tolist() == want["right"].tolist()
    np.testing.assert_array_equal(tree.threshold.view(np.int64), want["threshold"].astype(np.float64).view(np.int64))
    np.testing.assert_array_equal(tree.counts, np.array(want["counts"], np.float64).reshape(tree.counts.shape))
    np.testing.assert_array_equal(tree.impurity.view(np.int64), want["impurity"].astype(np.float64).view(np.int64))
    np.testing.assert_array_equal(tree.gain.view(np.int64), want["gain"].astype(np.float64).view(np.int64))


def _data(n, k, C, seed, distinct=None):
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(n, k))
    if distinct:
        x = np.round(x * distinct / 6) / 4
    w = rng.normal(size=(k, C))
    y = (x @ w + rng.gumbel(size=(n, C))).argmax(1).astype(np.float64)
    return x, y


@pytest.mark.parametrize("kind", ["gini", "entropy"])
@pytest.mark.parametrize("params", [dict(), dict(max_depth=0), dict(max_depth=2, max_bins=4), dict(min_inst=40),
                                    dict(min_gain=0.05), dict(max_depth=8, max_bins=7)])
def test_growth_matches_the_oracle(kind, params):
    x, y = _data(1500, 4, 3, seed=len(params) + len(kind))
    oracle = dict(max_depth=params.get("max_depth", 5), max_bins=params.get("max_bins", 32),
                  min_inst=params.get("min_inst", 1), min_gain=params.get("min_gain", 0.0), kind=kind)
    root, _thr = to.fit(x, y, **oracle)
    _assert_same_tree(_host_tree(x, y, oracle["max_depth"], oracle["max_bins"], oracle["min_inst"], oracle["min_gain"],
                                 kind), to.arrays(root))


def test_growth_edges():
    x, y = _data(300, 3, 2, seed=5)
    for xx, yy in ((x, np.zeros(300)), (np.ones((300, 3)), y), (x[:5], y[:5])):
        root, _ = to.fit(xx, yy)
        _assert_same_tree(_host_tree(xx, yy), to.arrays(root))
    root, _ = to.fit(np.ones((300, 3)), y)
    assert root["leaf"] and root["impurity"] == -1.0          # no feature has a split: invalid stats


def test_pruning_merges_leaves_of_one_prediction():
    rng = np.random.default_rng(11)
    x = rng.uniform(size=(2000, 2))
    y = ((x[:, 0] > 0.5) & (rng.uniform(size=2000) < 0.9)).astype(np.float64)   # class 0 dominates one side
    root, _ = to.fit(x, y, max_depth=6)
    tree = _host_tree(x, y, max_depth=6)
    _assert_same_tree(tree, to.arrays(root))
    unpruned = T.grow(_numpy_level(x, y, [to.splits(x[:, j], 32) for j in range(2)], 2), [to.splits(x[:, j], 32)
                      for j in range(2)], 2, 6, "gini", 1, 0.0)[1]
    assert sum(unpruned) * 2 + 1 > tree.num_nodes              # the growth made more nodes than the pruned tree keeps


@pytest.mark.parametrize("kind", ["gini", "entropy"])
@pytest.mark.parametrize("depth", [1, 2, 3])
def test_oracle_agrees_with_scikit_learn(kind, depth):
    tree_mod = pytest.importorskip("sklearn.tree")
    x, y = _data(3000, 5, 3, seed=depth, distinct=20)
    assert all(len(np.unique(x[:, j])) <= 32 for j in range(5))    # every midpoint is a candidate on both sides
    ties = []
    root, _ = to.fit(x, y, max_depth=depth, kind=kind, ties=ties)
    assert min(ties) > 1e-12                                      # no two candidates of a node within 1e-12
    sk = tree_mod.DecisionTreeClassifier(criterion=kind, max_depth=depth, random_state=0).fit(x, y)
    _raw, _prob, pred = to.transform(root, x)
    np.testing.assert_array_equal(pred, sk.predict(x))


# ---- parameters, caps and the classifier with stand-in engines ---------------------------------------------------
@pytest.mark.parametrize("kw", [dict(max_depth=-1), dict(max_depth=31), dict(max_depth=2.5), dict(max_depth=True),
                                dict(max_bins=1), dict(max_bins=257), dict(min_instances_per_node=0),
                                dict(min_info_gain=-0.1), dict(min_info_gain=float("nan")), dict(impurity="variance"),
                                dict(impurity=None)])
def test_parameters_are_refused_as_spark_refuses_them(kw):
    with pytest.raises(ValueError):
        DecisionTreeClassifier(**kw)


def test_parameter_bounds_are_accepted():
    DecisionTreeClassifier(max_depth=0, max_bins=2)
    DecisionTreeClassifier(max_depth=30, max_bins=256, impurity="Entropy", min_info_gain=0.0)


def test_equal_midpoints_give_equal_thresholds_and_java_bins():
    thr = T.greedy(EQUAL_MIDPOINTS, [1, 1, 1], 31, 3)
    assert thr == [1.0, 1.0] == to.splits(EQUAL_MIDPOINTS, 32)
    # java.util.Arrays.binarySearch on [1.0, 1.0] lands on index 0 (mid = 0 first); the others are insertion points
    assert to.binary_search(thr, EQUAL_MIDPOINTS).tolist() == [0, 0, 2]
    assert to.binary_search([0.5, 1.0, 1.0, 1.0, 2.0], np.array([1.0])).tolist() == [2]
    assert to.binary_search([1.0, 1.0, 1.0], np.array([1.0])).tolist() == [1]
    assert to.binary_search([0.0], np.array([-0.0])).tolist() == [0]          # -0.0's bits order below 0.0's
    rng = np.random.default_rng(8)
    for _ in range(50):                                 # without equal thresholds: the count of thresholds below x
        t = np.unique(rng.integers(-20, 20, int(rng.integers(1, 30))).astype(np.float64) / 2)
        x = rng.integers(-25, 25, 300).astype(np.float64) / 2
        np.testing.assert_array_equal(to.binary_search(t, x), np.searchsorted(t, x, side="left"))
    x = np.concatenate([np.repeat(EQUAL_MIDPOINTS, 30), np.linspace(-2, 3, 50)])[:, None]
    y = (x[:, 0] >= 1.0).astype(np.float64)
    root, _ = to.fit(x, y)
    _assert_same_tree(_host_tree(x, y), to.arrays(root))


class StandInEngine:
    """An Engine's dt_* and lr_stats on numpy rows: every call made on the host, for the classifier's plumbing."""

    def __init__(self):
        self.calls = []

    def lr_stats(self, part):
        x, y = part
        counts = np.bincount(y.astype(np.int64), minlength=N.LO_NB_MAX_CLASSES)
        return len(y), x.sum(0), np.zeros(x.shape[1]), counts

    def dt_sort(self, part, j0, kc, cap):
        x, _y = part
        self.calls.append(("sort", j0, kc))
        distinct = []
        for c in range(kc):
            v, n = to.value_counts(x[:, j0 + c])
            distinct.append((len(v), v if len(v) <= cap else None, n if len(v) <= cap else None))
        return SimpleNamespace(distinct=distinct, x=x[:, j0:j0 + kc], free=lambda: None)

    def dt_rank(self, s, cols, probes):
        codes = [np.sort(np.array([T.encode(float(v), False) for v in s.x[:, c]], np.uint64)) for c in range(s.x.shape[1])]
        lt = np.array([np.searchsorted(codes[c], p, "left") for c, p in zip(cols, probes)], np.int64)
        le = np.array([np.searchsorted(codes[c], p, "right") for c, p in zip(cols, probes)], np.int64)
        return lt, le

    def dt_bin(self, part, thr):
        x, y = part
        return SimpleNamespace(level=None, rows=(x, y, thr), free=lambda: None)

    def dt_level(self, part, binned, nbins, C, splits, nnodes, shape=None):
        if binned.level is None:                        # the level's shape is the caller's, as on the device
            binned.level = _numpy_level(*binned.rows, C, nbins)
        return binned.level(splits, nnodes)

    def dt_predict(self, part, tree, raw=False, labels=None):
        from learningorchestra_b200.engine import InvalidCellError
        x, y = part
        node = np.zeros(len(y), np.int64)
        for _ in range(tree.num_nodes):
            f = tree.feature[node]
            inner = f >= 0
            go_left = x[np.arange(len(y)), np.maximum(f, 0)] <= tree.threshold[node]
            node = np.where(inner, np.where(go_left, tree.left[node], tree.right[node]), node)
        prob = tree.counts[node] / tree.counts[node].sum(1, keepdims=True)
        pred = prob.argmax(1)
        if labels is None:
            return SimpleNamespace(prob=prob, pred=pred, free=lambda: None)
        slot = np.searchsorted(labels, y)
        bad = np.flatnonzero((slot >= len(labels)) | (labels[np.minimum(slot, len(labels) - 1)] != y))
        if len(bad):
            raise InvalidCellError(bad[0], x.shape[1], reason="row {row}: its label is not one of the evaluated labels")
        conf = np.zeros((len(labels), tree.num_classes), np.int64)
        np.add.at(conf, (slot, pred), 1)
        return conf


def _stand_in_features(x, y):
    engine = StandInEngine()
    parts = [SimpleNamespace(x=SimpleNamespace(dtype_code=N.LO_F64))]
    feats = SimpleNamespace(_frame=SimpleNamespace(_cache=SimpleNamespace(engine=engine)), _parts=parts,
                            fields=[f"f{j}" for j in range(x.shape[1])], label="y", row_ids=np.arange(len(y)))
    feats._parts = [_Part((x, y))]
    return feats, engine


class _Part(tuple):
    x = SimpleNamespace(dtype_code=N.LO_F64)

    @property
    def nkept(self):
        return len(self[1])


def test_classifier_fits_the_oracles_tree_through_stand_in_engines():
    x, y = _data(800, 3, 3, seed=2)
    x[:, 1] = np.round(x[:, 1] * 3)                    # a column with few distinct values: the listed path
    feats, engine = _stand_in_features(x, y)
    m = DecisionTreeClassifier(max_depth=4, max_bins=10).fit(feats)
    root, thr = to.fit(x, y, max_depth=4, max_bins=10)
    _assert_same_tree(m.tree, to.arrays(root))
    assert m.thresholds == thr and m.num_classes == 3 and m.depth <= 4


def test_classifier_refuses_caps_before_any_pass():
    x, y = _data(100, 2, 2, seed=1)
    feats, engine = _stand_in_features(x, y * 101)     # labels 0 and 101: 102 classes
    with pytest.raises(N.LoexecError, match="LO_DT_MAX_CLASSES"):
        DecisionTreeClassifier().fit(feats)
    assert not engine.calls
    wide = np.zeros((256, 5243))                       # 5243 x 256 bins x 100 classes x 8 bytes: just above 2^30
    assert 5242 * 256 * 100 * 8 <= N.LO_DT_PASS_HIST < 5243 * 256 * 100 * 8
    feats, engine = _stand_in_features(wide, (np.arange(256) % 100).astype(np.float64))
    with pytest.raises(N.LoexecError, match="LO_DT_PASS_HIST"):
        DecisionTreeClassifier(max_bins=256).fit(feats)
    assert not engine.calls
    feats, _ = _stand_in_features(np.zeros((0, 2)), np.zeros(0))
    feats._frame._cache.engine.lr_stats = lambda part: (0, np.zeros(2), np.zeros(2), np.zeros(1024, np.int64))
    with pytest.raises(N.LoexecError, match="at least one row"):
        DecisionTreeClassifier().fit(feats)


def test_sharded_merges_add_in_shard_order():
    from learningorchestra_b200.sharding import ShardedEngine
    x, y = _data(600, 2, 2, seed=4)
    members = [StandInEngine() for _ in range(3)]
    sh = object.__new__(ShardedEngine)
    sh._N, sh.world, sh.nlocal, sh.engines = N, 3, 3, members
    bounds = [0, 100, 350, 600]
    parts = [(x[a:b], y[a:b]) for a, b in zip(bounds[:-1], bounds[1:])]
    sorted_ = sh.dt_sort(parts, 0, 2, 400)
    cols, probes = np.array([0, 1]), np.array([T.encode(0.0, False), T.encode(0.5, False)], np.uint64)
    lt, le = sh.dt_rank(sorted_, cols, probes)
    assert lt.tolist() == [int((x[:, 0] < 0).sum()), int((x[:, 1] < 0.5).sum())]
    assert le.tolist() == [int((x[:, 0] <= 0).sum()), int((x[:, 1] <= 0.5).sum())]
    thr = [to.splits(x[:, j], 32) for j in range(2)]
    binned = [m.dt_bin(p, thr) for m, p in zip(members, parts)]
    hist = sh.dt_level(parts, binned, 32, 2, None, 1)
    whole = _numpy_level(x, y, thr, 2)(None, 1)
    np.testing.assert_array_equal(hist, whole)


# ---- launch shape, header, SASS -----------------------------------------------------------------------------------
def _constant(name, text):
    return int(eval(re.search(rf"constexpr \w+(?: \w+)? {name} = ([^;]+);", text).group(1).replace("ll", "")))


def shape(k, nbins, C, nnodes, hist_smem, pass_hist, vec=16):
    """Python restatement of dt_shape (loexec.cu): (16-byte loads, features per chunk, nodes per pass, passes)."""
    cell = nbins * C * 4
    cells = hist_smem // cell
    kpad = (k + vec - 1) // vec * vec
    use_vec = cells >= vec
    fc = min(kpad, cells // vec * vec) if use_vec else min(k, cells)
    gn = max(1, min(max(nnodes, 1), cells // fc, pass_hist // (k * nbins * C * 8)))
    return int(use_vec), fc, gn, (max(nnodes, 1) + gn - 1) // gn


def test_launch_shape_restatement_is_pinned_to_the_sources():
    text = (CSRC / "tree.cuh").read_text()
    hist_smem, pass_hist = _constant("kDtHistSmem", text), _constant("kDtPassHist", text)
    assert hist_smem == 112 * 1024 and pass_hist == N.LO_DT_PASS_HIST and _constant("kDtVec", text) == 16
    cu = (CSRC / "loexec.cu").read_text()
    body = cu[cu.index("DtShape dt_shape("):cu.index("template <typename K>\nvoid dt_sort_columns")]
    for piece in ("cells >= lo::kDtVec", "cells / lo::kDtVec * lo::kDtVec", "std::min<int64_t>(k, cells)",
                  "lo::kDtPassHist / ((int64_t)k * nbins * C * 8)", "cells / sh.fc"):
        assert piece in body, piece
    assert shape(20, 32, 2, 1, hist_smem, pass_hist) == (1, 32, 1, 1)
    assert shape(20, 32, 2, 64, hist_smem, pass_hist) == (1, 32, 14, 5)
    assert shape(3, 256, 100, 4, hist_smem, pass_hist) == (0, 1, 1, 4)
    assert shape(2000, 32, 2, 1, hist_smem, pass_hist)[1] == 448


def test_header_mirror_matches():
    text = (ROOT / "include" / "loexec.h").read_text()
    for name in ("LO_DT_MAX_BINS", "LO_DT_MAX_CLASSES", "LO_DT_PASS_HIST"):
        assert int(re.search(rf"#define {name}\s+(\d+)", text).group(1)) == getattr(N, name)
    assert N.LO_DT_MAX_BINS == T.MAX_BINS and N.LO_DT_MAX_CLASSES == T.MAX_CLASSES
    for fn in ("lo_dt_sort", "lo_dt_rank", "lo_dt_bin", "lo_dt_level", "lo_dt_predict"):
        decl = re.search(rf"int {fn}\(([^;]*)\);", text, re.S).group(1)
        assert len(decl.split(",")) == len(N.SIGNATURES[fn][1]), fn
    assert N.LO_ABI_VERSION == 7


def _sass(built, prefix):
    from learningorchestra_b200 import _native
    full = subprocess.run(["cuobjdump", "-sass", str(_native.LIB_PATH)], capture_output=True, text=True).stdout
    funcs = [f for f in full.split("Function : ")[1:] if f.startswith(prefix)]
    assert funcs, prefix
    return funcs


def test_sass_of_the_tree_kernels(built):
    for prefix in ("_ZN2lo9k_dt_keys", "_ZN2lo13k_dt_distinct", "_ZN2lo9k_dt_rank", "_ZN2lo8k_dt_bin",
                   "_ZN2lo10k_dt_level", "_ZN2lo12k_dt_predict"):
        for f in _sass(built, prefix):
            assert "LDL" not in f and "STL" not in f, prefix          # no local memory
    vec_bin = [f for f in _sass(built, "_ZN2lo8k_dt_bin") if "Li1EE" not in f.split("\n")[0]]
    vec_level = [f for f in _sass(built, "_ZN2lo10k_dt_level") if "Lb1EE" in f.split("\n")[0]]
    assert vec_bin and vec_level
    for f in vec_bin + vec_level:
        assert "LDG.E.NA.128" in f                                    # 16-byte read-once loads


def _stand_in_sharded(x, y, bounds):
    from learningorchestra_b200.sharding import ShardedEngine
    sh = object.__new__(ShardedEngine)
    sh._N, sh.world, sh.nlocal, sh.engines = N, len(bounds) - 1, len(bounds) - 1, [StandInEngine() for _ in bounds[1:]]
    parts = [_Part((x[a:b], y[a:b])) for a, b in zip(bounds[:-1], bounds[1:])]
    feats = SimpleNamespace(_frame=SimpleNamespace(_cache=SimpleNamespace(engine=sh)), _parts=parts,
                            fields=[f"f{j}" for j in range(x.shape[1])], label="y", row_ids=np.arange(100, 100 + len(y)))
    return feats, sh, parts


def test_sharded_fit_and_predict_through_stand_in_engines():
    x, y = _data(900, 3, 3, seed=12)
    x[:, 0] = np.round(x[:, 0] * 2)
    feats, sh, parts = _stand_in_sharded(x, y, [0, 200, 201, 900])
    m = DecisionTreeClassifier(max_depth=4).fit(feats)
    root, thr = to.fit(x, y, max_depth=4)
    _assert_same_tree(m.tree, to.arrays(root))
    assert m.thresholds == thr
    labels = np.unique(y)
    conf = sh.dt_predict(parts, m.tree, labels=labels)           # the members' counts summed
    _raw, _prob, pred = to.transform(root, x)
    want = np.zeros((len(labels), m.num_classes), np.int64)
    np.add.at(want, (np.searchsorted(labels, y), pred.astype(np.int64)), 1)
    np.testing.assert_array_equal(conf, want)
    y2 = y.copy()
    y2[[450, 899]] = 7.0                                  # unknown labels in the last shard: the lowest, made global
    feats, sh, parts = _stand_in_sharded(x, y2, [0, 200, 201, 900])
    from learningorchestra_b200.engine import InvalidCellError
    with pytest.raises(InvalidCellError) as e:
        sh.dt_predict(parts, m.tree, labels=labels)
    assert e.value.row == 450 and e.value.position == 3
