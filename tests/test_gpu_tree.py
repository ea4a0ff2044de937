"""GPU: the builder's "DT" classifier (Spark 2.4's DecisionTreeClassifier) over the feature matrix in HBM against the
numpy restatement in tests/tree_oracle.py — thresholds and bin codes bit for bit, every level's histogram exactly on
every launch route, whole trees node for node, transform and evaluate, the edges, refused cells, the caps, on one GPU
and on shard cuts."""
import numpy as np
import pytest

import tree_oracle as to
from learningorchestra_b200 import _native as N
from learningorchestra_b200 import tree as T
from learningorchestra_b200.classifier import DecisionTreeClassifier
from learningorchestra_b200.engine import InvalidCellError
from test_gpu_logistic import _cut, _sharded
from test_gpu_naive_bayes import _features, _free, _host, _part

pytestmark = pytest.mark.gpu


def _data(n, k, C, seed, dtype=np.float64, distinct=None):
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(n, k)) * rng.uniform(0.5, 3.0, k)
    if distinct:
        x = np.round(x * distinct / 6)
    w = rng.normal(size=(k, C))
    y = (x.astype(dtype).astype(np.float64) @ w + 2 * rng.gumbel(size=(n, C))).argmax(1).astype(np.float64)
    return x.astype(dtype), y


def _on(engine, x, y, cuts):
    """(features, parts, engine) of x, y on one GPU (cuts 1) or cut into `cuts` shards of this device."""
    if cuts == 1:
        parts = [_part(engine, x, y)]
        return _features(engine, parts, x.shape[1]), parts
    parts = _cut(engine, x, y, cuts)
    return _features(_sharded(engine, cuts), parts, x.shape[1]), parts


def _same_tree(tree, want):
    assert tree.feature.tolist() == want["feature"].tolist()
    assert tree.left.tolist() == want["left"].tolist() and tree.right.tolist() == want["right"].tolist()
    np.testing.assert_array_equal(tree.threshold.view(np.int64), want["threshold"].astype(np.float64).view(np.int64))
    np.testing.assert_array_equal(tree.counts, np.array(want["counts"], np.float64).reshape(tree.counts.shape))
    np.testing.assert_array_equal(tree.impurity.view(np.int64), want["impurity"].astype(np.float64).view(np.int64))
    np.testing.assert_array_equal(tree.gain.view(np.int64), want["gain"].astype(np.float64).view(np.int64))


def _check_fit(engine, x, y, cuts=1, **params):
    feats, parts = _on(engine, x, y, cuts)
    try:
        m = DecisionTreeClassifier(**params).fit(feats)
        o = dict(max_depth=params.get("max_depth", 5), max_bins=params.get("max_bins", 32),
                 min_inst=params.get("min_instances_per_node", 1), min_gain=params.get("min_info_gain", 0.0),
                 kind=params.get("impurity", "gini"))
        root, thr = to.fit(x, y, **o)
        for got, want in zip(m.thresholds, thr):
            np.testing.assert_array_equal(np.array(got, np.float64).view(np.int64), np.array(want, np.float64).view(np.int64))
        _same_tree(m.tree, to.arrays(root))
        raw, prob, pred = to.transform(root, x)
        with m.transform(feats, raw=True) as out:
            d = feats.devices[0]
            got_raw = np.concatenate([_host(r, d) for r in out.raw])
            got_prob = np.concatenate([_host(p, d) for p in out.probability])
            got_pred = np.concatenate([_host(p, d) for p in out.prediction])
        np.testing.assert_array_equal(got_raw.view(np.int64), raw.view(np.int64))
        np.testing.assert_array_equal(got_prob.view(np.int64), prob.view(np.int64))
        np.testing.assert_array_equal(got_pred, pred)
        ev = m.evaluate(feats)
        labels = np.unique(y)
        want_conf = np.zeros((len(labels), m.num_classes), np.int64)
        np.add.at(want_conf, (np.searchsorted(labels, y), pred.astype(np.int64)), 1)
        np.testing.assert_array_equal(ev["confusion"], want_conf)
        return m, root
    finally:
        _free(parts)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("cuts", [1, 2, 3, 8])
def test_fit_transform_evaluate_match_the_oracle(engine, dtype, cuts):
    x, y = _data(6007, 5, 3, seed=cuts, dtype=dtype)
    x[:, 2] = np.round(x[:, 2])                      # few distinct values: the listed path beside the rank path
    x[:100, 3] = -0.0
    x[100:200, 3] = 0.0
    m, _root = _check_fit(engine, x, y, cuts)
    assert m.num_nodes > 7 and m.rank_rounds >= 2


@pytest.mark.parametrize("impurity", ["gini", "entropy"])
def test_entropy_and_gini_trees(engine, impurity):
    x, y = _data(5000, 4, 4, seed=7)
    _check_fit(engine, x, y, impurity=impurity, max_depth=7)


@pytest.mark.parametrize("params", [dict(max_depth=0), dict(min_instances_per_node=300), dict(min_info_gain=0.02),
                                    dict(max_bins=2), dict(max_bins=256, max_depth=3), dict(max_depth=12)])
def test_edges(engine, params):
    x, y = _data(4000, 3, 2, seed=len(params))
    _check_fit(engine, x, y, **params)


def test_constant_label_and_constant_columns(engine):
    x, y = _data(1000, 3, 2, seed=9)
    m, root = _check_fit(engine, x, np.zeros(1000))
    assert m.num_nodes == 1
    m, root = _check_fit(engine, np.full((1000, 3), 0.1), y)
    assert m.num_nodes == 1 and m.tree.impurity[0] == -1.0


def test_pruning_merges_leaves(engine):
    rng = np.random.default_rng(11)
    x = rng.uniform(size=(3000, 2))
    y = ((x[:, 0] > 0.5) & (rng.uniform(size=3000) < 0.9)).astype(np.float64)
    _check_fit(engine, x, y, max_depth=6)


def test_fewer_rows_than_bins(engine):
    x, y = _data(20, 3, 2, seed=3)
    _check_fit(engine, x, y)
    _check_fit(engine, x[:1], y[:1])


def _level_routes(engine, x, y, thr, C, cuts=1):
    """Every level of a tree grown through the device, compared with a numpy restatement of the same routing; the
    launch shapes met."""
    feats, parts = _on(engine, x, y, cuts)
    eng = feats._frame._cache.engine
    rows = parts if cuts > 1 else parts[0]
    codes = to.bins(x, thr)
    nbins = max(len(t) for t in thr) + 1
    shapes = []
    try:
        binned = eng.dt_bin(rows, thr)
        try:
            got_codes = np.concatenate([b.codes.to_numpy(0)[:p.nkept * ((x.shape[1] + 15) // 16 * 16)]
                                        .reshape(p.nkept, -1)[:, :x.shape[1]]
                                        for b, p in zip(binned if cuts > 1 else [binned], parts)])
            np.testing.assert_array_equal(got_codes, codes)
            state = {}

            def level(splits, nnodes):
                sh = []
                hist = eng.dt_level(rows, binned, nbins, C, splits, nnodes, sh)
                shapes.append(tuple(sh))
                if splits is None:
                    slot = np.zeros(len(y), np.int64)
                else:
                    p = state["slot"]
                    s = splits[np.maximum(p, 0)]
                    f = np.where(p >= 0, s[:, 0], -1)
                    c = codes[np.arange(len(y)), np.maximum(f, 0)]
                    slot = np.where(f >= 0, np.where(c <= s[:, 1], s[:, 2], s[:, 3]), -1)
                state["slot"] = slot
                want = np.zeros_like(hist)
                live = slot >= 0
                for j in range(x.shape[1]):
                    np.add.at(want, (slot[live], j, codes[live, j], y[live].astype(np.int64)), 1)
                np.testing.assert_array_equal(hist, want)
                return hist

            T.grow(level, thr, C, 8, "gini", 1, 0.0)
        finally:
            for b in binned if cuts > 1 else [binned]:
                b.free()
    finally:
        _free(parts)
    return shapes


def test_every_level_on_every_route(engine):
    routes = set()
    cases = [(_data(20_000, 6, 3, seed=1), 32, 1),                    # 16-byte loads, one chunk, node groups of many
             (_data(20_000, 6, 3, seed=2, dtype=np.float32), 32, 3),
             (_data(5_000, 600, 2, seed=3), 32, 1),                    # wide k: several feature chunks
             (_data(30_000, 3, 100, seed=4), 256, 2)]                  # 256 bins x 100 classes: scalar route
    for (x, y), bins, cuts in cases:
        thr = [to.splits(x[:, j], bins) for j in range(x.shape[1])]
        C = int(y.max()) + 1
        for vec, fc, gn, passes in _level_routes(engine, x, y, thr, C, cuts):
            routes.add((vec, fc < ((x.shape[1] + 15) // 16 * 16 if vec else x.shape[1]), passes > 1))
    assert {r[0] for r in routes} == {0, 1}                          # 16-byte and scalar code loads
    assert any(r[1] for r in routes)                                 # more than one feature chunk
    assert any(r[2] for r in routes)                                 # more than one node group


def test_refused_cells_name_the_id_and_field(engine):
    x, y = _data(3000, 3, 2, seed=5)
    x[1234, 1] = np.nan
    for cuts in (1, 2, 3, 8):
        feats, parts = _on(engine, x, y, cuts)
        try:
            with pytest.raises(InvalidCellError, match="DecisionTreeClassifier: field 'f1' of the row with _id 1334"):
                DecisionTreeClassifier().fit(feats)
        finally:
            _free(parts)
    y2 = y.copy()
    y2[77] = 0.5
    feats, parts = _on(engine, np.nan_to_num(x), y2, 3)
    try:
        with pytest.raises(InvalidCellError, match="_id 177"):
            DecisionTreeClassifier().fit(feats)
    finally:
        _free(parts)


def test_class_cap_at_its_boundary(engine):
    x, y = _data(500, 2, 2, seed=6)
    y[0] = 99
    _check_fit(engine, x, y, max_depth=2)
    y[0] = 100
    feats, parts = _on(engine, x, y, 1)
    try:
        with pytest.raises(N.LoexecError, match="LO_DT_MAX_CLASSES"):
            DecisionTreeClassifier().fit(feats)
    finally:
        _free(parts)


@pytest.mark.parametrize("cuts", [1, 3])
def test_evaluate_counts_on_both_routes(engine, cuts):
    """100 classes: their 100 labels' counts (39 KiB) sit in shared memory beside the tree; 300 evaluated labels (117
    KiB, past kDtTreeSmem = 96 KiB) are counted straight into global memory."""
    x, y = _data(3000, 3, 2, seed=8)
    y[:98] = np.arange(2, 100)
    m, root = _check_fit(engine, x, y, cuts, max_depth=3)
    assert m.num_classes == 100
    _raw, _prob, pred = to.transform(root, x)
    y_eval = (np.arange(len(y)) % 300) * 0.5
    feats, parts = _on(engine, x, y_eval, cuts)
    try:
        ev = m.evaluate(feats)
    finally:
        _free(parts)
    labels = np.unique(y_eval)
    want = np.zeros((len(labels), 100), np.int64)
    np.add.at(want, (np.searchsorted(labels, y_eval), pred.astype(np.int64)), 1)
    np.testing.assert_array_equal(ev["confusion"], want)


def test_equal_adjacent_thresholds_fit_like_spark(engine):
    """Midpoints of three neighbouring doubles round to one value: two equal thresholds, binned by Java's binary search."""
    rng = np.random.default_rng(21)
    trio = np.array([np.nextafter(1.0, 0.0), 1.0, np.nextafter(1.0, 2.0)])
    x = np.stack([np.repeat(trio, 700), rng.normal(size=2100)], 1)
    y = ((x[:, 0] >= 1.0) ^ (rng.uniform(size=2100) < 0.1)).astype(np.float64)
    m, _root = _check_fit(engine, x, y)
    assert list(m.thresholds[0]) == [1.0, 1.0]
    x2 = np.concatenate([x, np.stack([rng.normal(size=500), rng.normal(size=500)], 1)])
    y2 = np.concatenate([y, (rng.uniform(size=500) < 0.5).astype(np.float64)])
    for cuts in (1, 3):
        _check_fit(engine, x2, y2, cuts, max_depth=6)


def test_the_c_abi_refuses_before_any_launch(engine):
    import ctypes as C
    x, y = _data(300, 3, 2, seed=13)
    part = _part(engine, x, y)
    try:
        with pytest.raises(N.LoexecError, match="cap = 258"):
            engine.dt_sort(part, 0, 3, 258)
        with pytest.raises(N.LoexecError, match="outside"):
            engine.dt_sort(part, 2, 2, 32)
        nd = np.zeros(3, np.int64)
        with pytest.raises(N.LoexecError, match="2\\^31"):
            N.check(engine._lib.lo_dt_sort(engine._ctx, part.x._h, 3, 3, 1 << 31, 0, 3, part.x._h, 0,
                                           nd.ctypes.data_as(C.c_void_p), None, None, None))
        s = engine.dt_sort(part, 0, 3, 32)
        try:
            with pytest.raises(N.LoexecError, match="cols\\[0\\] = 3"):
                engine.dt_rank(s, [3], [0])
        finally:
            s.free()
        with pytest.raises(N.LoexecError, match="not ascending"):
            engine.dt_bin(part, [[2.0, 1.0], [], []])
        with pytest.raises(N.LoexecError, match="not ascending"):
            engine.dt_bin(part, [[np.nan, 1.0], [], []])
        thr = [to.splits(x[:, j], 8) for j in range(3)]
        binned = engine.dt_bin(part, thr)
        try:
            with pytest.raises(N.LoexecError, match="code >= nbins = 2"):
                engine.dt_level(part, binned, 2, 2, None, 1)
            with pytest.raises(N.LoexecError, match="its label is not a class in \\[0, 1\\)"):
                engine.dt_level(part, binned, 8, 1, None, 1)
            engine.dt_level(part, binned, 8, 2, None, 1)
            for bad in ([[3, 0, 0, 0]], [[0, 8, 0, 0]], [[0, 0, 2, 0]], [[0, 0, 0, -2]]):
                with pytest.raises(N.LoexecError, match="out of range"):
                    engine.dt_level(part, binned, 8, 2, np.array(bad, np.int32), 2)
            with pytest.raises(N.LoexecError, match="LO_DT_PASS_HIST"):
                N.check(engine._lib.lo_dt_level(
                    engine._ctx, binned.codes._h, 5248, 5243, part.y._h, 0, 256, 100, None, 0, None, 0, None, 1,
                    np.zeros(1, np.int64).ctypes.data_as(C.c_void_p), None, None))
        finally:
            binned.free()

        def tree(feature, left, right):
            M = len(feature)
            return T.Tree(feature, np.zeros(M), left, right, np.ones((M, 2)), np.zeros(M), np.zeros(M), 2)

        for t in (tree([0, -1, -1], [0, -1, -1], [2, -1, -1]), tree([0, -1, -1], [1, -1, -1], [3, -1, -1]),
                  tree([3, -1, -1], [1, -1, -1], [2, -1, -1])):
            with pytest.raises(N.LoexecError, match="node 0"):
                engine.dt_predict(part, t)
    finally:
        part.free()


NUMBER_FIELDS = ["PassengerId", "Survived", "Pclass", "Age", "SibSp", "Parch", "Fare"]


@pytest.mark.parametrize("sharded", [False, True])
def test_titanic_end_to_end(engine, tmp_path, sharded):
    """Ingest, the field types, DeviceFrame.features and fit / transform / evaluate: the oracle's tree node for node,
    its predictions, and MulticlassMetrics' f1 and accuracy of them."""
    import csv
    import json
    from pathlib import Path
    from werkzeug.test import Client
    from learningorchestra_b200 import builder_frontend, server
    from learningorchestra_b200.column_store import ColumnarDatabase
    from learningorchestra_b200.sharding import ShardedEngine
    from oracle import naive_bayes as nb
    g = json.loads((Path(__file__).resolve().parent / "golden" / "titanic_shaped_input.json").read_text())
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
                m = DecisionTreeClassifier().fit(feats)
                root, thr = to.fit(x, y)
                _same_tree(m.tree, to.arrays(root))
                assert m.num_classes == 2 and m.num_nodes > 3
                _raw, prob, pred = to.transform(root, x)
                with m.transform(feats) as out:
                    got = np.concatenate([_host(v, d) for v, d in zip(out.prediction, out.devices)])
                    np.testing.assert_array_equal(got, pred)
                    p = np.concatenate([_host(v, d) for v, d in zip(out.probability, out.devices)])
                    np.testing.assert_array_equal(p.view(np.int64), prob.view(np.int64))
                ev = m.evaluate(feats)
                f1, acc = nb.metrics(y, pred)
                assert abs(ev["f1"] - f1) <= 1e-15 and ev["accuracy"] == acc
        eng.resident.clear()
    finally:
        if sharded:
            eng.close()
