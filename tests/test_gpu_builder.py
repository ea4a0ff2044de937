"""GPU: the builder route end to end (``POST /models``) and its two kernels — ``lo_random_split`` (Spark's randomSplit
over the feature matrix) bit for bit against a numpy restatement, and ``lo_text_codes_in`` (test cells coded by the
training dictionary) against a host lookup — on one GPU and on shard cuts."""
import csv
import json
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pyarrow as pa
import pytest
from werkzeug.test import Client

from learningorchestra_b200 import _native as N
from learningorchestra_b200 import builder_frontend, server
from learningorchestra_b200.classifier import (DecisionTreeClassifier, GBTClassifier, LogisticRegression, NaiveBayes,
                                               RandomForestClassifier)
from learningorchestra_b200.column_store import ColumnarDatabase
from learningorchestra_b200.engine import SPLIT_SEED, split_bounds
from learningorchestra_b200.sharding import ShardedEngine, ShardedText
from learningorchestra_b200.tree import splitmix
from test_gpu_logistic import _sharded
from test_gpu_naive_bayes import _part

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).resolve().parent / "golden"


# ---- random_split ---------------------------------------------------------------------------------------------------
def _draw(seed, ids):
    key = splitmix(np.uint64(~int(seed) & 0xFFFFFFFFFFFFFFFF))
    z = splitmix(np.asarray(ids, np.int64).view(np.uint64) ^ key)
    return (z >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def _oracle_split(ids, bounds, seed):
    """Per split, the indices (into ids) of its rows, in order: int64 arithmetic and boolean indexing."""
    u = _draw(seed, ids)
    return [np.nonzero((u >= bounds[s]) & (u < bounds[s + 1]))[0] for s in range(len(bounds) - 1)]


def _host(part):
    x = part.x.to_numpy(0, nrows=part.nkept * part.k).reshape(part.nkept, part.k)
    y = part.y.to_numpy(0, nrows=part.nkept) if part.y is not None else None
    return x, y


def _check_split(engine, x, y, ids, weights, seed, cuts=1, bounds=None):
    bounds = split_bounds(weights) if bounds is None else np.asarray(bounds, np.float64)
    want = _oracle_split(ids, bounds, seed)
    cut = np.linspace(0, len(ids), cuts + 1).astype(int)
    parts = [_part(engine, x[a:b], y[a:b]) for a, b in zip(cut[:-1], cut[1:])]
    for p, a in zip(parts, cut[:-1]):
        p.first = int(a)
    try:
        if cuts == 1:
            got = [[s] for s in engine.random_split(parts[0], ids, bounds, seed)]
        else:
            got = _sharded(engine, cuts).random_split(parts, [ids[a:b] for a, b in zip(cut[:-1], cut[1:])], bounds, seed)
        assert len(got) == len(weights)
        for rows, per_part in zip(want, got):
            gx = np.concatenate([_host(p)[0] for p in per_part])
            gy = np.concatenate([_host(p)[1] for p in per_part])
            np.testing.assert_array_equal(np.concatenate([p.rows for p in per_part]), rows)
            assert gx.dtype == x.dtype
            np.testing.assert_array_equal(gx.view(np.uint8), x[rows].view(np.uint8))
            np.testing.assert_array_equal(gy.view(np.uint8), y[rows].view(np.uint8))
            for p in per_part:
                p.free()
        return [len(r) for r in want]
    finally:
        for p in parts:
            p.free()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("cuts", [1, 2, 3])
def test_split_against_the_oracle(engine, dtype, cuts):
    rng = np.random.default_rng(11)
    n, k = 50_021, 7
    x = rng.normal(size=(n, k)).astype(dtype)
    x[::97, 3] = np.nan
    y = rng.integers(0, 3, n).astype(dtype)
    ids = np.arange(1, n + 1, dtype=np.int64) * 3 - (np.arange(n) % 2)          # not dense: skipped rows
    sizes = _check_split(engine, x, y, ids, [0.7, 0.2, 0.1], 1234, cuts)
    assert sum(sizes) == n and all(s > 0 for s in sizes)
    _check_split(engine, x, y, ids, [1.0], SPLIT_SEED, cuts)                  # one weight: every row, in order
    sizes = _check_split(engine, x, y, ids, [0.5, 0.0, 0.5], -5, cuts)         # a zero weight: an empty split
    assert sizes[1] == 0


def test_rows_at_or_above_the_last_bound_go_nowhere(engine):
    """A last bound below 1 (as one that rounded below 1.0 is) leaves the rows drawn above it out of every split."""
    rng = np.random.default_rng(3)
    n = 20_000
    x, y = rng.normal(size=(n, 3)), rng.integers(0, 2, n).astype(np.float64)
    ids = np.arange(1, n + 1)
    sizes = _check_split(engine, x, y, ids, [0, 0], 7, bounds=[0.0, 0.5, 0.9])
    assert sum(sizes) == int((_draw(7, ids) < 0.9).sum()) < n
    assert split_bounds([1.0] * 7)[-1] < 1.0


def test_split_of_features_keeps_the_input_and_tile_edges(engine):
    for n in (1, 1023, 1024, 1025, 3 * 1024 + 17):
        rng = np.random.default_rng(n)
        x, y = rng.normal(size=(n, 300)), rng.integers(0, 2, n).astype(np.float64)       # k > 256 threads
        _check_split(engine, x, y, np.arange(1, n + 1), [0.3, 0.7], 99)
    x, y = np.zeros((0, 2)), np.zeros(0)
    assert _check_split(engine, x, y, np.zeros(0, np.int64), [0.5, 0.5], 1) == [0, 0]


def test_split_refusals_launch_nothing(engine):
    part = _part(engine, np.ones((4, 2)), np.zeros(4))
    try:
        before = engine.launch_count
        for bad in ([0.0, 0.5, 0.4], [0.0, float("nan")], [0.5, 1.0], [0.0, float("inf")]):
            with pytest.raises(N.LoexecError):
                engine.random_split(part, np.arange(4), bad, 1)
        with pytest.raises(N.LoexecError):
            engine.random_split(part, np.arange(4), np.linspace(0, 1, N.LO_SPLIT_MAX + 2), 1)
        assert engine.launch_count == before
    finally:
        part.free()


# ---- text codes against a dictionary --------------------------------------------------------------------------------
def _lookup(cells, dictionary):
    index = {s: i for i, s in enumerate(dictionary)}
    return np.array([-1 if c is None else index.get(c, -1) for c in cells], np.int32)


def _codes_in(engine, cells, dictionary, cuts=1):
    arr = pa.array(cells, type=pa.large_string())
    d = pa.array(dictionary, type=pa.large_string())
    cut = np.linspace(0, len(cells), cuts + 1).astype(int)
    pieces = [engine.text(arr.slice(a, b - a)) for a, b in zip(cut[:-1], cut[1:])]
    tables = [engine.table("i32", p.n, 1) for p in pieces]
    try:
        if cuts == 1:
            unseen = engine.text_codes_in(pieces[0], d, tables[0], 0)
        else:
            text = ShardedText(pieces, list(cut[:-1]), arr)
            unseen = _sharded(engine, cuts).text_codes_in(text, d, SimpleNamespace(offsets=list(cut[:-1]), shards=tables), 0)
        return np.concatenate([t.to_numpy(0) for t in tables]), unseen
    finally:
        for t in tables + pieces:
            t.free()


@pytest.mark.parametrize("cuts", [1, 2, 3])
def test_codes_against_a_host_lookup(engine, cuts):
    rng = np.random.default_rng(5)
    words = [f"w{i}" for i in range(3000)] + ["", "é", "日本語", "x" * 5000, "\x00nul"]
    dictionary = list(rng.permutation(words[:2500])) + ["", "日本語", "x" * 5000]
    cells = [None if i % 13 == 0 else words[int(rng.integers(len(words)))] for i in range(40_003)]
    got, unseen = _codes_in(engine, cells, dictionary, cuts)
    want = _lookup(cells, dictionary)
    np.testing.assert_array_equal(got, want)
    assert unseen == sum(1 for c, w in zip(cells, want) if c is not None and w < 0) and unseen > 0


def test_codes_of_colliding_strings_and_edges(engine):
    g = json.loads((GOLD / "hash_collisions.json").read_text())
    strings = [p[k] for p in g["pairs"] for k in ("a", "b")]
    dictionary = strings[::2]
    cells = strings + [None] + strings[::-1]
    got, unseen = _codes_in(engine, cells, dictionary)
    np.testing.assert_array_equal(got, _lookup(cells, dictionary))
    got, unseen = _codes_in(engine, ["a", None, "b"], [])                 # an empty dictionary: every cell unseen
    assert got.tolist() == [-1, -1, -1] and unseen == 2
    got, unseen = _codes_in(engine, [], ["a"])
    assert got.size == 0 and unseen == 0
    with pytest.raises(N.LoexecError, match="more than once"):
        _codes_in(engine, ["a"], ["a", "b", "a"])
    with pytest.raises(N.LoexecError, match="null"):
        _codes_in(engine, ["a"], ["a", None])


# ---- POST /models end to end ----------------------------------------------------------------------------------------
NUMBER_FIELDS = ["Survived", "Pclass", "Age", "SibSp", "Parch", "Fare"]
MODELING_CODE = """
assembled = training_df.features(["Pclass", "Sex", "Age", "SibSp", "Parch", "Fare", "Embarked"], label="Survived",
                                 handle_invalid="skip")
features_training, features_evaluation = assembled.random_split([0.8, 0.2], seed=17)
features_testing = testing_df.features(["Pclass", "Sex", "Age", "SibSp", "Parch", "Fare", "Embarked"],
                                       handle_invalid="skip")
"""
ALL = ["NB", "LR", "DT", "GB", "RF"]
MODELS = {"NB": NaiveBayes, "LR": LogisticRegression, "DT": DecisionTreeClassifier, "GB": GBTClassifier,
          "RF": RandomForestClassifier}


def _datasets(tmp_path, train_rows=700):
    g = json.loads((GOLD / "titanic_shaped_input.json").read_text())
    h = g["headers"]
    train, test = tmp_path / "train.csv", tmp_path / "test.csv"
    with open(train, "w", newline="") as f:
        csv.writer(f).writerows([h] + g["rows"][:train_rows])
    s = h.index("Survived")
    with open(test, "w", newline="") as f:
        csv.writer(f).writerows([h[:s] + h[s + 1:]] + [r[:s] + r[s + 1:] for r in g["rows"][train_rows:]])
    return g, str(train), str(test)


def _app(eng, tmp_path):
    g, train, test = _datasets(tmp_path)
    db = ColumnarDatabase()
    c = Client(server.create_app(db, eng, synchronous=True))
    for name, path in (("train", train), ("test", test)):
        assert c.post("/files", json={"datasetName": name, "datasetURI": path}).status_code == 201
        fields = [f for f in NUMBER_FIELDS if f != "Survived" or name == "train"]
        assert c.patch("/fieldTypes", json={"inputDatasetName": name, "types": {f: "number" for f in fields}}).status_code == 200
    return g, db, c


def _pages(c, name):
    out, skip = [], 0
    while True:
        page = c.get(f"/files/{name}?limit=100&skip={skip}").get_json()["result"]
        if not page:
            return out
        out += page
        skip += len(page)


def _leases(eng):
    return sum(e.users for e in eng.resident._entries.values())


def _by_hand(db, eng, name):
    """The job's steps run by hand: the predictions (probability, prediction) of each classifier and its metrics."""
    out = {}
    with builder_frontend.device_frame(db, "train", eng, text=True) as tr, \
            builder_frontend.device_frame(db, "test", eng, text=True, dictionaries=tr.dictionaries) as te:
        scope = {"training_df": tr, "testing_df": te}
        exec(MODELING_CODE, {}, scope)
        try:
            model = MODELS[name]().fit(scope["features_training"])
            r = model.evaluate(scope["features_evaluation"])
            with model.transform(scope["features_testing"]) as p:
                import torch
                prob = np.concatenate([torch.as_tensor(v, device=f"cuda:{d}").cpu().numpy() for v, d in zip(p.probability, p.devices)])
                pred = np.concatenate([torch.as_tensor(v, device=f"cuda:{d}").cpu().numpy() for v, d in zip(p.prediction, p.devices)])
                ids = p.row_ids.copy()
            codes = np.concatenate([torch.as_tensor(col, device=f"cuda:{col.table.engine.device}").cpu().numpy()
                                    for col in te.columns["Sex"]])
            words = tr.dictionaries["Sex"].to_pylist()
            out = dict(prob=prob, pred=pred, ids=ids, f1=str(float(r["f1"])), accuracy=str(float(r["accuracy"])),
                       test_sex=[None if c < 0 else words[c] for c in codes],
                       stored_sex=db.column("test", "Sex").to_pylist())
        finally:
            for f in tr.made + te.made:
                f.release()
    return out


def _tables_alive(eng):
    import gc
    from learningorchestra_b200.engine import DeviceTable
    gc.collect()
    engines = set(eng.engines if isinstance(eng, ShardedEngine) else [eng])
    from learningorchestra_b200.engine import DeviceText
    return sum(1 for o in gc.get_objects()
               if isinstance(o, (DeviceTable, DeviceText)) and o._h is not None and o.engine in engines)


@pytest.mark.parametrize("sharded", [False, True])
def test_models_end_to_end(engine, tmp_path, sharded):
    eng = ShardedEngine.local() if sharded else engine
    try:
        eng.resident.clear()
        g, db, c = _app(eng, tmp_path)
        wants = {name: _by_hand(db, eng, name) for name in ALL}          # also makes both datasets resident
        before = _tables_alive(eng)
        r = c.post("/models", json={"trainDatasetName": "train", "testDatasetName": "test", "modelingCode": MODELING_CODE,
                                    "classifiersList": ALL + ["NB"]})
        assert r.status_code == 201
        assert r.get_json()["result"] == [f"/api/learningOrchestra/v1/builder/sparkml/test{n}?query={{}}&limit=10&skip=0"
                                          for n in ALL + ["NB"]]
        assert _tables_alive(eng) == before and _leases(eng) == 0           # every table the job made is freed
        test_rows = g["rows"][700:]
        h = g["headers"]
        for name in ALL:
            meta = db.find_one(f"test{name}", {"_id": 0})
            assert meta["finished"] is True, meta.get("exception")
            assert meta["type"] == "builder/sparkml" and meta["parentDatasetName"] == ["train", "test"]
            assert meta["classifier"] == name and meta["datasetName"] == f"test{name}" and meta["fitTime"] > 0
            want = wants[name]
            assert meta["F1"] == want["f1"] and meta["accuracy"] == want["accuracy"]
            rows = [d for d in _pages(c, f"test{name}") if d["_id"] != 0]
            assert [d["_id"] for d in rows] == list(range(1, len(want["ids"]) + 1))
            for d, row_id, p, q in zip(rows, want["ids"], want["pred"], want["prob"]):
                src = test_rows[row_id - 1]
                assert d["Name"] == src[h.index("Name")] and d["Sex"] == src[h.index("Sex")] and "Survived" not in d
                assert d["prediction"] == float(p) and d["probability"] == q.tolist()
                assert "features" not in d and "rawPrediction" not in d
            assert want["test_sex"] == want["stored_sex"]                    # each test cell has its training code
        eng.resident.clear()
    finally:
        if sharded:
            eng.close()


def test_models_failures_and_replacement(engine, tmp_path):
    engine.resident.clear()
    g, db, c = _app(engine, tmp_path)
    _by_hand(db, engine, "NB")                                            # both datasets resident
    before = _tables_alive(engine)
    body = {"trainDatasetName": "train", "testDatasetName": "test", "classifiersList": ["NB", "DT"]}
    for code in ("raise ValueError('no features')", "features_training = training_df.features(label='Survived', "
                                                    "handle_invalid='skip')"):
        assert c.post("/models", json=dict(body, modelingCode=code)).status_code == 201
        for name in ("NB", "DT"):
            meta = db.find_one(f"test{name}", {"_id": 0})
            assert meta["finished"] is False and ("no features" in meta["exception"] or "features_testing" in meta["exception"])
        assert _tables_alive(engine) == before and _leases(engine) == 0
    three = MODELING_CODE.replace('label="Survived"', 'label="Pclass"').replace('"Pclass", "Sex"', '"Sex"')
    r = c.post("/models", json=dict(body, classifiersList=["GB", "NB", "DT"], modelingCode=three))
    assert r.status_code == 201
    gb = db.find_one("testGB", {"_id": 0})
    assert gb["finished"] is False and "0 or 1" in gb["exception"]
    assert all(db.find_one(f"test{n}", {"_id": 0})["finished"] is True for n in ("NB", "DT"))
    assert _tables_alive(engine) == before and _leases(engine) == 0
    n_before = len(_pages(c, "testNB"))
    r = c.post("/models", json=dict(body, classifiersList=["NB"], modelingCode=MODELING_CODE))
    assert r.status_code == 201 and len(_pages(c, "testNB")) == n_before         # replaced, not appended
    assert sum(1 for d in db.find("testNB", {}) if d["_id"] == 0) == 1
    assert _tables_alive(engine) == before and _leases(engine) == 0
    engine.resident.clear()
