"""CPU: ``POST /models`` — its validators and their order, its URIs, the prediction datasets' metadata written before the
job runs, a job without an engine, the ``probability`` column of a prediction dataset, and the bounds and refusals of
``Features.random_split``."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
from werkzeug.test import Client

from learningorchestra_b200 import _native as N
from learningorchestra_b200 import server
from learningorchestra_b200.builder import source_columns
from learningorchestra_b200.column_store import ColumnarDatabase, NumberColumn, ProbabilityColumn, TextColumn
from learningorchestra_b200.builder_frontend import DeviceFrame, Features
from learningorchestra_b200.engine import AssembledRows, SPLIT_SEED, split_bounds
from learningorchestra_b200.utils import Database

BODY = {"trainDatasetName": "train", "testDatasetName": "test", "modelingCode": "", "classifiersList": ["NB"]}


def _app(finished=True):
    db = ColumnarDatabase()
    for name in ("train", "test"):
        db.ingest_columns(name, {"a": np.arange(4.0), "s": TextColumn(["x", "y", None, "x"])})
    if not finished:
        db.update_one("test", {"finished": False}, {"_id": 0})
    return db, Client(server.create_app(db, None, synchronous=True))


def _post(c, **changes):
    r = c.post("/models", json=dict(BODY, **changes))
    return r.status_code, r.get_json()["result"]


def test_validators_in_the_reference_order():
    db, c = _app(finished=False)
    assert _post(c, trainDatasetName="nope", classifiersList=["XX"]) == (406, "invalid input dataset name")
    assert _post(c, testDatasetName="nope") == (406, "invalid input dataset name")
    assert _post(c, classifiersList=["NB", "SVM"]) == (406, "invalid classifier name")     # before unfinished
    assert _post(c) == (406, "unfinished processing in input dataset")
    assert not any(n.startswith("test") and n != "test" for n in db.get_filenames())


def test_uris_one_per_entry_with_duplicates_and_metadata_before_the_job():
    db, c = _app()
    status, uris = _post(c, classifiersList=["NB", "LR", "NB", "RF"])
    assert status == 201
    assert uris == [f"/api/learningOrchestra/v1/builder/sparkml/test{n}?query={{}}&limit=10&skip=0"
                    for n in ("NB", "LR", "NB", "RF")]
    for name in ("NB", "LR", "RF"):
        docs = db.find(f"test{name}", {})
        assert len(docs) == 1
        meta = docs[0]
        assert {k: meta[k] for k in ("_id", "type", "finished", "parentDatasetName", "classifier", "datasetName")} == {
            "_id": 0, "type": "builder/sparkml", "finished": False, "parentDatasetName": ["train", "test"],
            "classifier": name, "datasetName": f"test{name}"}
        assert meta["timeCreated"].endswith("-00:00")
        assert "needs an Engine" in meta["exception"]          # no engine: recorded, and the dataset stays unfinished
    assert "testDT" not in db.get_filenames()
    assert Database.create_prediction_filename("test", "GB") == "testGB"


def test_a_second_request_replaces_the_dataset():
    db, c = _app()
    db.ingest_columns("testNB", {"old": np.arange(3.0)})
    assert _post(c)[0] == 201
    assert db.find("testNB", {}) == [d for d in db.find("testNB", {}) if d["_id"] == 0] and len(db.find("testNB", {})) == 1


def test_probability_column_pages_takes_and_finds():
    db = ColumnarDatabase()
    m = np.array([[0.25, 0.75], [1.0, 0.0], [0.5, 0.5]])
    db.insert_one_in_file("p", {"_id": 0, "datasetName": "p", "finished": True})
    db.create_table("p", np.arange(1, 4), {"probability": ProbabilityColumn(m), "prediction": NumberColumn([1.0, 0.0, 0.0])})
    c = Client(server.create_app(db, None))
    page = c.get("/files/p?limit=2&skip=1").get_json()["result"]
    assert page == [{"probability": [0.25, 0.75], "prediction": 1.0, "_id": 1},
                    {"probability": [1.0, 0.0], "prediction": 0.0, "_id": 2}]
    assert db.find_in_file("p", {"_id": 3}, 0, 10) == [{"probability": [0.5, 0.5], "prediction": 0.0, "_id": 3}]
    col = db.column("p", "probability")
    assert col.kind == "object" and len(col) == 3 and col.take([2, 0]).to_pylist() == [[0.5, 0.5], [0.25, 0.75]]
    with pytest.raises(ValueError):
        ProbabilityColumn(np.zeros(3))


def test_source_columns_share_or_take():
    db, _c = _app()
    same = source_columns(db, "test", np.arange(1, 5))
    assert list(same) == ["a", "s"] and same["a"] is db.column("test", "a")
    some = source_columns(db, "test", np.array([4, 2]))
    assert some["a"].to_pylist() == [3, 1] and some["s"].to_pylist() == ["x", "y"]


def _spark_bounds(weights):
    """Dataset.randomSplit: normalized = weights / sum; scanLeft(0.0)(_ + _) over them, in float64."""
    total = 0.0
    for w in weights:
        total += w
    out = [0.0]
    for w in weights:
        out.append(out[-1] + w / total)
    return np.array(out)


@pytest.mark.parametrize("weights", [[1.0], [0.7, 0.3], [0.1] * 10, [3, 0, 1e-300, 2], [1e308, 1e308], [0.2, 0.3, 0.5]])
def test_split_bounds_as_spark_computes_them(weights):
    got = split_bounds(weights)
    np.testing.assert_array_equal(got.view(np.int64), _spark_bounds(weights).view(np.int64))
    assert got[0] == 0.0 and np.all(np.diff(got) >= 0)


def test_split_bounds_may_end_below_or_above_one():
    assert split_bounds([1.0] * 7)[-1] < 1.0 < split_bounds([0.7, 0.2, 0.1])[-1]


@pytest.mark.parametrize("weights", [[], [-0.1, 1.0], [math.nan], [math.inf, 1.0], [0.0, 0.0], [1.0] * (N.LO_SPLIT_MAX + 1)])
def test_split_refusals(weights):
    with pytest.raises(ValueError):
        split_bounds(weights)


def test_random_split_hands_each_part_its_ids_and_registers_the_splits():
    """Features.random_split through a stand-in engine: the bounds, the seed and each part's _ids reach the engine, and
    every split is a Features of the same frame, listed in ``frame.made``."""
    calls = []
    table = SimpleNamespace(engine=SimpleNamespace(device=0), base_ptr=0, dtype_code=N.LO_F32, free=lambda: None)

    def random_split(part, ids, bounds, seed):
        calls.append((ids.tolist(), bounds.tolist(), seed))
        return [AssembledRows(table, None, np.array([0]), part.k, 1), AssembledRows(table, None, np.zeros(0, int), part.k, 0)]

    engine = SimpleNamespace(random_split=random_split)
    frame = object.__new__(DeviceFrame)
    frame._cache, frame.ids, frame.made = SimpleNamespace(engine=engine), np.array([5, 7, 9]), []
    feats = Features(frame, [AssembledRows(table, None, np.array([0, 2]), 2, 2)], ["a", "b"], None, "float32")
    first, second = feats.random_split([3, 1])
    assert calls == [([5, 9], [0.0, 0.75, 1.0], SPLIT_SEED)]
    assert first.row_ids.tolist() == [5] and second.row_ids.tolist() == []
    assert frame.made == [feats, first, second]
    with pytest.raises(ValueError):
        feats.random_split([0.0])
