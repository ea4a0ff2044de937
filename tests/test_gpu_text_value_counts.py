"""GPU: ``$group`` of text columns resident in HBM (``lo_text_upload`` / ``lo_value_counts_text``, the reworked
``k_hash_count_str`` with its null skipping and per-CTA shared-memory stage) and the ``/histograms`` route over them.

Results are multisets of (key, count), compared with ``collections.Counter`` over ``columnar.group_key`` and with the
host route (``lo_value_counts_str_host``, no validity); every representative row must be a non-null cell equal to its
key."""
import csv
import ctypes as C
import json
import threading
from collections import Counter
from pathlib import Path

import numpy as np
import pyarrow as pa
import pytest
from werkzeug.test import Client

from learningorchestra_b200 import _native as N
from learningorchestra_b200 import columnar, server, utils
from learningorchestra_b200.column_store import ColumnarDatabase
from learningorchestra_b200.data_type_update import DataType
from learningorchestra_b200.histogram import Histogram
from oracle import rsem

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).resolve().parent / "golden"


def _multiset(keys, counts):
    return sorted(Counter({columnar.group_key(k): int(c) for k, c in zip(keys, counts)}).items())


def _check(engine, arr):
    """Count ``arr`` (an Arrow string array) from HBM; returns the upload's and the count's timing."""
    up, t = {}, {}
    text = engine.text(arr, timing=up)
    try:
        rep, counts = engine.value_counts_text(text, timing=t)
    finally:
        text.free()
    cells = arr if isinstance(arr, list) else arr.to_pylist()
    present = [c for c in cells if c is not None]
    assert text.n == len(cells) and text.nulls == len(cells) - len(present)
    keys = []
    for r in rep:
        assert 0 <= r < len(cells) and cells[int(r)] is not None
        keys.append(cells[int(r)])
    assert len(set(keys)) == len(keys)
    want = sorted(Counter(columnar.group_key(c) for c in present).items())
    assert _multiset(keys, counts) == want
    if present:                                              # the host route, same kernel without validity
        hrep, hcounts = engine.value_counts_str_host(present)
        assert _multiset([present[int(r)] for r in hrep], hcounts) == want
    if t:
        assert t["h2d_bytes"] == 0 and t["launches"] == 2
    return up, t


def test_empty_strings_are_not_nulls(engine):
    _check(engine, pa.array(["", None, "", "a", None, "", "a", None], type=pa.large_string()))


def test_sliced_array_with_offset_offsets_and_bit_offset(engine):
    rng = np.random.default_rng(7)
    cells = [None if rng.random() < 0.3 else "k%d" % rng.integers(0, 9) for _ in range(300)]
    full = pa.array(cells, type=pa.large_string())
    for start, length in ((13, 200), (3, 1), (21, 279), (8, 64)):
        arr = full.slice(start, length)
        assert arr.offset % 8 != 0 or start == 8
        assert columnar.text_buffers(arr)[1][0] != 0 or start == 0
        _check(engine, arr)
    _check(engine, pa.array(cells[13:213], type=pa.string()))      # a 32-bit-offset array is widened first
    _check(engine, cells[5:50])                                    # a list of str / None


def test_non_ascii_cells_and_a_two_mib_cell(engine):
    big = "x" * (2 << 20)
    _check(engine, pa.array(["é", "日本語", big, "é", big + "y", big, "😀", None, "é"], type=pa.large_string()))


def test_zero_and_one_cells(engine):
    for cells in ([], ["a"], [None], [""]):
        up, t = _check(engine, pa.array(cells, type=pa.large_string()))
        assert up["h2d_bytes"] >= 8


def test_constant_three_value_and_all_distinct_columns(engine):
    n = 5_000_000
    const = pa.array(np.full(n, "S", dtype=object), type=pa.large_string())
    _check(engine, const)
    three = pa.array(np.array(["S", "C", "Q"], dtype=object)[np.arange(3_000_001) % 3], type=pa.large_string())
    _check(engine, three)
    m = 1_000_000
    # every CTA of the count kernel (at most 8 per SM, 256 rows per stride) sees more distinct cells than its stage
    # holds, so the stage overflows and the spill path runs
    assert m // (engine.sm_count * 8 * 256) * 256 > N.LO_TEXT_STAGE_SLOTS
    distinct = pa.array([str(i) for i in range(m)], type=pa.large_string())
    _check(engine, distinct)
    text = engine.text(distinct)
    try:
        rep, counts = engine.value_counts_text(text)
        assert len(rep) == m and int(counts.sum()) == m and np.array_equal(np.sort(rep), np.arange(m))
    finally:
        text.free()


def test_hash_collisions_meet_inside_one_cta(engine):
    fx = json.loads((GOLD / "hash_collisions.json").read_text())
    pairs = [(p["a"], p["b"]) for p in fx["pairs"]]
    cells = []
    for k in range(40):               # a, b, a, b ... within a few rows: the same warp and the same CTA
        for a, b in pairs:
            cells += [a, b, a, None, b] if k % 2 else [b, a]
    _check(engine, pa.array(cells, type=pa.large_string()))
    # the colliding pairs spread over one CTA's rows, one pair per warp: they meet in the stage, not in a warp
    spread = []
    for k in range(8):
        for a, b in pairs:
            spread += [a] * 31 + [b]
    _check(engine, pa.array(spread, type=pa.large_string()))


def test_capacity_contract(engine):
    arr = pa.array(["a", "b", None, "c", "a", "d"], type=pa.large_string())
    text = engine.text(arr)
    lib = engine._lib
    try:
        rows, counts, nd = np.zeros(4, np.int64), np.zeros(4, np.uint64), C.c_int64()
        rc = lib.lo_value_counts_text(engine._ctx, text._h, rows.ctypes.data_as(C.c_void_p),
                                      counts.ctypes.data_as(C.c_void_p), 2, C.byref(nd), None)
        assert rc == N.LO_ERR_INVALID and nd.value == 4 and "capacity" in lib.lo_last_error().decode()
        rc = lib.lo_value_counts_text(engine._ctx, text._h, None, None, 0, C.byref(nd), None)
        assert rc == N.LO_ERR_INVALID and nd.value == 4
        t = N.HostTiming()
        N.check(lib.lo_value_counts_text(engine._ctx, text._h, rows.ctypes.data_as(C.c_void_p),
                                         counts.ctypes.data_as(C.c_void_p), 4, C.byref(nd), C.byref(t)))
        assert nd.value == 4 and t.h2d_bytes == 0 and int(counts.sum()) == 5
        assert sorted(arr[int(r)].as_py() for r in rows) == ["a", "b", "c", "d"]
    finally:
        text.free()
    size = C.c_size_t()
    assert lib.lo_text_info(None, None, None, None, C.byref(size)) == N.LO_ERR_INVALID


# ---- /histograms ------------------------------------------------------------------------------------------------
TEXT_FIELDS = ["Sex", "Embarked", "Pclass", "Name", "Ticket", "Cabin"]


def _titanic():
    return json.loads((GOLD / "titanic_shaped_input.json").read_text())


def _expected(db, name, fields):
    """The reference's $group over every document of the collection (metadata document included)."""
    docs = db.find(name, {})
    return {f: sorted(Counter(columnar.group_key(d.get(f)) for d in docs).items()) for f in fields}


def _results(db, out):
    got = {}
    for d in db.find(out, {}):
        if d["_id"] != 0:
            (f, groups), = [(k, v) for k, v in d.items() if k != "_id"]
            got[f] = sorted((columnar.group_key(g["_id"]), g["count"]) for g in groups)
    return got


def _stores(tmp_path):
    g = _titanic()
    docs = utils.Database()
    hdr, documents = rsem.csv_rows_to_documents(g["headers"], g["rows"])
    docs.insert_one_in_file("t", rsem.dataset_metadata("t", hdr))
    docs.insert_many_in_file("t", documents)
    path = tmp_path / "t.csv"
    with open(path, "w", newline="") as f:
        csv.writer(f).writerows([g["headers"]] + g["rows"])
    return [("documents", docs), ("columnar", ColumnarDatabase())], path


def _post_files(db, engine, path):
    c = Client(server.create_app(db, engine, synchronous=True))
    assert c.post("/files", json={"datasetName": "t", "datasetURI": f"file://{path}"}).status_code == 201
    return c


def _count(c, name, out, fields):
    r = c.post("/histograms", json={"inputDatasetName": name, "outputDatasetName": out, "names": fields})
    assert r.status_code == 201, r.get_data(as_text=True)


class _Spy:
    """Records the timing of every value_counts_text call of an engine."""

    def __init__(self, engine, monkeypatch):
        self.calls, real = [], engine.value_counts_text

        def spy(text, timing=None):
            t = {}
            out = real(text, timing=t)
            self.calls.append(t)
            return out
        monkeypatch.setattr(engine, "value_counts_text", spy)


def test_post_files_then_histograms_on_text_fields(engine, tmp_path, monkeypatch):
    engine.resident.clear()
    _, path = _stores(tmp_path)
    db = ColumnarDatabase()
    c = _post_files(db, engine, path)
    spy = _Spy(engine, monkeypatch)
    _count(c, "t", "h1", TEXT_FIELDS)
    got = _results(db, "h1")
    assert got == _expected(db, "t", TEXT_FIELDS)
    assert len(spy.calls) == len(TEXT_FIELDS)                # every field took the resident route, Sex included
    # the host route on the same cells gives the same groups
    for f in TEXT_FIELDS:
        arr = db.column("t", f).arr
        present = [x for x in arr.to_pylist() if x is not None]
        rep, counts = engine.value_counts_str_host(present)
        host = _multiset([present[int(r)] for r in rep], counts)
        assert [kv for kv in got[f] if kv[0] != ("null",)] == host, f
    # a second request: a cache hit, and no cell crosses PCIe
    h0 = engine.resident.hits
    spy.calls.clear()
    _count(c, "t", "h2", TEXT_FIELDS)
    assert _results(db, "h2") == got and engine.resident.hits == h0 + 1
    assert len(spy.calls) == len(TEXT_FIELDS) and all(t["h2d_bytes"] == 0 for t in spy.calls)
    # /fieldTypes "number" on a counted field: the next request rebuilds, the field takes the number route
    assert c.patch("/fieldTypes", json={"inputDatasetName": "t", "types": {"Pclass": "number"}}).status_code == 200
    spy.calls.clear()
    _count(c, "t", "h3", ["Pclass", "Sex"])
    got3 = _results(db, "h3")
    assert got3 == _expected(db, "t", ["Pclass", "Sex"]) and len(spy.calls) == 1
    assert sorted(n for _k, n in got3["Pclass"]) == sorted(n for _k, n in got["Pclass"])
    assert all(k[0] in ("num", "null") for k, _n in got3["Pclass"])
    assert engine.resident._entries["t"].texts["Pclass"] is None
    engine.resident.clear()


def test_titanic_document_store_matches_the_reference_histogram(engine, monkeypatch):
    """The document store of test_titanic_histogram_value_counts_match_reference_execution: Embarked and Sex are text
    after the number cast, and their documents equal those the reference's histogram.py made."""
    engine.resident.clear()
    db = utils.Database()
    g = _titanic()
    headers, docs = rsem.csv_rows_to_documents(g["headers"], g["rows"])
    db.insert_one_in_file("titanic", rsem.dataset_metadata("titanic", headers))
    db.insert_many_in_file("titanic", docs)
    job = DataType(db, utils.DataTypeMetadata(db), engine)
    job.convert_existent_file("titanic", {"Survived": "number", "Pclass": "number", "Age": "number", "Fare": "number"})
    job.wait()
    gold = json.loads((GOLD / "reference_histogram.json").read_text())
    ref = {next(k for k in d if k != "_id"): d for d in gold["documents"] if d["_id"] != 0}
    spy = _Spy(engine, monkeypatch)
    h = Histogram(db, utils.HistogramMetadata(db), engine)
    h.create_file("titanic", "titanic_hist", list(gold["fields"]))
    h.wait()
    got = {next(k for k in d if k != "_id"): d for d in db.find("titanic_hist", {}) if d["_id"] != 0}
    for f in ("Embarked", "Sex"):
        assert f in ref
        assert rsem.normalise_group_result(got[f][f]) == rsem.normalise_group_result(ref[f][f]), f
        assert engine.resident._entries["titanic"].texts[f] is not None, f      # the resident route
    numbers = [f for f in gold["fields"] if f in ("Survived", "Pclass", "Age", "Fare")]
    assert all(engine.resident._entries["titanic"].texts[f] is None for f in numbers)
    assert len(spy.calls) == sum(1 for f in gold["fields"] if engine.resident._entries["titanic"].texts.get(f) is not None)
    for f in gold["fields"]:
        assert rsem.normalise_group_result(got[f][f]) == rsem.normalise_group_result(ref[f][f]), f
    engine.resident.clear()


def test_database_without_version_uploads_and_frees_per_request(engine):
    class Foreign:                     # a database object without version(): never cached
        def __init__(self, db):
            self._db = db

        def find(self, *a):
            return self._db.find(*a)

        def insert_one_in_file(self, *a):
            return self._db.insert_one_in_file(*a)

        def update_one(self, *a):
            return self._db.update_one(*a)

    engine.resident.clear()
    db = utils.Database()
    g = _titanic()
    hdr, documents = rsem.csv_rows_to_documents(g["headers"], g["rows"])
    db.insert_one_in_file("t", rsem.dataset_metadata("t", hdr))
    db.insert_many_in_file("t", documents)
    f = Foreign(db)
    h = Histogram(f, utils.HistogramMetadata(f), engine)
    h.file_processing("t", "out", ["Sex", "Embarked"])
    assert _results(db, "out") == _expected(db, "t", ["Sex", "Embarked"])
    assert not engine.resident._entries


def test_sharded_engine_counts_text_on_its_first_device(tmp_path):
    from learningorchestra_b200.sharding import ShardedEngine
    _, path = _stores(tmp_path)
    with ShardedEngine.local([0]) as sh:
        db = ColumnarDatabase()
        c = _post_files(db, sh, path)
        _count(c, "t", "h", TEXT_FIELDS)
        assert _results(db, "h") == _expected(db, "t", TEXT_FIELDS)
        assert all(sh.resident._entries["t"].texts[f] is not None for f in TEXT_FIELDS)
        sh.resident.clear()


def test_eviction_under_a_small_budget_keeps_results_correct(engine, tmp_path):
    engine.resident.clear()
    _, path = _stores(tmp_path)
    db = ColumnarDatabase()
    c = _post_files(db, engine, path)
    assert c.post("/files", json={"datasetName": "u", "datasetURI": f"file://{path}"}).status_code == 201
    old = engine.resident.max_bytes
    engine.resident.max_bytes = 1
    try:
        want = _expected(db, "t", TEXT_FIELDS)
        for k in range(3):
            for name in ("t", "u"):
                _count(c, name, f"e{name}{k}", TEXT_FIELDS)
                assert _results(db, f"e{name}{k}") == want
                assert len(engine.resident._entries) == 1
    finally:
        engine.resident.max_bytes = old
        engine.resident.clear()


def test_counting_threads_while_a_binned_request_rebuilds(engine, tmp_path, monkeypatch):
    """Two threads count text fields while a third keeps rebuilding the same dataset with binned requests on new
    fields: no entry is freed while a lease holds it, and every result is correct."""
    from learningorchestra_b200.table_cache import ResidentDataset
    engine.resident.clear()
    _, path = _stores(tmp_path)
    db = ColumnarDatabase()
    _post_files(db, engine, path)
    want = _expected(db, "t", ["Sex", "Embarked", "Name"])
    errors, leased_frees = [], []
    real_free = ResidentDataset.free

    def free(self):
        if self.users > 0:
            leased_frees.append(self.users)
        real_free(self)
    monkeypatch.setattr(ResidentDataset, "free", free)

    def counter(k):
        try:
            for i in range(6):
                out = f"c{k}_{i}"
                h = Histogram(db, utils.HistogramMetadata(db), engine)
                h.file_processing("t", out, ["Sex", "Embarked", "Name"])
                if _results(db, out) != want:
                    errors.append(out)
        except BaseException as exc:          # noqa: BLE001 — reported below
            errors.append(repr(exc))

    def binner():
        try:
            for i, fields in enumerate([["Age"], ["Fare"], ["Age", "SibSp"], ["Parch"], ["Fare", "Survived"], ["Age"]]):
                h = Histogram(db, utils.HistogramMetadata(db), engine)
                h.file_processing("t", f"b{i}", fields, bins=8)
                if i % 2:
                    engine.resident.invalidate("t")
        except BaseException as exc:          # noqa: BLE001
            errors.append(repr(exc))

    threads = [threading.Thread(target=counter, args=(k,)) for k in range(2)] + [threading.Thread(target=binner)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    assert not leased_frees
    engine.resident.clear()
