"""CPU: ``/histograms`` without ``bins`` on both stores, through the resident route, the host route and a rank group's
mix of the two, with a test double standing in for the device.  Every field shape the routes classify differently is
here: int and float numbers, NaN beside None, ints stored as floats, text with ``""``, mixed types, all-null, absent,
a field the metadata document also sets, and a field named twice.  The expected result documents and engine calls are
literals: a change to how a field is read or classified shows up as a changed group, key type or call."""
import itertools
import math
from collections import Counter

import numpy as np
import pyarrow as pa
import pytest

from learningorchestra_b200 import columnar, utils
from learningorchestra_b200.column_store import ColumnarDatabase, NumberColumn, ObjectColumn, TextColumn
from learningorchestra_b200.histogram import Histogram
from learningorchestra_b200.table_cache import ResidentTables

NAN = math.nan
ROWS = {
    "I": [3, 1, 3, None, 2, 3, 1],
    "F": [1.5, NAN, None, 2.0, -0.0, 0.0, 1.5],
    "C": [1.0, 2.0, 2.0, 3.5, 1.0, None, 4.0],
    "T": ["a", "", None, "a", "b", "", "a"],
    "M": [1, 1.0, "1", True, None, 1, "1"],
    "N": [None] * 7,
    "NT": [None] * 7,
    "S": [1, 2, 2, None, 1, 3, 2],
    "B": [0, 1, 1.5, None, 1, 0, 1],
}
META = {"S": "x", "B": True}                 # the metadata document sets these two fields too
FIELDS = ["I", "F", "C", "T", "M", "N", "NT", "S", "B", "A", "I"]
_OUT = itertools.count()


def _documents():
    db = utils.Database()
    db.insert_one_in_file("d", {"_id": 0, "finished": True, "fields": list(ROWS), **META})
    db.insert_many_in_file("d", [{"_id": i + 1, **{f: c[i] for f, c in ROWS.items() if c[i] is not None}}
                                 for i in range(7)])
    return db


def _number(values, is_int):
    valid = [v is not None for v in values]
    return NumberColumn([NAN if v is None else v for v in values], valid, [ok and is_int for ok in valid])


def _columns():
    db = ColumnarDatabase()
    db.ingest_columns("d", {
        "I": _number(ROWS["I"], True), "F": _number(ROWS["F"], False),
        "C": _number(ROWS["C"], False),          # integral values stored as floats: keys are floats
        "T": TextColumn(pa.array(ROWS["T"], type=pa.large_string())), "M": ObjectColumn(ROWS["M"]),
        "N": _number(ROWS["N"], False), "NT": TextColumn(pa.array(ROWS["NT"], type=pa.large_string())),
        "S": _number(ROWS["S"], True), "B": NumberColumn([0.0, 1.0, 1.5, NAN, 1.0, 0.0, 1.0],
                                                         [True, True, True, False, True, True, True],
                                                         [True, True, False, False, True, True, True])})
    db.update_one("d", META, {"_id": 0})
    return db


# ---- a test double for the device: every call that reaches it is recorded with its input size -------------------
class _Obj:
    def __init__(self, owner):
        self.owner = owner
        owner.live.add(id(self))

    def free(self):
        self.owner.live.discard(id(self))


class _Table(_Obj):
    def __init__(self, owner, nrows, ncols):
        super().__init__(owner)
        self.nrows, self.ncols, self.pitch_bytes = nrows, ncols, nrows * 8
        self.cols = [np.full(nrows, NAN) for _ in range(ncols)]

    def upload(self, col, values):
        self.owner.calls.append(("upload", col, len(values)))
        self.cols[col] = np.array(values, np.float64)


class _Text(_Obj):
    def __init__(self, owner, cells):
        super().__init__(owner)
        self.arr = pa.array(cells.to_pylist() if hasattr(cells, "to_pylist") else list(cells), type=pa.large_string())
        self.n, self.nulls, self.nbytes = len(self.arr), self.arr.null_count, 8


def _canon(v):
    b = np.where(v == 0, 0.0, v).view(np.uint64).copy()
    b[np.isnan(v)] = 0x7FF8000000000000
    return b


def _first_seen(cells):
    first, counts = {}, Counter()
    for i, c in enumerate(cells):
        if c is not None:
            first.setdefault(c, i)
            counts[c] += 1
    return np.array(list(first.values()), np.int64), np.array([counts[c] for c in first], np.uint64)


class _Engine:
    """The engine methods ``Histogram`` calls, computed on the host.  As in ``Engine``, a text count with no cells
    returns before anything reaches the device, and ``value_counts_str_host`` is ``pack_cells`` then
    ``value_counts_str_packed``, so ``calls`` holds what the device would see."""

    def __init__(self, world=1):
        self.live, self.calls, self.world, self.nlocal = set(), [], world, 1
        self.resident = ResidentTables(self)

    def table(self, dtype, nrows, ncols):
        self.calls.append(("table", nrows, ncols))
        return _Table(self, nrows, ncols)

    def text(self, cells):
        t = _Text(self, cells)
        self.calls.append(("text", t.n))
        return t

    def value_counts_text(self, text):
        if text.n == text.nulls:
            return np.zeros(0, np.int64), np.zeros(0, np.uint64)
        self.calls.append(("value_counts_text", text.n - text.nulls))
        return _first_seen(text.arr.to_pylist())

    def value_counts_column(self, table, col):
        self.calls.append(("value_counts_column", table.nrows))
        u, c = np.unique(_canon(table.cols[col]), return_counts=True)
        return u.view(np.float64), c.astype(np.uint64)

    def value_counts_f64_host(self, values):
        self.calls.append(("value_counts_f64_host", len(values)))
        u, c = np.unique(_canon(np.asarray(values, np.float64)), return_counts=True)
        return u.view(np.float64), c.astype(np.uint64)

    def value_counts_str_host(self, cells):
        return self.value_counts_str_packed(*columnar.pack_cells(cells))

    def value_counts_str_packed(self, chars, offsets):
        n = offsets.size - 1
        if n == 0:
            return np.zeros(0, np.int64), np.zeros(0, np.uint64)
        self.calls.append(("value_counts_str_packed", n, int(offsets[-1] - offsets[0])))
        return _first_seen([bytes(chars[offsets[i]:offsets[i + 1]]) for i in range(n)])


def _host_engine():
    eng = _Engine()
    eng.resident = None                      # the host route alone
    return eng


ENGINES = {"resident": _Engine, "host": _host_engine, "rank_group": lambda: _Engine(world=2)}


def _run(db, eng, fields=FIELDS):
    out = f"out{next(_OUT)}"
    Histogram(db, utils.HistogramMetadata(db), eng).file_processing("d", out, fields)
    docs = sorted((d for d in db.find(out, {}) if d["_id"] != 0), key=lambda d: d["_id"])
    return [next((k, v) for k, v in d.items() if k != "_id") for d in docs]


def _typed(groups, mixed):
    """(group key, key type, count) of each group, in an order-free form; a mixed field's representative of a group
    is unspecified (1 or 1.0), so its key type is not compared."""
    return sorted(((columnar.group_key(g["_id"]), None if mixed else type(g["_id"]).__name__, g["count"])
                   for g in groups), key=repr)


# what the routes return: field -> [(group key, key type, count)] in _typed's order, per store.  A field the metadata
# document also sets is classified with that document on a document store and beside it on a column store.
_NUM = "num"
GROUPS = {
    "documents": {
        "I": [(("null",), "NoneType", 2), ((_NUM, 1), "int", 2), ((_NUM, 2), "int", 1), ((_NUM, 3), "int", 3)],
        "F": [(("null",), "NoneType", 2), ((_NUM, "nan"), "float", 1), ((_NUM, 0), "float", 2),
              ((_NUM, 1.5), "float", 2), ((_NUM, 2), "float", 1)],
        "C": [(("null",), "NoneType", 2), ((_NUM, 1), "float", 2), ((_NUM, 2), "float", 2),
              ((_NUM, 3.5), "float", 1), ((_NUM, 4), "float", 1)],
        "T": [(("null",), "NoneType", 2), (("str", ""), "str", 2), (("str", "a"), "str", 3), (("str", "b"), "str", 1)],
        "M": [(("bool", True), None, 1), (("null",), None, 2), ((_NUM, 1), None, 3), (("str", "1"), None, 2)],
        "N": [(("null",), "NoneType", 8)],
        "NT": [(("null",), "NoneType", 8)],
        "S": [(("null",), None, 1), ((_NUM, 1), None, 2), ((_NUM, 2), None, 3), ((_NUM, 3), None, 1),
              (("str", "x"), None, 1)],
        "B": [(("bool", True), None, 1), (("null",), None, 1), ((_NUM, 0), None, 2), ((_NUM, 1), None, 3),
              ((_NUM, 1.5), None, 1)],
        "A": [(("null",), "NoneType", 8)],
    },
    "columnar": {
        "I": [(("null",), "NoneType", 2), ((_NUM, 1), "int", 2), ((_NUM, 2), "int", 1), ((_NUM, 3), "int", 3)],
        "F": [(("null",), "NoneType", 2), ((_NUM, "nan"), "float", 1), ((_NUM, 0), "float", 2),
              ((_NUM, 1.5), "float", 2), ((_NUM, 2), "float", 1)],
        "C": [(("null",), "NoneType", 2), ((_NUM, 1), "float", 2), ((_NUM, 2), "float", 2),
              ((_NUM, 3.5), "float", 1), ((_NUM, 4), "float", 1)],
        "T": [(("null",), "NoneType", 2), (("str", ""), "str", 2), (("str", "a"), "str", 3), (("str", "b"), "str", 1)],
        "M": [(("bool", True), None, 1), (("null",), None, 2), ((_NUM, 1), None, 3), (("str", "1"), None, 2)],
        "N": [(("null",), "NoneType", 8)],
        "NT": [(("null",), "NoneType", 8)],
        "S": [(("null",), "NoneType", 1), ((_NUM, 1), "int", 2), ((_NUM, 2), "int", 3), ((_NUM, 3), "int", 1),
              (("str", "x"), "str", 1)],
        "B": [(("bool", True), "bool", 1), (("null",), "NoneType", 1), ((_NUM, 0), "int", 2), ((_NUM, 1), "int", 3),
              ((_NUM, 1.5), "float", 1)],
        "A": [(("null",), "NoneType", 8)],
    },
}
MIXED = {"documents": {"M", "S", "B"}, "columnar": {"M"}}

# the calls each route makes, in order: the resident build and counts first, then the host route's counts.  The host
# route counts a field named twice twice; a mixed field goes up as tagged cells (9 bytes a number, 2 for "x" or True).
_F64, _STR, _COL = "value_counts_f64_host", "value_counts_str_packed", "value_counts_column"
CALLS = {
    ("documents", "resident"): [("table", 7, 6), *(("upload", j, 7) for j in range(6)), ("text", 7),
                                (_COL, 7), (_COL, 7), (_COL, 7), ("value_counts_text", 6), (_COL, 7), (_COL, 7), (_COL, 7),
                                (_STR, 6, 33), (_STR, 7, 56), (_STR, 7, 56)],
    ("documents", "host"): [(_F64, 6), (_F64, 6), (_F64, 6), (_STR, 6, 4), (_STR, 6, 33), (_STR, 7, 56), (_STR, 7, 56),
                            (_F64, 6)],
    ("documents", "rank_group"): [("table", 0, 1), ("text", 7), ("value_counts_text", 6), (_F64, 6), (_F64, 6),
                                  (_F64, 6), (_STR, 6, 33), (_STR, 7, 56), (_STR, 7, 56), (_F64, 6)],
    ("columnar", "resident"): [("table", 7, 4), *(("upload", j, 7) for j in range(4)), ("text", 7), ("text", 7),
                               (_COL, 7), (_COL, 7), (_COL, 7), ("value_counts_text", 6), (_COL, 7),
                               (_STR, 6, 33), (_F64, 6), (_STR, 1, 1), (_F64, 6), (_STR, 1, 2)],
    ("columnar", "host"): [(_F64, 6), (_F64, 6), (_F64, 6), (_STR, 6, 4), (_STR, 6, 33), (_F64, 6), (_STR, 1, 1),
                           (_F64, 6), (_STR, 1, 2), (_F64, 6)],
    ("columnar", "rank_group"): [("table", 0, 1), ("text", 7), ("text", 7), ("value_counts_text", 6), (_F64, 6),
                                 (_F64, 6), (_F64, 6), (_STR, 6, 33), (_F64, 6), (_STR, 1, 1), (_F64, 6), (_STR, 1, 2),
                                 (_F64, 6)],
}


@pytest.mark.parametrize("engine", list(ENGINES))
@pytest.mark.parametrize("store", ["documents", "columnar"])
def test_result_documents_and_engine_calls(store, engine):
    db = _documents() if store == "documents" else _columns()
    eng = ENGINES[engine]()
    got = _run(db, eng)
    assert [f for f, _g in got] == FIELDS
    for f, groups in got:
        assert _typed(groups, f in MIXED[store]) == GROUPS[store][f], (f, groups)
        assert all(g["_id"] is not None for g in groups[:-1]), f              # the null group comes last
    assert eng.calls == CALLS[store, engine]
    if eng.resident is not None:
        eng.resident.clear()
    assert not eng.live


# 70 values: ``numeric_column`` packs 64 and more with Arrow, where NaN is a value and None a null
LONG = [1.5, NAN, None, 2.0, 1.5, -0.0, 0.0] * 10
LONG_CALLS = {"resident": [("table", 70, 1), ("upload", 0, 70), (_COL, 70)], "host": [(_F64, 60)],
              "rank_group": [("table", 0, 1), (_F64, 60)]}


@pytest.mark.parametrize("engine", list(ENGINES))
@pytest.mark.parametrize("store", ["documents", "columnar"])
def test_a_long_number_field_with_nan_and_none(store, engine):
    if store == "documents":
        db = utils.Database()
        db.insert_one_in_file("d", {"_id": 0, "finished": True, "fields": ["W"]})
        db.insert_many_in_file("d", [{"_id": i + 1, **({"W": v} if v is not None else {})} for i, v in enumerate(LONG)])
    else:
        db = ColumnarDatabase()
        db.ingest_columns("d", {"W": _number(LONG, False)})
    eng = ENGINES[engine]()
    (f, groups), = _run(db, eng, ["W"])
    assert _typed(groups, False) == [(("null",), "NoneType", 11), ((_NUM, "nan"), "float", 10),
                                     ((_NUM, 0), "float", 20), ((_NUM, 1.5), "float", 20), ((_NUM, 2), "float", 10)]
    assert groups[-1]["_id"] is None and eng.calls == LONG_CALLS[engine]


def test_a_document_store_is_read_once_per_request(monkeypatch):
    """A cold request that needs the resident route and the host route reads the documents once; a warm request that
    the resident route answers alone reads none."""
    db, eng, reads = _documents(), _Engine(), []
    find = db.find
    monkeypatch.setattr(db, "find", lambda name, query: reads.append(name) or find(name, query))
    Histogram(db, utils.HistogramMetadata(db), eng).file_processing("d", "cold", FIELDS)
    assert reads.count("d") == 1
    Histogram(db, utils.HistogramMetadata(db), eng).file_processing("d", "warm", ["I", "T"])
    assert reads.count("d") == 1 and eng.resident.hits == 1
    eng.resident.clear()
    assert not eng.live
