"""CPU: ``/projections`` with ``castTo: "float32"`` on both stores, with a test double standing in for the device
(``float()`` for the parser, ``oracle.bsem_numpy`` for the fp32 cast and the bins).  The fields cover ints and floats
with None, NaN beside None, all-null, absent, text with ``""``, None, ``"nan"``, padded exponent and a non-ASCII digit,
text with bad cells, a mixed field and a numeric object column.  The expected values, histograms and refusals are
literals: a change to how a field is read, ordered or refused shows up here."""
import itertools
import math

import numpy as np
import pyarrow as pa
import pytest

from learningorchestra_b200 import utils
from learningorchestra_b200.column_store import ColumnarDatabase, NumberColumn, ObjectColumn, TextColumn
from learningorchestra_b200.projection import Projection
from learningorchestra_b200.table_cache import ResidentTables
from oracle import bsem_numpy as bn

NAN, INF = math.nan, math.inf
ROWS = {                                             # _id 1..6
    "I": [3, None, 1, 2, None, 7],
    "F": [0.1, NAN, None, -0.0, 2.25, 1e300],
    "N": [None] * 6,
    "T": ["1", "", None, "nan", " 1e3 ", "١٢"],
    "X": ["1", "2", "x", None, "y", "5"],
    "M": [1, "2", 3.5, None, True, "a"],
    "O": [1, 2.5, None, 4, 5, 6],
}
_OUT = itertools.count()


class _Documents(utils.Database):
    """The document store, counting the reads of the dataset."""
    finds = 0

    def find(self, filename, query):
        self.finds += filename == "d"
        return super().find(filename, query)


def _documents(order=range(1, 7)):
    db = _Documents()
    docs = {i: {"_id": i, **{f: c[i - 1] for f, c in ROWS.items() if c[i - 1] is not None}} for i in range(1, 7)}
    docs[0] = {"_id": 0, "finished": True, "fields": list(ROWS)}
    for i in order:
        db.insert_one_in_file("d", docs[i])
    return db


def _number(values, is_int):
    valid = [v is not None for v in values]
    return NumberColumn([NAN if v is None else v for v in values], valid, [ok and is_int for ok in valid])


def _columns():
    db = ColumnarDatabase()
    text = {f: TextColumn(pa.array(ROWS[f], type=pa.large_string())) for f in ("T", "X")}
    db.ingest_columns("d", {"I": _number(ROWS["I"], True), "F": _number(ROWS["F"], False),
                            "N": _number(ROWS["N"], False), **text, "M": ObjectColumn(ROWS["M"]),
                            "O": ObjectColumn(ROWS["O"])})
    return db


# ---- a test double for the device ----------------------------------------------------------------------------------
class _Obj:
    def __init__(self, owner):
        self.owner = owner
        owner.live.add(id(self))

    def free(self):
        self.owner.live.discard(id(self))


class _Table(_Obj):
    def __init__(self, owner, dtype, nrows, ncols):
        super().__init__(owner)
        self.nrows, self.ncols, self.pitch_bytes = nrows, ncols, nrows * 8
        self.data = np.full((ncols, nrows), NAN, np.float64 if dtype == "f64" else np.float32)

    def upload(self, col, values):
        self.owner.calls.append("upload")
        self.data[col] = values

    def to_numpy(self, col):
        return self.data[col].copy()


class _Counts(_Obj):
    def __init__(self, owner, counts):
        super().__init__(owner)
        self.counts = counts

    def to_numpy(self):
        return self.counts


def _minmax(cols):
    fin = [x[np.isfinite(x)] for x in (bn.cast_f64_f32(c) for c in cols)]
    return (np.array([x.min() if x.size else 0 for x in fin], np.float32),
            np.array([x.max() if x.size else 0 for x in fin], np.float32), np.array([x.size for x in fin], np.uint64))


class _Engine:
    """The engine calls a ``castTo`` makes, on the host: the resident route's and the chunked host pipeline's."""

    def __init__(self):
        self.live, self.calls = set(), []
        self.resident = ResidentTables(self)

    def table(self, dtype, nrows, ncols):
        return _Table(self, dtype, nrows, ncols)

    def parse_number_into(self, table, col, chars, offsets, nulls=None):
        self.calls.append("parse")
        out = {"first_invalid": None, "first_unsupported": None, "nulls": 0, "integer": True}
        for i in range(offsets.shape[0] - 1):
            null = nulls is not None and not (nulls[0][(nulls[1] + i) >> 3] >> ((nulls[1] + i) & 7)) & 1
            cell = chars[offsets[i]:offsets[i + 1]].tobytes().decode()
            if null or cell == "":
                table.data[col, i] = NAN
                out["nulls"] += 1
                continue
            try:
                table.data[col, i] = v = float(cell)
            except ValueError:
                out["first_invalid"] = i if out["first_invalid"] is None else out["first_invalid"]
                continue
            out["integer"] = out["integer"] and math.isfinite(v) and v.is_integer()
        return out

    def project_cast(self, table, idx, out=None):
        out = out if out is not None else self.table("f32", table.nrows, len(idx))
        out.data[:] = bn.project_cast_hist(table.data, idx)[0]
        return out

    def project_cast_hist(self, table, idx, nbins, lo, hi, out=None):
        o, counts = bn.project_cast_hist(table.data, idx, nbins, lo, hi)
        if out is not None:
            out.data[:] = o
        return _Counts(self, counts)

    def minmax_cast(self, table, idx):
        return _minmax([table.data[c] for c in idx])

    def project_cast_hist_host(self, cols, nbins=None, lo=None, hi=None, out=None):
        o, counts = bn.project_cast_hist(np.array(cols, np.float64).reshape(len(cols), -1), range(len(cols)), nbins,
                                         lo, hi)
        for j, x in enumerate(o):
            out[j][:] = x
        return counts, {}

    def minmax_cast_host(self, cols):
        return _minmax(cols)


REQUESTS = {"plain": {}, "bins": {"bins": 4}, "range": {"bins": 4, "value_range": [0, 4]}}


def _run(db, eng, fields, request="plain"):
    """(the output rows as (_id, {field: value}) in the order the store holds them, the histogram document or None,
    the exception recorded or None); the job's ``finished`` flag is checked against the exception."""
    out = f"out{next(_OUT)}"
    job = Projection(utils.ProjectionMetadata(db), eng)
    job.create("d", out, list(fields), "mongodb://h/database.d?r", f"mongodb://h/database.{out}?r",
               cast_to="float32", **REQUESTS[request])
    try:
        job.wait()
    except Exception:
        pass                     # the job records it in the output's metadata document, read below
    meta = db.find_one(out, {"_id": 0})
    assert meta["finished"] is ("exception" not in meta), meta
    rows = [(d["_id"], {f: v for f, v in d.items() if f != "_id"}) for d in db.find(out, {}) if d["_id"] != 0]
    for i, row in rows:
        assert type(i) is int and all(v is None or type(v) is float for v in row.values()), (i, row)
    return rows, meta.get("histogram"), meta.get("exception")


def _bits(v):
    return None if v is None else int(np.float32(v).view(np.uint32))


def _columns_of(rows, fields):
    return {f: [_bits(r[f]) for _i, r in sorted(rows, key=lambda x: x[0])] for f in dict.fromkeys(fields)}


# what castTo writes for each field, in _id order: fp32 values as Python floats, None where the cell holds no number
VALUES = {
    "I": [3.0, None, 1.0, 2.0, None, 7.0],
    "F": [0.10000000149011612, NAN, None, -0.0, 2.25, INF],
    "N": [None] * 6,
    "T": [1.0, None, None, NAN, 1000.0, 12.0],
    "O": [1.0, 2.5, None, 4.0, 5.0, 6.0],
    "A": [None] * 6,
}
# the histogram document of a ``bins`` request without and with ``range``: field -> request -> (range, counts)
HISTOGRAMS = {
    "I": {"bins": ([1.0, 7.0], [2, 1, 0, 1]), "range": ([0.0, 4.0], [0, 1, 1, 1])},
    "F": {"bins": ([-0.0, 2.25], [2, 0, 0, 1]), "range": ([0.0, 4.0], [2, 0, 1, 0])},
    "N": {"bins": ([0.0, 1.0], [0, 0, 0, 0]), "range": ([0.0, 4.0], [0, 0, 0, 0])},
    "T": {"bins": ([1.0, 1000.0], [2, 0, 0, 1]), "range": ([0.0, 4.0], [0, 1, 0, 0])},
    "O": {"bins": ([1.0, 6.0], [1, 1, 1, 2]), "range": ([0.0, 4.0], [0, 1, 1, 1])},
    "A": {"bins": ([0.0, 1.0], [0, 0, 0, 0]), "range": ([0.0, 4.0], [0, 0, 0, 0])},
}
# every field both stores can cast, one named twice; a document store casts an absent field to None, a column store
# refuses it (below), and holds O as an object column
GOOD = {"documents": ["I", "F", "N", "T", "O", "A", "I"], "columnar": ["I", "F", "N", "T", "I"]}
_STORES = {"documents": _documents, "columnar": _columns}


def _expected(fields, request):
    values = {f: [_bits(v) for v in VALUES[f]] for f in fields}
    hist = None if request == "plain" else {
        f: {"bins": 4, "range": HISTOGRAMS[f][request][0], "counts": HISTOGRAMS[f][request][1]} for f in fields}
    return values, hist


@pytest.mark.parametrize("request_kind", list(REQUESTS))
@pytest.mark.parametrize("store", list(_STORES))
def test_cast_values_and_histograms(store, request_kind):
    db, eng = _STORES[store](), _Engine()
    version = db.version("d")
    rows, hist, exc = _run(db, eng, GOOD[store], request_kind)
    assert exc is None and [i for i, _r in rows] == [1, 2, 3, 4, 5, 6]
    assert (_columns_of(rows, GOOD[store]), hist) == _expected(GOOD[store], request_kind)
    assert db.version("d") == version
    eng.resident.clear()
    assert not eng.live


# the first refusal of a request; on a document store a field that is not numeric now wins over a bad text cell, as it
# already did on a column store
REFUSALS = {
    ("X", "M"): "field 'M' is not numeric; run /fieldTypes first",
    ("X",): "could not convert string to float: 'x'",
    ("M",): "field 'M' is not numeric; run /fieldTypes first",
}


@pytest.mark.parametrize("fields", [*REFUSALS, ("A",)])
@pytest.mark.parametrize("store", list(_STORES))
def test_refusals(store, fields):
    db, eng = _STORES[store](), _Engine()
    rows, hist, exc = _run(db, eng, fields, "bins")
    if fields == ("A",) and store == "documents":
        assert exc is None and _columns_of(rows, fields) == _expected(fields, "plain")[0]
        return
    message = REFUSALS.get(fields, "field 'A' is not numeric; run /fieldTypes first")
    assert exc is not None and message in exc and rows == [] and hist is None, exc
    assert not eng.resident._entries and not eng.live


def test_numeric_object_column_on_a_column_store():
    rows, _hist, exc = _run(_columns(), _Engine(), ["O"])
    assert exc is None and _columns_of(rows, ["O"]) == _expected(["O"], "plain")[0]


def test_document_store_out_of_id_order():
    """Rows are written in the order the store holds them; the first bad cell is the first in ``_id`` order."""
    db = _documents([4, 2, 0, 6, 1, 5, 3])
    rows, hist, exc = _run(db, _Engine(), GOOD["documents"], "bins")
    assert exc is None and [i for i, _r in rows] == [4, 2, 6, 1, 5, 3]
    assert (_columns_of(rows, GOOD["documents"]), hist) == _expected(GOOD["documents"], "bins")
    assert "could not convert string to float: 'x'" in _run(db, _Engine(), ["X"])[2]


@pytest.mark.parametrize("store", list(_STORES))
def test_a_repeat_cast_is_a_resident_hit(store):
    """The selected fields stay resident for the dataset's version: a repeat request uploads and parses nothing.  A
    document store is read once per request, cold or warm."""
    db, eng = _STORES[store](), _Engine()
    version = db.version("d")
    rows, hist, exc = _run(db, eng, GOOD[store], "bins")
    assert eng.calls.count("parse") == 1 and eng.resident.hits == 0
    assert getattr(db, "finds", 1) == 1
    eng.calls.clear()
    again = _run(db, eng, GOOD[store], "bins")
    assert (_columns_of(again[0], GOOD[store]), *again[1:]) == (_columns_of(rows, GOOD[store]), hist, exc)
    assert eng.calls == [] and eng.resident.hits == 1 and db.version("d") == version
    assert getattr(db, "finds", 2) == 2
    eng.resident.clear()
    assert not eng.live
