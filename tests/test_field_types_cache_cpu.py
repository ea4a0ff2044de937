"""CPU: ``/fieldTypes`` on a column store with an engine that keeps datasets resident, and the cache rule that carries
resident objects across versions: an object made from store column ``c`` with row ids ``ids`` serves every later version
that still holds the same ``c`` and ``ids`` objects.  Test doubles stand in for the device (those of
``test_table_cache_cpu``: slabs are numpy columns, parsing is CPython's ``float()``, text columns are lists of cells)."""
import math
import random

import numpy as np
import pyarrow as pa
import pytest

from learningorchestra_b200 import utils
from learningorchestra_b200.column_store import ColumnarDatabase, NumberColumn, TextColumn
from learningorchestra_b200.data_type_update import DataType
from learningorchestra_b200.table_cache import ResidentTables
from oracle_engine import OracleEngine
from test_table_cache_cpu import _check_against_fresh, _Engine, _Table, _Text


def _float(cell):
    try:
        return math.nan if cell is None or cell == "" else float(cell), None
    except ValueError:
        return math.nan, "invalid"


class _Device(_Engine):
    """The double of test_table_cache_cpu with what the resident conversions call; every call is recorded."""

    def __init__(self):
        super().__init__()
        self.calls = []

    def table(self, dtype, nrows, ncols):
        t = super().table(dtype, nrows, ncols)
        t.nrows = nrows
        real = t.upload
        t.upload = lambda col, values: (self.calls.append("upload"), real(col, values))[1]
        return t

    def text(self, cells):
        self.calls.append("text")
        t = super().text(cells)
        t.arr, t.n, t.nulls = pa.array(t.cells, type=pa.large_string()), len(t.cells), sum(c is None for c in t.cells)
        return t

    def parse_number_into(self, table, col, chars, offsets, nulls=None):
        self.calls.append("parse_number_into")
        return super().parse_number_into(table, col, chars, offsets, nulls)

    def copy_column(self, src, src_col, dst, dst_col):
        dst.cols[dst_col] = src.cols[src_col].copy()

    def parse_text_into(self, table, col, text):
        self.calls.append("parse_text_into")
        out = {"first_invalid": None, "first_unsupported": None, "nulls": 0, "integer": True}
        for i, cell in enumerate(text.cells):
            v, bad = _float(cell)
            if bad and out["first_invalid"] is None:
                out["first_invalid"] = i
            table.cols[col][i] = v
            out["nulls"] += cell is None or cell == ""
            out["integer"] = out["integer"] and (bad is not None or math.isnan(v) and cell in (None, "") or
                                                 (math.isfinite(v) and v.is_integer()))
        return out

    def to_numpy(self, table, col):
        return table.cols[col].copy()

    def format_column(self, table, col, valid, is_int):
        self.calls.append("format_column")
        cells = ["" if not ok else (str(int(v)) if ii else repr(float(v)))
                 for v, ok, ii in zip(table.cols[col].tolist(), valid, is_int)]
        t = _Text(self.live, cells)
        t.arr, t.n, t.nulls = pa.array(cells, type=pa.large_string()), len(cells), 0
        return t

    def parse_number_packed(self, chars, offsets):
        self.calls.append("parse_number_packed")
        cells = [chars[offsets[i]:offsets[i + 1]].tobytes().decode() for i in range(offsets.shape[0] - 1)]
        parsed = [_float(c) for c in cells]
        status = [3 if bad else 2 if c == "" else 1 if math.isfinite(v) and v.is_integer() else 0
                  for c, (v, bad) in zip(cells, parsed)]
        return np.array([v for v, _ in parsed]), np.array(status, np.uint8)


_Table.to_numpy = lambda self, col: self.cols[col].copy()


# ---- the cache rule over seeded sequences of writes and adoptions ------------------------------------------------
FIELDS = ["n", "t", "u", "w"]


def _cells(rng, n, words=False):
    pick = ["a", "b", None] if words else ["1", "2.5", "", "-3", None, "7"]
    return pa.array([rng.choice(pick) for _ in range(n)], type=pa.large_string())


def _number_of(arr):
    v = np.array([_float(c)[0] for c in arr.to_pylist()], np.float64)
    valid = np.array([c not in (None, "") for c in arr.to_pylist()], bool)
    return NumberColumn(v, valid, valid & np.isfinite(v) & (v == np.floor(v)))


@pytest.mark.parametrize("seed", range(20))
def test_entries_carried_across_writes_equal_a_fresh_build_and_nothing_leaks(seed):
    rng = random.Random(seed)
    n = rng.randint(0, 9)
    db = ColumnarDatabase()
    db.ingest_columns("d", {"n": NumberColumn([float(rng.randint(-2, 3)) for _ in range(n)]), "t": _cells(rng, n),
                            "u": _cells(rng, n), "w": _cells(rng, n, words=True)})
    engine = _Device()
    cache = ResidentTables(engine, max_bytes=rng.choice([1 << 30, 300]))
    held = []
    for _ in range(30):
        r = rng.random()
        if r < 0.55:
            kinds = {f: db.column("d", f).kind for f in FIELDS}
            fields = rng.sample([f for f in FIELDS if kinds[f] == "number" or f != "w"], rng.randint(0, 2))
            text, numbers = rng.sample(FIELDS, rng.randint(0, 3)), rng.sample(FIELDS, rng.randint(0, 3))
            entry = cache.ensure(db, "d", fields, text, numbers)
            _check_against_fresh(db, entry, fields, text, numbers)
            held.append(entry)
        elif r < 0.7:            # "number" of a text field: the parsed slab adopted, or the entry's own slab
            f = rng.choice(["t", "u"])
            col = db.column("d", f)
            if col.kind == "text":
                new = _number_of(col.arr)
                db.set_column("d", f, new)
                if rng.random() < 0.5:
                    slab = engine.table("f64", n, 1)
                    slab.cols[0] = np.where(new.valid, new.values, np.nan)
                    kind = "int" if bool((new.is_int | ~new.valid).all()) else "float"
                    cache.adopt("d", f, new, slab, slab=(kind, int((~new.valid).sum())))
                else:
                    cache.adopt("d", f, new, same_as=col)
        elif r < 0.85:           # "string" of a number field: the text column adopted
            f = rng.choice(["n", "t", "u"])
            col = db.column("d", f)
            if col.kind == "number":
                cells = ["" if not ok else (str(int(v)) if ii else repr(v))
                         for v, ok, ii in zip(col.values.tolist(), col.valid, col.is_int)]
                new = TextColumn(pa.array(cells, type=pa.large_string()))
                db.set_column("d", f, new)
                cache.adopt("d", f, new, engine.text(new.arr))
        elif r < 0.92:           # a text column replaced by another
            db.set_column("d", "w", TextColumn(_cells(rng, n, words=True)))
        elif r < 0.95:
            cache.invalidate("d")
        if held and rng.random() < 0.5:
            cache.release(held.pop(rng.randrange(len(held))))
    while held:
        cache.release(held.pop())
    cache.clear()
    assert not engine.live


# ---- the /fieldTypes routes --------------------------------------------------------------------------------------
def _db(columns):
    db = ColumnarDatabase()
    db.ingest_columns("d", {f: pa.array(c, type=pa.large_string()) for f, c in columns.items()})
    return db


COLS = {"A": ["1", "2.5", None, "", "4"], "B": ["x", "y", None, "x", "z"], "C": ["7", "8", "9", "10", "-1"]}


def _convert(db, engine, types):
    job = DataType(db, utils.DataTypeMetadata(db), engine)
    for f, t in types.items():
        job.field_converter("d", f, t)


def test_number_on_a_resident_text_column_moves_no_cell_and_the_next_requests_neither():
    db, eng = _db(COLS), _Device()
    eng.resident = ResidentTables(eng)
    with eng.resident.lease(db, "d", (), text=list(COLS)):        # a /histograms without bins made them resident
        pass
    eng.calls.clear()
    _convert(db, eng, {"A": "number", "C": "number"})
    assert eng.calls == ["parse_text_into", "parse_text_into"]
    want, _ = _db(COLS), None
    _convert(want, OracleEngine(), {"A": "number", "C": "number"})
    for f in ("A", "C"):
        a, b = db.column("d", f), want.column("d", f)
        assert np.array_equal(a.values.view(np.uint64), b.values.view(np.uint64)), f
        assert np.array_equal(a.valid, b.valid) and np.array_equal(a.is_int, b.is_int), f
    eng.calls.clear()
    m0 = eng.resident.misses
    with eng.resident.lease(db, "d", (), text=list(COLS), numbers=list(COLS)) as data:      # without bins
        assert data.texts["B"] is not None and data.numbers["A"] is not None and "C" in data.column
    with eng.resident.lease(db, "d", ["A", "C"]) as data:                                     # with bins
        assert np.array_equal(data.table.cols[data.column["A"]].view(np.uint64),
                              np.where(want.column("d", "A").valid, want.column("d", "A").values, np.nan).view(np.uint64))
    assert eng.calls == [] and eng.resident.misses == m0 + 1
    # "string" back: formatted from the slab, and the text column is counted with no upload
    _convert(db, eng, {"A": "string"})
    assert eng.calls == ["format_column"]
    assert db.column("d", "A").arr.to_pylist() == ["1", "2.5", "", "", "4"]
    with eng.resident.lease(db, "d", (), text=["A"]) as data:
        assert data.texts["A"].cells == ["1", "2.5", "", "", "4"]
    assert eng.calls == ["format_column"]
    eng.resident.clear()
    assert not eng.live


def test_a_slab_parsed_for_a_binned_request_is_the_result():
    db, eng = _db(COLS), _Device()
    eng.resident = ResidentTables(eng)
    with eng.resident.lease(db, "d", ["A"]):
        pass
    eng.calls.clear()
    h0, m0 = eng.resident.hits, eng.resident.misses
    _convert(db, eng, {"A": "number"})
    assert eng.calls == [] and eng.resident.hits == h0 + 1 and eng.resident.misses == m0
    with eng.resident.lease(db, "d", ["A"]) as data:
        shared = data.table
    assert eng.calls == [] and eng.resident.misses == m0 + 1 and shared is not None
    eng.resident.clear()
    assert not eng.live


def test_a_bad_cell_writes_what_the_packed_route_writes():
    cols = {"A": ["1", "2", "oops", "4", None]}
    db, eng = _db(cols), _Device()
    eng.resident = ResidentTables(eng)
    with pytest.raises(ValueError, match="could not convert string to float: 'oops'"):
        _convert(db, eng, {"A": "number"})
    assert db.column("d", "A").to_pylist() == [1, 2, "oops", "4", None]
    eng.resident.clear()
    assert not eng.live


class _RankGroup(_Device):
    world, nlocal = 2, 1


@pytest.mark.parametrize("case", ["non_ascii", "no_resident", "rank_group"])
def test_other_engines_and_non_ascii_text_keep_the_packed_route(case):
    cols = {"A": ["１２", "3", None]} if case == "non_ascii" else {"A": ["12", "3", None]}
    db = _db(cols)
    eng = _RankGroup() if case == "rank_group" else _Device()
    if case != "no_resident":
        eng.resident = ResidentTables(eng)
    _convert(db, eng, {"A": "number"})
    assert eng.calls == ["parse_number_packed"]
    assert db.column("d", "A").to_pylist() == [12, 3, None]
