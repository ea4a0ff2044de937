"""CPU: the sharing rules of ``table_cache.ResidentTables`` over seeded request sequences.  An entry rebuilt at the same
version shares its predecessor's table and text columns where it can; whatever a lease returns must hold exactly what a
fresh cache builds for the same request, and nothing may outlive ``clear()``.  A test double stands in for the device:
slabs are numpy columns, parsing is CPython's ``float()``, text columns are lists of cells."""
import math
import random

import numpy as np
import pyarrow as pa
import pytest

from learningorchestra_b200 import utils
from learningorchestra_b200.column_store import ColumnarDatabase, NumberColumn, ObjectColumn
from learningorchestra_b200.table_cache import ResidentTables


class _Obj:
    def __init__(self, live):
        self.live = live
        live.add(id(self))

    def free(self):
        assert id(self) in self.live, "freed twice"
        self.live.discard(id(self))


class _Table(_Obj):
    def __init__(self, live, nrows, ncols):
        super().__init__(live)
        self.ncols, self.pitch_bytes = ncols, nrows * 8
        self.cols = [np.full(nrows, np.nan) for _ in range(ncols)]

    def upload(self, col, values):
        self.cols[col] = np.array(values, np.float64)


class _Text(_Obj):
    def __init__(self, live, cells):
        super().__init__(live)
        self.cells = cells.to_pylist() if hasattr(cells, "to_pylist") else list(cells)
        self.nbytes = 8 * len(self.cells) + 8


class _Engine:
    def __init__(self):
        self.live = set()

    def table(self, dtype, nrows, ncols):
        return _Table(self.live, nrows, ncols)

    def text(self, cells):
        return _Text(self.live, cells)

    def parse_number_into(self, table, col, chars, offsets, nulls=None):
        out = {"first_invalid": None, "first_unsupported": None, "nulls": 0, "integer": True}
        for i in range(offsets.shape[0] - 1):
            null = nulls is not None and (not (nulls[0][(nulls[1] + i) >> 3] >> ((nulls[1] + i) & 7)) & 1
                                          if isinstance(nulls, tuple) else bool(nulls[i]))
            cell = chars[offsets[i]:offsets[i + 1]].tobytes().decode()
            try:
                v = math.nan if null or cell == "" else float(cell)
            except ValueError:
                out["first_invalid"] = i if out["first_invalid"] is None else out["first_invalid"]
                continue
            table.cols[col][i] = v
            out["nulls"] += null or cell == ""
            out["integer"] = out["integer"] and (math.isnan(v) or v.is_integer())
        return out


FIELDS = ["n", "f", "t", "w", "m", "meta", "none"]


def _value(rng, f):
    if rng.random() < 0.15 or f == "none":
        return None
    return {"n": lambda: rng.randint(-2, 3), "f": lambda: rng.choice([0.5, -0.0, float("nan"), 2.0]),
            "t": lambda: rng.choice(["1", "2.5", "", "-3"]), "w": lambda: rng.choice(["male", "female", "x"]),
            "m": lambda: rng.choice([1, "1"]), "meta": lambda: rng.randint(0, 3)}[f]()


def _dataset(rng, store):
    rows = [{f: _value(rng, f) for f in FIELDS} for _ in range(rng.randint(0, 9))]
    if store == "documents":
        db = utils.Database()
        db.insert_one_in_file("d", {"_id": 0, "finished": True, "fields": FIELDS, "meta": 7})
        db.insert_many_in_file("d", [{"_id": i + 1, **{f: v for f, v in r.items() if v is not None}}
                                     for i, r in enumerate(rows)])
        return db
    db = ColumnarDatabase()
    cols = {}
    for f in FIELDS:
        vals = [r[f] for r in rows]
        if f in ("t", "w"):
            cols[f] = pa.array(vals, type=pa.large_string())
        elif f == "m":
            cols[f] = ObjectColumn(vals)
        else:
            cols[f] = NumberColumn([math.nan if v is None else v for v in vals], [v is not None for v in vals],
                                   [type(v) is int for v in vals])
    db.ingest_columns("d", cols)
    db.update_one("d", {"meta": 7}, {"_id": 0})
    return db


def _same_slab(a, b):
    return np.array_equal(np.asarray(a).view(np.uint64), np.asarray(b).view(np.uint64))


def _check_against_fresh(db, entry, fields, text, numbers):
    fresh_engine = _Engine()
    fresh_cache = ResidentTables(fresh_engine)
    with fresh_cache.lease(db, "d", fields, text, numbers) as fresh:
        assert entry.version == fresh.version and np.array_equal(entry.ids, fresh.ids)
        slab_fields = list(fields) + [f for f in numbers if fresh.numbers[f] is not None]
        for f in slab_fields:
            i, j = entry.column[f], fresh.column[f]
            assert _same_slab(entry.table.cols[i], fresh.table.cols[j]), f
            assert (entry.kinds[i], entry.nulls[i]) == (fresh.kinds[j], fresh.nulls[j]), f
        for f in text:
            got, want = entry.texts[f], fresh.texts[f]
            assert (got is None) == (want is None), f
            if want is not None:
                assert got.cells == want.cells and entry.absent[f] == fresh.absent[f], f
        for f in numbers:
            assert entry.numbers[f] == fresh.numbers[f], f
            if fresh.numbers[f] is not None:
                assert entry.absent[f] == fresh.absent[f], f
    fresh_cache.clear()
    assert not fresh_engine.live


@pytest.mark.parametrize("store", ["documents", "columnar"])
@pytest.mark.parametrize("seed", range(20))
def test_leased_entries_equal_a_fresh_build_and_nothing_leaks(store, seed):
    rng = random.Random(seed)
    db = _dataset(rng, store)
    engine = _Engine()
    cache = ResidentTables(engine, max_bytes=rng.choice([1 << 30, 300]))
    held = []
    for _ in range(25):
        r = rng.random()
        if r < 0.7:
            fields = rng.sample(["n", "f", "t", "none"], rng.randint(0, 2))
            text = rng.sample(FIELDS, rng.randint(0, 3))
            numbers = rng.sample(FIELDS, rng.randint(0, 3))
            entry = cache.ensure(db, "d", fields, text, numbers)
            _check_against_fresh(db, entry, fields, text, numbers)
            held.append(entry)
        elif r < 0.8:
            db.update_one("d", {"t": rng.choice(["4", "", "0.25"])}, {"_id": rng.randint(1, 3)})
        elif r < 0.85:
            cache.invalidate("d")
        if held and rng.random() < 0.5:
            cache.release(held.pop(rng.randrange(len(held))))
    while held:
        cache.release(held.pop())
    cache.clear()
    assert not engine.live
