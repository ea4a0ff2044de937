"""CPU: the host side of counting number fields from HBM — the ctypes mirror of ``lo_value_counts_f64_table``, the
binary64 group-by kernel's build (both instantiations, 16-byte loads, no local memory), the exact merge of shard groups,
the number residency of ``table_cache`` and the ``/histograms`` route over it with a test double standing in for the
device, and the typing of keys and the NaN / ``null`` split on both stores."""
import ctypes as C
import math
import re
import subprocess
import itertools
from collections import Counter
from pathlib import Path

import numpy as np
import pyarrow as pa
import pytest

from learningorchestra_b200 import _native, columnar, utils
from learningorchestra_b200.column_store import ColumnarDatabase, NumberColumn
from learningorchestra_b200.histogram import Histogram, number_groups
from learningorchestra_b200.sharding import merge_value_counts
from learningorchestra_b200.table_cache import ResidentTables

ROOT = Path(__file__).resolve().parent.parent
HEADER = ROOT / "include" / "loexec.h"
CANON_NAN = 0x7FF8000000000000
_OUT = itertools.count()


def test_ctypes_mirror_of_the_table_entry_point_matches_the_header():
    text = re.sub(r"/\*.*?\*/", "", HEADER.read_text(), flags=re.S)
    assert int(re.search(r"#define LO_ABI_VERSION (\d+)", text).group(1)) == _native.LO_ABI_VERSION == 7
    params = [p.strip() for p in re.search(r"lo_value_counts_f64_table\s*\(([^)]*)\)", text).group(1).split(",")]
    res, args = _native.SIGNATURES["lo_value_counts_f64_table"]
    assert res is C.c_int and len(args) == len(params) == 8
    expect = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64),
              C.POINTER(_native.HostTiming)]
    assert params[2].startswith("int32_t ") and params[5].startswith("int64_t ")
    assert args == expect


def _sass_functions():
    sass = subprocess.run(["cuobjdump", "-sass", str(_native.LIB_PATH)], capture_output=True, text=True, check=True).stdout
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = out.setdefault(m.group(1), [])
        elif cur is not None:
            m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
            if m:
                cur.append(m.group(1).strip())
    return out


def test_group_kernel_instantiations_load_16_bytes_and_never_touch_local_memory(built):
    fns = _sass_functions()
    assert not [f for f in fns if "k_hash_count_f64" in f]                   # the old kernel is gone
    vec = fns["_ZN2lo11k_group_f64ILb1EEEvPKdxPyS3_y"]
    scalar = fns["_ZN2lo11k_group_f64ILb0EEEvPKdxPyS3_y"]
    assert any("LDG.E.128" in t for t in vec)                                 # two doubles per load
    assert not any("LDG.E.128" in t for t in scalar) and any("LDG.E.64" in t for t in scalar)
    for ins in (vec, scalar):
        assert not any(re.search(r"\b(LDL|STL)\b", t) for t in ins)
        assert any("ATOMS.CAS.64" in t for t in ins) and any("MATCH.ANY.U64" in t for t in ins)


def _bits(x):
    return np.asarray(x, np.float64).view(np.uint64)


def test_shard_merge_is_exact():
    rng = np.random.default_rng(3)
    big = (1 << 53) + 1
    shards = [
        (np.array([1.0, 0.0, 2.5, np.nan]), np.array([3, 4, big, 7], np.uint64)),
        (np.array([0.0, 7.0, np.nan]), np.array([1, 1, big], np.uint64)),      # NaN on two shards, 7 on this one only
        (np.array([2.5, 1.0]), np.array([big, 2], np.uint64)),
        (np.zeros(0), np.zeros(0, np.uint64)),                                 # an empty shard
    ]
    shards[0][0][3] = np.uint64(CANON_NAN).view(np.float64)
    shards[1][0][2] = np.uint64(CANON_NAN).view(np.float64)
    keys, counts = merge_value_counts(shards)
    exp = Counter()
    for k, c in shards:
        for b, n in zip(_bits(k).tolist(), c.tolist()):
            exp[b] += n
    got = dict(zip(_bits(keys).tolist(), counts.tolist()))
    assert got == dict(exp) and counts.dtype == np.uint64
    assert got[_bits([2.5])[0]] == 2 * big and got[CANON_NAN] == 7 + big     # above 2^53: not rounded
    # many random shards against Counter
    pool = np.concatenate([rng.integers(-50, 50, 60).astype(np.float64), [0.0, np.inf, -np.inf]])
    parts, exp = [], Counter()
    for _ in range(5):
        k = np.unique(pool[rng.integers(0, pool.size, 40)])
        c = rng.integers(1, 1 << 62, k.size, dtype=np.uint64)
        parts.append((k, c))
        for b, n in zip(_bits(k).tolist(), c.tolist()):
            exp[b] = (exp[b] + n) % (1 << 64)
    keys, counts = merge_value_counts(parts)
    assert dict(zip(_bits(keys).tolist(), counts.tolist())) == dict(exp)
    assert merge_value_counts([])[0].size == 0


# ---- a test double for the device: slabs kept as numpy columns, counted on the host ------------------------------
class _Table:
    def __init__(self, owner, nrows, ncols):
        self.owner, self.nrows, self.ncols, self.pitch_bytes = owner, nrows, ncols, nrows * 8
        self.cols = [np.full(nrows, np.nan) for _ in range(ncols)]
        owner.live.add(id(self))

    def upload(self, col, values):
        self.owner.uploads.append(col)
        self.cols[col] = np.array(values, np.float64)

    def free(self):
        self.owner.live.discard(id(self))


class _Text:
    def __init__(self, owner, cells):
        self.owner, self.cells = owner, cells.to_pylist() if hasattr(cells, "to_pylist") else list(cells)
        self.n, self.nulls, self.nbytes = len(self.cells), sum(c is None for c in self.cells), 8
        self.arr = pa.array(self.cells, type=pa.large_string())
        owner.live.add(id(self))

    def free(self):
        self.owner.live.discard(id(self))


def _canon(v):
    b = _bits(np.where(v == 0, 0.0, v)).copy()
    b[np.isnan(v)] = CANON_NAN
    return b


class _NumberEngine:
    """``table`` / ``value_counts_column`` / ``parse_number_into`` on the host; uploads and counts are recorded."""

    def __init__(self):
        self.live, self.uploads, self.counted, self.host_packed = set(), [], [], []
        self.resident = ResidentTables(self)

    def table(self, dtype, nrows, ncols):
        return _Table(self, nrows, ncols)

    def parse_number_into(self, table, col, chars, offsets, nulls=None):
        n = offsets.shape[0] - 1
        cells = [bytes(chars[offsets[i]:offsets[i + 1]]).decode() for i in range(n)]
        valid = np.ones(n, bool) if nulls is None else ~np.asarray(nulls, bool) if not isinstance(nulls, tuple) else \
            np.array([(nulls[0][(nulls[1] + i) >> 3] >> ((nulls[1] + i) & 7)) & 1 for i in range(n)], bool)
        vals = [float(c) if ok and c else math.nan for c, ok in zip(cells, valid)]
        table.cols[col] = np.array(vals)
        return {"first_invalid": None, "first_unsupported": None, "nulls": int(np.isnan(vals).sum()),
                "integer": all(math.isnan(v) or v.is_integer() for v in vals)}

    def text(self, cells):
        self.uploads.append("text")
        return _Text(self, cells)

    def value_counts_text(self, text):
        return self.value_counts_str_host(text.cells)

    def value_counts_column(self, table, col):
        self.counted.append(col)
        u, c = np.unique(_canon(table.cols[col]), return_counts=True)
        return u.view(np.float64), c.astype(np.uint64)

    def value_counts_f64_host(self, values):
        self.host_packed.append(len(values))
        u, c = np.unique(_canon(np.asarray(values, np.float64)), return_counts=True)
        return u.view(np.float64), c.astype(np.uint64)

    def value_counts_str_host(self, cells):
        first, counts = {}, Counter()
        for i, c in enumerate(cells):
            if c is None:
                continue
            first.setdefault(c, i)
            counts[c] += 1
        return np.array(list(first.values()), np.int64), np.array([counts[c] for c in first], np.uint64)

    def value_counts_str_packed(self, chars, offsets):
        return self.value_counts_str_host([bytes(chars[offsets[i]:offsets[i + 1]]) for i in range(offsets.size - 1)])


NAN = float("nan")
AGE = [22.0, None, 38.0, NAN, 22.0, -0.0, 0.0, None, 1.5, NAN]
PCLASS = [3, 1, 3, 2, None, 3, 1, 3, 3, 2]


def _column_db():
    db = ColumnarDatabase()
    age = np.array([NAN if v is None else v for v in AGE])
    db.ingest_columns("d", {
        "Age": NumberColumn(age, np.array([v is not None for v in AGE])),
        "Pclass": NumberColumn(np.array([NAN if v is None else v for v in PCLASS]),
                               np.array([v is not None for v in PCLASS]), np.array([v is not None for v in PCLASS])),
        "Sex": pa.array(["m", "f", "m", None, "f", "m", "m", "f", "m", "m"], type=pa.large_string()),
        "Fare": pa.array(["7.25", "71.3", "8", "", "8", None, "7.25", "9", "8", "1e3"], type=pa.large_string()),
    })
    return db


def _document_db(extra_meta=None):
    db = utils.Database()
    db.insert_one_in_file("d", {"_id": 0, "finished": True, "fields": ["Age", "Pclass"], **(extra_meta or {})})
    db.insert_many_in_file("d", [{"_id": i + 1, **({"Age": a} if a is not None else {}),
                                  **({"Pclass": p} if p is not None else {})} for i, (a, p) in enumerate(zip(AGE, PCLASS))])
    return db


def _reference(db, f):
    """The reference's $group over every document, metadata included: (group key, type of the key, count)."""
    docs = list(db.find("d", {})) if not hasattr(db, "has_columns") else \
        [{}] + [{f: v} for v in db.column("d", f).to_pylist()]
    c = Counter(columnar.group_key(d.get(f)) for d in docs)
    return sorted(c.items(), key=repr)


def _typed(groups):
    return sorted(((columnar.group_key(g["_id"]), type(g["_id"]).__name__, g["count"]) for g in groups), key=repr)


def _run(db, eng, fields):
    h = Histogram(db, utils.HistogramMetadata(db), eng)
    out = f"out{next(_OUT)}"
    h.file_processing("d", out, fields)
    return {next(k for k in d if k != "_id"): d[next(k for k in d if k != "_id")] for d in db.find(out, {}) if d["_id"] != 0}


def _host_route(db, fields):
    """What the same request returns through the host packing route (an engine without ``resident``)."""
    class _Host(_NumberEngine):
        resident = None

        def __init__(self):
            self.live, self.uploads, self.counted, self.host_packed = set(), [], [], []
    return _run(db, _Host(), fields)


@pytest.mark.parametrize("store", ["columnar", "documents"])
def test_number_fields_are_counted_from_the_slab_with_the_host_routes_key_types(store):
    db = _column_db() if store == "columnar" else _document_db()
    eng = _NumberEngine()
    got = _run(db, eng, ["Age", "Pclass"])
    host = _host_route(db, ["Age", "Pclass"])
    assert len(eng.counted) == 2 and not eng.host_packed                 # both from the slabs
    for f in ("Age", "Pclass"):
        assert _typed(got[f]) == _typed(host[f]), (store, f)
        assert sorted(((k, n) for k, _t, n in _typed(got[f])), key=repr) == _reference(db, f)
    age = {columnar.group_key(g["_id"]): g for g in got["Age"]}
    assert age[("num", "nan")]["count"] == 2 and age[("null",)]["count"] == 3   # two real NaNs; 2 nulls + metadata
    assert age[("num", 0)]["count"] == 2 and type(age[("num", 22)]["_id"]) is float
    assert all(type(g["_id"]) is int for g in got["Pclass"] if g["_id"] is not None)


def test_key_types_follow_integers_collapsed_on_a_column_store():
    db = ColumnarDatabase()
    vals = np.array([1.0, 2.0, 2.5, 1.0, np.inf])
    db.ingest_columns("d", {"A": NumberColumn(vals, None, np.array([True, True, False, True, False])),   # collapsed
                            "B": NumberColumn(vals, None, np.array([True, False, False, True, False]))})  # 2.0 a float
    eng = _NumberEngine()
    got = _run(db, eng, ["A", "B"])
    host = _host_route(db, ["A", "B"])
    assert _typed(got["A"]) == _typed(host["A"]) and _typed(got["B"]) == _typed(host["B"])
    assert {g["_id"]: type(g["_id"]) for g in got["A"]} == {1: int, 2: int, 2.5: float, math.inf: float, None: type(None)}
    assert {type(g["_id"]) for g in got["B"] if g["_id"] is not None} == {float}


def test_number_groups_split_nan_from_null():
    keys = np.array([np.uint64(CANON_NAN).view(np.float64), 3.0, 0.0])
    g = number_groups(keys, np.array([5, 2, 1], np.uint64), True, 3, 1)
    assert _typed(g) == sorted([(("num", "nan"), "float", 2), (("num", 3), "int", 2), (("num", 0), "int", 1),
                                (("null",), "NoneType", 4)], key=repr)
    g = number_groups(keys[:1], np.array([3], np.uint64), False, 3, 0)   # every NaN a null: no NaN group
    assert g == [{"_id": None, "count": 3}]
    assert number_groups(np.zeros(0), np.zeros(0, np.uint64), False, 0, 0) == []


def test_cache_counts_numbers_from_slabs_and_keeps_text_and_mixed_on_their_routes():
    db = _column_db()
    eng = _NumberEngine()
    cache = eng.resident
    with cache.lease(db, "d", ["Fare"]) as data:                          # a binned request parses the text field Fare
        assert data.numbers["Fare"] is None and "Fare" in data.column
    with cache.lease(db, "d", (), numbers=["Fare", "Age", "Sex", "Nope"]) as data:
        assert data.numbers == {"Fare": None, "Age": False, "Sex": None, "Nope": None}
        assert data.absent["Age"] == 1 and "Age" in data.column and "Fare" in data.column
    ups = len(eng.uploads)
    with cache.lease(db, "d", (), numbers=["Age", "Sex"]):                 # a hit: nothing uploaded
        pass
    assert len(eng.uploads) == ups and cache.hits == 1
    with cache.lease(db, "d", ["Age"]) as data:                           # a binned request on the counted slab: a hit
        assert data.numbers["Age"] is False
    assert len(eng.uploads) == ups and cache.hits == 2
    eng2 = _NumberEngine()
    got = _run(db, eng2, ["Fare", "Sex", "Age"])
    assert eng2.counted == [eng2.resident._entries["d"].column["Age"]]    # Fare and Sex are text: not from a slab
    host = _host_route(db, ["Fare", "Sex", "Age"])
    for f in ("Fare", "Sex", "Age"):
        assert _typed(got[f]) == _typed(host[f]), f


def test_a_slab_made_resident_by_a_binned_request_is_counted_without_an_upload():
    for db in (_column_db(), _document_db()):
        eng = _NumberEngine()
        with eng.resident.lease(db, "d", ["Age", "Pclass"]):
            pass
        ups = len(eng.uploads)
        got = _run(db, eng, ["Age"])
        assert len(eng.uploads) == ups and len(eng.counted) == 1 and eng.resident.hits == 1
        assert _typed(got["Age"]) == _typed(_host_route(db, ["Age"])["Age"])


def test_mixed_fields_and_fields_set_on_the_metadata_document_take_the_host_route():
    db = _document_db({"Age": 5})                                         # the metadata document sets Age
    db.insert_many_in_file("d", [{"_id": 11, "Mixed": 1}, {"_id": 12, "Mixed": "1"}])
    eng = _NumberEngine()
    with eng.resident.lease(db, "d", (), numbers=["Age", "Mixed", "Pclass"]) as data:
        assert data.numbers["Age"] is None and data.numbers["Mixed"] is None and data.numbers["Pclass"] is True
    got = _run(db, eng, ["Age", "Mixed", "Pclass"])
    host = _host_route(db, ["Age", "Mixed", "Pclass"])
    for f in ("Age", "Mixed", "Pclass"):
        assert _typed(got[f]) == _typed(host[f]), f
    assert len(eng.counted) == 1 and eng.host_packed                      # Pclass from its slab, Age packed
    cdb = ColumnarDatabase()
    cdb.ingest_columns("d", {"X": np.array([1.0, 2.0])})
    cdb.update_one("d", {"X": 9}, {"_id": 0})                            # the metadata document sets X
    with _NumberEngine().resident.lease(cdb, "d", (), numbers=["X"]) as data:
        assert data.numbers["X"] is None


def test_field_types_rebuilds_the_entry():
    db = utils.Database()
    db.insert_one_in_file("d", {"_id": 0, "finished": True, "fields": ["A"]})
    db.insert_many_in_file("d", [{"_id": i + 1, "A": s} for i, s in enumerate(["1", "2", "2", "x"])])
    eng = _NumberEngine()
    with eng.resident.lease(db, "d", (), numbers=["A"]) as data:
        assert data.numbers["A"] is None                                   # text before /fieldTypes
    for i, v in enumerate([1, 2, 2, None]):                               # what /fieldTypes "number" writes
        db.update_one("d", {"A": v}, {"_id": i + 1})
    misses = eng.resident.misses
    with eng.resident.lease(db, "d", (), numbers=["A"]) as data:
        assert data.numbers["A"] is True and eng.resident.misses == misses + 1
    got = _run(db, eng, ["A"])
    assert _typed(got["A"]) == _typed(_host_route(db, ["A"])["A"])
