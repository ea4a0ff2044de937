"""CPU: the host side of counting text fields from HBM — the ctypes mirror of the lo_text_* / lo_value_counts_text
entry points, the text residency of ``table_cache`` and the ``/histograms`` route over it with a test double standing in
for the device, and the assembly of group keys and the ``null`` group from representative rows."""
import re
from collections import Counter
from pathlib import Path

import ctypes as C
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from learningorchestra_b200 import _native, columnar, utils
from learningorchestra_b200.column_store import ColumnarDatabase
from learningorchestra_b200.histogram import Histogram, text_groups
from learningorchestra_b200.table_cache import ResidentTables, is_text_field

ROOT = Path(__file__).resolve().parent.parent
HEADER = ROOT / "include" / "loexec.h"


def test_ctypes_mirror_of_the_text_entry_points_matches_the_header():
    text = re.sub(r"/\*.*?\*/", "", HEADER.read_text(), flags=re.S)
    assert int(re.search(r"#define LO_ABI_VERSION (\d+)", text).group(1)) == _native.LO_ABI_VERSION
    assert int(re.search(r"#define LO_TEXT_STAGE_SLOTS (\d+)", text).group(1)) == _native.LO_TEXT_STAGE_SLOTS
    for name in ("lo_text_upload", "lo_text_info", "lo_text_free", "lo_value_counts_text"):
        decl = re.search(name + r"\s*\(([^)]*)\)", text).group(1)
        params = [p.strip() for p in decl.split(",")]
        res, args = _native.SIGNATURES[name]
        assert res is C.c_int and len(args) == len(params), name
        for p, a in zip(params, args):
            if "lo_validity" in p:
                assert a is C.POINTER(_native.Validity), (name, p)
            elif "lo_host_timing" in p:
                assert a is C.POINTER(_native.HostTiming), (name, p)
            elif p.startswith("int64_t *"):
                assert a in (C.POINTER(C.c_int64), C.c_void_p), (name, p)
            elif p.startswith("size_t *"):
                assert a is C.POINTER(C.c_size_t), (name, p)
            elif p.startswith("int64_t "):
                assert a is C.c_int64, (name, p)
            elif "**" in p:
                assert a is C.POINTER(C.c_void_p), (name, p)
            else:
                assert a is C.c_void_p, (name, p)


# ---- a test double for the device: text columns "uploaded" as the Arrow arrays themselves -----------------------
class _Text:
    def __init__(self, owner, arr):
        self.owner, self.arr = owner, arr
        self.n, self.nulls = len(arr), arr.null_count
        self.nbytes = 8 * (len(arr) + 1) + int(pc.sum(pc.binary_length(arr)).as_py() or 0)
        owner.live.add(id(self))

    def free(self):
        self.owner.live.discard(id(self))


class _Table:
    def __init__(self, owner, nrows, ncols):
        self.owner, self.nrows, self.ncols, self.pitch_bytes = owner, nrows, ncols, nrows * 8
        owner.live.add(id(self))

    def upload(self, col, values):
        pass

    def free(self):
        self.owner.live.discard(id(self))


class _TextEngine:
    """``table`` / ``text`` / ``value_counts_text`` computed on the host: every upload is recorded."""

    def __init__(self):
        self.live, self.uploads = set(), []
        self.resident = ResidentTables(self)

    def table(self, dtype, nrows, ncols):
        return _Table(self, nrows, ncols)

    def text(self, cells):
        arr = cells if isinstance(cells, pa.Array) else pa.array(cells, type=pa.large_string())
        self.uploads.append(arr)
        return _Text(self, arr)

    def value_counts_text(self, text):
        first, counts = {}, Counter()
        for i, c in enumerate(text.arr.to_pylist()):
            if c is not None:
                first.setdefault(c, i)
                counts[c] += 1
        return np.array(list(first.values()), np.int64), np.array([counts[c] for c in first], np.uint64)


def _dbs(columns):
    docs = utils.Database()
    docs.insert_one_in_file("d", {"_id": 0, "finished": True, "fields": list(columns)})
    n = len(next(iter(columns.values())))
    docs.insert_many_in_file("d", [{"_id": i + 1, **{f: c[i] for f, c in columns.items() if c[i] is not None}}
                                   for i in range(n)])
    cdb = ColumnarDatabase()
    cdb.ingest_columns("d", {f: (pa.array(c, type=pa.large_string()) if is_text_field(c) else np.array(c, float))
                             for f, c in columns.items()})
    return [("documents", docs), ("columnar", cdb)]


COLS = {"Sex": ["male", "female", None, "male", "", "female", "male"],
        "Name": ["a", "b", "c", "d", "e", "f", "g"],
        "Age": [1.0, 2.0, 3.0, 4.0, 5.0, 6.0, 7.0]}


def test_text_columns_are_uploaded_once_and_rebuilt_after_a_write():
    for kind, db in _dbs(COLS):
        eng = _TextEngine()
        cache = eng.resident
        with cache.lease(db, "d", (), text=["Sex", "Age"]) as data:
            assert data.texts["Age"] is None                  # a number field is not kept as text
            assert data.texts["Sex"].arr.to_pylist() == COLS["Sex"]
            assert data.absent == {"Sex": 1, "Age": 1}        # the metadata document lacks both
        assert len(eng.uploads) == 1, kind
        with cache.lease(db, "d", (), text=["Sex"]):
            pass
        assert len(eng.uploads) == 1 and cache.hits == 1, kind
        with cache.lease(db, "d", (), text=["Sex"]) as held:     # a lease on the old entry across the rebuilds
            with cache.lease(db, "d", (), text=["Name"]) as data:   # a new field: only it is uploaded, Sex is shared
                assert set(f for f, t in data.texts.items() if t is not None) == {"Sex", "Name"}
                assert data.texts["Sex"] is held.texts["Sex"]
            assert len(eng.uploads) == 2, kind
            with cache.lease(db, "d", ["Age"]) as data:             # a number field (a binned request): no text upload
                assert data.texts["Sex"] is held.texts["Sex"] and "Age" in data.column
            assert len(eng.uploads) == 2 and cache.misses == 3, kind
            assert id(held.texts["Sex"]) in eng.live                # still held by the newest entry and the lease
        db.update_one("d", {"Sex": "x"}, {"_id": 3})
        with cache.lease(db, "d", (), text=["Sex"]) as data:   # the version moved: uploaded again
            assert "x" in data.texts["Sex"].arr.to_pylist(), kind
        assert len(eng.uploads) == 3, kind                   # only the requested field: the stale entry keeps nothing
        assert len(eng.live) == 2, kind                      # the stale entry's table and columns are all freed
        cache.clear()
        assert not eng.live, kind


def test_a_text_field_float_rejects_is_kept_and_does_not_raise():
    for kind, db in _dbs({"Sex": ["male", "female", "male"]}):
        eng = _TextEngine()
        with eng.resident.lease(db, "d", (), text=["Sex"]) as data:
            rep, counts = eng.value_counts_text(data.texts["Sex"])
        assert sorted(zip(data.texts["Sex"].arr.take(pa.array(rep)).to_pylist(), counts.tolist())) == \
            [("female", 1), ("male", 2)], kind


def test_byte_budget_counts_text_columns():
    for kind, db in _dbs(COLS):
        if kind == "documents":
            db.insert_many_in_file("e", [{"_id": i + 1, "Name": c} for i, c in enumerate(COLS["Name"])])
        else:
            db.ingest_columns("e", {"Name": pa.array(COLS["Name"], type=pa.large_string())})
        eng = _TextEngine()
        with eng.resident.lease(db, "d", (), text=["Name"]) as data:
            size = data.nbytes
            assert size == data.table.pitch_bytes * data.table.ncols + data.texts["Name"].nbytes > 0
        eng.resident.max_bytes = size                        # room for one dataset: the text column is what counts
        with eng.resident.lease(db, "e", (), text=["Name"]):
            pass
        assert list(eng.resident._entries) == ["e"] and len(eng.live) == 2, kind    # "d" evicted and freed


def test_a_field_set_on_a_non_data_document_is_not_taken_as_text():
    db = utils.Database()
    db.insert_one_in_file("d", {"_id": 0, "finished": True, "Sex": "meta"})
    db.insert_many_in_file("d", [{"_id": 1, "Sex": "male"}])
    eng = _TextEngine()
    with eng.resident.lease(db, "d", (), text=["Sex"]) as data:
        assert data.texts["Sex"] is None and not eng.uploads


def _groups(gs):
    return sorted((columnar.group_key(g["_id"]), g["count"]) for g in gs)


def test_histogram_counts_text_fields_from_the_resident_columns():
    """The route a real engine takes, with the host double: text fields from resident columns, the number field on its
    own route; the result documents equal the reference's $group (Counter over every document, metadata included)."""
    for kind, db in _dbs(COLS):
        eng = _TextEngine()
        eng.value_counts_f64_host = lambda v: (np.unique(v), np.unique(v, return_counts=True)[1].astype(np.uint64))
        h = Histogram(db, utils.HistogramMetadata(db), eng)
        h.file_processing("d", "out", ["Sex", "Name", "Age"])
        docs = {next(k for k in d if k != "_id"): d for d in db.find("out", {}) if d["_id"] != 0}
        for f in ("Sex", "Name", "Age"):
            values = [None] + COLS[f]                                  # the metadata document first
            expect = Counter(columnar.group_key(v) for v in values)
            assert _groups(docs[f][f]) == sorted(expect.items()), (kind, f)
        assert len(eng.uploads) == 2, kind                          # Sex and Name; Age is a number field


def test_text_groups_from_representative_rows_of_a_sliced_array_with_nulls():
    full = pa.array(["x", None, "y", "", "x", None, "é", "y", "x", "", None, "z"], type=pa.large_string())
    for start, length in ((0, 12), (3, 7), (1, 9), (5, 0)):
        arr = full.slice(start, length)
        cells = arr.to_pylist()
        first, counts = {}, Counter()
        for i, c in enumerate(cells):
            if c is not None:
                first.setdefault(c, i); counts[c] += 1
        rep = np.array(list(first.values()), np.int64)
        cnt = np.array([counts[c] for c in first], np.uint64)
        for r in rep:
            assert arr[int(r)].is_valid
        groups = text_groups(arr, rep, cnt, arr.null_count + 1)
        expect = Counter(columnar.group_key(c) for c in cells + [None])
        assert _groups(groups) == sorted(expect.items()), (start, length)
        assert groups[-1] == {"_id": None, "count": arr.null_count + 1}
