"""CPU: the host side of dictionary codes of text columns — the header <-> ctypes mirror of ``LO_I32``,
``lo_text_codes`` and ``lo_text_codes_shards``, the SASS of their kernels, the dictionary read from first rows (one
column and the shard merge's order, against ``pyarrow.compute.dictionary_encode``), and the builder front-end's
``device_frame(..., text=True)`` with a test double standing in for the device."""
import ctypes as C
import re
from types import SimpleNamespace

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from learningorchestra_b200 import _native, builder_frontend, utils
from learningorchestra_b200.engine import _DTYPES, _NP, DeviceColumn, text_dictionary
from learningorchestra_b200.sharding import ShardedEngine, all_shard_bounds

from test_text_shards_cpu import HEADER, _sass_functions


def _params(text, name):
    return [p.strip() for p in re.search(r"\b%s\s*\(([^)]*)\)" % name, text).group(1).split(",")]


def test_ctypes_mirror_of_the_codes_entry_points_matches_the_header():
    text = re.sub(r"/\*.*?\*/", "", HEADER.read_text(), flags=re.S)
    assert int(re.search(r"#define LO_ABI_VERSION (\d+)", text).group(1)) == _native.LO_ABI_VERSION == 7
    dtypes = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define (LO_(?:F64|F32|U8|U32|I32))\s+(\d+)", text)}
    assert dtypes == {"LO_F64": 1, "LO_F32": 2, "LO_U8": 3, "LO_U32": 4, "LO_I32": 5}
    assert all(getattr(_native, k) == v for k, v in dtypes.items())
    assert _params(text, "lo_text_codes") == ["lo_ctx *ctx", "const lo_text *t", "lo_table *out", "int32_t col",
                                              "int64_t *first_rows_out", "int64_t capacity", "int64_t *ndistinct",
                                              "lo_host_timing *timing"]
    assert _params(text, "lo_text_codes_shards") == [
        "lo_ctx *root", "const lo_text *const *shards", "const int64_t *row0", "int32_t nshards", "lo_table *const *out",
        "int32_t col", "int64_t *first_rows_out", "int64_t capacity", "int64_t *ndistinct", "lo_host_timing *timing"]
    P = C.c_void_p
    assert _native.SIGNATURES["lo_text_codes"] == (C.c_int, [P, P, P, C.c_int32, P, C.c_int64, C.POINTER(C.c_int64),
                                                            C.POINTER(_native.HostTiming)])
    assert _native.SIGNATURES["lo_text_codes_shards"] == (C.c_int, [
        P, C.POINTER(P), C.POINTER(C.c_int64), C.c_int32, C.POINTER(P), C.c_int32, P, C.c_int64, C.POINTER(C.c_int64),
        C.POINTER(_native.HostTiming)])


def test_code_tables_are_int32_for_every_consumer():
    assert _DTYPES["i32"] == _native.LO_I32 and _NP[_native.LO_I32] is np.int32
    table = SimpleNamespace(ncols=1, base_ptr=4096, pitch_bytes=256, nrows=10, dtype_code=_native.LO_I32)
    col = DeviceColumn(table, 0)
    assert col.__cuda_array_interface__["typestr"] == "<i4" and col.__cuda_array_interface__["shape"] == (10,)


def test_kernels_never_touch_local_memory_and_the_slot_pass_never_inserts(built):
    fns = _sass_functions()

    def one(name):
        found = [f for f in fns if re.search(r"\d%s[A-Z]" % name, f)]
        assert len(found) == 1, (name, found)
        return fns[found[0]]

    for name in ("k_text_slots", "k_hash_min_str", "k_compact_first", "k_rank_slots", "k_remap_codes"):
        assert not any(re.search(r"\b(LDL|STL)\b", t) for t in one(name)), name
    slots = one("k_text_slots")
    assert not any("CAS" in t for t in slots)                                  # a lookup: the table is never written
    assert any(re.search(r"\b(RED|ATOM)G?\.E\.MIN\.64\b", t) for t in slots)   # the first row
    merge = one("k_hash_min_str")
    assert any("ATOMG.E.CAS.64" in t for t in merge)
    assert any(re.search(r"\b(RED|ATOM)G?\.E\.MIN\.64\b", t) for t in merge)


# ---- dictionaries from first rows --------------------------------------------------------------------------------
def _first_rows(cells):
    """The first row of each distinct non-null cell, ascending: what lo_text_codes returns."""
    seen = {}
    for i, c in enumerate(cells):
        if c is not None and c not in seen:
            seen[c] = i
    return sorted(seen.values())


def _codes(cells, first):
    index = {cells[r]: k for k, r in enumerate(first)}
    return np.array([-1 if c is None else index[c] for c in cells], np.int32)


def _merged_first_rows(cells, bounds):
    """The shard merge: each shard's distinct cells with their GLOBAL first rows in the shard (in an arbitrary order,
    as a hash table compacts them), merged by the lowest first row of each cell, then sorted."""
    rng = np.random.default_rng(len(bounds))
    lowest = {}
    for b, e in bounds:
        local = [(cells[b + r], b + r) for r in _first_rows(cells[b:e])]
        for j in rng.permutation(len(local)):
            cell, row = local[j]
            lowest[cell] = min(lowest.get(cell, row), row)
    return sorted(lowest.values())


COLUMNS = {
    "mixed": ["b", None, "a", "", "b", None, "", "c", "a", "é", "日本", "é"] * 9,
    "empty": [],
    "all_null": [None] * 40,
    "one": ["S"] * 33,
    "late_words": [None] * 70 + ["z", "y", "x", "z"] * 5,
}


@pytest.mark.parametrize("name", list(COLUMNS))
def test_dictionary_from_first_rows_is_dictionary_encode(name):
    cells = COLUMNS[name]
    arr = pa.array(cells, type=pa.large_string())
    enc = pc.dictionary_encode(arr)
    first = _first_rows(cells)
    assert text_dictionary(arr, first).equals(enc.dictionary)
    np.testing.assert_array_equal(_codes(cells, first),
                                  enc.indices.fill_null(-1).to_numpy(zero_copy_only=False).astype(np.int32))
    sliced = pa.array([None, "q"] + cells, type=pa.large_string()).slice(2)      # offsets and a bit offset past 0
    assert text_dictionary(sliced, first).equals(enc.dictionary)
    for world in (1, 2, 3, 8, 16):
        assert _merged_first_rows(cells, all_shard_bounds(len(cells), world, align=1)) == first, world


# ---- device_frame(..., text=True) with a test double for the device ------------------------------------------------
class _Table:
    def __init__(self, log, nrows):
        self.log, self.nrows, self._h = log, nrows, object()
        log["made"].append(self)

    def column_view(self, col, keepalive=None):
        return ("view", self, col)

    def free(self):
        self._h = None


class _Cache:
    def __init__(self, log, data):
        self.log, self.data = log, data

    def ensure(self, database, filename, fields, text=(), numbers=(), snapshot=None):
        self.log["ensure"].append((list(fields), list(text), snapshot is not None))
        return self.data

    def release(self, entry):
        self.log["released"] += 1


class _Engine:
    def __init__(self, data, fail_on=None):
        self.log = {"made": [], "ensure": [], "released": 0, "codes": []}
        self.resident, self.fail_on = _Cache(self.log, data), fail_on

    def table(self, dtype, nrows, ncols):
        assert dtype == "i32" and ncols == 1
        return _Table(self.log, nrows)

    def text_codes(self, text, table, col):
        if text.arr is self.fail_on:
            raise RuntimeError("LO_ERR_NOMEM")
        self.log["codes"].append((text, table, col))
        return np.array(_first_rows(text.arr.to_pylist()), np.int64)


def _store():
    db = utils.Database()
    db.insert_one_in_file("d", {"_id": 0, "datasetName": "d", "finished": True, "fields": ["s", "a", "m", "t"]})
    for i in range(80):
        db.insert_one_in_file("d", {"_id": i + 1, "s": ["x", "y", None][i % 3], "a": float(i), "m": (i if i % 2 else "w"),
                                    "t": "k%d" % (i % 5)})
    return db


def _data(db):
    rows = sorted((d for d in db.find("d", {}) if d["_id"] != 0), key=lambda d: d["_id"])
    texts = {f: SimpleNamespace(arr=pa.array([d.get(f) for d in rows], type=pa.large_string()),
                                nulls=sum(d.get(f) is None for d in rows), n=len(rows)) for f in ("s", "t")}
    return SimpleNamespace(ids=np.arange(1, 81), table=_Table({"made": []}, 80), column={"a": 0}, kinds=["float"],
                           nulls=[0], texts=texts)


def test_device_frame_without_text_is_unchanged():
    db = _store()
    eng = _Engine(_data(db))
    frame = builder_frontend.device_frame(db, "d", eng)
    assert frame.fields == ["a"] and eng.log["ensure"] == [(["a"], [], False)] and not eng.log["made"]
    assert frame.dictionaries == {} and frame.kinds == {"a": "float"}
    frame.release()
    assert eng.log["released"] == 1


def test_device_frame_with_text_numbers_words_in_store_order():
    db = _store()
    data = _data(db)
    eng = _Engine(data)
    with builder_frontend.device_frame(db, "d", eng, text=True) as frame:
        assert eng.log["ensure"] == [(["a"], ["s", "t"], True)]             # the mixed field is not asked for
        assert frame.fields == ["s", "a", "t"]
        assert frame.kinds["s"] == frame.kinds["t"] == "text" and frame.kinds["a"] == "float"
        assert frame.nulls["s"] == data.texts["s"].nulls and frame.nulls["t"] == 0
        for f in ("s", "t"):
            enc = pc.dictionary_encode(data.texts[f].arr)
            assert frame.dictionaries[f].equals(enc.dictionary)
            (_v, table, col), = frame.columns[f]
            assert col == 0 and table.nrows == 80 and table._h is not None
        tables = list(eng.log["made"])
    assert len(tables) == 2 and all(t._h is None for t in tables) and eng.log["released"] == 1


def test_device_frame_frees_its_code_tables_when_a_field_fails():
    db = _store()
    data = _data(db)
    eng = _Engine(data, fail_on=data.texts["t"].arr)
    with pytest.raises(RuntimeError):
        builder_frontend.device_frame(db, "d", eng, text=True)
    assert len(eng.log["made"]) == 2 and all(t._h is None for t in eng.log["made"]) and eng.log["released"] == 1


def test_a_rank_group_refuses_to_number_a_part_of_a_column():
    sh = object.__new__(ShardedEngine)
    sh._N, sh.world, sh.nlocal = _native, 4, 1
    with pytest.raises(_native.LoexecError) as e:
        sh.text_codes(None, None, 0)
    assert e.value.code == _native.LO_ERR_INVALID and "every row" in e.value.message
