"""GPU: ``$group`` of number columns with the staged binary64 group-by kernel (``k_group_f64``) on both of its entry
points — ``lo_value_counts_f64_host`` (a host column copied per call) and ``lo_value_counts_f64_table`` (rows of a device
table, nothing copied) — and the ``/histograms`` route that counts number fields from their HBM-resident slabs.

Kernel results are compared with ``collections.Counter`` over ``oracle.rsem.group_key`` of the exact bit patterns; the
route's result documents with the host packing route's, as multisets of (group key, type of the key, count)."""
import csv
import ctypes as C
import json
import threading
from collections import Counter
from pathlib import Path

import numpy as np
import pytest
from werkzeug.test import Client

from edge_values import f64 as _f64
from learningorchestra_b200 import _native as N
from learningorchestra_b200 import columnar, server, utils
from learningorchestra_b200.column_store import ColumnarDatabase, NumberColumn
from learningorchestra_b200.histogram import Histogram
from learningorchestra_b200.sharding import merge_value_counts
from oracle import rsem
from test_gpu_groupby_prepass import _last_slot_keys, _special_f64, _table_slots

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).resolve().parent / "golden"
STAGE_SLOTS = 1024            # kF64StageSlots (csrc/kernels.cuh)


def _oracle(x):
    u, uc = np.unique(np.asarray(x, np.float64).view(np.uint64), return_counts=True)
    exp = Counter()
    for b, c in zip(u.view(np.float64), uc):
        exp[rsem.group_key(float(b))] += int(c)
    return dict(exp)


def _groups(keys, counts):
    kb = keys.view(np.uint64)
    assert 0x8000000000000000 not in kb.tolist()                           # canonical keys: no -0.0, one NaN
    assert (kb[np.isnan(keys)] == 0x7FF8000000000000).all()
    got = {rsem.group_key(float(k)): int(c) for k, c in zip(keys, counts)}
    assert len(got) == len(keys)
    return got


def _both(engine, x, table=None):
    """Both entry points on the same column against the oracle; returns the table call's timing."""
    x = np.ascontiguousarray(x, np.float64)
    exp = _oracle(x)
    assert _groups(*engine.value_counts_f64_host(x)) == exp
    own = table is None
    if own:
        table = engine.table("f64", x.size, 1)
        if x.size:
            table.upload(0, x)
    t = {}
    try:
        assert _groups(*engine.value_counts_column(table, 0, timing=t)) == exp
    finally:
        if own:
            table.free()
    assert t["h2d_bytes"] == 0 and t["launches"] == (2 if x.size else 0)
    return t


def test_nan_zero_and_empty_marker_bit_patterns_and_keys_one_ulp_apart(engine):
    rng = np.random.default_rng(31)
    sp = np.concatenate([_special_f64(), _f64([0xFFFFFFFFFFFFFFFF, 0x7FFFFFFFFFFFFFFF])])   # the empty marker too
    x = np.concatenate([np.repeat(sp, rng.integers(1, 40, sp.size)), sp])
    rng.shuffle(x)
    _both(engine, x)


@pytest.mark.parametrize("n", [0, 1, 2, 3, 4, 5, 31, 32, 33, 63, 64, 65, 511, 512, 513, 1025])
def test_lengths_and_every_tail(engine, n):
    rng = np.random.default_rng(n)
    pool = np.concatenate([_special_f64(), rng.integers(-20, 20, 40).astype(np.float64) * 0.25])
    x = pool[rng.integers(0, pool.size, n)] if n else np.zeros(0)
    if n == 1:
        x = _f64([0xFFFFFFFFFFFFFFFF])                                      # the empty marker as the only value
    _both(engine, x)


def test_constant_three_value_and_twenty_thousand_value_columns(engine):
    n = 4_000_001
    _both(engine, np.full(n, 7.25))
    _both(engine, np.array([1.0, 2.0, 3.0])[np.arange(n) % 3])
    rng = np.random.default_rng(5)
    x = rng.integers(0, 20_000, n).astype(np.float64) * 0.5
    x[::1001] = np.nan
    x[::997] = -0.0
    _both(engine, x)


def test_all_distinct_column_overflows_every_ctas_stage(engine):
    m = 4_000_000
    grid = min((m + 511) // 512, engine.sm_count * 8)
    assert m // grid > 2 * STAGE_SLOTS                  # every CTA sees more distinct keys than its stage holds
    rng = np.random.default_rng(6)
    x = rng.permutation(m).astype(np.float64) * 1.5 - 1e6
    _both(engine, x)
    keys, counts = engine.value_counts_column(engine.table_from_numpy([x]), 0)
    assert keys.size == m and (counts == 1).all()


def test_last_slot_keys_meet_in_the_stage_flush(engine):
    keys = _last_slot_keys(2048, 16384, 17)
    rng = np.random.default_rng(18)
    mult = rng.choice([1, 1, 2, 3], keys.size)           # at most 8192 rows: a table of at most 16384 slots
    x = np.repeat(keys, mult)
    rng.shuffle(x)
    mask = np.uint64(_table_slots(x.size) - 1)
    from oracle import bsem_numpy as bn
    assert ((bn.splitmix64(keys.view(np.uint64)) & mask) == mask).all()
    _both(engine, x)
    _both(engine, np.tile(keys[:64], 5000))              # a few last-slot keys in every CTA: all staged, all flushed


def _kernel_names(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if "k_group_f64" in e.name]


def test_aligned_table_and_a_table_wrapped_at_an_8_byte_offset(engine):
    rng = np.random.default_rng(7)
    n = 1_000_003
    x = rng.integers(0, 300, n).astype(np.float64)
    x[::50] = np.nan
    base = engine.table("f64", n + 1, 2)
    base.upload(1, np.concatenate([[12345.0], x]))
    aligned = engine.table_from_numpy([x])
    wrapped = engine.wrap("f64", n, 1, base.base_ptr + base.pitch_bytes + 8, base.pitch_bytes, keepalive=base)
    assert (wrapped.base_ptr % 16) == 8 and (aligned.base_ptr % 256) == 0
    _both(engine, x, aligned)
    _both(engine, x, wrapped)
    names = _kernel_names(lambda: engine.value_counts_column(aligned, 0))
    assert names and all("<true>" in k for k in names), names
    names = _kernel_names(lambda: engine.value_counts_column(wrapped, 0))
    assert names and all("<false>" in k for k in names), names
    wrapped.free()
    aligned.free()
    base.free()


def test_contract_capacity_and_refusals_launch_nothing(engine):
    lib, ctx = engine._lib, engine._ctx
    x = np.arange(1000, dtype=np.float64) % 10
    t = engine.table_from_numpy([x])
    keys, counts, nd, tm = np.zeros(16), np.zeros(16, np.uint64), C.c_int64(-1), N.HostTiming()
    p = lambda a: a.ctypes.data_as(C.c_void_p)                               # noqa: E731
    N.check(lib.lo_value_counts_f64_table(ctx, t._h, 0, p(keys), p(counts), 16, C.byref(nd), C.byref(tm)))
    assert nd.value == 10 and tm.h2d_bytes == 0 and tm.launches == 2 and tm.kernel_ms > 0
    assert tm.d2h_bytes == 8 + 2 * 10 * 8
    rc = lib.lo_value_counts_f64_table(ctx, t._h, 0, p(keys), p(counts), 4, C.byref(nd), None)
    assert rc == N.LO_ERR_INVALID and nd.value == 10 and b"do not fit" in lib.lo_last_error()
    assert all(counts[i] == 100 for i in range(4))                          # what was written is exact
    f32 = engine.table("f32", 10, 1)
    before = engine.launch_count
    for args, msg in (((f32._h, 0, p(keys), p(counts), 16), b"LO_F64"),
                      ((t._h, 1, p(keys), p(counts), 16), b"column 1"),
                      ((t._h, -1, p(keys), p(counts), 16), b"column -1"),
                      ((t._h, 0, None, None, 16), b"NULL"),
                      ((None, 0, p(keys), p(counts), 16), b"NULL")):
        rc = lib.lo_value_counts_f64_table(ctx, *args, C.byref(nd), None)
        assert rc == N.LO_ERR_INVALID and msg in lib.lo_last_error(), (args, lib.lo_last_error())
    assert lib.lo_value_counts_f64_table(ctx, t._h, 0, p(keys), p(counts), 16, None, None) == N.LO_ERR_INVALID
    assert engine.launch_count == before
    f32.free()
    t.free()


# ---- /histograms ------------------------------------------------------------------------------------------------
NUMBER_FIELDS = ["PassengerId", "Survived", "Pclass", "Age", "SibSp", "Parch", "Fare"]


class _HostRoute:
    """The engine without ``resident``: /histograms packs every field per request (the route before this one)."""

    resident = None

    def __init__(self, engine):
        self._engine = engine

    def __getattr__(self, name):
        return getattr(self._engine, name)


def _typed(db, out):
    got = {}
    for d in db.find(out, {}):
        if d["_id"] != 0:
            (f, groups), = [(k, v) for k, v in d.items() if k != "_id"]
            got[f] = sorted(((columnar.group_key(g["_id"]), type(g["_id"]).__name__, g["count"]) for g in groups), key=repr)
    return got


def _host_route(db, name, fields, engine):
    out = f"host_{name}_{'_'.join(fields)}_{len(list(db.find(name, {})))}"
    Histogram(db, utils.HistogramMetadata(db), _HostRoute(engine)).file_processing(name, out, fields)
    return _typed(db, out)


class _Spy:
    """Records the timing of every value_counts_column call of an engine."""

    def __init__(self, engine, monkeypatch):
        self.calls, real = [], engine.value_counts_column

        def spy(table, col, timing=None):
            t = {}
            out = real(table, col, timing=t)
            self.calls.append(t)
            return out
        monkeypatch.setattr(engine, "value_counts_column", spy)


def _titanic_csv(tmp_path):
    g = json.loads((GOLD / "titanic_shaped_input.json").read_text())
    path = tmp_path / "t.csv"
    with open(path, "w", newline="") as f:
        csv.writer(f).writerows([g["headers"]] + g["rows"])
    return g, path


def test_post_files_field_types_then_histograms_on_number_fields(engine, tmp_path, monkeypatch):
    engine.resident.clear()
    _g, path = _titanic_csv(tmp_path)
    db = ColumnarDatabase()
    c = Client(server.create_app(db, engine, synchronous=True))
    assert c.post("/files", json={"datasetName": "t", "datasetURI": f"file://{path}"}).status_code == 201
    r = c.patch("/fieldTypes", json={"inputDatasetName": "t", "types": {f: "number" for f in NUMBER_FIELDS}})
    assert r.status_code == 200, r.get_data(as_text=True)
    spy = _Spy(engine, monkeypatch)
    fields = NUMBER_FIELDS + ["Sex"]
    r = c.post("/histograms", json={"inputDatasetName": "t", "outputDatasetName": "h1", "names": fields})
    assert r.status_code == 201, r.get_data(as_text=True)
    got = _typed(db, "h1")
    assert got == _host_route(db, "t", fields, engine)
    assert len(spy.calls) == len(NUMBER_FIELDS) and all(t["h2d_bytes"] == 0 for t in spy.calls)
    entry = engine.resident._entries["t"]
    assert all(entry.numbers[f] is not None for f in NUMBER_FIELDS) and entry.numbers["Sex"] is None
    hits = engine.resident.hits
    spy.calls.clear()
    r = c.post("/histograms", json={"inputDatasetName": "t", "outputDatasetName": "h2", "names": fields})
    assert r.status_code == 201 and _typed(db, "h2") == got and engine.resident.hits == hits + 1
    assert len(spy.calls) == len(NUMBER_FIELDS)
    engine.resident.clear()


def _nan_null_db():
    rng = np.random.default_rng(12)
    n = 200_003
    v = rng.integers(-50, 50, n).astype(np.float64) * 0.5
    v[rng.random(n) < 0.02] = np.nan                                          # real NaNs
    valid = rng.random(n) >= 0.03                                             # nulls (NaN in the slab)
    v[~valid] = np.nan
    whole = rng.integers(0, 9, n).astype(np.float64)
    is_int = rng.random(n) < 0.5                                              # ints and floats mixed: not collapsed
    db = ColumnarDatabase()
    db.ingest_columns("c", {"NaNs": NumberColumn(v, valid), "Mixed": NumberColumn(whole, None, is_int),
                            "Ints": NumberColumn(whole, None, np.ones(n, bool))})
    return db


def test_column_store_nans_nulls_and_key_types(engine, monkeypatch):
    engine.resident.clear()
    db = _nan_null_db()
    assert not db.column("c", "Mixed").integers_collapsed and db.column("c", "Ints").integers_collapsed
    spy = _Spy(engine, monkeypatch)
    fields = ["NaNs", "Mixed", "Ints"]
    Histogram(db, utils.HistogramMetadata(db), engine).file_processing("c", "out", fields)
    got = _typed(db, "out")
    assert got == _host_route(db, "c", fields, engine) and len(spy.calls) == 3
    nans = {k: (t, n) for k, t, n in got["NaNs"]}
    col = db.column("c", "NaNs")
    assert nans[("num", "nan")][1] == int((np.isnan(col.values) & col.valid).sum())
    assert nans[("null",)][1] == int((~col.valid).sum()) + 1                # + the metadata document
    assert {t for k, t, _n in got["Mixed"] if k != ("null",)} == {"float"}
    assert {t for k, t, _n in got["Ints"] if k != ("null",)} == {"int"}
    engine.resident.clear()


def _document_db():
    rng = np.random.default_rng(13)
    db = utils.Database()
    db.insert_one_in_file("d", {"_id": 0, "finished": True, "fields": ["A", "B", "C"]})
    docs = []
    for i in range(5000):
        d = {"_id": i + 1, "A": int(rng.integers(0, 40))}
        b = rng.random()
        if b < 0.9:
            d["B"] = float(rng.integers(0, 30)) * 0.25 if b > 0.05 else float("nan")
        if i % 7:
            d["C"] = int(rng.integers(0, 5)) if i % 2 else float(rng.integers(0, 5))
        docs.append(d)
    db.insert_many_in_file("d", docs)
    return db


def test_document_store_and_a_database_without_version(engine, monkeypatch):
    engine.resident.clear()
    db = _document_db()
    spy = _Spy(engine, monkeypatch)
    Histogram(db, utils.HistogramMetadata(db), engine).file_processing("d", "out", ["A", "B", "C"])
    want = _host_route(db, "d", ["A", "B", "C"], engine)
    assert _typed(db, "out") == want and len(spy.calls) == 3
    engine.resident.clear()

    class Foreign:                     # a database object without version(): never cached
        def __init__(self, db):
            self._db = db

        def find(self, *a):
            return self._db.find(*a)

        def insert_one_in_file(self, *a):
            return self._db.insert_one_in_file(*a)

        def update_one(self, *a):
            return self._db.update_one(*a)

    f = Foreign(db)
    Histogram(f, utils.HistogramMetadata(f), engine).file_processing("d", "out2", ["A", "B", "C"])
    assert _typed(db, "out2") == want and not engine.resident._entries and len(spy.calls) == 6


def test_a_slab_made_resident_by_a_binned_request_is_counted_without_an_upload(engine, monkeypatch):
    engine.resident.clear()
    db = _nan_null_db()
    Histogram(db, utils.HistogramMetadata(db), engine).file_processing("c", "b", ["NaNs", "Ints"], bins=16)
    entry = engine.resident._entries["c"]
    misses = engine.resident.misses
    uploads = []
    monkeypatch.setattr(type(entry.table), "upload", lambda self, *a, **k: uploads.append(a))
    spy = _Spy(engine, monkeypatch)
    Histogram(db, utils.HistogramMetadata(db), engine).file_processing("c", "out", ["NaNs", "Ints"])
    assert engine.resident._entries["c"] is entry and engine.resident.misses == misses and not uploads
    assert len(spy.calls) == 2 and all(t["h2d_bytes"] == 0 for t in spy.calls)
    monkeypatch.undo()
    assert _typed(db, "out") == _host_route(db, "c", ["NaNs", "Ints"], engine)
    engine.resident.clear()


def test_counting_threads_while_a_binned_request_rebuilds(engine, monkeypatch):
    from learningorchestra_b200.table_cache import ResidentDataset
    engine.resident.clear()
    db = _nan_null_db()
    want = _host_route(db, "c", ["NaNs", "Mixed"], engine)
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
                Histogram(db, utils.HistogramMetadata(db), engine).file_processing("c", out, ["NaNs", "Mixed"])
                if _typed(db, out) != want:
                    errors.append(out)
        except BaseException as exc:          # noqa: BLE001 — reported below
            errors.append(repr(exc))

    def binner():
        try:
            for i, fields in enumerate([["Ints"], ["NaNs"], ["Mixed", "Ints"], ["Ints"]]):
                Histogram(db, utils.HistogramMetadata(db), engine).file_processing("c", f"b{i}", fields, bins=8)
                if i % 2:
                    engine.resident.invalidate("c")
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


# ---- several devices ----------------------------------------------------------------------------------------------
def _column(n=3_000_001):
    rng = np.random.default_rng(14)
    x = rng.integers(0, 5000, n).astype(np.float64) * 0.125
    x[::333] = np.nan
    x[::777] = -0.0
    return x


def test_shard_groups_merged_from_tables_cut_from_one_column(engine):
    x = _column()
    cuts = [0, 1_000_032, 1_000_032, 2_500_000, x.size]                    # an empty cut included
    parts = []
    for a, b in zip(cuts, cuts[1:]):
        t = engine.table("f64", b - a, 1)
        if b > a:
            t.upload(0, x[a:b])
        parts.append(engine.value_counts_column(t, 0))
        t.free()
    assert _groups(*merge_value_counts(parts)) == _oracle(x)


def test_sharded_engine_over_every_visible_gpu_equals_one_device(engine):
    from learningorchestra_b200.sharding import ShardedEngine
    n = C.c_int()
    N.check(engine._lib.lo_device_count(C.byref(n)))
    x = _column()
    want = _groups(*engine.value_counts_column(engine.table_from_numpy([x]), 0))
    with ShardedEngine.local() as sh:
        t = sh.table_from_numpy([x])
        assert _groups(*sh.value_counts_column(t, 0)) == want == _oracle(x)
        t.free()
        db = _nan_null_db()
        Histogram(db, utils.HistogramMetadata(db), sh).file_processing("c", "out", ["NaNs", "Mixed"])
        assert _typed(db, "out") == _host_route(db, "c", ["NaNs", "Mixed"], engine)
        assert all(sh.resident._entries["c"].numbers[f] is not None for f in ("NaNs", "Mixed"))
        sh.resident.clear()
    if n.value < 2:
        pytest.skip("one visible GPU: the local group of two or more devices is unverified")
