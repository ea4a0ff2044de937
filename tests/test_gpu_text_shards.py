"""GPU: ``$group`` of a text column cut into row-range shards (``lo_value_counts_text_shards``: per-shard count and key
gather, the copy to the root, the ``k_hash_sum_str`` merge) and the ``/histograms`` route of a ``ShardedEngine`` over
it.

One H100 is enough for the entry point: several pieces of one column are uploaded on the same context and counted as
shards.  Results are multisets of (key, count), compared with ``collections.Counter`` over ``columnar.group_key`` and
with ``value_counts_text`` on the whole column; every representative row must be a GLOBAL row whose cell equals its
group's key."""
import ctypes as C
import json
import threading
from collections import Counter

import numpy as np
import pyarrow as pa
import pytest

from learningorchestra_b200 import _native as N
from learningorchestra_b200 import columnar
from learningorchestra_b200.column_store import ColumnarDatabase

from test_gpu_text_value_counts import GOLD, TEXT_FIELDS, _count, _expected, _post_files, _results, _stores, _titanic

pytestmark = pytest.mark.gpu


def _multiset(keys, counts):
    return sorted(Counter({columnar.group_key(k): int(c) for k, c in zip(keys, counts)}).items())


def _call(engine, pieces, row0, capacity, outputs=True, timing=None, root=None, nshards=None):
    """One raw lo_value_counts_text_shards call: (rc, rows, counts, *ndistinct)."""
    k = len(pieces)
    handles = (C.c_void_p * max(k, 1))(*[p._h if p is not None else None for p in pieces])
    r0 = (C.c_int64 * max(k, 1))(*row0)
    rows, counts, nd = np.full(max(capacity, 1), -1, np.int64), np.zeros(max(capacity, 1), np.uint64), C.c_int64(-1)
    rc = engine._lib.lo_value_counts_text_shards(
        engine._ctx if root is None else root, handles, r0, k if nshards is None else nshards,
        rows.ctypes.data_as(C.c_void_p) if outputs else None, counts.ctypes.data_as(C.c_void_p) if outputs else None,
        capacity, C.byref(nd), C.byref(timing) if timing is not None else None)
    take = max(0, min(nd.value, capacity))
    return rc, rows[:take], counts[:take], nd.value


def _pieces(engine, arr, cuts):
    return [engine.text(arr.slice(b, e - b)) for b, e in zip(cuts, cuts[1:])]


def _check(engine, arr, cuts):
    """Count ``arr`` cut at ``cuts`` (0 = cuts[0] <= ... <= cuts[-1] = len(arr)) as shards on one context."""
    cells = arr.to_pylist()
    n = len(cells)
    assert cuts[0] == 0 and cuts[-1] == n and list(cuts) == sorted(cuts)
    pieces, whole = _pieces(engine, arr, cuts), engine.text(arr)
    try:
        present = [c for c in cells if c is not None]
        want = sorted(Counter(columnar.group_key(c) for c in present).items())
        wrep, wcounts = engine.value_counts_text(whole)
        assert _multiset([cells[int(r)] for r in wrep], wcounts) == want
        t, l0 = N.HostTiming(), engine.launch_count
        rc, rows, counts, nd = _call(engine, pieces, cuts[:-1], max(len(present), 1), timing=t)
        assert rc == N.LO_OK, engine._lib.lo_last_error()
        live = sum(1 for p in pieces if p.n > p.nulls)
        assert engine.launch_count - l0 == t.launches == (5 * live + 3 if present else 0)
        assert t.h2d_bytes == 0 and t.d2h_bytes == (8 + 16 * nd if present else 0)
        keys = []
        for r in rows:
            assert 0 <= r < n and cells[int(r)] is not None
            keys.append(cells[int(r)])
        assert len(set(keys)) == len(keys) == nd
        assert _multiset(keys, counts) == want
    finally:
        for p in pieces + [whole]:
            p.free()


def test_small_cuts_empty_all_null_and_one_row_pieces(engine):
    base = pa.array(["x", "y"] * 3 + [None] * 40 + ["é", "", "x", None, "z", "x"] * 20, type=pa.large_string())
    arr = base.slice(3, len(base) - 5)          # offsets past 0 and a bit offset of 3 under every piece
    n = len(arr)
    for cuts in ([0, n], [0, 0, n], [0, n, n], [0, 1, n], [0, 3, 43, n], [0, 0, 1, 2, 3, 43, 44, 90, n],
                 [0, 5, 5, 9, 17, 18, n]):
        _check(engine, arr, cuts)
    _check(engine, pa.array([None] * 50, type=pa.large_string()), [0, 20, 50])
    _check(engine, pa.array([], type=pa.large_string()), [0, 0, 0])


def test_constant_three_value_20000_value_and_all_distinct_columns(engine):
    n = 2_000_003
    const = pa.array(np.full(n, "S", dtype=object), type=pa.large_string())
    _check(engine, const, [0, 0, 1, 1000, 1_000_001, n])            # every cut inside the one run
    three = pa.array(np.array(["S", "C", "Q"], dtype=object)[np.arange(n) % 3], type=pa.large_string())
    _check(engine, three, [0, 7, 600_013, 1_200_000, n])
    rng = np.random.default_rng(11)
    keys = np.array(["v%d" % i for i in range(20_000)], dtype=object)
    many = pa.array(keys[rng.integers(0, 20_000, 1_000_000)], type=pa.large_string())
    _check(engine, many, [0, 250_001, 500_000, 750_003, 1_000_000])
    m = 1_000_000
    distinct = pa.array([str(i) for i in range(m)], type=pa.large_string())
    _check(engine, distinct, [0, 1, 125_000, 250_001, 375_000, 500_003, 625_000, 750_000, 875_007, m])


def test_titanic_shaped_fields(engine):
    g = _titanic()
    n = len(g["rows"])
    for j, f in enumerate(g["headers"]):
        cells = [None if (i * 7 + j) % 11 == 0 else row[j] for i, row in enumerate(g["rows"])]   # and some nulls
        arr = pa.array(cells, type=pa.large_string())
        _check(engine, arr, [0, 13, 300, 300, 301, 777, n])


def test_colliding_keys_meet_only_in_the_merge(engine):
    fx = json.loads((GOLD / "hash_collisions.json").read_text())
    pairs = [(p["a"], p["b"]) for p in fx["pairs"]]
    left = [a for a, _b in pairs for _ in range(5)] + [None, "only-left"]
    right = [None] + [b for _a, b in pairs for _ in range(3)] + ["only-right"]
    arr = pa.array(left + right, type=pa.large_string())
    assert len(arr) * 2 <= fx["table_slots"]           # each shard and the merge use a table of table_slots slots
    _check(engine, arr, [0, len(left), len(arr)])
    # the other way round, and each key split over both pieces as well
    _check(engine, pa.array(right + left, type=pa.large_string()), [0, len(right), len(arr)])
    both = pa.array(left + right + left, type=pa.large_string())
    _check(engine, both, [0, len(left) + 4, len(both)])


def test_one_shard_is_value_counts_text_with_an_offset(engine):
    arr = pa.array(["a", None, "b", "a", "c", "a"], type=pa.large_string())
    piece = engine.text(arr)
    try:
        rc, rows, counts, nd = _call(engine, [piece], [1000], 8)
        assert rc == N.LO_OK and nd == 3
        assert sorted((arr[int(r) - 1000].as_py(), int(c)) for r, c in zip(rows, counts)) == [("a", 3), ("b", 1), ("c", 1)]
    finally:
        piece.free()


def test_capacity_contract(engine):
    arr = pa.array(["a", "b", None, "c", "a", "d", "b"], type=pa.large_string())
    pieces = _pieces(engine, arr, [0, 3, 7])
    lib = engine._lib
    try:
        rc, _rows, _counts, nd = _call(engine, pieces, [0, 3], 3)
        assert rc == N.LO_ERR_INVALID and nd == 4 and "capacity" in lib.lo_last_error().decode()
        rc, _rows, _counts, nd = _call(engine, pieces, [0, 3], 0, outputs=False)
        assert rc == N.LO_ERR_INVALID and nd == 4
        rc, rows, counts, nd = _call(engine, pieces, [0, 3], 4)
        assert rc == N.LO_OK and nd == 4 and int(counts.sum()) == 6
        assert sorted(arr[int(r)].as_py() for r in rows) == ["a", "b", "c", "d"]
    finally:
        for p in pieces:
            p.free()


def test_refusals_launch_nothing(engine):
    arr = pa.array(["a", "b", "c", "a"] * 4, type=pa.large_string())
    pieces = _pieces(engine, arr, [0, 8, 16])
    lib = engine._lib
    cases = [
        (dict(pieces=pieces, row0=[0, 8], capacity=4, root=C.c_void_p(0)), "root"),
        (dict(pieces=[pieces[0], None], row0=[0, 8], capacity=4), "shards[1]"),
        (dict(pieces=pieces, row0=[0, 8], capacity=4, nshards=0), "nshards"),
        (dict(pieces=[pieces[0]] * 17, row0=list(range(0, 17 * 8, 8)), capacity=4), "nshards"),
        (dict(pieces=pieces, row0=[0, 7], capacity=4), "row0[1]"),             # overlapping
        (dict(pieces=pieces, row0=[8, 0], capacity=4), "row0[1]"),             # decreasing
        (dict(pieces=pieces, row0=[-1, 8], capacity=4), "row0[0]"),
        (dict(pieces=pieces, row0=[0, 8], capacity=4, outputs=False), "NULL"),
    ]
    try:
        for kw, word in cases:
            l0 = engine.launch_count
            rc, _rows, _counts, _nd = _call(engine, **kw)
            assert rc == N.LO_ERR_INVALID and word in lib.lo_last_error().decode(), (word, lib.lo_last_error())
            assert engine.launch_count == l0, word
        nd = C.c_int64()
        r0 = (C.c_int64 * 2)(0, 8)
        assert lib.lo_value_counts_text_shards(engine._ctx, None, r0, 2, None, None, 0, C.byref(nd), None) == N.LO_ERR_INVALID
        handles = (C.c_void_p * 2)(pieces[0]._h, pieces[1]._h)
        assert lib.lo_value_counts_text_shards(engine._ctx, handles, None, 2, None, None, 0, C.byref(nd), None) == N.LO_ERR_INVALID
        rc, _rows, _counts, nd = _call(engine, pieces, [0, 8], 3)             # the success path still works
        assert rc == N.LO_OK and nd == 3
    finally:
        for p in pieces:
            p.free()


def test_concurrent_calls_on_the_same_pieces(engine):
    rng = np.random.default_rng(5)
    keys = np.array(["k%d" % i for i in range(300)], dtype=object)
    arr = pa.array(keys[rng.integers(0, 300, 300_000)], type=pa.large_string())
    want = sorted(Counter(arr.to_pylist()).items())
    pieces = _pieces(engine, arr, [0, 100_000, 200_001, 300_000])
    errors = []

    def run():
        try:
            for _ in range(3):
                rc, rows, counts, _nd = _call(engine, pieces, [0, 100_000, 200_001], 300)
                got = sorted((arr[int(r)].as_py(), int(c)) for r, c in zip(rows, counts))
                if rc != N.LO_OK or got != want:
                    errors.append((rc, len(got)))
        except BaseException as exc:          # noqa: BLE001 — reported below
            errors.append(repr(exc))

    threads = [threading.Thread(target=run) for _ in range(4)]
    try:
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        assert not errors, errors
    finally:
        for p in pieces:
            p.free()


# ---- /histograms on a ShardedEngine over every visible GPU ----------------------------------------------------------
def test_sharded_engine_over_every_visible_gpu_equals_one_engine(engine, tmp_path):
    from learningorchestra_b200.sharding import ShardedEngine, ShardedText
    _, path = _stores(tmp_path)
    engine.resident.clear()
    one = ColumnarDatabase()
    _count(_post_files(one, engine, path), "t", "h", TEXT_FIELDS)
    single = _results(one, "h")
    engine.resident.clear()
    with ShardedEngine.local() as sh:
        db = ColumnarDatabase()
        c = _post_files(db, sh, path)
        _count(c, "t", "h", TEXT_FIELDS)
        assert _results(db, "h") == single == _expected(db, "t", TEXT_FIELDS)
        nrows = len(db.column("t", TEXT_FIELDS[0]).arr)
        bounds = sh.bounds(nrows)
        for f in TEXT_FIELDS:
            t = sh.resident._entries["t"].texts[f]
            assert isinstance(t, ShardedText) and len(t.pieces) == sh.nlocal
            assert [(o, o + p.n) for o, p in zip(t.offsets, t.pieces)] == bounds
            assert [p.engine for p in t.pieces] == sh.engines and t.n == nrows
        assert c.post("/files", json={"datasetName": "u", "datasetURI": f"file://{path}"}).status_code == 201
        sh.resident.max_bytes = 1
        for k in range(2):
            for name in ("t", "u"):
                _count(c, name, f"e{name}{k}", TEXT_FIELDS)
                assert _results(db, f"e{name}{k}") == single
                assert len(sh.resident._entries) == 1
        sh.resident.clear()
        nlocal = sh.nlocal
    if nlocal < 2:
        pytest.skip("one visible GPU: text shards on two or more devices are unverified")
