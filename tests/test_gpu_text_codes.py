"""GPU: dictionary codes of resident text columns (``lo_text_codes`` / ``lo_text_codes_shards``: the slot pass after
``k_hash_count_str``, the first-row order, the shard merge by lowest first row) and the builder front-end's device frame
with ``text=True``.

The oracle is ``pyarrow.compute.dictionary_encode`` on the same ``large_string`` array: its indices with null -> -1, and
its dictionary.  Several shards of one column run on one context on a one-GPU box, across devices when there are more."""
import ctypes as C
import json

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest
import torch

from learningorchestra_b200 import _native as N
from learningorchestra_b200 import builder_frontend, utils
from learningorchestra_b200.column_store import ColumnarDatabase
from learningorchestra_b200.engine import text_dictionary

from test_gpu_text_value_counts import GOLD, _count, _post_files, _stores, _titanic

pytestmark = pytest.mark.gpu


def _oracle(arr):
    enc = pc.dictionary_encode(arr)
    return enc.indices.fill_null(-1).to_numpy(zero_copy_only=False).astype(np.int32), enc.dictionary


def _codes(engine, arr):
    """(codes, dictionary, timing) of ``arr`` numbered on the device from one resident text column."""
    text = engine.text(arr)
    table = engine.table("i32", len(arr), 1)
    try:
        t = {}
        first = engine.text_codes(text, table, 0, timing=t)
        assert np.all(np.diff(first) > 0)
        return table.to_numpy(0), text_dictionary(text.arr, first), t
    finally:
        table.free()
        text.free()


def _check(engine, arr):
    want_codes, want_dict = _oracle(arr)
    codes, dictionary, t = _codes(engine, arr)
    np.testing.assert_array_equal(codes, want_codes)
    assert dictionary.equals(want_dict)
    live = len(arr) - arr.null_count
    assert t["h2d_bytes"] == 0 and t["launches"] == (6 if live else 0)
    assert t["d2h_bytes"] == (8 + 8 * len(want_dict) if live else 0)
    return codes, dictionary


def _cuts(n, k):
    """k + 1 cut points of an n-row column into k uneven row ranges, the first of them empty when k > 2."""
    cuts = [0] + [n * j * 7 // (8 * k) for j in range(1, k)] + [n]
    if k > 2:
        cuts[1] = 0
    return cuts


def _call_shards(engine, pieces, tables, row0, capacity, col=0, first=True, root=None, nshards=None, out=True):
    k = len(pieces)
    handles = (C.c_void_p * max(k, 1))(*[p._h if p is not None else None for p in pieces])
    outs = (C.c_void_p * max(k, 1))(*[t._h if t is not None else None for t in tables])
    r0 = (C.c_int64 * max(k, 1))(*row0)
    rows, nd, t = np.full(max(capacity, 1), -1, np.int64), C.c_int64(-1), N.HostTiming()
    rc = engine._lib.lo_text_codes_shards(engine._ctx if root is None else root, handles, r0,
                                          k if nshards is None else nshards, outs if out else None, col,
                                          rows.ctypes.data_as(C.c_void_p) if first else None, capacity, C.byref(nd),
                                          C.byref(t))
    return rc, rows[:max(0, min(nd.value, capacity))], nd.value, t


def _check_shards(engine, arr, cuts):
    """The codes of ``arr`` cut at ``cuts`` as shards on one context equal the oracle's, launches as documented."""
    want_codes, want_dict = _oracle(arr)
    pieces = [engine.text(arr.slice(b, e - b)) for b, e in zip(cuts, cuts[1:])]
    tables = [engine.table("i32", e - b, 1) for b, e in zip(cuts, cuts[1:])]
    try:
        l0 = engine.launch_count
        rc, first, nd, t = _call_shards(engine, pieces, tables, cuts[:-1], max(len(arr) - arr.null_count, 1))
        assert rc == N.LO_OK, engine._lib.lo_last_error()
        live = sum(1 for p in pieces if p.n > p.nulls)
        assert engine.launch_count - l0 == t.launches == (8 * live + 5 if live else 0)
        assert t.h2d_bytes == 0
        np.testing.assert_array_equal(np.concatenate([tb.to_numpy(0) for tb in tables]), want_codes)
        assert nd == len(want_dict) and text_dictionary(arr, first).equals(want_dict)
    finally:
        for x in pieces + tables:
            x.free()


def _columns():
    fx = json.loads((GOLD / "hash_collisions.json").read_text())
    pairs = [c for p in fx["pairs"] for c in (p["a"], p["b"])]
    rng = np.random.default_rng(3)
    big = "q" * (70 << 10)
    base = pa.array([None if rng.random() < 0.2 else "k%d" % rng.integers(0, 12) for _ in range(2000)], type=pa.large_string())
    return {
        "empty": pa.array([], type=pa.large_string()),
        "all_null": pa.array([None] * 777, type=pa.large_string()),
        "one_value": pa.array(["S"] * 100_003, type=pa.large_string()),
        "empty_next_to_null": pa.array(["", None, "", "a", None, "", "a", None, "b", ""], type=pa.large_string()),
        "over_64_kib": pa.array([big, big + "x", None, big, big[:-1], big + "x", "", big], type=pa.large_string()),
        "last_byte": pa.array(["prefix-%03d" % (i % 7) for i in range(500)] + ["prefix-00\x00", "prefix-00\xff"],
                              type=pa.large_string()),
        "collisions": pa.array([pairs[(i * 5) % len(pairs)] for i in range(3 * len(pairs))] + [None] + pairs[::-1],
                               type=pa.large_string()),
        "non_ascii": pa.array(["é", "日本語", None, "😀", "e", "é", "日本", "日本語", "́e", "😀"] * 31, type=pa.large_string()),
        "bit_offset": base.slice(13, 1500),
    }


@pytest.mark.parametrize("name", list(_columns()))
def test_codes_match_dictionary_encode(engine, name):
    arr = _columns()[name]
    if name == "bit_offset":
        assert arr.offset % 8 != 0 and arr.null_count > 0
    codes, dictionary = _check(engine, arr)
    if name == "collisions":
        assert len(dictionary) == len(set(arr.to_pylist()) - {None})
    if name == "empty_next_to_null":
        assert dictionary.to_pylist() == ["", "a", "b"] and codes.tolist()[:3] == [0, -1, 0]


def test_all_distinct_million_rows(engine):
    n = 1_000_000
    rng = np.random.default_rng(9)
    arr = pa.array(np.array([str(i) for i in rng.permutation(n)], dtype=object), type=pa.large_string())
    codes, _dictionary = _check(engine, arr)
    np.testing.assert_array_equal(codes, np.arange(n, dtype=np.int32))


@pytest.mark.parametrize("k", [1, 2, 3, 8])
def test_shards_give_the_same_codes(engine, k):
    cols = _columns()
    n = 1_000_000
    rng = np.random.default_rng(k)
    cols["many"] = pa.array(np.array(["v%d" % i for i in range(5000)], dtype=object)[rng.integers(0, 5000, n)],
                            type=pa.large_string())
    cols["distinct"] = pa.array([str(i) for i in range(200_000)], type=pa.large_string())
    for name, arr in cols.items():
        _check_shards(engine, arr, _cuts(len(arr), k))


def test_sharded_engine_over_every_visible_gpu(engine):
    from learningorchestra_b200.sharding import ShardedEngine
    rng = np.random.default_rng(4)
    arr = pa.array([None if rng.random() < 0.1 else "c%d" % rng.integers(0, 3000) for _ in range(300_001)],
                   type=pa.large_string())
    want_codes, want_dict = _oracle(arr)
    with ShardedEngine.local() as sh:
        text = sh.text(arr)
        table = sh.table("i32", len(arr), 1)
        try:
            first = sh.text_codes(text, table, 0)
            np.testing.assert_array_equal(table.to_numpy(0), want_codes)
            assert text_dictionary(arr, first).equals(want_dict)
            assert [t.engine for t in table.shards] == sh.engines
        finally:
            table.free()
            text.free()


def test_capacity_contract(engine):
    arr = pa.array(["a", "b", None, "c", "a", "d"], type=pa.large_string())
    want_codes, _ = _oracle(arr)
    text, table = engine.text(arr), engine.table("i32", len(arr), 1)
    lib = engine._lib
    try:
        rows, nd = np.zeros(4, np.int64), C.c_int64()
        rc = lib.lo_text_codes(engine._ctx, text._h, table._h, 0, rows.ctypes.data_as(C.c_void_p), 2, C.byref(nd), None)
        assert rc == N.LO_ERR_INVALID and nd.value == 4 and "capacity" in lib.lo_last_error().decode()
        assert rows[:2].tolist() == [0, 1]
        np.testing.assert_array_equal(table.to_numpy(0), want_codes)          # written all the same
        pieces = [engine.text(arr.slice(0, 3)), engine.text(arr.slice(3, 3))]
        tables = [engine.table("i32", 3, 1), engine.table("i32", 3, 1)]
        try:
            rc, first, nd2, _t = _call_shards(engine, pieces, tables, [0, 3], 3)
            assert rc == N.LO_ERR_INVALID and nd2 == 4 and first.tolist() == [0, 1, 3]
        finally:
            for x in pieces + tables:
                x.free()
    finally:
        table.free()
        text.free()


def test_refusals_launch_nothing(engine):
    from learningorchestra_b200.engine import Engine
    arr = pa.array(["a", "b", "c", "a"] * 4, type=pa.large_string())
    lib = engine._lib
    text = engine.text(arr)
    good, f64, short, wide = (engine.table("i32", 16, 1), engine.table("f64", 16, 1), engine.table("i32", 15, 1),
                              engine.table("i32", 16, 2))
    pieces = [engine.text(arr.slice(0, 8)), engine.text(arr.slice(8, 8))]
    halves = [engine.table("i32", 8, 1), engine.table("i32", 8, 1)]
    other = Engine(0)                                    # a second context on the same device
    foreign = other.text(arr)
    rows, nd = np.zeros(16, np.int64), C.c_int64()
    rp = rows.ctypes.data_as(C.c_void_p)

    def single(t=text, out=good, col=0, first=True, cap=16, ndp=True):
        return lib.lo_text_codes(engine._ctx, t._h if t is not None else None, out._h if out is not None else None, col,
                                 rp if first else None, cap, C.byref(nd) if ndp else None, None)

    cases = [
        (lambda: single(t=None), "text"),
        (lambda: single(out=None), "out"),
        (lambda: single(out=f64), "LO_I32"),
        (lambda: single(out=short), "rows"),
        (lambda: single(col=1), "column"),
        (lambda: single(out=wide, col=-1), "column"),
        (lambda: single(t=foreign), "context"),
        (lambda: single(cap=-1), "negative"),
        (lambda: single(ndp=False), "ndistinct"),
        (lambda: single(first=False), "first_rows_out"),
        (lambda: _call_shards(engine, pieces, halves, [0, 8], 4, root=C.c_void_p(0))[0], "root"),
        (lambda: _call_shards(engine, [pieces[0], None], halves, [0, 8], 4)[0], "shards[1]"),
        (lambda: _call_shards(engine, pieces, [halves[0], None], [0, 8], 4)[0], "out[1]"),
        (lambda: _call_shards(engine, pieces, halves, [0, 8], 4, out=False)[0], "out"),
        (lambda: _call_shards(engine, pieces, [halves[0], f64], [0, 8], 4)[0], "LO_I32"),
        (lambda: _call_shards(engine, pieces, [halves[0], short], [0, 8], 4)[0], "rows"),
        (lambda: _call_shards(engine, pieces, halves, [0, 8], 4, col=1)[0], "column"),
        (lambda: _call_shards(engine, pieces, halves, [0, 8], 4, nshards=0)[0], "nshards"),
        (lambda: _call_shards(engine, [pieces[0]] * 17, [halves[0]] * 17, list(range(0, 17 * 8, 8)), 4)[0], "nshards"),
        (lambda: _call_shards(engine, pieces, halves, [0, 7], 4)[0], "row0[1]"),              # overlapping
        (lambda: _call_shards(engine, pieces, halves, [8, 0], 4)[0], "row0[1]"),              # decreasing
        (lambda: _call_shards(engine, pieces, halves, [-1, 8], 4)[0], "row0[0]"),
        (lambda: _call_shards(engine, pieces, halves, [0, 8], 4, first=False)[0], "first_rows_out"),
    ]
    if torch.cuda.device_count() > 1:
        far = Engine(1)
        elsewhere = far.table("i32", 16, 1)
        cases.append((lambda: single(out=elsewhere), "device"))
    try:
        for call, word in cases:
            l0 = engine.launch_count
            rc = call()
            assert rc == N.LO_ERR_INVALID and word in lib.lo_last_error().decode(), (word, lib.lo_last_error())
            assert engine.launch_count == l0, word
        r0 = (C.c_int64 * 2)(0, 8)
        outs = (C.c_void_p * 2)(halves[0]._h, halves[1]._h)
        handles = (C.c_void_p * 2)(pieces[0]._h, pieces[1]._h)
        assert lib.lo_text_codes_shards(engine._ctx, None, r0, 2, outs, 0, rp, 4, C.byref(nd), None) == N.LO_ERR_INVALID
        assert lib.lo_text_codes_shards(engine._ctx, handles, None, 2, outs, 0, rp, 4, C.byref(nd), None) == N.LO_ERR_INVALID
        # the compute entries refuse a code table
        for fn in (lambda: engine.value_counts_column(good, 0), lambda: engine.minmax_cast(good, [0]),
                   lambda: engine.project_cast(good, [0]), lambda: engine.hist_u8_cols(good, [0]),
                   lambda: good.checksum(0), lambda: engine.parse_text_into(good, 0, text)):
            with pytest.raises(N.LoexecError) as e:
                fn()
            assert e.value.code == N.LO_ERR_INVALID
        rc, first, nd2, _t = _call_shards(engine, pieces, halves, [0, 8], 4)      # the success path still works
        assert rc == N.LO_OK and nd2 == 3 and first.tolist() == [0, 1, 2]
    finally:
        for x in [text, good, f64, short, wide, foreign] + pieces + halves:
            x.free()
        other.close()
        if torch.cuda.device_count() > 1:
            elsewhere.free()
            far.close()


# ---- the builder front-end's device frame -----------------------------------------------------------------------------
def _frame_matches(frame, arrays):
    """Every text field of ``frame`` read in place by torch equals the oracle on ``arrays[field]``."""
    for f in frame.fields:
        if frame.kinds[f] != "text":
            continue
        parts = []
        for col in frame.columns[f]:
            t = torch.as_tensor(col, device=f"cuda:{col.table.engine.device}")
            assert t.dtype == torch.int32 and t.data_ptr() == col.data_ptr      # in place
            parts.append(t.cpu().numpy())
        want_codes, want_dict = _oracle(arrays[f])
        np.testing.assert_array_equal(np.concatenate(parts), want_codes)
        assert frame.dictionaries[f].equals(want_dict), f
        assert frame.nulls[f] == arrays[f].null_count


def _code_tables(frame):
    return [t for t, _d in frame._codes.values()]


def test_device_frame_with_text_after_post_files(engine, tmp_path, monkeypatch):
    g = _titanic()
    stores, path = _stores(tmp_path)
    engine.resident.clear()
    db = ColumnarDatabase()
    c = _post_files(db, engine, path)
    arrays = {f: db.column("t", f).arr for f in g["headers"]}
    with builder_frontend.device_frame(db, "t", engine) as plain:
        assert plain.fields == []                                          # every field of an upload is text
    with builder_frontend.device_frame(db, "t", engine, text=True) as frame:
        assert frame.fields == list(g["headers"]) and all(frame.kinds[f] == "text" for f in frame.fields)
        _frame_matches(frame, arrays)
        codes = {f: np.concatenate([torch.as_tensor(col, device="cuda").cpu().numpy() for col in frame.columns[f]])
                 for f in frame.fields}
        dictionaries = {f: frame.dictionaries[f].to_pylist() for f in frame.fields}
        tables = _code_tables(frame)
    assert tables and all(t._h is None for t in tables)                    # freed by release()
    # after a /histograms on the same fields the frame is a cache hit and uploads no text
    engine.resident.clear()
    _count(c, "t", "h", list(g["headers"]))
    uploads = []
    real = engine.text
    monkeypatch.setattr(engine, "text", lambda cells, timing=None: uploads.append(1) or real(cells, timing))
    h0 = engine.resident.hits
    with builder_frontend.device_frame(db, "t", engine, text=True) as frame:
        assert engine.resident.hits == h0 + 1 and not uploads
        _frame_matches(frame, arrays)
    monkeypatch.undo()
    # the same frame on a document store
    docs = dict(stores)["documents"]
    with builder_frontend.device_frame(docs, "t", engine, text=True) as frame:
        assert frame.fields == list(g["headers"])
        for f in frame.fields:
            got = np.concatenate([torch.as_tensor(col, device="cuda").cpu().numpy() for col in frame.columns[f]])
            np.testing.assert_array_equal(got, codes[f])
            assert frame.dictionaries[f].to_pylist() == dictionaries[f], f
    engine.resident.clear()


def test_device_frame_numbers_and_words_in_store_order(engine):
    db = utils.Database()
    db.insert_one_in_file("d", {"_id": 0, "datasetName": "d", "finished": True, "fields": ["s", "a", "m", "b"],
                                "timeCreated": "t"})
    rng = np.random.default_rng(2)
    a = rng.normal(size=5000)
    words = np.array(["male", "female", "", "x"], dtype=object)
    for i in range(5000):
        db.insert_one_in_file("d", {"_id": i + 1, "s": None if i % 9 == 0 else str(words[i % 4]), "a": float(a[i]),
                                    "m": (i if i % 2 else "w%d" % i), "b": (int(i) if i % 7 else None)})
    engine.resident.clear()
    with builder_frontend.device_frame(db, "d", engine) as plain:          # without text: as before
        assert plain.fields == ["a", "b"] and plain.dictionaries == {} and not plain._codes
        ptr = {f: plain.columns[f][0].data_ptr for f in plain.fields}
    with builder_frontend.device_frame(db, "d", engine, text=True) as frame:
        assert frame.fields == ["s", "a", "b"]                              # store order; the mixed field stays out
        assert frame.kinds["s"] == "text" and frame.kinds["a"] != "text" and frame.kinds["b"] != "text"
        assert {f: frame.columns[f][0].data_ptr for f in ("a", "b")} == ptr   # the same resident slabs
        s = pa.array([None if i % 9 == 0 else str(words[i % 4]) for i in range(5000)], type=pa.large_string())
        _frame_matches(frame, {"s": s})
        np.testing.assert_array_equal(torch.as_tensor(frame.columns["a"][0], device="cuda").cpu().numpy(), a)
    engine.resident.clear()


def test_device_frame_on_a_sharded_engine(engine, tmp_path):
    from learningorchestra_b200.sharding import ShardedEngine, ShardedTable
    g = _titanic()
    _, path = _stores(tmp_path)
    with ShardedEngine.local() as sh:
        db = ColumnarDatabase()
        _post_files(db, sh, path)
        arrays = {f: db.column("t", f).arr for f in g["headers"]}
        with builder_frontend.device_frame(db, "t", sh, text=True) as frame:
            assert frame.fields == list(g["headers"])
            assert all(len(frame.columns[f]) == sh.nlocal for f in frame.fields)
            _frame_matches(frame, arrays)
            tables = _code_tables(frame)
        assert all(isinstance(t, ShardedTable) and not t.shards for t in tables)
        sh.resident.clear()
