"""GPU: the feature matrix (``lo_assemble_rows``, ``Engine`` / ``ShardedEngine.assemble_rows``,
``DeviceFrame.features``): Spark 2.4's ``VectorAssembler`` rows and label from f64 slabs and int32 code columns.

The oracle is numpy: ``np.stack`` of the sources as float64, invalid cells (NaN, code -1) found per row, rows dropped
(skip) or invalid codes set to NaN (keep), then ``.astype(np.float32)`` with every NaN made 0x7fc00000 (the K2 rule).
Results are compared bit for bit."""
import csv
import ctypes as C
import json
from pathlib import Path

import numpy as np
import pytest
import torch
from werkzeug.test import Client

from learningorchestra_b200 import _native as N
from learningorchestra_b200 import builder_frontend, server
from learningorchestra_b200.column_store import ColumnarDatabase
from learningorchestra_b200.engine import InvalidCellError
from learningorchestra_b200.sharding import ShardedEngine

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).resolve().parent / "golden"

F64_EDGES = np.array([0.0, -0.0, 5e-324, -5e-324, 2.2250738585072009e-308, 1e-40, -1e-45, 2.0 ** -150,
                      3 * 2.0 ** -150, 2.0 ** -149 * 1.5, 3.4028235677973366e38, -3.4028235677973366e38,
                      3.4028234663852886e38, 1e300, -1e300, np.inf, -np.inf, 1.0 + 2.0 ** -24, 1.0 + 3 * 2.0 ** -24,
                      -(1.0 + 2.0 ** -24), 16777217.0, 0.1, np.nan], np.float64)
NAN_PAYLOAD = np.array([0x7FF8000000000001, 0xFFF8000000000000, 0x7FFC000000000000], np.uint64).view(np.float64)
CODE_EDGES = np.array([-1, 0, 1, 2 ** 24 - 1, 2 ** 24, 2 ** 24 + 1, 2 ** 24 + 3, 2 ** 31 - 1, 123456789], np.int32)


def _columns(n, kinds, seed, invalid=True):
    """n-row source columns, one per kind ("f" f64, "i" int32 codes), edge values sprinkled in; with ``invalid``, a few
    NaN cells and -1 codes (about one row in three has one, whatever the number of columns)."""
    rng = np.random.default_rng(seed)
    p = 0.3 / max(len(kinds), 1) if invalid else 0.0
    cols = []
    for kind in kinds:
        if kind == "f":
            c = rng.normal(scale=1e3, size=n)
            pick = rng.random(n) < 0.2
            c[pick] = rng.choice(np.concatenate([F64_EDGES[:-1], NAN_PAYLOAD if invalid else []]), size=int(pick.sum()))
            if not invalid:
                c[np.isnan(c)] = 1.5
            c[rng.random(n) < p] = np.nan
        else:
            c = rng.integers(0, 60, size=n).astype(np.int32)
            pick = rng.random(n) < 0.2
            c[pick] = rng.choice(CODE_EDGES[1:], size=int(pick.sum()))
            c[rng.random(n) < p] = -1
        cols.append(c)
    return cols


def _bad(c):
    return c == -1 if c.dtype == np.int32 else np.isnan(c)


def _as_f64(c, mode):
    v = c.astype(np.float64)
    if c.dtype == np.int32 and mode == "keep":
        v[c == -1] = np.nan
    return v


def _cast(v, dtype):
    if dtype == "float64":
        return v
    with np.errstate(over="ignore"):
        out = v.astype(np.float32)
    out[np.isnan(out)] = np.uint32(0x7FC00000).view(np.float32)
    return out


def _oracle(cols, label, dtype, mode):
    """(x, y, kept rows) or ("error", row, position)."""
    n = cols[0].shape[0]
    bad = np.stack([_bad(c) for c in cols], 1) if n else np.zeros((0, len(cols)), bool)
    if label is not None:
        bad = np.concatenate([bad, _bad(label)[:, None]], 1)
    rowbad = bad.any(1)
    if mode == "error" and rowbad.any():
        r = int(np.argmax(rowbad))
        return "error", r, int(np.argmax(bad[r]))
    keep = ~rowbad if mode == "skip" else np.ones(n, bool)
    x = np.stack([_as_f64(c, mode) for c in cols], 1) if n else np.zeros((0, len(cols)))
    y = _as_f64(label, mode) if label is not None else None
    rows = np.flatnonzero(keep)
    return _cast(x[keep], dtype), None if y is None else _cast(y[keep], dtype), rows


def _tables(engine, cols, unaligned=False):
    """(sources, owned tables): the f64 columns in one f64 table (or each in a table wrapped one element past a
    16-byte boundary), each code column in an i32 table of its own, as a device frame holds them."""
    n = cols[0].shape[0]
    f = [j for j, c in enumerate(cols) if c.dtype == np.float64]
    owned, src = [], [None] * len(cols)
    if f and not unaligned:
        t = engine.table_from_numpy([cols[j] for j in f]) if n else engine.table("f64", 0, len(f))
        owned.append(t)
        for i, j in enumerate(f):
            src[j] = (t, i)
    for j, c in enumerate(cols):
        if src[j] is not None:
            continue
        if c.dtype == np.float64:
            buf = torch.empty(n + 1, dtype=torch.float64, device=f"cuda:{engine.device}")
            buf[1:] = torch.from_numpy(c)
            t = engine.wrap("f64", n, 1, buf.data_ptr() + 8, 8 * n + 8, keepalive=buf)
        else:
            t = engine.table("i32", n, 1)
            if n:
                t.upload(0, c)
        owned.append(t)
        src[j] = (t, 0)
    return src, owned


def _check(engine, cols, label=None, dtype="float32", mode="keep", unaligned=False):
    want = _oracle(cols, label, dtype, mode)
    src, owned = _tables(engine, cols + ([label] if label is not None else []), unaligned)
    lab = src.pop() if label is not None else None
    try:
        l0, t = engine.launch_count, {}
        if isinstance(want[0], str):
            with pytest.raises(InvalidCellError) as e:
                engine.assemble_rows(src, lab, dtype, mode)
            assert (e.value.row, e.value.position) == want[1:] and e.value.code == N.LO_ERR_INVALID
            assert engine.launch_count - l0 == 1
            return want
        res = engine.assemble_rows(src, lab, dtype, mode, timing=t)
        try:
            n = cols[0].shape[0]
            assert engine.launch_count - l0 == (0 if n == 0 else 3 if mode == "skip" else 1)
            x, y, rows = want
            got = torch.as_tensor(res.matrix(), device=f"cuda:{engine.device}")
            assert tuple(got.shape) == x.shape
            assert x.size == 0 or got.data_ptr() == res.x.base_ptr                          # zero-copy
            bits = np.uint32 if dtype == "float32" else np.uint64
            np.testing.assert_array_equal(got.cpu().numpy().view(bits), x.view(bits))
            if label is not None:
                gy = torch.as_tensor(res.vector(), device=f"cuda:{engine.device}").cpu().numpy()
                np.testing.assert_array_equal(gy.view(bits), y.view(bits))
            else:
                assert res.vector() is None
            np.testing.assert_array_equal(res.rows, rows)
            return want
        finally:
            res.free()
    finally:
        for o in owned:
            o.free()


@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("mode", ["keep", "skip", "error"])
def test_every_mode_and_dtype_against_the_oracle(engine, dtype, mode):
    cols = _columns(5000, "fifffiif", 1)
    label = _columns(5000, "f", 2)[0]
    _check(engine, cols, label, dtype, mode)
    _check(engine, cols, None, dtype, mode)
    if mode == "error":                               # without an invalid cell the matrix is made
        clean = _columns(5000, "fifffiif", 3, invalid=False)
        assert not isinstance(_check(engine, clean, _columns(5000, "i", 4, invalid=False)[0], dtype, mode)[0], str)


@pytest.mark.parametrize("k", [1, 3, 31, 32, 33, 100])
@pytest.mark.parametrize("n", [0, 1, 127, 128, 129, 255, 257, 4097])
def test_shapes_and_tile_edges(engine, k, n):
    kinds = ("fi" * k)[:k] if k > 1 else "f"
    cols = _columns(n, kinds, 10 * k + n)
    label = _columns(n, "i", n)[0]
    for mode in ("keep", "skip"):
        _check(engine, cols, label if k % 2 else None, "float32", mode)
    _check(engine, cols, None, "float64", "skip")


@pytest.mark.parametrize("k", [1, 3, 33])
def test_unaligned_sources_take_scalar_loads(engine, k):
    cols = _columns(1000, ("ffi" * k)[:k], 7 + k)
    for mode in ("keep", "skip", "error"):
        _check(engine, cols, None, "float32", mode, unaligned=True)
        _check(engine, cols, cols[-1].copy(), "float64", mode, unaligned=True)


def test_edge_values_bit_for_bit(engine):
    f = np.concatenate([F64_EDGES, NAN_PAYLOAD])
    codes = np.resize(CODE_EDGES, f.size)
    for dtype in ("float32", "float64"):
        want = _check(engine, [f, codes, -f], None, dtype, "keep")
        assert np.isinf(want[0][10, 0]) == (dtype == "float32")            # rounds to +inf in f32 only


def test_error_names_the_lowest_row_and_its_first_invalid_source(engine):
    n = 1000
    a, b = np.arange(n, dtype=np.float64), np.arange(n, dtype=np.int32)
    a[700], b[600], b[900] = np.nan, -1, -1
    label = np.zeros(n)
    label[500] = np.nan
    assert _check(engine, [a, b], label, "float32", "error") == ("error", 500, 2)          # the label
    assert _check(engine, [a, b], None, "float32", "error") == ("error", 600, 1)
    a[600] = np.nan
    assert _check(engine, [a, b], None, "float64", "error") == ("error", 600, 0)


def _refusals(engine, peer=None):
    """(description, argument overrides) of lo_assemble_rows calls that must be refused before any launch."""
    n = 300
    f64 = engine.table_from_numpy([np.zeros(n), np.ones(n)])
    i32 = engine.table("i32", n, 1)
    f32 = engine.table("f32", n, 1)
    u8 = engine.table("u8", n, 1)
    short = engine.table("f64", n - 1, 1)
    x = engine.table("f32", 2 * n, 1)
    x64 = engine.table("f64", 2 * n, 1)
    small = engine.table("f32", 2 * n - 1, 1)
    y, y_small, y64 = engine.table("f32", n, 1), engine.table("f32", n - 1, 1), engine.table("f64", n, 1)
    x8 = engine.table("u8", 2 * n, 1)
    P = C.c_void_p

    def srcs(*ts):
        return (P * len(ts))(*[t._h for t in ts])

    def cols(*cs):
        return (C.c_int32 * len(cs))(*cs)

    base = dict(src=srcs(f64, i32), src_col=cols(0, 0), k=2, label=None, label_col=0, mode=N.LO_INVALID_KEEP, x=x._h,
                ld=2, y=None, kept=None, info=True)
    cases = [("NULL src", dict(src=None)), ("NULL src_col", dict(src_col=None)), ("k = 0", dict(k=0)),
             ("k < 0", dict(k=-1)), ("ld < k", dict(ld=1)), ("f32 source", dict(src=srcs(f64, f32))),
             ("u8 source", dict(src=srcs(u8, i32))), ("column out of range", dict(src_col=cols(2, 0))),
             ("negative column", dict(src_col=cols(0, -1))), ("mismatched rows", dict(src=srcs(f64, short))),
             ("NULL source", dict(src=(P * 2)(f64._h, None))), ("unknown mode", dict(mode=3)),
             ("negative mode", dict(mode=-1)), ("NULL x", dict(x=None)), ("x too small", dict(x=small._h)),
             ("x of i32", dict(x=i32._h)), ("x of u8", dict(x=x8._h)),
             ("ld too large for x", dict(ld=3)), ("label without y", dict(label=f64._h, label_col=1)),
             ("y without label", dict(y=y._h)), ("y too small", dict(label=f64._h, y=y_small._h)),
             ("y of another dtype", dict(label=f64._h, y=y64._h)), ("y dtype with f64 x", dict(x=x64._h, label=f64._h, y=y._h)),
             ("f32 label", dict(label=f32._h, y=y._h)), ("label column out of range", dict(label=f64._h, label_col=2, y=y._h)),
             ("label of other rows", dict(label=short._h, y=y._h)), ("NULL info", dict(info=None))]
    held = [f64, i32, f32, u8, short, x, x64, small, y, y_small, y64, x8]
    if peer is not None:
        other, px = peer.table_from_numpy([np.zeros(n)]), peer.table("f32", 2 * n, 1)
        cases += [("source on another device", dict(src=srcs(f64, other), src_col=cols(0, 0))),
                  ("x on another device", dict(x=px._h))]
        held += [other, px]
    return base, cases, held


def test_every_refusal_launches_nothing(engine):
    peer = None
    count = C.c_int()
    N.check(N.load().lo_device_count(C.byref(count)))
    if count.value > 1:
        from learningorchestra_b200.engine import Engine
        peer = Engine(1)
    try:
        base, cases, _keep = _refusals(engine, peer)
        lib = engine._lib
        for name, over in cases:
            a = {**base, **over}
            info = N.AssembleInfo()
            l0 = engine.launch_count
            rc = lib.lo_assemble_rows(engine._ctx, a["src"], a["src_col"], a["k"], a["label"], a["label_col"], a["mode"],
                                      a["x"], a["ld"], a["y"], a["kept"], C.byref(info) if a["info"] else None, None)
            assert rc == N.LO_ERR_INVALID, name
            assert engine.launch_count == l0, name
        a = base
        info = N.AssembleInfo()
        assert lib.lo_assemble_rows(engine._ctx, a["src"], a["src_col"], 2, None, 0, a["mode"], a["x"], 2, None, None,
                                    C.byref(info), None) == N.LO_OK and info.nkept == 300
    finally:
        if peer is not None:
            peer.close()


def test_python_refusals_before_any_launch(engine):
    t = engine.table_from_numpy([np.zeros(10)])
    l0 = engine.launch_count
    for kw in (dict(dtype="float16"), dict(handle_invalid="drop")):
        with pytest.raises(ValueError):
            engine.assemble_rows([(t, 0)], **kw)
    with pytest.raises(ValueError):
        engine.assemble_rows([])
    assert engine.launch_count == l0
    t.free()


def test_sharded_result_concatenates_to_the_single_device_one(engine):
    n = 70_001
    cols = _columns(n, "ffif", 21)
    label = _columns(n, "f", 22)[0]
    with ShardedEngine.local() as sh:
        st = sh.table_from_numpy([cols[0], cols[1], cols[3], label])
        codes = sh.table("i32", n, 1)
        codes.upload(0, cols[2])
        src = [(st, 0), (st, 1), (codes, 0), (st, 2)]
        for dtype, mode in (("float32", "skip"), ("float64", "keep"), ("float32", "error")):
            want = _oracle(cols, label, dtype, mode)
            if isinstance(want[0], str):
                with pytest.raises(InvalidCellError) as e:
                    sh.assemble_rows(src, (st, 3), dtype, mode)
                assert (e.value.row, e.value.position) == want[1:]
                continue
            parts = sh.assemble_rows(src, (st, 3), dtype, mode)
            try:
                assert len(parts) == sh.nlocal
                x = np.concatenate([torch.as_tensor(p.matrix(), device=f"cuda:{p.x.engine.device}").cpu().numpy()
                                    for p in parts])
                y = np.concatenate([torch.as_tensor(p.vector(), device=f"cuda:{p.x.engine.device}").cpu().numpy()
                                    for p in parts])
                bits = np.uint32 if dtype == "float32" else np.uint64
                np.testing.assert_array_equal(x.view(bits), want[0].view(bits))
                np.testing.assert_array_equal(y.view(bits), want[1].view(bits))
                np.testing.assert_array_equal(np.concatenate([p.rows for p in parts]), want[2])
            finally:
                for p in parts:
                    p.free()
        st.free()
        codes.free()


NUMBER_FIELDS = ["PassengerId", "Survived", "Pclass", "Age", "SibSp", "Parch", "Fare"]


@pytest.mark.parametrize("sharded", [False, True])
def test_titanic_features_end_to_end(engine, tmp_path, sharded):
    g = json.loads((GOLD / "titanic_shaped_input.json").read_text())
    path = tmp_path / "t.csv"
    with open(path, "w", newline="") as f:
        csv.writer(f).writerows([g["headers"]] + g["rows"])
    eng = ShardedEngine.local() if sharded else engine
    try:
        eng.resident.clear()
        db = ColumnarDatabase()
        db.ingest_csv("t", str(path), engine=eng)
        c = Client(server.create_app(db, eng, synchronous=True))
        r = c.patch("/fieldTypes", json={"inputDatasetName": "t", "types": {f: "number" for f in NUMBER_FIELDS}})
        assert r.status_code == 200, r.get_data(as_text=True)
        host = builder_frontend.file_processor(db, "t")
        with builder_frontend.device_frame(db, "t", eng, text=True) as frame:
            fields = [f for f in frame.fields if f != "Survived"]
            with frame.features(label="Survived", handle_invalid="skip") as feats:
                assert feats.fields == fields and feats.label == "Survived"
                cols = {}
                for f in frame.fields:
                    if frame.kinds[f] == "text":
                        index = {s: i for i, s in enumerate(frame.dictionaries[f].to_pylist())}
                        cols[f] = np.array([-1 if v is None else index[v] for v in host.column(f).to_pylist()], np.int32)
                    else:
                        cols[f] = np.array([np.nan if v is None else v for v in host.column(f).to_pylist()], np.float64)
                x, y, rows = _oracle([cols[f] for f in fields], cols["Survived"], "float32", "skip")
                got = np.concatenate([torch.as_tensor(v, device=f"cuda:{d}").cpu().numpy()
                                      for v, d in zip(feats.x, feats.devices)])
                np.testing.assert_array_equal(got.view(np.uint32), x.view(np.uint32))
                gy = np.concatenate([torch.as_tensor(v, device=f"cuda:{d}").cpu().numpy()
                                     for v, d in zip(feats.y, feats.devices)])
                np.testing.assert_array_equal(gy.view(np.uint32), y.view(np.uint32))
                ids = np.array([d["_id"] for d in sorted(db.find("t", {}), key=lambda d: d["_id"]) if d["_id"] != 0])
                np.testing.assert_array_equal(feats.row_ids, ids[rows])
                kept = {int(i) for i in feats.row_ids}
                empty = {i + 1 for i, row in enumerate(g["rows"])
                         if any(row[g["headers"].index(f)] == "" for f in NUMBER_FIELDS)}
                assert kept == set(range(1, len(g["rows"]) + 1)) - empty and len(kept) < len(g["rows"])
                assert any(row[g["headers"].index("Embarked")] == "" for row in g["rows"] if int(row[0]) in kept) or \
                    not any(row[g["headers"].index("Embarked")] == "" for row in g["rows"])
                tables = [p.x for p in feats._parts] + [p.y for p in feats._parts]
            assert all(t._h is None for t in tables)
            with pytest.raises(N.LoexecError) as e:
                frame.features(label="Survived")
            assert "'Age'" in str(e.value) and "_id" in str(e.value) and e.value.code == N.LO_ERR_INVALID
            with pytest.raises(KeyError):
                frame.features(["Age", "nope"])
        eng.resident.clear()
    finally:
        if sharded:
            eng.close()
