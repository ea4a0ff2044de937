"""GPU: the "string" cast's number -> text formatter (lo_format_number_host -> k_format_number_len / _write) against
CPython's repr(float) / str(int), its round trip through the GPU parser, the C ABI's edges, and the DataType / REST
paths on both stores against the reference's own converted documents."""
import ctypes as C
import json
import math
from pathlib import Path

import numpy as np
import pytest
from werkzeug.test import Client

from learningorchestra_b200 import _native as N
from learningorchestra_b200 import server, utils
from learningorchestra_b200._native import LoexecError
from learningorchestra_b200.column_store import ColumnarDatabase, NumberColumn, TextColumn
from learningorchestra_b200.data_type_update import DataType
from oracle import rsem
from test_format_cpu import EDGES, SPECIAL_BITS, bits_to_float, expected, with_neighbours

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).resolve().parent / "golden"
FLOAT, INTEGER, EMPTY = N.LO_NUM_FLOAT, N.LO_NUM_INTEGER, N.LO_NUM_EMPTY


def _load(name):
    return json.loads((GOLD / name).read_text())


def _value_sets():
    """(values, status): the specials, edges, powers of ten and two with neighbours as FLOAT, integral doubles of every
    exponent as INTEGER, and a few EMPTY cells."""
    floats = [bits_to_float(b) for b in SPECIAL_BITS] + with_neighbours(EDGES)
    floats += with_neighbours([float(f"1e{k}") for k in range(-323, 309)] + [math.ldexp(1.0, k) for k in range(-1074, 1024)])
    floats += [-v for v in floats]
    rng = np.random.default_rng(11)
    ints = [0.0, -0.0, 1e22, 1.7976931348623157e308, -1.7976931348623157e308] + with_neighbours([2.0 ** 53, 2.0 ** 63, 2.0 ** 64])
    for e in range(0, 1024):
        m = int(rng.integers(2 ** 52, 2 ** 53))
        ints += [math.ldexp(1.0, e), float(math.floor(math.ldexp(float(m), e - 52))) * (1 if e % 2 else -1)]
    values = np.array(floats + ints + [0.0] * 5, dtype=np.float64)
    status = np.array([FLOAT] * len(floats) + [INTEGER] * len(ints) + [EMPTY] * 5, dtype=np.uint8)
    return values, status


def _check(values, status, chars, offsets):
    exp = [expected(v, s) for v, s in zip(values.tolist(), status.tolist())]
    assert offsets[0] == 0 and offsets.shape == (len(exp) + 1,)
    assert np.array_equal(np.diff(offsets), [len(e) for e in exp])
    raw = chars.tobytes()
    if raw != "".join(exp).encode():
        for i, e in enumerate(exp):
            assert raw[offsets[i]:offsets[i + 1]].decode() == e, (i, float(values[i]).hex(), int(status[i]), e)


def test_formatter_equals_python_on_edge_sets_and_5m_random_cells(engine):
    values, status = _value_sets()
    chars, offsets = engine.format_number_host(values, status)
    _check(values, status, chars, offsets)
    # one call of > 5 M cells: many blocks of each kernel, a multi-tile scan
    rng = np.random.default_rng(20261015)
    n = 5_000_003
    rand = rng.integers(0, 2 ** 64, size=n, dtype=np.uint64).view(np.float64)
    big_values = np.concatenate([rand, values])
    big_status = np.concatenate([np.full(n, FLOAT, dtype=np.uint8), status])
    timing = {}
    chars, offsets = engine.format_number_host(big_values, big_status, timing)
    _check(big_values, big_status, chars, offsets)
    assert timing["kernel_ms"] > 0 and timing["launches"] == 3


def _mixed(n, seed):
    """n values as the "number" cast leaves them: random bit patterns, %.6f-shaped decimals, integers (some beyond
    2^64), nulls; status INTEGER exactly where the value is finite and integral (is_integer())."""
    rng = np.random.default_rng(seed)
    kind = rng.integers(0, 5, n)
    v = rng.integers(0, 2 ** 64, size=n, dtype=np.uint64).view(np.float64).copy()
    v[kind == 1] = np.round(rng.uniform(-1e6, 1e6, (kind == 1).sum()), 6)
    v[kind == 2] = rng.integers(-10 ** 15, 10 ** 15, (kind == 2).sum()).astype(np.float64)
    v[kind == 3] = np.floor(rng.uniform(-1.0, 1.0, (kind == 3).sum()) * 10.0 ** rng.integers(19, 308, (kind == 3).sum()))
    with np.errstate(invalid="ignore"):
        status = np.where(np.isfinite(v) & (v == np.floor(v)), INTEGER, FLOAT).astype(np.uint8)
    status[kind == 4] = EMPTY
    v[v == 0] = 0.0                       # int(-0.0) is 0: a zero reads back as +0.0
    return v, status


def test_parser_reads_the_formatter_back_bit_for_bit(engine):
    values, status = _mixed(1_000_000, 3)
    chars, offsets = engine.format_number_host(values, status)
    back, back_status = engine.parse_number_packed(chars, offsets)
    assert np.array_equal(back_status, status)
    keep = status != EMPTY
    nan = np.isnan(values) & keep
    assert np.array_equal(np.isnan(back) & keep, nan)
    ok = keep & ~nan
    assert np.array_equal(back[ok].view(np.uint64), values[ok].view(np.uint64))


def _call(engine, values, status, chars_capacity, with_chars=True):
    values = np.ascontiguousarray(values, dtype=np.float64)
    status = np.ascontiguousarray(status, dtype=np.uint8)
    n = values.shape[0]
    offsets = np.full(n + 1, -7, dtype=np.int64)
    chars = np.zeros(max(chars_capacity, 1), dtype=np.uint8)
    rc = engine._lib.lo_format_number_host(engine._ctx, values.ctypes.data_as(C.c_void_p), status.ctypes.data_as(C.c_void_p), n,
                                           offsets.ctypes.data_as(C.c_void_p),
                                           chars.ctypes.data_as(C.c_void_p) if with_chars else None, chars_capacity, None)
    return rc, offsets, chars


def test_abi_edges(engine):
    rc, offsets, _ = _call(engine, [], [], 0, with_chars=False)
    assert rc == N.LO_OK and offsets.tolist() == [0]
    values, status = [1.5, 3.0, 0.0, 1e22], [FLOAT, INTEGER, EMPTY, FLOAT]
    rc, offsets, _ = _call(engine, values, status, 0, with_chars=False)                 # sizes only
    assert rc == N.LO_OK and offsets.tolist() == [0, 3, 4, 4, 9]
    rc, offsets, chars = _call(engine, values, status, 8)                                # one byte short
    assert rc == N.LO_ERR_INVALID and offsets.tolist() == [0, 3, 4, 4, 9]
    assert "9 bytes" in N.load().lo_last_error().decode()
    assert not chars.any()
    rc, offsets, chars = _call(engine, values, status, 9)
    assert rc == N.LO_OK and chars[:9].tobytes() == b"1.531e+22"
    for bad_status, bad_value, what in [(3, 1.0, "status 3"), (4, 1.0, "status 4"), (INTEGER, 0.5, "not finite and integral"),
                                        (INTEGER, math.inf, "not finite and integral")]:
        v = [1.0] * 6 + [bad_value] + [2.0] * 3
        s = [FLOAT] * 6 + [bad_status] + [INTEGER] * 3
        rc, _, _ = _call(engine, v, s, 1000)
        msg = N.load().lo_last_error().decode()
        assert rc == N.LO_ERR_INVALID and "row 6" in msg and what in msg, msg
    with pytest.raises(LoexecError, match="row 1"):
        engine.format_number_host(np.array([1.0, 2.5]), np.array([INTEGER, INTEGER], dtype=np.uint8))


def _titanic_documents():
    db = utils.Database()
    g = _load("titanic_shaped_input.json")
    headers, docs = rsem.csv_rows_to_documents(g["headers"], g["rows"])
    db.insert_one_in_file("titanic", rsem.dataset_metadata("titanic", headers))
    db.insert_many_in_file("titanic", docs)
    return db


def _titanic_columns(tmp_path):
    import csv
    g = _load("titanic_shaped_input.json")
    path = tmp_path / "titanic.csv"
    with path.open("w", newline="") as f:
        csv.writer(f, lineterminator="\n").writerows([g["headers"]] + g["rows"])
    db = ColumnarDatabase()
    db.ingest_csv("titanic", str(path))
    return db


def _cast(db, name, types, engine):
    job = DataType(db, utils.DataTypeMetadata(db), engine)
    job.convert_existent_file(name, types)
    job.wait(120)
    assert db.find_one(name, {"_id": 0})["finished"] is True


def test_number_then_string_equals_the_reference_on_both_stores(engine, tmp_path):
    gold_s = _load("reference_datatype_string.json")
    vec = _load("reference_cast_vectors.json")
    for db in (_titanic_documents(), _titanic_columns(tmp_path)):
        _cast(db, "titanic", {f: "number" for f in gold_s["fields"]}, engine)
        before = engine.launch_count
        _cast(db, "titanic", {f: "string" for f in gold_s["fields"]}, engine)
        assert engine.launch_count >= before + 3 * len(gold_s["fields"])      # the numbers went to the device
        got = sorted([d["_id"]] + [d[f] for f in gold_s["fields"]] for d in db.find("titanic", {}) if d["_id"] != 0)
        assert got == gold_s["rows"]
    # the per-value vectors produced by the reference's own converter: "number" then back to "string"
    docs = utils.Database()
    docs.insert_one_in_file("vec", rsem.dataset_metadata("vec", ["v"]))
    docs.insert_many_in_file("vec", [{"_id": i + 1, "v": v} for i, v in enumerate(vec["in"])])
    cols = ColumnarDatabase()
    import pyarrow as pa
    cols.ingest_columns("vec", {"v": TextColumn(pa.array(vec["in"], type=pa.large_string()))})
    for db in (docs, cols):
        _cast(db, "vec", {"v": "number"}, engine)
        before = engine.launch_count
        _cast(db, "vec", {"v": "string"}, engine)
        assert engine.launch_count > before
        out = [d["v"] for d in sorted(db.find("vec", {}), key=lambda d: d["_id"]) if d["_id"] != 0]
        assert out == vec["back_to_string"]
    assert isinstance(cols.column("vec", "v"), TextColumn)


def test_rest_field_types_string_on_a_columnar_dataset(engine, tmp_path):
    db = _titanic_columns(tmp_path)
    c = Client(server.create_app(db, engine, synchronous=True))
    gold_s = _load("reference_datatype_string.json")
    types = {f: "number" for f in gold_s["fields"]}
    assert c.patch("/fieldTypes", json={"inputDatasetName": "titanic", "types": types}).status_code == 200
    assert all(isinstance(db.column("titanic", f), NumberColumn) for f in gold_s["fields"])
    r = c.patch("/fieldTypes", json={"inputDatasetName": "titanic", "types": {f: "string" for f in gold_s["fields"]}})
    assert r.status_code == 200
    assert r.get_json() == {"result": "/api/learningOrchestra/v1/dataset/titanic?query={}&limit=20&skip=0"}
    assert db.find_one("titanic", {"_id": 0})["finished"] is True
    assert all(isinstance(db.column("titanic", f), TextColumn) for f in gold_s["fields"])
    got = sorted([d["_id"]] + [d[f] for f in gold_s["fields"]] for d in db.find("titanic", {}) if d["_id"] != 0)
    assert got == gold_s["rows"]
