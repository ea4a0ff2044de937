"""GPU: ``/fieldTypes`` on a column store with an engine that keeps datasets in HBM.  ``"number"`` parses the field's
resident text column on every device (``lo_parse_text_to_table``), ``"string"`` formats its resident slab into a new
resident text column (``lo_format_table_to_text`` / ``lo_text_download``), and the cache carries what a conversion left
unchanged to the next version.  Every result column must equal, bit for bit, what the packed host route
(``parse_number_packed`` / ``format_number_host``, called on the same cells) writes, on one device and on a
``ShardedEngine`` over every visible GPU."""
import csv
import ctypes as C
import itertools
import json
import math
from pathlib import Path

import numpy as np
import pyarrow as pa
import pytest
from werkzeug.test import Client

from learningorchestra_b200 import _native as N
from learningorchestra_b200 import columnar, server, utils
from learningorchestra_b200.column_store import ColumnarDatabase
from learningorchestra_b200.data_type_update import DataType
from learningorchestra_b200.engine import DeviceTable
from learningorchestra_b200.sharding import ShardedEngine, ShardedTable
from edge_values import NAN_BITS, SPECIALS
from oracle import rsem

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).resolve().parent / "golden"


@pytest.fixture(scope="module")
def sharded(built):
    eng = ShardedEngine.local()          # every visible GPU; a group of one on a one-GPU box
    yield eng
    eng.close()


@pytest.fixture(params=["engine", "sharded"])
def any_engine(request, engine, sharded):
    eng = engine if request.param == "engine" else sharded
    eng.resident.clear()
    yield eng
    eng.resident.clear()


class _Packed:
    """The route without resident datasets: the same engine's host-buffer parse and format."""

    def __init__(self, eng):
        self.parse_number_packed, self.format_number_host = eng.parse_number_packed, eng.format_number_host


_NAMES = itertools.count()


def _convert(eng, cells, field_type, name="c"):
    """The column store of ``cells`` (an Arrow array, or a NumberColumn) after ``field_type`` with ``eng``: (column,
    error or None).  Each call has a dataset name of its own: the engine's resident datasets are keyed by name."""
    db, filename = ColumnarDatabase(), f"d{next(_NAMES)}"
    db.ingest_columns(filename, {name: cells})
    job = DataType(db, utils.DataTypeMetadata(db), eng)
    try:
        job.field_converter(filename, name, field_type)
        err = None
    except (ValueError, RuntimeError) as exc:
        err = exc
    return db.column(filename, name), err


def _same_column(a, b):
    assert a.kind == b.kind
    if a.kind == "number":
        assert np.array_equal(a.values.view(np.uint64), b.values.view(np.uint64))
        assert np.array_equal(a.valid, b.valid) and np.array_equal(a.is_int, b.is_int)
    elif a.kind == "text":
        (ca, oa, _), (cb, ob, _) = columnar.text_buffers(a.arr), columnar.text_buffers(b.arr)
        assert np.array_equal(oa - oa[0], ob - ob[0]) and a.arr.null_count == b.arr.null_count == 0
        assert ca[oa[0]:oa[-1]].tobytes() == cb[ob[0]:ob[-1]].tobytes()
    else:
        assert repr(a.values) == repr(b.values)


def _both_ways(eng, cells):
    """``"number"`` on ``cells`` through the resident route and the packed route, then ``"string"`` on the result: the
    columns and failures agree at each step.  Returns the number column."""
    got, err = _convert(eng, cells, "number")
    want, want_err = _convert(_Packed(eng), cells, "number")
    assert repr(err) == repr(want_err)
    _same_column(got, want)
    if got.kind == "number":
        s_got, _ = _convert(eng, got, "string")
        s_want, _ = _convert(_Packed(eng), got, "string")
        _same_column(s_got, s_want)
    return got


def _text(cells):
    return pa.array(cells, type=pa.large_string())


def test_reference_goldens(any_engine):
    g = json.loads((GOLD / "titanic_shaped_input.json").read_text())
    gold = json.loads((GOLD / "reference_datatype_number.json").read_text())
    for f in gold["fields"]:
        j = g["headers"].index(f)
        col = _both_ways(any_engine, _text([r[j] for r in g["rows"]]))
        assert [None if not ok else (int(v) if ii else v) for v, ok, ii in
                zip(col.values.tolist(), col.valid, col.is_int)] == [r[gold["fields"].index(f) + 1] for r in gold["rows"]]
    sg = json.loads((GOLD / "reference_datatype_string.json").read_text())
    for f in sg["fields"]:
        got, _ = _convert(any_engine, _convert(any_engine, _text([r[g["headers"].index(f)] for r in g["rows"]]),
                                               "number")[0], "string")
        assert got.arr.to_pylist() == [r[sg["fields"].index(f) + 1] for r in sg["rows"]], f


def test_edge_values_and_a_million_random_doubles(any_engine):
    edge = [repr(float(v)) for v in SPECIALS] + [repr(float(v)) for v in np.array(NAN_BITS, np.uint64).view(np.float64)]
    edge += ["1e22", "-0", "1_000", " 7 ", "9007199254740993", "1e-400", "inf", "-Infinity", "nan", "", None]
    _both_ways(any_engine, _text(edge))
    rng = np.random.default_rng(7)
    v = rng.standard_normal(1_000_000) * 10.0 ** rng.integers(-30, 30, 1_000_000)
    v[::7] = np.round(v[::7])
    cells = [repr(float(x)) for x in v]
    for i in range(0, len(cells), 97):
        cells[i] = None if i % 2 else ""
    _both_ways(any_engine, _text(cells))


def test_a_sliced_array_and_a_non_ascii_column(any_engine):
    full = _text([None if i % 11 == 0 else str(i * 0.25) for i in range(5000)])
    _both_ways(any_engine, full.slice(37, 4000))
    col = _both_ways(any_engine, _text(["１２", "٣.٥", "7", None, ""] * 50))      # the packed route: Unicode mapping
    assert col.values[0] == 12.0 and col.values[1] == 3.5


def test_bad_cells_after_a_shard_boundary_and_over_one_mib(any_engine):
    n = 100_003
    cells = [str(i) for i in range(n)]
    cut = any_engine.bounds(n)[-1][0] if hasattr(any_engine, "bounds") else n // 2
    bad = list(cells)
    bad[cut + 1], bad[n - 2] = "12abc", "x"
    col = _both_ways(any_engine, _text(bad))
    assert col.kind == "object" and col.values[cut] == cut and col.values[cut + 1] == "12abc"
    big = list(cells)
    big[cut + 3] = "1" * ((1 << 20) + 1)
    _both_ways(any_engine, _text(big))


class _Uploads:
    """Every cell the engine is asked to move to the device: text uploads, slab uploads and host parses."""

    def __init__(self, eng, monkeypatch):
        self.calls = []
        for name in ("text", "parse_number_into", "parse_number_packed", "format_number_host"):
            real = getattr(eng, name)
            monkeypatch.setattr(eng, name, lambda *a, _r=real, _n=name, **k: (self.calls.append(_n), _r(*a, **k))[1])
        for cls in (DeviceTable, ShardedTable):
            real = cls.upload
            monkeypatch.setattr(cls, "upload", lambda self_, *a, _r=real, **k: (self.calls.append("upload"), _r(self_, *a, **k))[1])


def _docs(db, name):
    return sorted((d for d in db.find(name, {}) if d["_id"] != 0), key=lambda d: d["_id"])


def test_titanic_flow_moves_no_cell_after_the_conversion(any_engine, tmp_path, monkeypatch):
    """upload -> /histograms -> /fieldTypes -> /histograms: the documents equal the oracle's, the conversion and the
    requests after it move no cell to the device, and the request after the write is one miss."""
    g = json.loads((GOLD / "titanic_shaped_input.json").read_text())
    path = tmp_path / "t.csv"
    with open(path, "w", newline="") as f:
        csv.writer(f).writerows([g["headers"]] + g["rows"])
    fields = ["Age", "Fare", "Pclass", "Survived"]
    db = ColumnarDatabase()
    c = Client(server.create_app(db, any_engine, synchronous=True))
    assert c.post("/files", json={"datasetName": "t", "datasetURI": f"file://{path}"}).status_code == 201
    assert c.post("/histograms", json={"inputDatasetName": "t", "outputDatasetName": "h1", "names": fields}).status_code == 201
    spy = _Uploads(any_engine, monkeypatch)
    assert c.patch("/fieldTypes", json={"inputDatasetName": "t", "types": {"Age": "number", "Fare": "number"}}).status_code == 200
    assert spy.calls == []
    m0 = any_engine.resident.misses
    assert c.post("/histograms", json={"inputDatasetName": "t", "outputDatasetName": "h2", "names": fields}).status_code == 201
    assert c.post("/histograms", json={"inputDatasetName": "t", "outputDatasetName": "h3", "names": ["Age", "Fare"],
                                       "bins": 8}).status_code == 201
    assert spy.calls == [] and any_engine.resident.misses == m0 + 1
    # the oracle: the same flow on documents, without an engine's resident datasets
    from oracle_engine import OracleEngine
    odb = ColumnarDatabase()
    oc = Client(server.create_app(odb, OracleEngine(), synchronous=True))
    assert oc.post("/files", json={"datasetName": "t", "datasetURI": f"file://{path}"}).status_code == 201
    assert oc.patch("/fieldTypes", json={"inputDatasetName": "t", "types": {"Age": "number", "Fare": "number"}}).status_code == 200
    assert oc.post("/histograms", json={"inputDatasetName": "t", "outputDatasetName": "h2", "names": fields}).status_code == 201
    for mine, theirs, f in zip(_docs(db, "h2"), _docs(odb, "h2"), fields):
        assert rsem.normalise_group_result(mine[f]) == rsem.normalise_group_result(theirs[f]), f
    # "string" back: the text column is handed to the cache, and counting it moves nothing
    assert c.patch("/fieldTypes", json={"inputDatasetName": "t", "types": {"Fare": "string"}}).status_code == 200
    assert c.post("/histograms", json={"inputDatasetName": "t", "outputDatasetName": "h4", "names": ["Fare"]}).status_code == 201
    assert spy.calls == []
    assert oc.patch("/fieldTypes", json={"inputDatasetName": "t", "types": {"Fare": "string"}}).status_code == 200
    assert oc.post("/histograms", json={"inputDatasetName": "t", "outputDatasetName": "h4", "names": ["Fare"]}).status_code == 201
    assert rsem.normalise_group_result(_docs(db, "h4")[0]["Fare"]) == rsem.normalise_group_result(_docs(odb, "h4")[0]["Fare"])
    _same_column(db.column("t", "Fare"), odb.column("t", "Fare"))


def test_c_abi_refuses_mismatches_before_launching(engine):
    lib = N.load()
    text = engine.text(_text(["1", "2", "3"]))
    table = engine.table("f64", 4, 1)
    f32 = engine.table("f32", 3, 1)
    s, t = N.ParseSummary(), N.HostTiming()
    launches = engine.launch_count
    for tab, col in ((table, 0), (f32, 0), (engine.table("f64", 3, 1), 1)):
        rc = lib.lo_parse_text_to_table(engine._ctx, text._h, tab._h, col, C.byref(s), C.byref(t))
        assert rc == N.LO_ERR_INVALID
    h = C.c_void_p()
    assert lib.lo_format_table_to_text(engine._ctx, f32._h, 0, None, None, C.byref(h), None) == N.LO_ERR_INVALID
    assert engine.launch_count == launches
    bad = engine.table_from_numpy([np.array([1.0, 2.5, math.inf])])
    with pytest.raises(N.LoexecError, match="row 1"):
        engine.format_column(bad, 0, np.ones(3, bool), np.ones(3, bool))
    for o in (text, table, f32, bad):
        o.free()
