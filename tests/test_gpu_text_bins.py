"""GPU: binned histograms and ``castTo`` projections straight from TEXT fields (``lo_parse_number_to_table``).

The definition: a text cell is ``float(cell)`` followed by the B-semantics cast and binning; None and ``""`` are null.
Every case is checked against two oracles — ``bn.hist_f32(bn.cast_f64_f32(float(cell)))`` and the same request made
after ``/fieldTypes {"f": "number"}`` on a copy of the dataset — on both store kinds (documents and columns), and the
dataset itself must stay text."""
import csv
import json
import os
import socket
from pathlib import Path

import numpy as np
import pyarrow as pa
import pytest
from werkzeug.test import Client

from learningorchestra_b200 import server, utils
from learningorchestra_b200.column_store import ColumnarDatabase, TextColumn
from oracle import bsem_numpy as bn
from oracle import rsem

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).resolve().parent / "golden"
FIELDS4 = ["Survived", "Pclass", "Age", "Fare"]
NAN = 0x7FF8000000000000


def _num(cell):
    return np.nan if cell is None or cell == "" else float(cell)


def _stores(name, headers, rows, tmp_path):
    """[("documents", db), ("columnar", db)] holding the same CSV rows, every cell text; the columnar one through
    POST /files."""
    docs = utils.Database()
    hdr, documents = rsem.csv_rows_to_documents(headers, rows)
    docs.insert_one_in_file(name, rsem.dataset_metadata(name, hdr))
    docs.insert_many_in_file(name, documents)
    path = tmp_path / f"{name}.csv"
    with open(path, "w", newline="") as f:
        csv.writer(f).writerows([headers] + rows)
    cdb = ColumnarDatabase()
    return [("documents", docs, None), ("columnar", cdb, str(path))]


def _client(db, engine, name, path):
    c = Client(server.create_app(db, engine, synchronous=True))
    if path is not None:
        assert c.post("/files", json={"datasetName": name, "datasetURI": f"file://{path}"}).status_code == 201
    return c


def _data(db, name):
    return sorted((d for d in db.find(name, {}) if d["_id"] != 0), key=lambda d: d["_id"])


def _outputs(db, name):
    return [d for d in db.find(name, {}) if d["_id"] != 0], db.find_one(name, {"_id": 0})


def _snapshot(db, name):
    if isinstance(db, ColumnarDatabase):
        return {f: (db.column(name, f), [b.address if b is not None else None for b in db.column(name, f).arr.buffers()])
                for f in db.column_names(name)}, db.version(name)
    return json.dumps(_data(db, name), sort_keys=True), db.version(name)


def _requests(c, name, tag):
    for out, body in ((f"{tag}_h", {"names": ["Age", "Fare"], "bins": 10, "range": [0, 100]}),
                      (f"{tag}_ha", {"names": ["Age", "Fare"], "bins": 10})):
        r = c.post("/histograms", json={"inputDatasetName": name, "outputDatasetName": out, **body})
        assert r.status_code == 201
    r = c.post("/projections", json={"inputDatasetName": name, "outputDatasetName": f"{tag}_p", "names": FIELDS4,
                                     "castTo": "float32", "bins": 10})
    assert r.status_code == 201


def _f32_bits(v):
    return None if v is None else int(np.float32(v).view(np.uint32))


def test_titanic_text_fields_equal_fieldtypes_then_request(engine, tmp_path):
    g = json.loads((GOLD / "titanic_shaped_input.json").read_text())
    for kind, db, path in _stores("t", g["headers"], g["rows"], tmp_path):
        engine.resident.clear()
        c = _client(db, engine, "t", path)
        before = _snapshot(db, "t")
        rows = _data(db, "t")
        _requests(c, "t", "a")
        after = _snapshot(db, "t")
        if kind == "columnar":       # the text columns are the very same Arrow arrays, not rewritten
            assert all(after[0][f][0] is before[0][f][0] and after[0][f][1] == before[0][f][1] for f in before[0]), kind
            assert all(isinstance(db.column("t", f), TextColumn) for f in FIELDS4)
        else:
            assert after[0] == before[0], kind
        assert after[1] == before[1], kind
        # oracle 1: float(cell) -> fp32 -> frozen binning
        for out, rng in (("a_h", (0.0, 100.0)), ("a_ha", None)):
            docs, meta = _outputs(db, out)
            assert meta["finished"] is True, (kind, meta)
            for d in docs:
                (f, res), = [(k, v) for k, v in d.items() if k != "_id"]
                x = bn.cast_f64_f32(np.array([_num(r[f]) for r in rows]))
                if rng is None:
                    fin = x[np.isfinite(x)]
                    lo, hi = bn.auto_range([fin.min()], [fin.max()], [fin.size], 10)
                    lo, hi = lo[0], hi[0]
                else:
                    lo, hi = np.float32(rng[0]), np.float32(rng[1])
                assert res["range"] == [float(lo), float(hi)], (kind, out, f)
                assert res["counts"] == bn.hist_f32(x, lo, hi, 10).tolist(), (kind, out, f)
        pdocs, pmeta = _outputs(db, "a_p")
        assert pmeta["finished"] is True, (kind, pmeta)
        pdocs.sort(key=lambda d: d["_id"])
        for f in FIELDS4:
            x = bn.cast_f64_f32(np.array([_num(r[f]) for r in rows]))
            got = [d[f] for d in pdocs]
            assert [(_f32_bits(v)) for v in got] == [None if r[f] in (None, "") else int(b) for r, b in
                                                     zip(rows, x.view(np.uint32))], (kind, f)
        # a repeat castTo reads the resident slabs: a hit that parses nothing, with the same output
        hits, misses = engine.resident.hits, engine.resident.misses
        r = c.post("/projections", json={"inputDatasetName": "t", "outputDatasetName": "a_p2", "names": FIELDS4,
                                         "castTo": "float32", "bins": 10})
        assert r.status_code == 201
        assert (engine.resident.hits, engine.resident.misses) == (hits + 1, misses), kind
        rdocs, rmeta = _outputs(db, "a_p2")
        assert rmeta["finished"] is True and rmeta["histogram"] == pmeta["histogram"], kind
        assert [[_f32_bits(d[f]) for f in FIELDS4] for d in sorted(rdocs, key=lambda d: d["_id"])] == \
            [[_f32_bits(d[f]) for f in FIELDS4] for d in pdocs], kind
        # oracle 2: the same requests after /fieldTypes "number" on a copy of the dataset
        _, db2, path2 = [s for s in _stores("n", g["headers"], g["rows"], tmp_path) if s[0] == kind][0]
        c2 = _client(db2, engine, "n", path2)
        assert c2.patch("/fieldTypes", json={"inputDatasetName": "n", "types": {f: "number" for f in FIELDS4}}).status_code == 200
        _requests(c2, "n", "b")
        for a, b in (("a_h", "b_h"), ("a_ha", "b_ha")):
            assert sorted(_outputs(db, a)[0], key=lambda d: d["_id"]) == sorted(_outputs(db2, b)[0], key=lambda d: d["_id"]), (kind, a)
        assert pmeta["histogram"] == _outputs(db2, "b_p")[1]["histogram"], kind
        qdocs = sorted(_outputs(db2, "b_p")[0], key=lambda d: d["_id"])
        assert [[_f32_bits(d[f]) for f in FIELDS4] for d in pdocs] == [[_f32_bits(d[f]) for f in FIELDS4] for d in qdocs], kind
    engine.resident.clear()


# ---- cell semantics ---------------------------------------------------------------------------------------------
def _parse(engine, arr_or_cells, nulls=None):
    from learningorchestra_b200 import columnar
    arr = columnar.number_text(arr_or_cells)
    chars, offsets, validity = columnar.text_buffers(arr)
    t = engine.table("f64", len(arr), 1)
    try:
        s = engine.parse_number_into(t, 0, chars, offsets, validity if nulls is None else nulls)
        return t.to_numpy(0).view(np.uint64), s
    finally:
        t.free()


def _expected_bits(cells, null=lambda c: c is None or c == ""):
    return [NAN if null(c) else int(np.float64(float(c)).view(np.uint64)) for c in cells]


def test_cell_semantics_equal_the_reference_vectors(engine):
    g = json.loads((GOLD / "reference_cast_vectors.json").read_text())
    cells = g["in"]
    bits, s = _parse(engine, cells)
    assert bits.tolist() == _expected_bits(cells)
    for c, b, ref in zip(cells, bits, g["number"]):           # the reference's own float(): value and int / float kind
        if ref is None:
            assert c in (None, "")
            continue
        v = np.uint64(b).view(np.float64)
        (k, text), = ref.items()
        assert (np.isnan(v) and text == "nan") or v == float(int(text) if k == "int" else float(text)), (c, ref)
    assert s["first_invalid"] is None and s["first_unsupported"] is None
    assert s["nulls"] == sum(c in (None, "") for c in cells) and s["integer"] is False
    _, s = _parse(engine, ["1", "-0.0", " 7 ", None, "", "1e22", "１２"])
    assert s["integer"] is True and s["nulls"] == 2
    # a bool null mask instead of the Arrow bitmap
    bits, s = _parse(engine, ["1.5", "zz", "2"], nulls=np.array([False, True, False]))
    assert bits.tolist() == [int(np.float64(1.5).view(np.uint64)), NAN, int(np.float64(2.0).view(np.uint64))]
    assert s["first_invalid"] is None and s["nulls"] == 1


def test_arrow_nulls_with_non_empty_slots_and_sliced_arrays(engine):
    text = b"12abc3.5junk-7"
    offsets = np.array([0, 2, 5, 8, 12, 14], np.int64)          # "12" | "abc" (null) | "3.5" | "junk" (null) | "-7"
    valid = np.packbits(np.array([1, 0, 1, 0, 1, 0, 0, 0], np.uint8), bitorder="little")
    arr = pa.LargeStringArray.from_buffers(5, pa.py_buffer(offsets), pa.py_buffer(text), pa.py_buffer(valid), null_count=2)
    bits, s = _parse(engine, arr)
    assert bits.tolist() == _expected_bits(["12", None, "3.5", None, "-7"])
    assert s["first_invalid"] is None and s["nulls"] == 2
    big = pa.array([None if i % 11 == 0 else ("" if i % 13 == 0 else repr(i * 0.37 - 5)) for i in range(1000)],
                   type=pa.large_string())
    for start, length in ((0, 1000), (3, 500), (77, 923), (999, 1), (500, 0)):
        sl = big.slice(start, length)
        assert length == 0 or sl.offset == start
        bits, s = _parse(engine, sl)
        cells = sl.to_pylist()
        assert bits.tolist() == _expected_bits(cells), (start, length)
        assert s["nulls"] == sum(c in (None, "") for c in cells)


# ---- failures ---------------------------------------------------------------------------------------------------
def _bad_rows(n=20):
    rows = [[str(i), repr(i * 1.5)] for i in range(n)]
    rows[7][1] = "abc"
    rows[3][1] = "x"
    rows[9][0] = "y"
    return rows


def _resident_bytes(engine):
    return sum(e.nbytes for e in engine.resident._entries.values())


def test_unparsable_cell_fails_the_job_and_changes_nothing(engine, tmp_path):
    for kind, db, path in _stores("bad", ["id", "v"], _bad_rows(), tmp_path):
        engine.resident.clear()
        c = _client(db, engine, "bad", path)
        before = _snapshot(db, "bad")
        for route, body in (("/histograms", {"bins": 10}), ("/projections", {"castTo": "float32"})):
            out = f"o{route[1]}"
            r = c.post(route, json={"inputDatasetName": "bad", "outputDatasetName": out, "names": ["v", "id"], **body})
            assert r.status_code == 201
            docs, meta = _outputs(db, out)
            assert meta["finished"] is False and docs == [], (kind, route, meta)
            assert "could not convert string to float: 'x'" in meta["exception"], (kind, route, meta["exception"])
        after = _snapshot(db, "bad")
        assert after[1] == before[1] and (after[0] == before[0] if kind == "documents" else
                                          all(after[0][f][0] is before[0][f][0] for f in before[0])), kind
        assert "bad" not in engine.resident._entries, kind
        # the first requested field that has a bad cell is named, whatever the row order across fields
        c.post("/histograms", json={"inputDatasetName": "bad", "outputDatasetName": "o2", "names": ["id", "v"], "bins": 4})
        assert "could not convert string to float: 'y'" in db.find_one("o2", {"_id": 0})["exception"], kind
    engine.resident.clear()


def test_cell_over_the_parser_limit_fails_loudly(engine):
    """A cell of 1 MiB + 1 bytes (longer than a CSV field may be, so the stores are filled directly)."""
    cells = ["2", "1" * ((1 << 20) + 1), "zz"]
    docs = utils.Database()
    docs.insert_one_in_file("big", rsem.dataset_metadata("big", ["b"]))
    docs.insert_many_in_file("big", [{"_id": i + 1, "b": v} for i, v in enumerate(cells)])
    cdb = ColumnarDatabase()
    cdb.ingest_columns("big", {"b": pa.array(cells, type=pa.large_string())})
    for kind, db in (("documents", docs), ("columnar", cdb)):
        engine.resident.clear()
        c = Client(server.create_app(db, engine, synchronous=True))
        c.post("/histograms", json={"inputDatasetName": "big", "outputDatasetName": "h", "names": ["b"], "bins": 4})
        meta = db.find_one("h", {"_id": 0})
        assert meta["finished"] is False and "1 MiB limit" in meta["exception"] and "no CPU fallback" in meta["exception"], kind
        assert "big" not in engine.resident._entries
    engine.resident.clear()


def test_failing_requests_leave_no_device_memory_behind(engine):
    import torch
    n = 1_000_000
    cells = pa.array([repr(i * 0.25) for i in range(n - 1)] + ["nope"], type=pa.large_string())
    db = ColumnarDatabase()
    db.ingest_columns("m", {"ok": pa.array([str(i) for i in range(n)], type=pa.large_string()), "bad": cells})
    c = Client(server.create_app(db, engine, synchronous=True))
    engine.resident.clear()

    def fail(i):
        c.post("/histograms", json={"inputDatasetName": "m", "outputDatasetName": f"h{i}", "names": ["ok", "bad"], "bins": 8})
        assert "could not convert string to float: 'nope'" in db.find_one(f"h{i}", {"_id": 0})["exception"]

    fail(0)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(engine.device)[0]
    for i in range(1, 6):
        fail(i)
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info(engine.device)[0]
    assert free0 - free1 < 4 * n * 8 // 2, (free0, free1)        # a leaked table would be 16 MB per request
    assert "m" not in engine.resident._entries and _resident_bytes(engine) == 0


# ---- residency ----------------------------------------------------------------------------------------------------
def test_second_request_is_a_cache_hit_and_fieldtypes_rebuilds(engine, tmp_path):
    g = json.loads((GOLD / "titanic_shaped_input.json").read_text())
    for kind, db, path in _stores("r", g["headers"], g["rows"], tmp_path):
        engine.resident.clear()
        c = _client(db, engine, "r", path)
        body = {"inputDatasetName": "r", "names": ["Age", "Fare"], "bins": 10}
        h0, m0, l0 = engine.resident.hits, engine.resident.misses, engine.launch_count
        c.post("/histograms", json={**body, "outputDatasetName": "r1"})
        l1 = engine.launch_count
        c.post("/histograms", json={**body, "outputDatasetName": "r2"})
        l2 = engine.launch_count
        assert engine.resident.misses == m0 + 1 and engine.resident.hits == h0 + 1, kind
        assert (l1 - l0) - (l2 - l1) == 2, kind           # the first request's two parse launches, none on the hit
        first = _outputs(db, "r1")[0]
        assert sorted(first, key=lambda d: d["_id"]) == sorted(_outputs(db, "r2")[0], key=lambda d: d["_id"])
        assert c.patch("/fieldTypes", json={"inputDatasetName": "r", "types": {"Age": "number"}}).status_code == 200
        c.post("/histograms", json={**body, "outputDatasetName": "r3"})
        assert engine.resident.misses == m0 + 2, kind    # the version moved: rebuilt (Age now numbers, Fare text)
        assert sorted(_outputs(db, "r3")[0], key=lambda d: d["_id"]) == sorted(first, key=lambda d: d["_id"]), kind
    engine.resident.clear()


# ---- several GPUs -------------------------------------------------------------------------------------------------
def _boundary_cells(n, cut):
    """Three text columns: clean (with nulls), bad cells either side of row ``cut``, bad cells after it only."""
    base = [None if i % 17 == 0 else ("" if i % 19 == 0 else repr(round((i * 7919 % 10007) * 0.1 - 500, 1)))
            for i in range(n)]
    both, after = list(base), list(base)
    both[cut + 3], both[cut - 2], both[n - 1] = "q", "w", "e"
    after[cut + 1], after[cut + 5] = "r", "t"
    return [pa.array(col, type=pa.large_string()) for col in (base, both, after)]


def _sharded_parse(sh, n, cols):
    from learningorchestra_b200 import columnar
    t = sh.table("f64", n, len(cols))
    summaries = []
    for j, arr in enumerate(cols):
        chars, offsets, validity = columnar.text_buffers(columnar.number_text(arr))
        summaries.append(sh.parse_number_into(t, j, chars, offsets, validity))
    return t, summaries


def _check_boundary(n, cut, summaries_per_rank, counts):
    cols = _boundary_cells(n, cut)
    firsts = [min(r for r in (s[j]["first_invalid"] for s in summaries_per_rank) if r is not None) for j in (1, 2)]
    assert firsts == [cut - 2, cut + 1]
    assert all(s[0]["first_invalid"] is None for s in summaries_per_rank)
    assert sum(s[0]["nulls"] for s in summaries_per_rank) == sum(c in (None, "") for c in cols[0].to_pylist())
    x = bn.cast_f64_f32(np.array([_num(c) for c in cols[0].to_pylist()]))
    np.testing.assert_array_equal(counts, bn.hist_f32(x, np.float32(-600), np.float32(600), 50)[None, :])


def test_local_group_parses_every_shard(engine):
    import torch
    from learningorchestra_b200.sharding import ShardedEngine
    n = 300_007
    with ShardedEngine.local(list(range(torch.cuda.device_count()))) as sh:
        cut = sh.bounds(n)[-1][0] if sh.nlocal > 1 else n // 2
        t, summaries = _sharded_parse(sh, n, _boundary_cells(n, cut))
        counts = sh.project_cast_hist(t, [0], 50, -600.0, 600.0).to_numpy()
        t.free()
        _check_boundary(n, cut, [summaries], counts)
        # the executors over the group: same counts as one GPU
        db = ColumnarDatabase()
        db.ingest_columns("g", dict(zip(["a", "b", "c"], _boundary_cells(n, cut))))
        for eng in (sh, engine):
            c = Client(server.create_app(db, eng, synchronous=True))
            c.post("/histograms", json={"inputDatasetName": "g", "outputDatasetName": f"h{id(eng)}", "names": ["a"],
                                        "bins": 50, "range": [-600, 600]})
        got = [_outputs(db, f"h{id(e)}")[0] for e in (sh, engine)]
        assert got[0] == got[1] and got[0][0]["a"]["counts"] == counts[0].tolist()
        c = Client(server.create_app(db, sh, synchronous=True))
        c.post("/histograms", json={"inputDatasetName": "g", "outputDatasetName": "hb", "names": ["a", "b"], "bins": 5})
        assert "could not convert string to float: 'w'" in db.find_one("hb", {"_id": 0})["exception"]
    engine.resident.clear()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _rank_worker(rank, world, port, n, ret):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = rank % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from learningorchestra_b200.engine import Engine
    from learningorchestra_b200.sharding import ShardedEngine, shard_bounds
    eng = Engine(dev)
    sh = ShardedEngine.from_torch_distributed(eng, merge="peer")
    cut = shard_bounds(n, world, 1)[0]
    t, summaries = _sharded_parse(sh, n, _boundary_cells(n, cut))
    counts = sh.project_cast_hist(t, [0], 50, -600.0, 600.0, bcast=True).to_numpy()
    t.free()
    dist.barrier()
    ret.put((rank, cut, summaries, counts))
    dist.barrier()
    sh.close()
    eng.close()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_rank_group_first_bad_row_is_global(built, world):
    import torch.multiprocessing as mp
    n = 200_003
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_rank_worker, args=(r, world, port, n, ret)) for r in range(world)]
    for p in procs:
        p.start()
    res = {}
    try:
        for _ in range(world):
            r, cut, summaries, counts = ret.get(timeout=300)
            res[r] = (cut, summaries, counts)
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    cut = res[0][0]
    for r in range(world):
        _check_boundary(n, cut, [res[q][1] for q in range(world)], res[r][2])


# ---- size -----------------------------------------------------------------------------------------------------------
def test_ten_million_rows_of_four_text_fields(engine):
    n, k = 10_000_000, 4
    rng = np.random.default_rng(20261016)
    db = ColumnarDatabase()
    values, cols = [], {}
    for j in range(k):
        x = rng.uniform(-1000, 1000, n)
        if j == 1:
            x = np.round(x)                                  # integer-valued cells: repr "12.0"
        if j == 2:
            x = np.round(x, 2)
        x[rng.random(n) < 0.01] = np.nan                     # nulls
        cells = [None if v != v else repr(v) for v in x.tolist()]
        cols[f"f{j}"] = pa.array(cells, type=pa.large_string())
        del cells
        values.append(x)
    db.ingest_columns("big", cols)
    engine.resident.clear()
    c = Client(server.create_app(db, engine, synchronous=True))
    r = c.post("/histograms", json={"inputDatasetName": "big", "outputDatasetName": "h", "names": list(cols), "bins": 64})
    assert r.status_code == 201 and db.find_one("h", {"_id": 0})["finished"] is True
    docs = {f: res for d in _outputs(db, "h")[0] for f, res in d.items() if f != "_id"}
    with engine.resident.lease(db, "big", list(cols)) as data:
        out = engine.project_cast(data.table, [data.column[f] for f in cols])
        sums = [out.checksum(j) for j in range(k)]
        out.free()
    r2 = np.arange(n, dtype=np.uint64) * np.uint64(2) + np.uint64(1)
    for j, f in enumerate(cols):
        x32 = bn.cast_f64_f32(values[j])
        fin = x32[np.isfinite(x32)]
        lo, hi = bn.auto_range([fin.min()], [fin.max()], [fin.size], 64)
        assert docs[f]["counts"] == bn.hist_f32(x32, lo[0], hi[0], 64).tolist(), f
        with np.errstate(over="ignore"):
            exp = int(np.sum(x32.view(np.uint32).astype(np.uint64) * r2, dtype=np.uint64))
        assert sums[j] == exp, f
    engine.resident.clear()
