"""GPU: the device CSV reader (lo_csv_read_host, csrc/csv.inc) against the reference's own csv.reader call
(csv_oracle.csv_reference_rows), and ColumnarDatabase.ingest_csv / POST /files with an engine."""
import io
import json
import random
from pathlib import Path

import numpy as np
import pytest

from csv_oracle import KINDS, csv_reference_rows
from learningorchestra_b200 import _native as N
from learningorchestra_b200.column_store import ColumnarDatabase
from test_csv_cpu import HAND

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden"


def device_rows(engine, body: bytes):
    header, nrows, chars, offsets, failure = engine.read_csv_host(body)
    raw = chars.tobytes()
    rows = [[raw[offsets[c, r]:offsets[c, r + 1]].decode("utf-8") for c in range(offsets.shape[0])] for r in range(1, nrows + 1)]
    return header, rows, (None if failure is None else (KINDS[failure[0]], failure[1]))


def test_hand_cases(engine):
    for body in HAND:
        assert device_rows(engine, body) == csv_reference_rows(body), body


def test_random_bodies(engine):
    rng = random.Random(20261016)
    alphabet = [b",", b"\"", b"\r", b"\n", b"a", b" ", "é".encode(), b"\xc3", b"\xa9", b"\x00", b"\xff"]
    weights = [6, 6, 3, 4, 6, 2, 2, 1, 1, 0.3, 0.3]
    for _ in range(3000):
        body = b"".join(rng.choices(alphabet, weights, k=rng.randint(0, 40)))
        assert device_rows(engine, body) == csv_reference_rows(body), body


def test_bodies_across_segment_and_cta_boundaries(engine):
    """Quoted runs, "" pairs, \\r\\n and multi-byte characters at every offset around the 256-byte segments and the
    128-thread CTAs (32 KiB); one 100 KB quoted field."""
    rng = random.Random(5)
    pieces = ['"a,b"', '""""', '"x\r\ny"', "\r\n", "é", "€", "😀", "plain", '"q""q"', ",", "\n"]
    for length in (255, 256, 257, 511, 32767, 32768, 32769, 100_000):
        for _ in range(3):
            text = "h1,h2,h3\r\n"
            while len(text.encode()) < length:
                text += ",".join(rng.choice(pieces[:9]) for _ in range(3)) + rng.choice(["\r\n", "\n", "\r"])
            body = text.encode()
            assert device_rows(engine, body) == csv_reference_rows(body)
    big = b'h,i\n1,"' + ("é,\"\"\n" * 20000).encode() + b'"\n2,3\n'
    exp = csv_reference_rows(big)
    assert exp[2] is None and len(exp[1][0][1]) == 60000 and len(big) > 100_000
    assert device_rows(engine, big) == exp


def test_failure_kinds_keep_the_rows_before(engine, tmp_path):
    cases = {
        N.LO_CSV_SHORT_ROW: b"a,b\n1,2\n3,4\n5\n6,7\n",
        N.LO_CSV_FIELD_LIMIT: b"a,b\n1,2\n3,4\n" + b"x" * 131073 + b",5\n",
        N.LO_CSV_BAD_UTF8: b"a,b\n1,2\n3,4\n\xff,5\n",
        N.LO_CSV_NUL: b"a,b\n1,2\n3,4\n\x00,5\n",
        N.LO_CSV_UNSUPPORTED: b"a,b\n1,2\n3,4\n\xc3\n\xa9,5\n",
    }
    for kind, body in cases.items():
        header, nrows, chars, offsets, failure = engine.read_csv_host(body)
        assert header == ["a", "b"] and nrows == 2 and failure[:2] == (kind, 3)
        path = tmp_path / f"k{kind}.csv"
        path.write_bytes(body)
        db = ColumnarDatabase()
        assert db.ingest_csv("f", str(path), url="file://f", engine=engine) == 2
        meta = db.find_one("f", {"_id": 0})
        assert meta["finished"] is False and meta["exception"]
        rows = sorted((d for d in db.find("f", {}) if d["_id"] != 0), key=lambda d: d["_id"])
        assert rows == [{"a": "1", "b": "2", "_id": 1}, {"a": "3", "b": "4", "_id": 2}]
    for body in (b"", b"\n\n", b"a\x00,b\n1,2\n"):       # empty body, failing header: nothing stored
        db = ColumnarDatabase()
        assert db.ingest_csv("f", io.BytesIO(body), engine=engine) == 0
        meta = db.find_one("f", {"_id": 0})
        assert meta["finished"] is False and meta["exception"] and not db.has_columns("f")


def _titanic_csv(tmp_path):
    import csv
    g = json.loads((GOLDEN / "titanic_shaped_input.json").read_text())
    buf = io.StringIO()
    w = csv.writer(buf, lineterminator="\n")
    w.writerow(g["headers"])
    w.writerows(g["rows"])
    path = tmp_path / "titanic.csv"
    path.write_text(buf.getvalue(), encoding="utf-8")
    return path


def test_ingest_matches_the_pyarrow_path_on_titanic(engine, tmp_path):
    path = _titanic_csv(tmp_path)
    a, b = ColumnarDatabase(), ColumnarDatabase()
    assert a.ingest_csv("t", str(path), url="u") == b.ingest_csv("t", str(path), url="u", engine=engine) == 891
    strip = lambda m: {k: v for k, v in m.items() if k != "timeCreated"}
    assert strip(a.find_one("t", {"_id": 0})) == strip(b.find_one("t", {"_id": 0}))
    assert a.column_names("t") == b.column_names("t")
    for name in a.column_names("t"):
        assert a.column("t", name).arr.to_pylist() == b.column("t", name).arr.to_pylist()
        b.column("t", name).arr.validate(full=True)
    by_id = lambda db: sorted(db.find("t", {}), key=lambda d: d["_id"])
    assert by_id(a) == by_id(b)


def test_body_over_2_31_bytes(engine):
    """A repeated block, so the columns are known by construction; every index above 2^31 is exercised."""
    block = 'id,"quoted, text","multi\r\nline ""é"""\n'.encode()
    header = b"a,b,c\n"
    reps = (2 ** 31 + 2 ** 20) // len(block) + 1
    body = np.empty(len(header) + reps * len(block), dtype=np.uint8)
    body[:len(header)] = np.frombuffer(header, np.uint8)
    body[len(header):] = np.tile(np.frombuffer(block, np.uint8), reps)
    assert body.size > 2 ** 31
    hdr, nrows, chars, offsets, failure = engine.read_csv_host(body)
    del body
    assert hdr == ["a", "b", "c"] and nrows == reps and failure is None
    cells = [b"id", b"quoted, text", b'multiline "\xc3\xa9"']
    for c, cell in enumerate(cells):
        lens = np.diff(offsets[c, 1:])
        assert (lens == len(cell)).all()
        for r in (1, reps // 2, reps):
            assert chars[offsets[c, r]:offsets[c, r + 1]].tobytes() == cell
    assert offsets[2, -1] == chars.size


def test_files_fieldtypes_histograms_over_http(engine, tmp_path):
    """POST /files -> PATCH /fieldTypes -> POST /histograms with an engine == the reference-executed goldens; a failing
    upload still answers 201 and shows finished False with the exception."""
    from werkzeug.test import Client

    from learningorchestra_b200.server import create_app
    from oracle import rsem
    path = _titanic_csv(tmp_path)
    gold = json.loads((GOLDEN / "reference_histogram.json").read_text())
    app = create_app(None, engine, synchronous=True)
    c = Client(app)
    r = c.post("/files", json={"datasetName": "titanic", "datasetURI": f"file://{path}"})
    assert r.status_code == 201
    assert app.database.find_one("titanic", {"_id": 0})["finished"] is True
    types = {f: "number" for f in ("Survived", "Pclass", "Age", "Fare")}
    assert c.patch("/fieldTypes", json={"inputDatasetName": "titanic", "types": types}).status_code == 200
    r = c.post("/histograms", json={"inputDatasetName": "titanic", "outputDatasetName": "titanic_hist", "names": gold["fields"]})
    assert r.status_code == 201
    got = sorted(app.database.find("titanic_hist", {}), key=lambda d: d["_id"])
    ref = sorted(gold["documents"], key=lambda d: d["_id"])
    assert got[0]["finished"] is True and [d["_id"] for d in got] == [d["_id"] for d in ref]
    for mine, theirs, f in zip(got[1:], ref[1:], gold["fields"]):
        assert rsem.normalise_group_result(mine[f]) == rsem.normalise_group_result(theirs[f]), f
    bad = tmp_path / "bad.csv"
    bad.write_bytes(b"a,b\n1,2\n3\n")
    r = c.post("/files", json={"datasetName": "bad", "datasetURI": f"file://{bad}"})
    assert r.status_code == 201
    meta = app.database.find_one("bad", {"_id": 0})
    assert meta["finished"] is False and "IndexError" in meta["exception"]
