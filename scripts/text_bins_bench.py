"""Binned histograms of TEXT fields: the two routes a user has, timed in one run, alternated.

    python scripts/text_bins_bench.py [--rows 10000000] [--fields 4] [--bins 64] [--reps 3] [--seed S] [--out FILE]

Dataset: ``--rows`` x ``--fields`` text columns (Arrow large_string, as POST /files stores them), every cell ``repr()``
of a seeded double, 1 % nulls.  Routes, through the executors on a column store:

* old: PATCH /fieldTypes "number" on a fresh copy (parse, binary64 back to the host, column replaced), then the binned
  /histograms (upload of the binary64 columns to HBM, bins);
* new cold: the binned /histograms on the text fields, nothing resident (parse straight into HBM, bins);
* new warm: the same request again (resident slabs, bins only).

For each: wall time per request and rows/s (dataset rows / time, all fields binned).  The new route's parse calls also report their
``kernel_ms`` (summed over the fields) and text bytes/s over it.  The counts of the routes must be equal.  The card's
name and power limit are read in the same run and printed with the numbers.  Writes nothing into the tree.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True)
    except OSError:
        return "unknown"
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def columns(rows, fields, seed):
    import pyarrow as pa
    rng = np.random.default_rng(seed)
    out = {}
    for j in range(fields):
        x = rng.uniform(-1000, 1000, rows)
        x[rng.random(rows) < 0.01] = np.nan
        out[f"f{j}"] = pa.array([None if v != v else repr(v) for v in x.tolist()], type=pa.large_string())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--fields", type=int, default=4)
    ap.add_argument("--bins", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=20261016)
    ap.add_argument("--out")
    a = ap.parse_args()

    from learningorchestra_b200.column_store import ColumnarDatabase
    from learningorchestra_b200.columnar import text_buffers
    from learningorchestra_b200.data_type_update import DataType
    from learningorchestra_b200.engine import Engine
    from learningorchestra_b200.histogram import Histogram
    from learningorchestra_b200.utils import DataTypeMetadata, HistogramMetadata

    cols = columns(a.rows, a.fields, a.seed)
    names = list(cols)
    text_bytes = sum(int(o[-1] - o[0]) for o in (text_buffers(c)[1] for c in cols.values()))
    res = {"card": card(), "rows": a.rows, "fields": a.fields, "bins": a.bins, "text_bytes": text_bytes,
           "old": [], "new_cold": [], "new_warm": [], "parse_kernel_ms": []}
    with Engine(0) as eng:
        parse = eng.parse_number_into
        kernel_ms = []

        def timed_parse(*args, **kw):          # collects each parse call's device time
            s = parse(*args, **kw)
            kernel_ms.append(s["kernel_ms"])
            return s
        eng.parse_number_into = timed_parse

        def histogram(db, out):
            h = Histogram(db, HistogramMetadata(db), eng)
            t0 = time.perf_counter()
            h.create_file("d", out, names, bins=a.bins)
            h.wait()
            dt = time.perf_counter() - t0
            assert db.find_one(out, {"_id": 0})["finished"] is True
            return dt, sorted((d for d in db.find(out, {}) if d["_id"] != 0), key=lambda d: d["_id"])

        counts = {}
        for rep in range(a.reps + 1):                  # rep 0 warms every shape up and is not reported
            db = ColumnarDatabase()
            db.ingest_columns("d", dict(cols))
            eng.resident.clear()
            kernel_ms.clear()
            cold, counts["new"] = histogram(db, f"c{rep}")
            parse_ms = sum(kernel_ms)
            warm, counts["warm"] = histogram(db, f"w{rep}")
            db2 = ColumnarDatabase()
            db2.ingest_columns("d", dict(cols))
            eng.resident.clear()
            t0 = time.perf_counter()
            job = DataType(db2, DataTypeMetadata(db2), eng)
            job.field_file_converter("d", {f: "number" for f in names})
            _, counts["old"] = histogram(db2, f"o{rep}")
            old = time.perf_counter() - t0
            assert counts["old"] == counts["new"] == counts["warm"]
            if rep:
                res["new_cold"].append(cold); res["new_warm"].append(warm); res["old"].append(old)
                res["parse_kernel_ms"].append(parse_ms)
        eng.resident.clear()
    for k in ("old", "new_cold", "new_warm"):
        t = float(np.median(res[k]))
        res[f"{k}_s"] = t
        res[f"{k}_rows_per_s"] = a.rows / t
    pk = float(np.median(res["parse_kernel_ms"]))
    res["parse_kernel_ms_median"] = pk
    res["parse_text_bytes_per_s"] = text_bytes / (pk * 1e-3) if pk > 0 else None
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
