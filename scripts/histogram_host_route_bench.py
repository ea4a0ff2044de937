"""`/histograms` without `bins` through the host route alone: `Histogram.file_processing` on an engine whose `resident`
is None, so every field is read from the store and packed per request.

    python scripts/histogram_host_route_bench.py [--rows 10000000] [--docs 200000] [--reps 7] [--out FILE]

Inputs, seeded: a column store of --rows rows (a number field of 1 000 integer values with 1 % nulls, a text field of
six words with 1 % nulls, and an all-null number field) and a document store of --docs documents (a number field, a
text field and a mixed field of 1, 1.0, "1", True and None).  Per field: the wall time of one request for that field
(best, median and worst of --reps after one warm-up request) and a digest of its result document (groups, counts and
key types), so runs of two builds can be checked to compute the same groups.  The card's name, power limit and max SM
clock are printed with the numbers (read-only nvidia-smi query).  Writes nothing into the tree.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))

from value_counts_bench import card  # noqa: E402


class HostRoute:
    """The engine without ``resident``: the host route counts every field."""

    resident = None

    def __init__(self, engine):
        self._engine = engine

    def __getattr__(self, name):
        return getattr(self._engine, name)


def column_store(n, rng):
    import pyarrow as pa
    from learningorchestra_b200.column_store import ColumnarDatabase, NumberColumn, TextColumn
    valid = rng.random(n) >= 0.01
    ints = rng.integers(0, 1000, n).astype(np.float64)
    words = pa.array(["male", "female", "", "S", "C", "Q"], type=pa.large_string())
    text = words.take(pa.array(rng.integers(0, 6, n), mask=rng.random(n) < 0.01))
    db = ColumnarDatabase()
    db.ingest_columns("c", {"number": NumberColumn(np.where(valid, ints, np.nan), valid, valid),
                            "text": TextColumn(text),
                            "null": NumberColumn(np.full(n, np.nan), np.zeros(n, bool))})
    return db, "c", ["number", "text", "null"]


def document_store(n, rng):
    from learningorchestra_b200 import utils
    mixed = [1, 1.0, "1", True, None]
    words = ["male", "female", "", "S", "C", "Q"]
    number, text, kind = rng.integers(0, 1000, n).tolist(), rng.integers(0, 6, n).tolist(), rng.integers(0, 5, n).tolist()
    db = utils.Database()
    db.insert_one_in_file("d", {"_id": 0, "finished": True, "fields": ["number", "text", "mixed"]})
    db.insert_many_in_file("d", [{"_id": i + 1, "number": number[i], "text": words[text[i]], "mixed": mixed[kind[i]]}
                                 for i in range(n)])
    return db, "d", ["number", "text", "mixed"]


def digest(groups, typed):
    """A mixed field's representative of a group is unspecified (1 or 1.0): its key types are left out."""
    from learningorchestra_b200 import columnar
    canon = sorted((repr(columnar.group_key(g["_id"])), type(g["_id"]).__name__ if typed else "", g["count"])
                   for g in groups)
    return hashlib.sha256(json.dumps(canon).encode()).hexdigest()[:16]


def run(db, name, fields, engine, reps):
    from learningorchestra_b200 import utils
    from learningorchestra_b200.histogram import Histogram
    job = Histogram(db, utils.HistogramMetadata(db), HostRoute(engine))
    out = {}
    for f in fields:
        ts, results = [], set()
        for r in range(reps + 1):
            target = f"h_{name}_{f}_{r}"
            t0 = time.perf_counter()
            job.file_processing(name, target, [f])
            dt = (time.perf_counter() - t0) * 1e3
            if r:                                       # the first request warms the engine and pyarrow
                ts.append(dt)
            (doc,) = [d for d in db.find(target, {}) if d["_id"] != 0]
            results.add(digest(doc[f], f != "mixed"))
            db.delete_file(target)
        assert len(results) == 1, f"{name}.{f}: the result changed between requests"
        ts.sort()
        out[f] = {"best_ms": round(ts[0], 2), "median_ms": round(ts[len(ts) // 2], 2), "worst_ms": round(ts[-1], 2),
                  "result": results.pop()}
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--docs", type=int, default=200_000)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", type=Path)
    args = ap.parse_args()
    from learningorchestra_b200.engine import Engine
    rng = np.random.default_rng(20261017)
    report = {"card": card(), "rows": args.rows, "docs": args.docs, "reps": args.reps}
    with Engine(0) as eng:
        report["column_store"] = run(*column_store(args.rows, rng), eng, args.reps)
        report["document_store"] = run(*document_store(args.docs, rng), eng, args.reps)
    line = json.dumps(report)
    print(line)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(line + "\n")


if __name__ == "__main__":
    main()
