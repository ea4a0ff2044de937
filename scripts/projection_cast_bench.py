"""`/projections` with `castTo: "float32"` on a document store: `Projection.create` cold and warm, with and without
`bins`.

    python scripts/projection_cast_bench.py [--docs 2000000] [--reps 3] [--out FILE]

Input, seeded: a document store of --docs data rows in `_id` order with two number fields (ints and floats, 5 % None
each) and two text fields (`repr()` of floats, 5 % `""` and 5 % None each).  Per mode (no `bins`; 64 bins without
`range`): the wall time of a cold request (the engine's resident copy cleared first) and of a warm one (the same request
again), best, median and worst of --reps, and a digest of the output rows and histogram document, so runs of two builds
can be checked to compute the same thing.  The card's name, power limit and max SM clock are printed with the numbers
(read-only nvidia-smi query).  Writes nothing into the tree.
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

FIELDS = ["ints", "floats", "text_a", "text_b"]
MODES = {"no_bins": {}, "bins_64": {"bins": 64}}


def document_store(n, rng):
    from learningorchestra_b200 import utils
    null = rng.random((4, n)) < 0.05
    empty = rng.random((2, n)) < 0.05
    ints = rng.integers(-10_000, 10_000, n).tolist()
    floats = np.round(rng.normal(30, 15, n), 3).tolist()
    text = [[None if null[2 + k, i] else ("" if empty[k, i] else repr(v)) for i, v in
             enumerate(rng.uniform(-1e4, 1e4, n).tolist())] for k in range(2)]
    db = utils.Database()
    db.insert_one_in_file("d", {"_id": 0, "finished": True, "fields": FIELDS})
    db.insert_many_in_file("d", [{"_id": i + 1, "ints": None if null[0, i] else ints[i],
                                  "floats": None if null[1, i] else floats[i], "text_a": text[0][i], "text_b": text[1][i]}
                                 for i in range(n)])
    return db


def digest(db, target):
    rows = [d for d in db.find(target, {}) if d["_id"] != 0]
    h = hashlib.sha256(json.dumps([d["_id"] for d in rows]).encode())
    for f in FIELDS:
        v = np.array([np.nan if d[f] is None else d[f] for d in rows], np.float32)
        h.update(v.view(np.uint32).tobytes())
        h.update(np.array([d[f] is None for d in rows]).tobytes())
    h.update(json.dumps(db.find_one(target, {"_id": 0}).get("histogram"), sort_keys=True).encode())
    return h.hexdigest()[:16]


def run(db, engine, reps):
    from learningorchestra_b200 import utils
    from learningorchestra_b200.projection import Projection
    out, k = {}, 0
    for mode, body in MODES.items():
        times, results = {"cold": [], "warm": []}, set()
        for r in range(reps + 1):
            engine.resident.clear()
            for temp in ("cold", "warm"):
                target, k = f"p{k}", k + 1
                job = Projection(utils.ProjectionMetadata(db), engine)
                t0 = time.perf_counter()
                job.create("d", target, list(FIELDS), "mongodb://h/database.d?r", f"mongodb://h/database.{target}?r",
                           cast_to="float32", **body)
                job.wait()
                dt = (time.perf_counter() - t0) * 1e3
                assert db.find_one(target, {"_id": 0})["finished"] is True
                if r:                                   # the first round warms the engine, numpy and pyarrow
                    times[temp].append(dt)
                if r == 1:
                    results.add(digest(db, target))
                db.delete_file(target)
        assert len(results) == 1, f"{mode}: cold and warm requests wrote different outputs"
        out[mode] = {temp: {"best_ms": round(min(ts), 1), "median_ms": round(sorted(ts)[len(ts) // 2], 1),
                            "worst_ms": round(max(ts), 1)} for temp, ts in times.items()}
        out[mode]["result"] = results.pop()
    engine.resident.clear()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--docs", type=int, default=2_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", type=Path)
    args = ap.parse_args()
    from learningorchestra_b200.engine import Engine
    rng = np.random.default_rng(20261017)
    report = {"card": card(), "docs": args.docs, "fields": FIELDS, "reps": args.reps}
    t0 = time.perf_counter()
    db = document_store(args.docs, rng)
    report["build_s"] = round(time.perf_counter() - t0, 1)
    with Engine(0) as eng:
        report["document_store"] = run(db, eng, args.reps)
    line = json.dumps(report)
    print(line)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(line + "\n")


if __name__ == "__main__":
    main()
