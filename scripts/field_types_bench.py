"""The upload -> /fieldTypes -> /histograms flow on a column store, step by step.

    python scripts/field_types_bench.py [--rows 10000000] [--fields 4] [--bins 64] [--reps 3] [--gpus 1 all]
                                        [--tree OTHER_CHECKOUT] [--out FILE]

Dataset: ``text_bins_bench.py``'s — ``--rows`` x ``--fields`` text columns of ``repr()`` of seeded doubles, 1 % nulls,
as POST /files stores them.  Steps, each timed by wall clock, with the bytes handed to calls that copy host cells or
values to the device (text uploads, slab uploads, host-buffer parses and formats):

1. /histograms without ``bins`` on the fields (their text columns become resident);
2. /fieldTypes "number" on the fields;
3. /histograms with ``bins``;
4. /histograms without ``bins``.

``--tree``: another checkout (built) to run the same flow from, alternated with this one rep by rep, each run in a
process of its own.  ``--gpus``: 1 runs an ``Engine`` on device 0, ``all`` a ``ShardedEngine`` over every visible GPU.
The card's name and power limit are printed with the numbers.  Writes nothing into the tree (the dataset is cached in
a temporary directory).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines() if q.returncode == 0 else ["unknown"]


def dataset(rows, fields, seed, cache: Path):
    import numpy as np
    import pyarrow as pa
    import pyarrow.feather as feather
    if not cache.exists():
        rng = np.random.default_rng(seed)
        cols = {}
        for j in range(fields):
            x = rng.uniform(-1000, 1000, rows)
            x[rng.random(rows) < 0.01] = np.nan
            cols[f"f{j}"] = pa.array([None if v != v else repr(v) for v in x.tolist()], type=pa.large_string())
        feather.write_feather(pa.table(cols), str(cache) + ".tmp")
        os.replace(str(cache) + ".tmp", cache)
    t = feather.read_table(str(cache), memory_map=False)
    return {n: t.column(n).combine_chunks() for n in t.column_names}


def child(a):
    """One run of the flow from the checkout this process imports."""
    sys.path.insert(0, a.tree_root)
    from learningorchestra_b200 import utils
    from learningorchestra_b200.column_store import ColumnarDatabase
    from learningorchestra_b200.data_type_update import DataType
    from learningorchestra_b200.engine import Engine
    from learningorchestra_b200.histogram import Histogram
    from learningorchestra_b200.sharding import ShardedEngine

    cols = dataset(a.rows, a.fields, a.seed, Path(a.cache))
    names = list(cols)
    eng = Engine(0) if a.gpus[0] == "1" else ShardedEngine.local()
    moved = [0]

    def count(obj, name, nbytes):
        real = getattr(obj, name, None)
        if real is not None:
            setattr(obj, name, lambda *x, **k: (moved.__setitem__(0, moved[0] + nbytes(*x)), real(*x, **k))[1])

    count(eng, "text", lambda cells, *r: len(cells) * 8 + int(cells.buffers()[2].size if cells.buffers()[2] else 0))
    count(eng, "parse_number_into", lambda t, c, chars, offsets, *r: int(offsets[-1] - offsets[0]) + offsets.nbytes)
    count(eng, "parse_number_packed", lambda chars, offsets: int(offsets[-1] - offsets[0]) + offsets.nbytes)
    count(eng, "format_number_host", lambda values, status, *r: values.nbytes + status.nbytes)
    from learningorchestra_b200 import engine as E, sharding as S
    for cls in (E.DeviceTable, S.ShardedTable):
        real = cls.upload
        cls.upload = lambda self, col, values, *r, _r=real: (moved.__setitem__(0, moved[0] + values.nbytes), _r(self, col, values, *r))[1]

    db = ColumnarDatabase()
    db.ingest_columns("d", cols)
    steps = []

    def step(name, fn):
        moved[0] = 0
        t0 = time.perf_counter()
        fn()
        steps.append({"step": name, "s": time.perf_counter() - t0, "h2d_bytes": moved[0]})

    hist = lambda out, bins=None: Histogram(db, utils.HistogramMetadata(db), eng).file_processing("d", out, names, bins)
    step("histograms", lambda: hist("h1"))
    job = DataType(db, utils.DataTypeMetadata(db), eng)
    step("fieldTypes number", lambda: [job.field_converter("d", f, "number") for f in names])
    step(f"histograms bins={a.bins}", lambda: hist("h2", a.bins))
    step("histograms", lambda: hist("h3"))
    import hashlib
    groups = {f: sorted(json.dumps(g, sort_keys=True, default=str) for g in d[f])
              for d in db.find("h3", {}) if d["_id"] != 0 for f in d if f != "_id"}
    eng.close()
    print(json.dumps({"tree": a.tree_root, "gpus": a.gpus, "steps": steps,
                      "h3": hashlib.sha256(json.dumps(groups, sort_keys=True).encode()).hexdigest()}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--fields", type=int, default=4)
    ap.add_argument("--bins", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=20261016)
    ap.add_argument("--gpus", nargs="+", default=["1", "all"])
    ap.add_argument("--tree", help="another built checkout to alternate with this one")
    ap.add_argument("--out")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--tree-root", default=str(ROOT), help=argparse.SUPPRESS)
    ap.add_argument("--cache", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        return child(a)
    trees = [str(Path(a.tree).resolve()), str(ROOT)] if a.tree else [str(ROOT)]
    results = {"card": card(), "rows": a.rows, "fields": a.fields, "bins": a.bins, "runs": []}
    with tempfile.TemporaryDirectory() as tmp:
        cache = Path(tmp) / "data.feather"
        for rep in range(a.reps):
            for gpus in a.gpus:
                for tree in trees:
                    p = subprocess.run([sys.executable, __file__, "--child", "--tree-root", tree, "--gpus", gpus,
                                        "--cache", str(cache), "--rows", str(a.rows), "--fields", str(a.fields),
                                        "--bins", str(a.bins), "--seed", str(a.seed)],
                                       capture_output=True, text=True, cwd=tree)
                    if p.returncode != 0:
                        raise RuntimeError(p.stderr[-4000:])
                    run = json.loads(p.stdout.strip().splitlines()[-1])
                    run["rep"] = rep
                    results["runs"].append(run)
                    print(json.dumps({k: run[k] for k in ("tree", "gpus", "rep", "steps")}), flush=True)
    outs = {}
    for run in results["runs"]:                 # every run must count the same groups
        outs.setdefault(run["gpus"][0], run["h3"])
        assert run["h3"] == outs[run["gpus"][0]], "the runs' /histograms documents differ"
    text = json.dumps(results, indent=1)
    if a.out:
        Path(a.out).write_text(text)
    print("card:", results["card"])


if __name__ == "__main__":
    main()
