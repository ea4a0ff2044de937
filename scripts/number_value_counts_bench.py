"""`$group` of number columns: the host route (lo_value_counts_f64_host: pack, copy, count) against the resident route
(lo_value_counts_f64_table on the slab kept in HBM), and /histograms end to end.

    python scripts/number_value_counts_bench.py [--titanic-mb 1024] [--rows 10000000] [--reps 5] [--out FILE]
                                                [--ab LIB.so ...]

Input: a Titanic-shaped CSV body (csv_bench.titanic_body) ingested with the engine, then /fieldTypes "number" on its
number fields, plus synthetic columns of --rows values (3 values, 20 000 values, all distinct, constant, 1 % NaN and
1 % null).  Per field: the host call's time and kernel_ms, the resident call's time and kernel_ms, GB/s of the slab over
the resident kernel_ms, and the /histograms wall time of one request for that field, cold (the slab uploaded by the
request) and warm (resident).  With two or more GPUs, ShardedEngine.value_counts_column and its host merge are timed
apart on the all-distinct column.
--ab: host-route kernel_ms of the given builds of libloexec.so on the four synthetic columns, each build in a fresh
process, alternating, --reps rounds (median): the parent commit's library against this one measures the kernel alone.
The card's name, power limit and max SM clock are printed with the numbers (read-only nvidia-smi query).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))

from value_counts_bench import best, card  # noqa: E402

NUMBER_FIELDS = ["PassengerId", "Survived", "Pclass", "Age", "SibSp", "Parch", "Fare"]

AB_CHILD = r'''
import ctypes as C, json, sys
import numpy as np
sys.path.insert(0, %r)
from learningorchestra_b200 import _native as N
from learningorchestra_b200.engine import Engine
n, reps = int(sys.argv[1]), int(sys.argv[2])
eng = Engine(0)
lib = eng._lib
rng = np.random.default_rng(1)
cols = {"three": (np.arange(n) %% 3).astype(np.float64), "k20000": rng.integers(0, 20000, n).astype(np.float64),
        "distinct": rng.permutation(n).astype(np.float64), "constant": np.full(n, 7.25)}
out = {}
for name, x in cols.items():
    card = int(np.unique(x).size)
    keys, counts, nd = np.empty(card), np.empty(card, np.uint64), C.c_int64()
    ks = []
    for r in range(reps + 1):
        t = N.HostTiming()
        N.check(lib.lo_value_counts_f64_host(eng._ctx, x.ctypes.data_as(C.c_void_p), n, keys.ctypes.data_as(C.c_void_p),
                                             counts.ctypes.data_as(C.c_void_p), card, C.byref(nd), C.byref(t)))
        assert nd.value == card and int(counts.sum()) == n
        if r:
            ks.append(t.kernel_ms)
    out[name] = sorted(ks)[len(ks) // 2]
print(json.dumps(out))
''' % str(ROOT)


def ab(libs, rows, reps):
    res = {lib: [] for lib in libs}
    for rnd in range(reps):
        for lib in libs:
            env = dict(os.environ, LOEXEC_LIB=lib, LOEXEC_LAX="1")
            p = subprocess.run([sys.executable, "-c", AB_CHILD, str(rows), "5"], env=env, capture_output=True, text=True)
            line = [x for x in p.stdout.splitlines() if x.startswith("{")]
            if not line:
                print("FAILED", lib, p.stderr[-800:], flush=True)
                continue
            res[lib].append(json.loads(line[-1]))
            print("ab", rnd, lib, line[-1], flush=True)
    out = {}
    for lib, runs in res.items():
        out[lib] = {k: {"median": sorted(r[k] for r in runs)[len(runs) // 2],
                        "min": min(r[k] for r in runs), "max": max(r[k] for r in runs)} for k in (runs[0] if runs else {})}
    return out


def host_call(eng, values):
    """lo_value_counts_f64_host as the host route calls it: the valid values packed, copied and counted."""
    from learningorchestra_b200 import _native as N
    x = np.ascontiguousarray(values, np.float64)
    cap = max(x.size, 1)
    keys, counts, nd, t = np.empty(cap), np.empty(cap, np.uint64), C.c_int64(), N.HostTiming()
    N.check(eng._lib.lo_value_counts_f64_host(eng._ctx, x.ctypes.data_as(C.c_void_p), x.size, keys.ctypes.data_as(C.c_void_p),
                                              counts.ctypes.data_as(C.c_void_p), cap, C.byref(nd), C.byref(t)))
    return t.kernel_ms, int(nd.value)


def field_numbers(eng, db, name, f, reps):
    from learningorchestra_b200 import utils
    from learningorchestra_b200.histogram import Histogram
    col = db.column(name, f)
    r = {"rows": len(col)}
    k = []

    def host():
        kk, d = host_call(eng, col.values[col.valid])
        k.append(kk)
        return d
    r["host_call_ms"], nd = best(host, reps)
    r["host_kernel_ms"] = min(k)
    eng.resident.clear()
    with eng.resident.lease(db, name, (), numbers=[f]) as data:
        j = data.column[f]
        t, kr = {}, []

        def resident():
            out = eng.value_counts_column(data.table, j, timing=t)
            kr.append(t["kernel_ms"])
            return out
        r["resident_call_ms"], (keys, counts) = best(resident, reps)
    r["resident_kernel_ms"] = min(kr)
    r["resident_h2d_bytes"] = t["h2d_bytes"]
    r["groups"] = int(keys.size)
    assert int(counts.sum()) == len(col)
    r["GBps_slab"] = len(col) * 8 / 1e9 / (r["resident_kernel_ms"] / 1e3)
    h = Histogram(db, utils.HistogramMetadata(db), eng)
    eng.resident.clear()
    for label in ("cold", "warm"):
        t0 = time.perf_counter()
        h.file_processing(name, f"{name}_{f}_{label}", [f])
        r[f"histograms_{label}_ms"] = (time.perf_counter() - t0) * 1e3
    return r


def synthetic(rows, seed):
    rng = np.random.default_rng(seed)
    nan_null = rng.integers(0, 1000, rows).astype(np.float64) * 0.5
    nan_null[rng.random(rows) < 0.01] = np.nan
    valid = rng.random(rows) >= 0.01
    nan_null[~valid] = np.nan
    from learningorchestra_b200.column_store import NumberColumn
    return {"three": NumberColumn((np.arange(rows) % 3).astype(np.float64)),
            "k20000": NumberColumn(rng.integers(0, 20_000, rows).astype(np.float64)),
            "distinct": NumberColumn(rng.permutation(rows).astype(np.float64)),
            "constant": NumberColumn(np.full(rows, 7.25)),
            "nan_null": NumberColumn(nan_null, valid)}


def sharded(rows, reps):
    from learningorchestra_b200 import _native as N
    from learningorchestra_b200.sharding import ShardedEngine, merge_value_counts
    n = C.c_int()
    N.check(N.load().lo_device_count(C.byref(n)))
    if n.value < 2:
        return "not measured (one visible GPU)"
    x = np.random.default_rng(3).permutation(rows).astype(np.float64)
    with ShardedEngine.local() as sh:
        t = sh.table_from_numpy([x])
        parts = []
        count_ms, _ = best(lambda: parts.append([e.value_counts_column(s, 0) for e, s in zip(sh.engines, t.shards)]), reps)
        merge_ms, (keys, counts) = best(lambda: merge_value_counts(parts[-1]), reps)
        total_ms, _ = best(lambda: sh.value_counts_column(t, 0), reps)
        assert keys.size == rows
        t.free()
        return {"gpus": sh.nlocal, "shards_counted_one_after_another_ms": count_ms, "host_merge_ms": merge_ms,
                "value_counts_column_ms": total_ms}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--titanic-mb", type=int, default=1024)
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ab", nargs="*", default=[])
    ap.add_argument("--seed", type=int, default=20261016)
    ap.add_argument("--out")
    a = ap.parse_args()
    results = {"card": card()}
    print("card:", results["card"], flush=True)
    if a.ab:
        results["ab_host_kernel_ms"] = ab(a.ab, a.rows, a.reps)
        print("ab", json.dumps(results["ab_host_kernel_ms"]), flush=True)
    from learningorchestra_b200 import utils
    from learningorchestra_b200.column_store import ColumnarDatabase
    from learningorchestra_b200.data_type_update import DataType
    from learningorchestra_b200.engine import Engine
    eng = Engine(0)
    fields = {}
    if a.titanic_mb:
        from csv_bench import titanic_body
        body = titanic_body(a.seed, a.titanic_mb)
        db = ColumnarDatabase()
        with tempfile.TemporaryDirectory() as tmp:
            path = Path(tmp) / "titanic.csv"
            path.write_bytes(body)
            results["body_bytes"] = len(body)
            del body
            db.ingest_csv("titanic", str(path), engine=eng)
        job = DataType(db, utils.DataTypeMetadata(db), eng)
        job.convert_existent_file("titanic", {f: "number" for f in NUMBER_FIELDS})
        job.wait()
        for f in NUMBER_FIELDS:
            fields[f] = field_numbers(eng, db, "titanic", f, a.reps)
            print(f, json.dumps(fields[f]), flush=True)
    sdb = ColumnarDatabase()
    sdb.ingest_columns("synthetic", synthetic(a.rows, a.seed))
    for f in ("three", "k20000", "distinct", "constant", "nan_null"):
        fields[f] = field_numbers(eng, sdb, "synthetic", f, a.reps)
        print(f, json.dumps(fields[f]), flush=True)
    results["fields"] = fields
    eng.close()
    results["sharded_distinct"] = sharded(a.rows, a.reps)
    print("sharded", json.dumps(results["sharded_distinct"]), flush=True)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
