"""`$group` of text columns: the host route (lo_value_counts_str_host: pack, copy, count) against the resident route
(lo_text_upload once, then lo_value_counts_text per request), and /histograms end to end.

    python scripts/value_counts_bench.py [--titanic-mb 1024] [--distinct-rows 10000000] [--reps 5] [--out FILE]
                                         [--ab LIB.so ...] [--ab-rows 10000000]

Input: a Titanic-shaped CSV body (csv_bench.titanic_body) ingested with the engine (POST /files' reader), plus an
all-distinct and a constant column of --distinct-rows cells.  Per field: the host call's time and kernel_ms, the
upload's time, the resident call's time and kernel_ms, GB/s of chars + offsets over the resident kernel_ms, and the
/histograms wall time of one request for that field, cold (the column uploaded by the request) and warm (resident).
--ab: host-route kernel_ms of the given builds of libloexec.so on synthetic columns (3 values, 20 000 values,
all distinct, constant), each build in a fresh process, alternating, --reps rounds: the parent commit's library against
this one measures the shared-memory stage alone.  The card's name, power limit and max SM clock are printed with the
numbers (read-only nvidia-smi query).
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
sys.path.insert(0, str(ROOT / "tests"))

AB_CHILD = r'''
import ctypes as C, json, sys
import numpy as np
sys.path.insert(0, %r)
from learningorchestra_b200 import _native as N
from learningorchestra_b200.engine import Engine
n, reps = int(sys.argv[1]), int(sys.argv[2])
eng = Engine(0)
lib = eng._lib
out = {}
for name, card in (("three", 3), ("k20000", 20000), ("distinct", n), ("constant", 1)):
    codes = np.arange(n, dtype=np.int64) %% card          # cell i: its code as 8 decimal digits
    chars = np.ascontiguousarray(((codes[:, None] // 10 ** np.arange(7, -1, -1)) %% 10 + 48).astype(np.uint8).ravel())
    off = np.arange(n + 1, dtype=np.int64) * 8
    rows, counts, nd = np.empty(card, np.int64), np.empty(card, np.uint64), C.c_int64()
    ks = []
    for r in range(reps + 1):
        t = N.HostTiming()
        N.check(lib.lo_value_counts_str_host(eng._ctx, chars.ctypes.data_as(C.c_void_p), off.ctypes.data_as(C.c_void_p), n,
                                             rows.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p), card,
                                             C.byref(nd), C.byref(t)))
        assert nd.value == card and int(counts.sum()) == n
        if r:
            ks.append(t.kernel_ms)
    out[name] = sorted(ks)[len(ks) // 2]
print(json.dumps(out))
''' % str(ROOT)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:            # the numbers are still printed, marked with what is missing
        return f"unknown ({e})"


def best(fn, reps):
    ts, out = [], None
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        ts.append(time.perf_counter() - t0)
    return min(ts) * 1e3, out


def host_call(eng, arr):
    """lo_value_counts_str_host as the host route calls it: non-null cells packed, copied and counted."""
    from learningorchestra_b200 import _native as N
    from learningorchestra_b200.column_store import TextColumn
    a = arr.drop_null() if arr.null_count else arr
    chars, offsets, _ = TextColumn(a).packed()
    n = len(a)
    cap = n
    rows, counts, nd, t = np.empty(cap, np.int64), np.empty(cap, np.uint64), C.c_int64(), N.HostTiming()
    N.check(eng._lib.lo_value_counts_str_host(eng._ctx, chars.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p),
                                              n, rows.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p), cap,
                                              C.byref(nd), C.byref(t)))
    return t.kernel_ms, int(nd.value)


def field_numbers(eng, db, name, f, arr, reps):
    from learningorchestra_b200 import utils
    from learningorchestra_b200.histogram import Histogram
    r = {"rows": len(arr), "bytes": int(arr.buffers()[2].size) if arr.buffers()[2] is not None else 0}
    k, nd = [], 0

    def host():
        kk, d = host_call(eng, arr)
        k.append(kk)
        return d
    r["host_call_ms"], nd = best(host, reps)
    r["host_kernel_ms"] = min(k)
    up = {}
    r["upload_ms"], text = best(lambda: eng.text(arr, timing=up), 1)
    t, kr = {}, []

    def resident():
        out = eng.value_counts_text(text, timing=t)
        kr.append(t["kernel_ms"])
        return out
    r["resident_call_ms"], (rep, counts) = best(resident, reps)
    r["resident_kernel_ms"] = min(kr)
    r["resident_h2d_bytes"] = t["h2d_bytes"]
    r["groups"] = int(len(rep))
    assert len(rep) == nd and int(counts.sum()) == len(arr) - arr.null_count
    r["GBps_chars_offsets"] = (r["bytes"] + 8 * (len(arr) + 1)) / 1e9 / (r["resident_kernel_ms"] / 1e3)
    text.free()
    if db is not None:
        h = Histogram(db, utils.HistogramMetadata(db), eng)
        eng.resident.clear()
        for label in ("cold", "warm"):
            t0 = time.perf_counter()
            h.file_processing(name, f"{name}_{f}_{label}", [f])
            r[f"histograms_{label}_ms"] = (time.perf_counter() - t0) * 1e3
    return r


def ab(libs, rows, reps):
    res = {lib: [] for lib in libs}
    for rnd in range(reps):
        for lib in libs:
            env = dict(os.environ, LOEXEC_LIB=lib, LOEXEC_LAX="1")
            p = subprocess.run([sys.executable, "-c", AB_CHILD, str(rows), "3"], env=env, capture_output=True, text=True)
            line = [x for x in p.stdout.splitlines() if x.startswith("{")]
            if not line:
                print("FAILED", lib, p.stderr[-800:], flush=True)
                continue
            res[lib].append(json.loads(line[-1]))
            print("ab", rnd, lib, line[-1], flush=True)
    summary = {}
    for lib, runs in res.items():
        summary[lib] = {k: sorted(r[k] for r in runs)[len(runs) // 2] for k in (runs[0] if runs else {})}
    return summary


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--titanic-mb", type=int, default=1024)
    ap.add_argument("--distinct-rows", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ab", nargs="*", default=[])
    ap.add_argument("--ab-rows", type=int, default=10_000_000)
    ap.add_argument("--seed", type=int, default=20261016)
    ap.add_argument("--out")
    a = ap.parse_args()
    results = {"card": card()}
    print("card:", results["card"], flush=True)
    if a.ab:
        results["ab_host_kernel_ms"] = ab(a.ab, a.ab_rows, a.reps)
        print("ab", json.dumps(results["ab_host_kernel_ms"]), flush=True)
    if a.titanic_mb:
        import pyarrow as pa
        from csv_bench import titanic_body
        from learningorchestra_b200.column_store import ColumnarDatabase
        from learningorchestra_b200.engine import Engine
        eng = Engine(0)
        body = titanic_body(a.seed, a.titanic_mb)
        with tempfile.TemporaryDirectory() as tmp:
            path = Path(tmp) / "titanic.csv"
            path.write_bytes(body)
            results["body_bytes"] = len(body)
            del body
            db = ColumnarDatabase()
            db.ingest_csv("titanic", str(path), engine=eng)
        fields = {}
        for f in ("Embarked", "Sex", "Pclass", "Name", "Ticket"):
            fields[f] = field_numbers(eng, db, "titanic", f, db.column("titanic", f).arr, a.reps)
            print(f, json.dumps(fields[f]), flush=True)
        m = a.distinct_rows
        for f, cells in (("distinct", np.char.add("d", np.arange(m).astype("U10")).astype(object)),
                         ("constant", np.full(m, "S", dtype=object))):
            fields[f] = field_numbers(eng, None, None, f, pa.array(cells, type=pa.large_string()), a.reps)
            print(f, json.dumps(fields[f]), flush=True)
        results["fields"] = fields
        eng.close()
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
