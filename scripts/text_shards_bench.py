"""`$group` of a text column cut into row-range shards (lo_value_counts_text_shards) against the whole column
(lo_value_counts_text), and the share of the call the root's merge takes.

    python scripts/text_shards_bench.py [--titanic-mb 256] [--rows 10000000] [--pieces 2 4 8] [--reps 7] [--out FILE]

Columns: the text fields of a Titanic-shaped CSV body (csv_bench.titanic_body, read by the engine as POST /files does),
plus a constant and an all-distinct column of --rows cells.  On device 0, each column is counted whole and as 2, 4 and
8 pieces uploaded to the SAME device, cut where ShardedEngine cuts them (sharding.all_shard_bounds).  Per column and
cut: the median call time over --reps calls (host clock around a call that ends in a synchronise), the median
kernel_ms (the whole column's count; the shards' root merge), and the merge's share of the call.  The pieces' groups
are checked against the whole column's.  With more than one visible GPU, the same columns are counted by a
ShardedEngine over every device (one piece per device); with one, multi-device time is reported as not measured.
The card's name, power limit and max SM clock are printed with the numbers (read-only nvidia-smi query).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))

from value_counts_bench import card  # noqa: E402


def median(xs):
    return sorted(xs)[len(xs) // 2]


def groups(arr, rows, counts):
    """{key: count} of a call's groups (keys read from the whole column at the representative rows)."""
    import pyarrow as pa
    keys = arr.take(pa.array(np.asarray(rows, np.int64))).to_pylist()
    return dict(zip(keys, (int(c) for c in counts)))


def timed(call, reps):
    """(median call ms, median kernel_ms, last output) of ``call(timing_dict)``, after one call that is not timed."""
    ms, kms, out = [], [], call({})
    for _ in range(reps):
        t = {}
        t0 = time.perf_counter()
        out = call(t)
        ms.append((time.perf_counter() - t0) * 1e3)
        kms.append(t["kernel_ms"])
    return median(ms), median(kms), out


def shards_call(eng, pieces, row0, n, timing):
    from learningorchestra_b200.engine import _value_counts
    k = len(pieces)
    handles = (C.c_void_p * k)(*[p._h for p in pieces])
    r0 = (C.c_int64 * k)(*row0)
    return _value_counts(lambda rows, counts, cap, nd, t: eng._lib.lo_value_counts_text_shards(
        eng._ctx, handles, r0, k, rows, counts, cap, nd, t), n, np.int64, timing)


def column_numbers(eng, arr, cuts, reps):
    from learningorchestra_b200.sharding import all_shard_bounds
    n = len(arr) - arr.null_count
    whole = eng.text(arr)
    r = {"rows": len(arr)}
    r["whole_call_ms"], r["whole_kernel_ms"], (rep, cnt) = timed(lambda t: eng.value_counts_text(whole, timing=t), reps)
    r["groups"] = int(len(rep))
    exact = len(rep) <= 1_000_000                  # above that, compare the group sizes only (a dict of every key is slow)
    want = groups(arr, rep, cnt) if exact else np.sort(cnt)
    whole.free()
    for w in cuts:
        bounds = all_shard_bounds(len(arr), w)
        pieces = [eng.text(arr.slice(b, e - b)) for b, e in bounds]
        ms, kms, (rows, counts) = timed(lambda t: shards_call(eng, pieces, [b for b, _ in bounds], n, t), reps)
        for p in pieces:
            p.free()
        same = groups(arr, rows, counts) == want if exact else \
            (np.array_equal(np.sort(counts), want) and np.unique(rows).size == rows.size)
        assert same, f"{w} pieces: the groups differ from the whole column's"
        r[f"p{w}"] = {"call_ms": ms, "merge_kernel_ms": kms, "merge_share": kms / ms}
    return r


def sharded_numbers(cols, reps):
    from learningorchestra_b200.sharding import ShardedEngine
    out = {}
    with ShardedEngine.local() as sh:
        out["devices"] = sh.nlocal
        for name, arr in cols.items():
            text = sh.text(arr)
            ms, kms, _ = timed(lambda t: sh.value_counts_text(text, timing=t), reps)
            text.free()
            out[name] = {"call_ms": ms, "merge_kernel_ms": kms, "merge_share": kms / ms}
            print("devices", name, json.dumps(out[name]), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--titanic-mb", type=int, default=256)
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--pieces", type=int, nargs="*", default=[2, 4, 8])
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--seed", type=int, default=20261017)
    ap.add_argument("--out")
    a = ap.parse_args()
    import pyarrow as pa
    from csv_bench import titanic_body
    from learningorchestra_b200 import _native as N
    from learningorchestra_b200.column_store import ColumnarDatabase
    from learningorchestra_b200.engine import Engine
    results = {"card": card()}
    print("card:", results["card"], flush=True)
    eng = Engine(0)
    cols = {}
    if a.titanic_mb:
        body = titanic_body(a.seed, a.titanic_mb)
        with tempfile.TemporaryDirectory() as tmp:
            path = Path(tmp) / "titanic.csv"
            path.write_bytes(body)
            results["body_bytes"] = len(body)
            del body
            db = ColumnarDatabase()
            db.ingest_csv("titanic", str(path), engine=eng)
        for f in ("Embarked", "Sex", "Pclass", "Name", "Ticket", "Cabin"):
            cols[f] = db.column("titanic", f).arr
    if a.rows:
        cols["constant"] = pa.array(np.full(a.rows, "S", dtype=object), type=pa.large_string())
        cols["distinct"] = pa.array(np.char.add("d", np.arange(a.rows).astype("U10")).astype(object), type=pa.large_string())
    fields = {}
    for name, arr in cols.items():
        fields[name] = column_numbers(eng, arr, a.pieces, a.reps)
        print(name, json.dumps(fields[name]), flush=True)
    results["one_device"] = fields
    eng.close()
    n = C.c_int()
    N.check(N.load().lo_device_count(C.byref(n)))
    if n.value > 1:
        results["devices"] = sharded_numbers(cols, a.reps)
    else:
        results["devices"] = "not measured: one visible GPU"
        print("multi-device time: not measured (one visible GPU)", flush=True)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
