"""The "string" cast's number -> text formatter (lo_format_number_host: k_format_number_len, a CUB scan of the lengths,
k_format_number_write) on 8 M cells: whole-call time with pageable and with pinned host buffers, the kernels' own device
time (lo_host_timing.kernel_ms), the same cells through Python's repr() / str(int) on the host, and the executor-level
"string" cast of a 10 M-row columnar collection with the host str() path (no device formatter) and with the GPU.

The kernel is bound by digit arithmetic (128-bit products, divisions by 10), not by HBM, so no share of HBM peak is
reported.  Prints the results as JSON, with the card's name and power limit read in the same run, and writes them to
--out (default format_bench.json in the current directory)."""
import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np

from learningorchestra_b200 import _native as N
from learningorchestra_b200 import utils
from learningorchestra_b200.column_store import ColumnarDatabase, NumberColumn
from learningorchestra_b200.data_type_update import DataType
from learningorchestra_b200.engine import Engine

MIX = {"random_bits": 0.25, "fixed_6_decimals": 0.35, "int_below_2^53": 0.30, "int_2^64_to_1e308": 0.02, "null": 0.08}


def cells(n, seed):
    """(values, status): what the "number" cast leaves in a column, drawn in the MIX proportions."""
    rng = np.random.default_rng(seed)
    kind = rng.choice(len(MIX), size=n, p=list(MIX.values()))
    v = rng.integers(0, 2 ** 64, size=n, dtype=np.uint64).view(np.float64).copy()
    m = kind == 1
    v[m] = np.round(rng.uniform(-1e4, 1e4, m.sum()), 6)
    m = kind == 2
    v[m] = rng.integers(-10 ** 9, 10 ** 9, m.sum()).astype(np.float64)
    m = kind == 3
    v[m] = np.floor(rng.uniform(1.0, 10.0, m.sum()) * 10.0 ** rng.integers(20, 308, m.sum()))
    with np.errstate(invalid="ignore"):
        integral = np.isfinite(v) & (v == np.floor(v))     # random bit patterns of |v| >= 2^52 are integral too
    status = np.where(integral, N.LO_NUM_INTEGER, N.LO_NUM_FLOAT).astype(np.uint8)
    status[kind == 4] = N.LO_NUM_EMPTY
    return v, status


def best(fn, n=5):
    fn()
    runs = []
    for _ in range(n):
        t0 = time.perf_counter()
        k = fn()
        runs.append((time.perf_counter() - t0, k))
    return min(runs)


def main():
    ap = argparse.ArgumentParser(description="GPU number -> text formatter: call, kernel and executor-level timings")
    ap.add_argument("--out", type=Path, default=Path("format_bench.json"), help="where the JSON result is written")
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    eng = Engine(0)
    res = {"gpu": smi, "mix": MIX}

    n = 8_000_000
    values, status = cells(n, 20261015)
    chars, offsets = eng.format_number_host(values, status)
    cap = int(offsets[-1])

    def call(v, s, off, ch):
        t = N.HostTiming()
        N.check(eng._lib.lo_format_number_host(eng._ctx, v.ctypes.data_as(C.c_void_p), s.ctypes.data_as(C.c_void_p), n,
                                               off.ctypes.data_as(C.c_void_p), ch.ctypes.data_as(C.c_void_p), cap, C.byref(t)))
        return t.kernel_ms

    off_p, ch_p = np.empty(n + 1, np.int64), np.empty(cap, np.uint8)
    t_page, k_page = best(lambda: call(values, status, off_p, ch_p))
    assert np.array_equal(off_p, offsets) and np.array_equal(ch_p, chars)
    pv, ps = eng.pinned_empty(n, np.float64), eng.pinned_empty(n, np.uint8)
    pv[...] = values
    ps[...] = status
    po, pc = eng.pinned_empty(n + 1, np.int64), eng.pinned_empty(cap, np.uint8)
    t_pin, k_pin = best(lambda: call(pv, ps, po, pc))
    assert np.array_equal(po, offsets) and np.array_equal(pc, chars)
    k = min(k_page, k_pin)
    res["format_number_host"] = {
        "cells": n, "text_bytes": cap,
        "share_float": float(np.mean(status == N.LO_NUM_FLOAT)), "share_integer": float(np.mean(status == N.LO_NUM_INTEGER)),
        "share_integer_ge_2^64": float(np.mean((status == N.LO_NUM_INTEGER) & (np.abs(values) >= 2.0 ** 64))), "host_bytes_moved": n * 9 + (n + 1) * 8 + cap,
        "call_s_pageable": t_page, "Mcells_per_s_pageable": n / t_page / 1e6,
        "call_s_pinned": t_pin, "Mcells_per_s_pinned": n / t_pin / 1e6,
        "kernel_ms": k, "kernel_Mcells_per_s": n / k / 1e3}

    # the same cells through Python, the way the host path formats them
    t0 = time.perf_counter()
    text = [repr(x) if s == N.LO_NUM_FLOAT else str(int(x)) if s == N.LO_NUM_INTEGER else ""
            for x, s in zip(values.tolist(), status.tolist())]
    t_py = time.perf_counter() - t0
    assert "".join(text).encode() == chars.tobytes()
    res["python_repr_loop"] = {"cells": n, "s": t_py, "Mcells_per_s": n / t_py / 1e6}

    # executor level: PATCH /fieldTypes "string" on a 10 M-row number column, host str() vs the GPU
    rows = 10_000_000
    v10, s10 = cells(rows, 7)
    col = NumberColumn(np.where(s10 == N.LO_NUM_EMPTY, np.nan, v10), s10 != N.LO_NUM_EMPTY, s10 == N.LO_NUM_INTEGER)
    out = {}
    for label, engine in (("host_str", None), ("gpu", eng)):
        db = ColumnarDatabase()
        db.ingest_columns("big", {"x": col})
        job = DataType(db, utils.DataTypeMetadata(db), engine=engine)
        t0 = time.perf_counter()
        job.convert_existent_file("big", {"x": "string"})
        job.wait(3600)
        out[label] = (time.perf_counter() - t0, db.column("big", "x").arr)
    assert out["host_str"][1].equals(out["gpu"][1])
    res["datatype_string_cast_10M_rows"] = {"rows": rows, "host_str_s": out["host_str"][0], "gpu_s": out["gpu"][0],
                                            "speedup": out["host_str"][0] / out["gpu"][0]}
    eng.close()
    print(json.dumps(res, indent=1))
    args.out.parent.mkdir(parents=True, exist_ok=True)
    args.out.write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
