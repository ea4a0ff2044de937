"""Device CSV reader (lo_csv_read_host) against pyarrow and the reference's own reader, on bodies generated from a seed.

    python scripts/csv_bench.py [--seed S] [--titanic-mb 1024] [--mnist-mb 256] [--reviews-mb 256] [--big-gb N]
                                [--small-window-mb 16] [--out FILE]

Bodies: Titanic-shaped rows (12 text columns with quoted names), MNIST as CSV (785 integer columns) and review-like
text (quoted commas, "" pairs, multi-line fields, non-ASCII text).  For each body, in one run: kernel_ms; the whole
call with pinned and with pageable input and GB/s of body for each; pyarrow.csv.read_csv (its thread count); the oracle
reader single-threaded on a sample; ingest_csv end to end with and without an engine; a full parity check of the
columns against the oracle.  The streaming reader (Engine.read_csv_stream, lo_csv_stream_*) from a file, at the default
window and at a smaller one: call time, GB/s of body, the peak device bytes it reports and a check that its columns
equal read_csv_host's; ingest_csv with an engine goes through the stream.  --big-gb N writes a body of N GB to disk,
records the single-shot reader's LO_ERR_NOMEM on it and streams it (skipped, with the reason, when the host has too
little RAM for its columns).  The card's name and power limit are printed with the numbers.
"""
from __future__ import annotations

import argparse
import io
import json
import shutil
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def _tile(header: bytes, rows: bytes, mb: int) -> bytes:
    reps = max(1, (mb << 20) // max(len(rows), 1))
    return header + rows * reps


def titanic_body(seed, mb):
    from oracle.rsem import TITANIC_HEADERS, titanic_shaped_rows
    import csv
    buf = io.StringIO()
    w = csv.writer(buf, lineterminator="\n")
    w.writerows(titanic_shaped_rows(20000, seed))
    return _tile((",".join(TITANIC_HEADERS) + "\n").encode(), buf.getvalue().encode(), mb)


def mnist_body(seed, mb):
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (2000, 785)) * (rng.random((2000, 785)) < 0.2)
    img[:, 0] = rng.integers(0, 10, 2000)
    rows = "\n".join(",".join(map(str, r)) for r in img.tolist()) + "\n"
    header = "label," + ",".join(f"pixel{i}" for i in range(784)) + "\n"
    return _tile(header.encode(), rows.encode(), mb)


def reviews_body(seed, mb):
    rng = np.random.default_rng(seed)
    words = ["good", "bad", "ok, fine", 'said "wow"', "naïve", "café", "日本語", "emoji 😀", "line\nbreak", "€5"]
    out = []
    for i in range(20000):
        text = " ".join(words[j] for j in rng.integers(0, len(words), rng.integers(3, 40)))
        out.append(f'{i},{rng.integers(1, 6)},"{text.replace(chr(34), chr(34) * 2)}"\r\n')
    return _tile(b"id,stars,review\r\n", "".join(out).encode(), mb)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:            # the numbers are still printed, marked with what is missing
        return f"unknown ({e})"


def timed(fn, reps=3):
    best = None
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        dt = time.perf_counter() - t0
        best = dt if best is None else min(best, dt)
    return best, out


def same_columns(stream_cols, chars, offsets, first=1):
    """The stream's Arrow columns == read_csv_host's chars / offsets (data rows from record `first`)."""
    for c, col in enumerate(stream_cols):
        off = np.frombuffer(col.buffers()[1], np.int64, count=len(col) + 1, offset=col.offset * 8)
        data = np.frombuffer(col.buffers()[2], np.uint8, count=int(off[-1]))
        ref = offsets[c, first:]
        if len(col) != ref.size - 1 or not np.array_equal(off - off[0], ref - ref[0]):
            return False
        if not np.array_equal(data[off[0]:off[-1]], chars[ref[0]:ref[-1]]):
            return False
    return True


def stream_numbers(eng, path, gb, window):
    t = {}
    t0 = time.perf_counter()
    header, nrows, cols, failure = eng.read_csv_stream(str(path), window, t)
    dt = time.perf_counter() - t0
    return {"call_ms": dt * 1e3, "GBps": gb / dt, "kernel_ms": t["kernel_ms"], "windows": t["windows"],
            "peak_device_bytes": t["peak_device_bytes"]}, (header, nrows, cols, failure)


def big_body(eng, a, tmp, results):
    """A body larger than the single-shot reader's ceiling, written to disk in blocks of the reviews body (long text
    cells, so the host can hold the columns of a body that large) and streamed."""
    import os
    from learningorchestra_b200 import _native as N
    block = reviews_body(a.seed, 64)
    header_len = block.index(b"\n") + 1
    rows = block[header_len:]
    reps = max(1, int(a.big_gb * 1e9) // len(rows))
    size = header_len + reps * len(rows)
    r = {"bytes": size}
    # the columns need about the body's text plus 8 bytes per cell on the host, twice while they grow
    cells = rows.count(b"\n") * reps * 3
    need = 2 * (size + 8 * cells)
    avail = os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    disk = shutil.disk_usage(tmp).free
    if need > avail or size > disk:
        r["skipped"] = (f"host has {avail / 1e9:.1f} GB of free RAM and {disk / 1e9:.1f} GB of disk; the body takes "
                        f"{size / 1e9:.1f} GB and its columns about {need / 1e9:.1f} GB")
        print("big", json.dumps(r), flush=True)
        results["bodies"]["big"] = r
        return
    path = Path(tmp) / "big.csv"
    with open(path, "wb") as f:
        f.write(block[:header_len])
        for _ in range(reps):
            f.write(rows)
    del block, rows
    try:
        body = np.memmap(path, dtype=np.uint8, mode="r")      # the single-shot call checks HBM before reading it
        t0 = time.perf_counter()
        try:
            eng.read_csv_host(body)
            r["single_shot"] = "ok"
        except N.LoexecError as e:
            r["single_shot"] = f"{e} ({(time.perf_counter() - t0) * 1e3:.0f} ms)"
        del body
        num, (header, nrows, cols, failure) = stream_numbers(eng, path, size / 1e9, None)
        r.update(stream=num, rows=nrows, failure=failure)
        del cols
    finally:
        path.unlink()
    results["bodies"]["big"] = r
    print("big", json.dumps(r), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seed", type=int, default=20261016)
    ap.add_argument("--titanic-mb", type=int, default=1024)
    ap.add_argument("--mnist-mb", type=int, default=256)
    ap.add_argument("--reviews-mb", type=int, default=256)
    ap.add_argument("--big-gb", type=float, default=0)
    ap.add_argument("--small-window-mb", type=int, default=16)
    ap.add_argument("--out")
    a = ap.parse_args()
    import pyarrow as pa
    import pyarrow.csv as pacsv

    from csv_oracle import csv_reference_rows
    from learningorchestra_b200.build import build_all
    from learningorchestra_b200.column_store import ColumnarDatabase
    from learningorchestra_b200.engine import Engine
    build_all()
    eng = Engine(0)
    results = {"card": card(), "pyarrow_threads": pa.cpu_count(), "bodies": {}}
    print("card:", results["card"], flush=True)
    tmp = tempfile.mkdtemp()
    for name, make, mb in (("titanic", titanic_body, a.titanic_mb), ("mnist", mnist_body, a.mnist_mb),
                           ("reviews", reviews_body, a.reviews_mb)):
        body = make(a.seed, mb)
        gb = len(body) / 1e9
        r = {"bytes": len(body)}
        host = np.frombuffer(body, np.uint8)
        pinned = eng.pinned_empty(len(body), np.uint8)
        pinned[:] = host
        eng.read_csv_host(host[: 1 << 20])                      # warm-up
        t = {}
        for label, buf in (("pinned", pinned), ("pageable", host)):
            dt, out = timed(lambda: eng.read_csv_host(buf, t))
            r[f"call_{label}_ms"] = dt * 1e3
            r[f"call_{label}_GBps"] = gb / dt
            r["kernel_ms"] = t["kernel_ms"]
        header, nrows, chars, offsets, failure = out
        r.update(rows=nrows, cols=len(header), failure=failure)
        dt, _ = timed(lambda: pacsv.read_csv(io.BytesIO(body), parse_options=pacsv.ParseOptions(newlines_in_values=True),
                                             convert_options=pacsv.ConvertOptions(
            column_types={h: pa.large_string() for h in header}, strings_can_be_null=False)), reps=1)
        r["pyarrow_ms"] = dt * 1e3
        r["pyarrow_GBps"] = gb / dt
        sample = body[: 16 << 20]
        sample = sample[: sample.rfind(b"\n") + 1]
        dt, _ = timed(lambda: csv_reference_rows(sample), reps=1)
        r["oracle_sample_bytes"] = len(sample)
        r["oracle_GBps"] = len(sample) / 1e9 / dt
        path = Path(tmp) / f"{name}.csv"
        path.write_bytes(body)
        stream_ok = True
        for label, window in (("stream", None), ("stream_small", a.small_window_mb << 20)):
            eng.read_csv_stream(str(path), window)                       # warm-up: pinned staging, the pool
            r[label], (sh, sn, scols, sfail) = stream_numbers(eng, path, gb, window)
            stream_ok = stream_ok and sh == header and sn == nrows and sfail == failure and \
                same_columns(scols, chars, offsets)
            del scols
        r["stream_equals_single_shot"] = bool(stream_ok)
        # ingest_csv with an engine streams the file (Engine.read_csv_stream)
        for label, e in (("ingest_engine_ms", eng), ("ingest_pyarrow_ms", None)):
            db = ColumnarDatabase()
            t0 = time.perf_counter()
            db.ingest_csv(name, str(path), engine=e)
            r[label] = (time.perf_counter() - t0) * 1e3
            del db
        path.unlink()
        # full parity: every cell of every row against the reference's reader
        eh, erows, efail = csv_reference_rows(body)
        raw = chars.tobytes()
        ok = eh == header and efail is None and failure is None and len(erows) == nrows
        for c in range(len(header)) if ok else ():
            col = [raw[offsets[c, i]:offsets[c, i + 1]].decode() for i in range(1, nrows + 1)]
            ok = ok and col == [row[c] for row in erows]
        r["parity"] = bool(ok and stream_ok)
        del erows, pinned
        results["bodies"][name] = r
        print(name, json.dumps(r), flush=True)
    if a.big_gb:
        big_body(eng, a, tmp, results)
    eng.close()
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(results, indent=1))
    if not all(b.get("parity", True) for b in results["bodies"].values()):
        sys.exit("parity FAILED")


if __name__ == "__main__":
    main()
