"""POST /models on the GPU: wall time per phase of one builder job over a synthetic train and test dataset, and the two
builder kernels against host or torch compositions.

  python scripts/builder_bench.py [--rows 10000000] [--test-rows 1000000] [--repeat 2] [--out results.json]

Prints one JSON line; ``--out`` also writes it to that file.

* The job: a train dataset of ``--rows`` rows x 20 number fields + 2 text fields + a 0/1 label, and a test dataset of
  ``--test-rows`` rows without the label, both in a ColumnarDatabase, through ``POST /models`` with all five classifiers
  and a modelingCode that assembles, splits 0.8 / 0.2 and skips invalid rows.  Wall seconds per phase: frames (both
  datasets resident and coded), modelingCode (assemble + split), and each classifier's fit, evaluate, transform and
  write-back (``Builder.timings``).
* ``lo_random_split`` against a torch composition that draws the same u in int64 arithmetic and splits by boolean
  indexing, alternated, outputs compared bit for bit; its kernel time and its bytes over that time.
* ``lo_text_codes_in`` of the test set's text column against ``pyarrow.compute.index_in`` on the host, alternated, codes
  compared.
* The card's name, power limit and SM clock, read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

K, WORDS = 20, 40
CODE = """
fields = [f"f{j}" for j in range(20)] + ["t0", "t1"]
assembled = training_df.features(fields, label="label", handle_invalid="skip")
features_training, features_evaluation = assembled.random_split([0.8, 0.2], seed=7)
features_testing = testing_df.features(fields, handle_invalid="skip")
"""


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def dataset(db, name, n, seed, label):
    import pyarrow as pa
    from learningorchestra_b200.column_store import NumberColumn, TextColumn
    rng = np.random.default_rng(seed)
    x = rng.random(size=(K, n)) * 10.0                   # >= 0: NaiveBayes refuses negative features
    cols = {f"f{j}": NumberColumn(x[j]) for j in range(K)}
    words = pa.array([f"word{i}" for i in range(WORDS)] + ["unseen"], type=pa.large_string())
    for t in range(2):
        cols[f"t{t}"] = TextColumn(words.take(pa.array(rng.integers(0, WORDS + (0 if label else 1), n))))
    if label:
        cols["label"] = NumberColumn((x[0] + x[1] + rng.normal(size=n) > 10.0).astype(np.float64))
    db.ingest_columns(name, cols)


def torch_split(x, y, ids, bounds, seed):
    """The same draw in int64 arithmetic (wrapping multiplies, logical shifts by masking) and boolean indexing."""
    import torch
    m64 = lambda v: torch.tensor(np.array(v, np.uint64).view(np.int64), device=x.device)

    def shr(z, s):
        return (z >> s) & ((1 << (64 - s)) - 1)

    def mix(z):
        z = z + m64(0x9E3779B97F4A7C15)
        z = (z ^ shr(z, 30)) * m64(0xBF58476D1CE4E5B9)
        z = (z ^ shr(z, 27)) * m64(0x94D049BB133111EB)
        return z ^ shr(z, 31)
    key = mix(m64(~seed & 0xFFFFFFFFFFFFFFFF))
    u = shr(mix(ids ^ key), 11).to(torch.float64) * 2.0 ** -53
    out = []
    for s in range(len(bounds) - 1):
        keep = (u >= float(bounds[s])) & (u < float(bounds[s + 1]))
        out.append((x[keep], y[keep], torch.nonzero(keep).flatten()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--test-rows", type=int, default=1_000_000)
    ap.add_argument("--repeat", type=int, default=2)
    ap.add_argument("--out", default=None, help="a file to write the JSON line to as well")
    a = ap.parse_args()
    import pyarrow.compute as pc
    import torch
    from werkzeug.test import Client

    from learningorchestra_b200 import builder_frontend, server
    from learningorchestra_b200.column_store import ColumnarDatabase
    from learningorchestra_b200.engine import Engine, split_bounds

    result = {"card": card(), "rows": a.rows, "test_rows": a.test_rows, "features": K + 2}
    db = ColumnarDatabase()
    dataset(db, "train", a.rows, 1, True)
    dataset(db, "test", a.test_rows, 2, False)
    with Engine(0) as eng:
        app = server.create_app(db, eng, synchronous=True)
        c = Client(app)
        jobs = []
        for _ in range(a.repeat):
            t0 = time.perf_counter()
            r = c.post("/models", json={"trainDatasetName": "train", "testDatasetName": "test", "modelingCode": CODE,
                                        "classifiersList": ["NB", "LR", "DT", "GB", "RF"]})
            assert r.status_code == 201, r.get_data(as_text=True)
            wall = time.perf_counter() - t0
            for name in ("NB", "LR", "DT", "GB", "RF"):
                meta = db.find_one(f"test{name}", {"_id": 0})
                assert meta["finished"], meta.get("exception")
            jobs.append({"wall_s": wall, **app.last_job.timings})
        result["job"] = jobs

        # the split kernel against the torch composition, alternated
        bounds = split_bounds([0.8, 0.2])
        with builder_frontend.device_frame(db, "train", eng, text=True) as frame:
            with frame.features([f"f{j}" for j in range(K)], label="label") as feats:
                part = feats._parts[0]
                ids_np = feats.row_ids
                xt = torch.as_tensor(feats.x[0], device="cuda:0")
                yt = torch.as_tensor(feats.y[0], device="cuda:0")
                idt = torch.as_tensor(ids_np, device="cuda:0")
                split, comp = [], []
                for _ in range(a.repeat + 1):
                    timing = {}
                    t0 = time.perf_counter()
                    got = eng.random_split(part, ids_np, bounds, 7, timing=timing)
                    split.append({"wall_ms": (time.perf_counter() - t0) * 1e3, "kernel_ms": timing["kernel_ms"]})
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    want = torch_split(xt, yt, idt, bounds, 7)
                    torch.cuda.synchronize()
                    comp.append({"wall_ms": (time.perf_counter() - t0) * 1e3})
                    for g, (wx, wy, wr) in zip(got, want):
                        gx = g.x.to_numpy(0, nrows=g.nkept * K)
                        assert np.array_equal(gx.view(np.uint32), wx.flatten().cpu().numpy().view(np.uint32))
                        assert np.array_equal(g.y.to_numpy(0, nrows=g.nkept).view(np.uint32), wy.cpu().numpy().view(np.uint32))
                        assert np.array_equal(g.rows, wr.cpu().numpy())
                        g.free()
                n = len(ids_np)
                nbytes = 8 * n + 8 * n + n * (K + 1) * 4 + n * ((K + 1) * 4 + 8)
                result["split"] = {"rows": n, "bytes": nbytes, "kernel": split[1:], "torch": comp[1:],
                                   "GBps": [nbytes / (s["kernel_ms"] * 1e-3) / 1e9 for s in split[1:]]}

        # the dictionary probe against pyarrow.compute.index_in on the host, alternated
        with builder_frontend.device_frame(db, "train", eng, text=True) as frame:
            dictionary = frame.dictionaries["t0"]
        cells = db.column("test", "t0").arr
        text = eng.text(cells)
        table = eng.table("i32", text.n, 1)
        probe, host = [], []
        try:
            for _ in range(a.repeat + 1):
                timing = {}
                t0 = time.perf_counter()
                eng.text_codes_in(text, dictionary, table, 0, timing=timing)
                probe.append({"wall_ms": (time.perf_counter() - t0) * 1e3, "kernel_ms": timing["kernel_ms"]})
                t0 = time.perf_counter()
                want = pc.index_in(cells, value_set=dictionary)
                host.append({"wall_ms": (time.perf_counter() - t0) * 1e3})
                assert np.array_equal(table.to_numpy(0), want.fill_null(-1).to_numpy().astype(np.int32))
        finally:
            table.free()
            text.free()
        result["dictionary"] = {"cells": len(cells), "words": len(dictionary), "device": probe[1:], "index_in": host[1:]}
    result["card_after"] = card()
    line = json.dumps(result)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    os.environ.setdefault("PYTHONHASHSEED", "0")
    main()
