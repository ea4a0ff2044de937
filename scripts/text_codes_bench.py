"""Dictionary codes of resident text columns (lo_text_codes / lo_text_codes_shards) against the same column's `$group`
(lo_value_counts_text): the codes add a slot pass, the ordering of the groups and a remap to what the count already does.

    python scripts/text_codes_bench.py [--rows 1000000 10000000] [--reps 7] [--out FILE]

Columns of --rows cells at low cardinality (10 distinct cells, uniformly mixed) and high cardinality (every cell
distinct, in shuffled order).  On device 0: the median call time over --reps calls (host clock around a call that ends
in a synchronise) and the median kernel_ms of value_counts_text and of text_codes on the same resident column, and
their ratio.  Then the same columns cut over every visible GPU (a ShardedEngine, one piece per device) through
ShardedEngine.text_codes / value_counts_text; with one visible GPU that is a group of one.  The codes are checked against
the whole column's on one device.  The card's name, power limit and max SM clock are printed with the numbers
(read-only nvidia-smi query).
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))

from text_shards_bench import timed  # noqa: E402
from value_counts_bench import card  # noqa: E402


def columns(rows, seed):
    import pyarrow as pa
    rng = np.random.default_rng(seed)
    words = np.array(["w%d" % i for i in range(10)], dtype=object)
    return {"low": pa.array(words[rng.integers(0, 10, rows)], type=pa.large_string()),
            "high": pa.array(np.char.add("d", rng.permutation(rows).astype("U10")).astype(object), type=pa.large_string())}


def numbers(eng, arr, reps):
    """value_counts_text and text_codes on one resident column of ``eng`` (an Engine or a ShardedEngine)."""
    text = eng.text(arr)
    table = eng.table("i32", len(arr), 1)
    try:
        count_ms, count_kms, _ = timed(lambda t: eng.value_counts_text(text, timing=t), reps)
        codes_ms, codes_kms, first = timed(lambda t: eng.text_codes(text, table, 0, timing=t), reps)
        codes = table.to_numpy(0)
    finally:
        table.free()
        text.free()
    r = {"rows": len(arr), "distinct": int(len(first)), "value_counts_ms": count_ms, "value_counts_kernel_ms": count_kms,
         "text_codes_ms": codes_ms, "text_codes_kernel_ms": codes_kms, "codes_over_counts": codes_ms / count_ms}
    return r, codes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, nargs="*", default=[1_000_000, 10_000_000])
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--seed", type=int, default=20261017)
    ap.add_argument("--out")
    a = ap.parse_args()
    from learningorchestra_b200.engine import Engine
    from learningorchestra_b200.sharding import ShardedEngine
    results = {"card": card(), "one_device": {}, "devices": {}}
    print("card:", results["card"], flush=True)
    eng = Engine(0)
    sh = ShardedEngine.local()
    results["devices"]["count"] = sh.nlocal
    try:
        for rows in a.rows:
            for name, arr in columns(rows, a.seed).items():
                key = f"{name}_{rows}"
                one, codes = numbers(eng, arr, a.reps)
                results["one_device"][key] = one
                print("one device", key, json.dumps(one), flush=True)
                many, sharded_codes = numbers(sh, arr, a.reps)
                assert np.array_equal(codes, sharded_codes), f"{key}: the sharded codes differ from one device's"
                results["devices"][key] = many
                print(f"{sh.nlocal} device(s)", key, json.dumps(many), flush=True)
    finally:
        sh.close()
        eng.close()
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
