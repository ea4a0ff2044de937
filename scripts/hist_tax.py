"""What the 256-bin histogram costs on top of the projection + cast, measured on the S100 table (100 M x 32 fp64 -> fp32).

Two arms per build on the same resident table, alternating, each in a fresh process (LOEXEC_LIB selects the build):

* ``fused``       project_cast_hist, the bench.py step;
* ``cast``        project_cast, the same launch without a histogram;
* ``fused_base`` / ``cast_base``  the same two with a second build of libloexec.so (``--base``, e.g. the parent commit's).

Each arm times ``--steps`` launches with CUDA events after ``--warmup`` launches, with SM clock / power / throttle
reasons sampled inside the timed window (bench.ClockSampler).  The histogram's cost of a build is its fused step's
excess over its cast-only step.  Prints one JSON object and writes it to ``--out``/hist_tax.json.

    python scripts/hist_tax.py --base /path/to/parent/libloexec.so --reps 3 --out /tmp/hist_tax
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent

CHILD = r'''
import json, sys
import numpy as np, torch
sys.path.insert(0, sys.argv[1])
import bench
from learningorchestra_b200.engine import Engine
arm, rows, steps, warmup = sys.argv[2], int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5])
eng = Engine(0); st = torch.cuda.Stream(); torch.cuda.set_stream(st)
t = eng.table("f64", rows, 32).fill_synthetic(0, bench.SEED, stream=st); out = eng.table("f32", rows, 32)
cols = bench.projected_columns(32); c = eng.counts(32, bench.NBINS)
lo, hi = np.full(32, bench.GEN_LO, np.float32), np.full(32, bench.GEN_HI, np.float32)
if arm == "fused":
    fn = lambda: eng.project_cast_hist(t, cols, bench.NBINS, lo, hi, out=out, counts=c, stream=st)
else:
    fn = lambda: eng.project_cast(t, cols, out=out, stream=st)
for _ in range(warmup): fn()
torch.cuda.synchronize()
sampler = bench.ClockSampler(0); sampler.start(); sampler.wait_ready()
a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
sampler.mark_start(); a.record(st)
for _ in range(steps): fn()
b.record(st); torch.cuda.synchronize(); sampler.mark_end()
ms = a.elapsed_time(b) / steps
print(json.dumps({"ms_per_step": ms, "gb_s": rows * 32 * 12 / (ms * 1e-3) / 1e9, "clocks": sampler.stop()}))
'''


def run_arm(lib: str | None, arm: str, a) -> dict:
    env = dict(os.environ)
    if lib:
        env.update(LOEXEC_LIB=lib, LOEXEC_LAX="1")
    p = subprocess.run([sys.executable, "-c", CHILD, str(ROOT), arm, str(a.rows), str(a.steps), str(a.warmup)],
                       env=env, capture_output=True, text=True)
    line = [x for x in p.stdout.splitlines() if x.startswith("{")]
    if p.returncode != 0 or not line:
        raise SystemExit(f"arm {arm} ({lib or 'in-tree'}) failed:\n{p.stderr[-2000:]}")
    return json.loads(line[-1])


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"nvidia_smi": q[0] if q else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", help="second libloexec.so (the one to compare against)")
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "hist_tax"))
    a = ap.parse_args()
    arms = [("fused", None, "fused"), ("cast", None, "cast")]
    if a.base:
        arms += [("fused_base", a.base, "fused"), ("cast_base", a.base, "cast")]
    runs = {name: [] for name, _, _ in arms}
    for rep in range(a.reps):
        for name, lib, arm in arms:
            r = run_arm(lib, arm, a)
            runs[name].append(r)
            print(rep, name, round(r["ms_per_step"], 3), "ms", (r["clocks"] or {}).get("sm_mhz"), "MHz", file=sys.stderr, flush=True)
    med = {name: statistics.median(r["ms_per_step"] for r in rs) for name, rs in runs.items()}
    res = {"card": card(), "rows": a.rows, "steps": a.steps, "reps": a.reps, "median_ms": med,
           "hist_cost_ms": med["fused"] - med["cast"], "runs": runs}
    if a.base:
        res["hist_cost_base_ms"] = med["fused_base"] - med["cast_base"]
    print(json.dumps({k: v for k, v in res.items() if k != "runs"}))
    Path(a.out).mkdir(parents=True, exist_ok=True)
    (Path(a.out) / "hist_tax.json").write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
