"""DecisionTreeClassifier fit / transform / evaluate on one H100: every phase of the library's fit timed by its CUDA
events (lo_host_timing.kernel_ms) and wall clock, against a torch composition, alternated: torch.sort per column, bucketize against the library's thresholds (the
composition does not search for thresholds itself: its split search is the library's, untimed), and per level the rows
routed through the library's splits and one bincount of (node, bin, class) per feature.  Records the card, its power
limit and SM clock in the same run and checks that both give the same histogram at every level.  A skewed shape (every
column rounded to three values, as categorical builder fields are) puts a warp's shared atomics on a few counters.

    python scripts/tree_bench.py [--shapes 10000000:20:0,100000000:32:0,10000000:20:1] [--reps 3]

Prints one JSON line per shape."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from learningorchestra_b200 import tree as T                          # noqa: E402
from learningorchestra_b200.classifier import _DT_SORT_BUDGET         # noqa: E402
from learningorchestra_b200.engine import AssembledRows, Engine       # noqa: E402

HBM_GBS = 3350.0          # H100 SXM5 HBM3 peak (GB/s), the yardstick of the passes' share of peak


def _card():
    q = "name,power.limit,clocks.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True).stdout.strip()
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def _ms(t):
    return t.get("kernel_ms", 0.0)


def library_fit(engine, part, max_depth=5, max_bins=32):
    """The classifier's fit, phase by phase, with every call's kernel time."""
    ph = {}
    t = {}
    n, _s, _m, counts = engine.lr_stats(part, timing=t)
    ph["stats"] = _ms(t)
    C = int(np.flatnonzero(counts)[-1]) + 1
    cap = T.num_splits(max_bins, n) + 1
    kc = max(1, min(part.k, _DT_SORT_BUDGET // (8 * n)))         # the classifier's column batches
    calls, thr, rounds, ph["sort"] = [], [], 0, 0.0
    for j0 in range(0, part.k, kc):
        w = min(kc, part.k - j0)
        t = {}
        s = engine.dt_sort(part, j0, w, cap, timing=t)
        ph["sort"] += _ms(t)

        def rank(cols, codes):
            t0 = time.perf_counter()
            out = engine.dt_rank(s, cols, codes)
            calls.append(time.perf_counter() - t0)
            return out

        distinct = [T.merge_distinct([s.distinct[c]]) for c in range(w)]
        got, r = T.column_thresholds(n, max_bins, distinct, rank, True, w)
        s.free()
        thr += got
        rounds += r
    ph["rank_ms"], ph["rank_rounds"], ph["rank_calls"] = 1e3 * sum(calls), rounds, len(calls)
    t = {}
    binned = engine.dt_bin(part, thr, timing=t)
    ph["bin"] = _ms(t)
    nbins = max(len(x) for x in thr) + 1
    levels, plan = [], []

    def level(splits, nnodes):
        tt = {}
        h = engine.dt_level(part, binned, nbins, C, splits, nnodes, timing=tt)
        levels.append(_ms(tt))
        plan.append((splits, nnodes, h))
        return h

    tree, _ = T.grow(level, thr, C, max_depth, "gini", 1, 0.0)
    binned.free()
    ph["levels"] = levels
    return tree, thr, ph, plan


def torch_fit(x, y, thr, plan):
    """The torch composition: sort every column, bucketize against the thresholds, and for every level of ``plan``
    ((splits, nnodes, library histogram) as the library's fit met them) route the rows by the splits and bincount (node,
    bin, class) per feature.  Returns its time (ms) and whether every level's histogram equals the library's."""
    n, k = x.shape
    C = int(y.max().item()) + 1
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for j in range(k):
        torch.sort(x[:, j])
    thr_t = [torch.tensor(t, dtype=torch.float64, device=x.device) for t in thr]
    codes = torch.stack([torch.bucketize(x[:, j].double(), thr_t[j], right=False) for j in range(k)], 1).to(torch.uint8)
    nbins = max(len(t) for t in thr) + 1
    yi = y.long()
    node = torch.zeros(n, dtype=torch.long, device=x.device)
    hists = []
    for splits, nnodes, _h in plan:
        if splits is not None:
            sp = torch.as_tensor(np.asarray(splits, np.int64), device=x.device)
            s = sp[node.clamp(min=0)]
            live = (node >= 0) & (s[:, 0] >= 0)
            c = codes.gather(1, s[:, 0].clamp(min=0)[:, None]).squeeze(1).long()
            node = torch.where(live, torch.where(c <= s[:, 1], s[:, 2], s[:, 3]), torch.full_like(node, -1))
        rows = node >= 0
        base = node[rows] * nbins
        hists.append([torch.bincount((base + codes[rows, j].long()) * C + yi[rows], minlength=nnodes * nbins * C)
                      for j in range(k)])
    torch.cuda.synchronize()
    ms = 1e3 * (time.perf_counter() - t0)
    same = all(np.array_equal(h[:, j].ravel(), level[j].cpu().numpy())
               for (_s, _n, h), level in zip(plan, hists) for j in range(k))
    return ms, same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="10000000:20:0,100000000:32:0,10000000:20:1")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    engine = Engine(0)
    card = _card()
    for shape in a.shapes.split(","):
        n, k, skew = (int(v) for v in shape.split(":"))
        g = torch.Generator(device="cuda").manual_seed(n + k)
        x = torch.randn(n, k, device="cuda", generator=g)
        if skew:
            x = x.round().clamp(-1.0, 1.0)
        w = torch.randn(k, 3, device="cuda", generator=g)
        y = (x @ w + torch.rand(n, 3, device="cuda", generator=g).log().neg().log().neg()).argmax(1).float()
        xt = engine.wrap("f32", n * k, 1, x.data_ptr(), n * k * 4, keepalive=x)
        yt = engine.wrap("f32", n, 1, y.data_ptr(), n * 4, keepalive=y)
        part = AssembledRows(xt, yt, None, k, n)
        lib, comp, same = [], [], True
        for _ in range(a.reps):
            torch.cuda.empty_cache()                          # the composition's cached blocks back to the device
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tree, thr, ph, plan = library_fit(engine, part)
            lib.append((1e3 * (time.perf_counter() - t0), ph))
            ms, ok = torch_fit(x, y, thr, plan)
            comp.append(ms)
            same = same and ok
        C = int(y.max().item()) + 1
        tp = {}
        engine.dt_predict(part, tree, timing=tp).free()
        te = {}
        engine.dt_predict(part, tree, labels=np.arange(C, dtype=np.float64), timing=te)
        best = min(lib, key=lambda r: r[0])
        ph = best[1]
        bin_bytes, level_bytes = n * k * 4 + n * ((k + 15) // 16 * 16), n * ((k + 15) // 16 * 16) + n * 4 * 3
        print(json.dumps({
            "card": card, "rows": n, "k": k, "skewed": bool(skew), "fit_ms": round(best[0], 2), "torch_ms": round(min(comp), 2),
            "phases_ms": {kk: (round(v, 3) if isinstance(v, float) else v) for kk, v in ph.items() if kk != "levels"},
            "level_ms": [round(v, 3) for v in ph["levels"]],
            "transform_ms": round(_ms(tp), 3), "evaluate_ms": round(_ms(te), 3),
            "bin_share_of_peak": round(bin_bytes / (ph["bin"] * 1e-3) / 1e9 / HBM_GBS, 3),
            "root_level_share_of_peak": round(level_bytes / (ph["levels"][0] * 1e-3) / 1e9 / HBM_GBS, 3),
            "predict_share_of_peak": round((n * k * 4 + n * 8 * (2 * C + 1)) / (_ms(tp) * 1e-3) / 1e9 / HBM_GBS, 3),
            "level_histograms_equal": bool(same)}), flush=True)
        part.free()


if __name__ == "__main__":
    main()
