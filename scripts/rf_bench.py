"""RandomForestClassifier fit / transform / evaluate on one H100: the library's fit timed per batch level — the level
passes by their CUDA events (lo_host_timing.kernel_ms) with their node-group passes, the host's split choice (the
split search and the subset draws) by wall clock — and the classifier's whole fit by wall clock, against a torch
composition, alternated.  The composition reuses the library's thresholds, bagging table and feature subsets (it
searches for none of them): it bucketizes every column once, draws every (row, tree) weight with the same splitmix64
hash in int64 arithmetic, and per level routes the rows through the library's splits and accumulates the weights per
(node, listed feature, bin, class) with index_add_; its histograms must equal the library's.  Records the card, its
power limit and SM clock in the same run.

    python scripts/rf_bench.py [--shapes 10000000:20,1000000:20] [--trees 20] [--depth 5] [--reps 2]

Prints one JSON line per shape."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from learningorchestra_b200 import classifier as CL                               # noqa: E402
from learningorchestra_b200 import tree as T                                       # noqa: E402
from learningorchestra_b200.classifier import RandomForestClassifier, split_thresholds  # noqa: E402
from learningorchestra_b200.engine import AssembledRows, Engine                    # noqa: E402

MIN64 = -(1 << 63)


def _card():
    q = "name,power.limit,clocks.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True).stdout.strip()
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def _ms(t):
    return t.get("kernel_ms", 0.0)


def _features(engine, part):
    return SimpleNamespace(_frame=SimpleNamespace(_cache=SimpleNamespace(engine=engine)), _parts=[part],
                           fields=[f"f{j}" for j in range(part.k)], label="y", row_ids=np.arange(part.nkept))


def _s64(v):
    v &= (1 << 64) - 1
    return v - (1 << 64) if v >> 63 else v


def _srl(z, s):
    return (z >> s) & ((1 << (64 - s)) - 1)


def _mix(z):
    """splitmix64's step on int64 tensors (two's complement wraps as uint64 does; shifts made logical)."""
    z = z + _s64(0x9E3779B97F4A7C15)
    z = (z ^ _srl(z, 30)) * _s64(0xBF58476D1CE4E5B9)
    z = (z ^ _srl(z, 27)) * _s64(0x94D049BB133111EB)
    return z ^ _srl(z, 31)


def library_fit(engine, part, est, thr, C, m, batch):
    """The classifier's batches phase by phase: per level the kernel time and node-group passes, per batch the host's
    split choice (the batch's wall time less its level calls' wall time).  Returns (trees, phases, plans)."""
    nbins = max(len(t) for t in thr) + 1
    draw = T.draw_table(est.num_trees, est.subsampling_rate)
    binned = engine.dt_bin(part, thr)
    trees, phases, plans = [], [], []
    try:
        for tree0 in range(0, est.num_trees, batch):
            nt = min(batch, est.num_trees - tree0)
            levels, passes, walls, plan = [], [], [], []

            def level(splits, nnodes, feats):
                tt, sh = {}, []
                t0 = time.perf_counter()
                hist = engine.rf_level(part, binned, nbins, C, est.seed, draw, tree0, nt, splits, feats, shape=sh,
                                       timing=tt)
                walls.append(time.perf_counter() - t0)
                levels.append(_ms(tt))
                passes.append(sh[3])
                plan.append((splits, feats, hist))
                return hist

            t0 = time.perf_counter()
            grown, _ = T.grow(level, thr, C, est.max_depth, est.impurity, 1, 0.0, trees=nt,
                              subsets=lambda t, node: T.feature_subset(est.seed, tree0 + t, node, part.k, m))
            host = time.perf_counter() - t0 - sum(walls)
            trees += grown
            plans.append((tree0, nt, plan))
            phases.append({"levels_ms": [round(v, 3) for v in levels], "passes": passes, "host_split_ms": 1e3 * host})
    finally:
        binned.free()
    return trees, phases, plans, draw


def torch_fit(x, y, thr, C, seed, draw, plans):
    """The composition over the library's thresholds, table and subsets; returns (ms, its histograms equal the
    library's)."""
    n, k = x.shape
    dev = x.device
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    thr_t = [torch.tensor(t, dtype=torch.float64, device=dev) for t in thr]
    codes = torch.stack([torch.bucketize(x[:, j].double(), thr_t[j], right=False) for j in range(k)], 1)
    nbins = max(len(t) for t in thr) + 1
    cls = y.long()
    rows = torch.arange(n, device=dev, dtype=torch.int64)
    key = _mix(torch.tensor(_s64(seed), dtype=torch.int64, device=dev))
    tab = torch.tensor([_s64(v ^ (1 << 63)) for v in draw], dtype=torch.int64, device=dev)   # unsigned order as signed
    hists = []
    for tree0, nt, plan in plans:
        w = torch.stack([((_mix(_mix(key ^ (tree0 + t)) ^ rows) ^ MIN64)[:, None] >= tab[None, :]).sum(1)
                         for t in range(nt)]).double()
        node = torch.arange(nt, device=dev)[:, None].expand(nt, n).clone()
        for splits, feats, _h in plan:
            if splits is not None:
                sp = torch.as_tensor(np.asarray(splits, np.int64), device=dev)
                s = sp[node.clamp(min=0)]
                live = (node >= 0) & (s[..., 0] >= 0)
                c = codes[rows[None, :].expand(nt, n), s[..., 0].clamp(min=0)]
                node = torch.where(live, torch.where(c <= s[..., 1], s[..., 2], s[..., 3]), torch.full_like(node, -1))
            fl = torch.as_tensor(np.asarray(feats, np.int64), device=dev)
            nnodes, mm = fl.shape
            live = (node >= 0) & (w > 0)
            tt, rr = live.nonzero(as_tuple=True)
            s = node[tt, rr]
            acc = torch.zeros(nnodes * mm * nbins * C, dtype=torch.float64, device=dev)
            for q in range(mm):
                idx = ((s * mm + q) * nbins + codes[rr, fl[s, q]]) * C + cls[rr]
                acc.index_add_(0, idx, w[tt, rr])
            hists.append(acc)
    torch.cuda.synchronize()
    ms = 1e3 * (time.perf_counter() - t0)
    lib = [h for _t0, _nt, plan in plans for _s, _f, h in plan]
    same = all(np.array_equal(a.cpu().numpy().astype(np.int64), b.ravel()) for a, b in zip(hists, lib))
    return ms, same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="10000000:20,1000000:20")
    ap.add_argument("--trees", type=int, default=20)
    ap.add_argument("--depth", type=int, default=5)
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    engine = Engine(0)
    card = _card()
    for shape in a.shapes.split(","):
        n, k = (int(v) for v in shape.split(":"))
        g = torch.Generator(device="cuda").manual_seed(n + k)
        x = torch.randn(n, k, device="cuda", generator=g)
        w = torch.randn(k, 3, device="cuda", generator=g)
        y = (x @ w + torch.randn(n, 3, device="cuda", generator=g)).argmax(1).float()
        xt = engine.wrap("f32", n * k, 1, x.data_ptr(), n * k * 4, keepalive=x)
        yt = engine.wrap("f32", n, 1, y.data_ptr(), n * 4, keepalive=y)
        part = AssembledRows(xt, yt, None, k, n)
        feats = _features(engine, part)
        est = RandomForestClassifier(num_trees=a.trees, max_depth=a.depth)
        thr, _rounds = split_thresholds(feats, n, k, 32, "RandomForestClassifier")
        m = T.subset_size(est.feature_subset_strategy, k, est.num_trees)
        batch = max(1, min(est.num_trees, CL._RF_SLOT_BUDGET // (8 * n)))
        fit, lib, comp, same = [], [], [], True
        for _ in range(a.reps):
            torch.cuda.empty_cache()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            model = est.fit(feats)
            fit.append(1e3 * (time.perf_counter() - t0))
            t0 = time.perf_counter()
            trees, phases, plans, draw = library_fit(engine, part, est, thr, 3, m, batch)
            lib.append((1e3 * (time.perf_counter() - t0), phases))
            ms, ok = torch_fit(x, y, thr, 3, est.seed, draw, plans)
            comp.append(ms)
            same = same and ok
        tp, te = {}, {}
        engine.rf_predict(part, model.trees, timing=tp).free()
        engine.rf_predict(part, model.trees, labels=np.array([0.0, 1.0, 2.0]), timing=te)
        best = min(lib, key=lambda r: r[0])
        ph = best[1]
        print(json.dumps({
            "card": card, "rows": n, "k": k, "trees": a.trees, "depth": a.depth, "m": m, "tree_batches": len(ph),
            "fit_wall_ms": round(min(fit), 1), "phased_fit_wall_ms": round(best[0], 1), "torch_ms": round(min(comp), 1),
            "levels_ms_per_batch": [p["levels_ms"] for p in ph], "passes_per_batch": [p["passes"] for p in ph],
            "levels_total_ms": round(sum(sum(p["levels_ms"]) for p in ph), 2),
            "host_split_total_ms": round(sum(p["host_split_ms"] for p in ph), 2),
            "total_nodes": model.total_num_nodes,
            "transform_ms": round(_ms(tp), 3), "evaluate_ms": round(_ms(te), 3),
            "torch_hist_equal": same}), flush=True)
        part.free()


if __name__ == "__main__":
    main()
