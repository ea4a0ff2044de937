"""GBTClassifier fit / transform / evaluate on one H100: the library's fit timed per tree — its level passes and its
update pass by their CUDA events (lo_host_timing.kernel_ms), the host's split choice (lo_gb_stats and the variance
search) by wall clock — and the classifier's whole fit by wall clock, against a torch composition, alternated.  The
composition reuses the library's thresholds and trees (it searches for neither): it bucketizes every column once, and
per tree routes the rows level by level through the library's splits and accumulates (count, r, r^2) per (node,
feature, bin) with index_add_ in f64, then walks the tree for the margins and writes the next residuals.  Records the
card, its power limit and SM clock in the same run, and checks that the composition's sums agree with the library's
exact ones (their largest relative difference: its f64 atomics are not exact) and its last residuals (their largest
absolute difference: the two exp functions may differ by an ulp).

    python scripts/gbt_bench.py [--shapes 10000000:20,1000000:20] [--trees 20] [--depth 5] [--reps 2]

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
from learningorchestra_b200 import tree as T                                  # noqa: E402
from learningorchestra_b200.classifier import GBTClassifier, split_thresholds  # noqa: E402
from learningorchestra_b200.engine import AssembledRows, Engine               # noqa: E402


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


def library_fit(engine, part, thr, trees, depth, step=0.1):
    """The classifier's boosting loop over the binned rows, phase by phase: per tree the level passes' kernel time,
    the update pass's kernel time and the host's split choice (the tree's wall time less its level calls' wall time).
    Returns (trees, per-tree phases, plan: per tree the (splits, nnodes, words) of every level)."""
    nbins = max(len(t) for t in thr) + 1
    binned = engine.dt_bin(part, thr)
    rows = engine.gb_update(part)
    out, phases, plans = [], [], []
    try:
        for m in range(trees):
            levels, walls, plan = [], [], []

            def level(splits, nnodes):
                tt = {}
                t0 = time.perf_counter()
                words = engine.gb_level(part, binned, rows, nbins, splits, nnodes, timing=tt)
                walls.append(time.perf_counter() - t0)
                levels.append(_ms(tt))
                plan.append((splits, nnodes, words))
                return words

            t0 = time.perf_counter()
            tree, _ = T.grow(level, thr, 0, depth, T.VARIANCE, 1, 0.0)
            host = time.perf_counter() - t0 - sum(walls)
            w = 1.0 if m == 0 else step
            tu = {}
            engine.gb_update(part, rows, tree, w, timing=tu)
            out.append(tree)
            plans.append(plan)
            phases.append({"levels_ms": sum(levels), "root_ms": levels[0], "update_ms": _ms(tu),
                           "host_split_ms": 1e3 * host, "nodes": tree.num_nodes})
        last_r = torch.as_tensor(rows.residual.to_numpy(0)[:part.nkept])
    finally:
        binned.free()
        rows.free()
    return out, phases, plans, last_r


def torch_fit(x, y, thr, trees, plans, step=0.1):
    """The torch composition over the library's thresholds and trees; returns (ms, max relative difference of its
    level sums from the library's, its last residuals)."""
    n, k = x.shape
    dev = x.device
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    thr_t = [torch.tensor(t, dtype=torch.float64, device=dev) for t in thr]
    codes = torch.stack([torch.bucketize(x[:, j].double(), thr_t[j], right=False) for j in range(k)], 1)
    nbins = max(len(t) for t in thr) + 1
    yp = 2.0 * y.double() - 1.0
    F = torch.zeros(n, dtype=torch.float64, device=dev)
    r = yp.clone()
    xd = x.double()
    fcol = torch.arange(k, device=dev)
    sums = []
    for m, (tree, plan) in enumerate(zip(trees, plans)):
        node = torch.zeros(n, dtype=torch.long, device=dev)
        for splits, nnodes, _w in plan:
            if splits is not None:
                sp = torch.as_tensor(np.asarray(splits, np.int64), device=dev)
                s = sp[node.clamp(min=0)]
                live = (node >= 0) & (s[:, 0] >= 0)
                c = codes.gather(1, s[:, 0].clamp(min=0)[:, None]).squeeze(1)
                node = torch.where(live, torch.where(c <= s[:, 1], s[:, 2], s[:, 3]), torch.full_like(node, -1))
            rows = node >= 0
            idx = ((node[rows, None] * k + fcol[None, :]) * nbins + codes[rows]).ravel()
            acc = torch.zeros(nnodes * k * nbins, 3, dtype=torch.float64, device=dev)
            rr = r[rows, None].expand(-1, k).ravel()
            acc.index_add_(0, idx, torch.stack([torch.ones_like(rr), rr, rr * rr], 1))
            sums.append(acc)
        feat = torch.as_tensor(tree.feature, device=dev, dtype=torch.long)
        thr_n = torch.as_tensor(tree.threshold, device=dev)
        left = torch.as_tensor(tree.left, device=dev, dtype=torch.long)
        right = torch.as_tensor(tree.right, device=dev, dtype=torch.long)
        pred = torch.as_tensor(tree.prediction, device=dev)
        leaf = torch.zeros(n, dtype=torch.long, device=dev)
        for _ in range(tree.depth):
            f = feat[leaf]
            v = xd.gather(1, f.clamp(min=0)[:, None]).squeeze(1)
            leaf = torch.where(f >= 0, torch.where(v <= thr_n[leaf], left[leaf], right[leaf]), leaf)
        F = F + pred[leaf] * (1.0 if m == 0 else step)
        r = (4.0 * yp) / (1.0 + torch.exp((2.0 * yp) * F))
    torch.cuda.synchronize()
    ms = 1e3 * (time.perf_counter() - t0)
    worst = 0.0
    at = 0
    for plan in plans:
        for _s, nnodes, words in plan:
            w64 = np.asarray(words, np.uint64)
            cnt = w64[..., 0].astype(np.float64).ravel()
            lib = np.stack([cnt, _bin_sums(w64, 1, cnt), _bin_sums(w64, 3, None)], 1)
            got = sums[at].cpu().numpy()
            at += 1
            scale = np.maximum(np.abs(lib), 1.0)
            worst = max(worst, float(np.max(np.abs(got - lib) / scale)))
    return ms, worst, r.cpu()


def _bin_sums(words, p, cnt):
    """Every bin's sum (word pair p) as f64, the 2^60 offset of q1 removed: Python ints, one rounding each."""
    lo, hi = words[..., p].ravel(), words[..., p + 1].ravel()
    out = np.empty(len(lo))
    for i, (a, b) in enumerate(zip(lo.tolist(), hi.tolist())):
        v = a + (b << 64)
        if cnt is not None:
            v -= int(cnt[i]) << 60
        out[i] = float(v) / 2 ** 58
    return out


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
        w = torch.randn(k, device="cuda", generator=g)
        u = torch.rand(n, device="cuda", generator=g)
        y = ((x @ w + torch.log(u / (1 - u))) > 0).float()
        xt = engine.wrap("f32", n * k, 1, x.data_ptr(), n * k * 4, keepalive=x)
        yt = engine.wrap("f32", n, 1, y.data_ptr(), n * 4, keepalive=y)
        part = AssembledRows(xt, yt, None, k, n)
        feats = _features(engine, part)
        thr, _rounds = split_thresholds(feats, n, k, 32, "GBTClassifier")
        fit, lib, comp = [], [], []
        worst, r_diff = 0.0, 0.0
        for _ in range(a.reps):
            torch.cuda.empty_cache()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            model = GBTClassifier(max_iter=a.trees, max_depth=a.depth).fit(feats)
            fit.append(1e3 * (time.perf_counter() - t0))
            t0 = time.perf_counter()
            trees, phases, plans, last_r = library_fit(engine, part, thr, a.trees, a.depth)
            lib.append((1e3 * (time.perf_counter() - t0), phases))
            ms, wdiff, r_t = torch_fit(x, y, thr, trees, plans)
            comp.append(ms)
            worst = max(worst, wdiff)
            r_diff = max(r_diff, float((r_t - last_r).abs().max()))
        tp, te = {}, {}
        engine.gb_predict(part, model.trees, model.tree_weights, timing=tp).free()
        engine.gb_predict(part, model.trees, model.tree_weights, labels=np.array([0.0, 1.0]), timing=te)
        best = min(lib, key=lambda r: r[0])
        ph = best[1]
        print(json.dumps({
            "card": card, "rows": n, "k": k, "trees": a.trees, "depth": a.depth,
            "fit_wall_ms": round(min(fit), 1), "phased_fit_wall_ms": round(best[0], 1), "torch_ms": round(min(comp), 1),
            "per_tree_mean_ms": {key: round(float(np.mean([p[key] for p in ph])), 3)
                                 for key in ("levels_ms", "root_ms", "update_ms", "host_split_ms")},
            "tree0": {key: round(v, 3) for key, v in ph[0].items()},
            "levels_total_ms": round(sum(p["levels_ms"] for p in ph), 2),
            "update_total_ms": round(sum(p["update_ms"] for p in ph), 2),
            "host_split_total_ms": round(sum(p["host_split_ms"] for p in ph), 2),
            "total_nodes": int(sum(p["nodes"] for p in ph)),
            "transform_ms": round(_ms(tp), 3), "evaluate_ms": round(_ms(te), 3),
            "torch_sums_max_rel_diff": worst, "torch_last_residual_max_abs_diff": r_diff}), flush=True)
        part.free()


if __name__ == "__main__":
    main()
