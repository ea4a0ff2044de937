"""Numpy restatement of Spark 2.4's GBTClassifier with its defaults (DESIGN.md §3.6.5), written node by node as
Spark's GradientBoostedTrees and RandomForest do, sharing no code with learningorchestra_b200: the label remap, the
regression trees with Variance impurity grown from exact fixed-point sums (Python ints, one rounding per statistic),
toNode(prune = true), LogLoss's residuals and the model's transform.  The split candidates and the bins are
tree_oracle's."""
import math

import numpy as np

import tree_oracle as to

EPS = 2.220446049250313e-16
DOUBLE_MIN = -1.7976931348623157e308
SCALE = 2 ** 58


def quantise(r):
    """(q1, q2) int64 of every residual: rint(r 2^58) and rint(fl(r r) 2^58)."""
    r = np.asarray(r, np.float64)
    return np.rint(r * SCALE).astype(np.int64), np.rint((r * r) * SCALE).astype(np.int64)


def exact_sum(q, groups, ngroups):
    """Exact Python-int sums of int64 values q per group (the values split in 32-bit halves, each half summed in int64)."""
    hi, lo = q >> 32, q & 0xFFFFFFFF
    sh, sl = np.zeros(ngroups, np.int64), np.zeros(ngroups, np.int64)
    np.add.at(sh, groups, hi)
    np.add.at(sl, groups, lo)
    return [int(a) * (1 << 32) + int(b) for a, b in zip(sh, sl)]


def stats_of(cnt, s1, s2):
    """(count, sum, sumSq) in f64 from integer sums: each rounded once (Python's int -> float), then scaled."""
    return float(cnt), float(s1) / SCALE, float(s2) / SCALE


def variance(st):
    c, s, sq = st
    if c == 0:
        return 0.0
    return (sq - (s * s) / c) / c


def _gain(parent_imp, left, right, min_inst, min_gain):
    lc, rc = left[0], right[0]
    if lc < min_inst or rc < min_inst:
        return DOUBLE_MIN, False, None, None
    limp, rimp = variance(left), variance(right)
    total = lc + rc
    gain = parent_imp - (lc / total) * limp - (rc / total) * rimp
    if gain < min_gain:
        return DOUBLE_MIN, False, None, None
    return gain, True, limp, rimp


def regression_tree(codes, thr, r, max_depth=5, min_inst=1, min_gain=0.0):
    """One regression tree on the bin codes (n, k) and residuals r, as nested dicts after pruning."""
    q1, q2 = quantise(r)
    n, k = codes.shape

    def node_stats(rows):
        return (len(rows), exact_sum(q1[rows], np.zeros(len(rows), np.int64), 1)[0],
                exact_sum(q2[rows], np.zeros(len(rows), np.int64), 1)[0])

    def node(rows, depth):
        tot = node_stats(rows)
        parent = stats_of(*tot)
        parent_imp = variance(parent)
        best = None
        for j in range(k):
            m = len(thr[j])
            if not m:
                continue
            b = codes[rows, j]
            cnt = np.bincount(b, minlength=m + 1).tolist()
            s1, s2 = exact_sum(q1[rows], b, m + 1), exact_sum(q2[rows], b, m + 1)
            lc = l1 = l2 = 0
            for i in range(m):
                lc, l1, l2 = lc + cnt[i], l1 + s1[i], l2 + s2[i]
                left = stats_of(lc, l1, l2)
                right = stats_of(tot[0] - lc, tot[1] - l1, tot[2] - l2)
                gain, valid, limp, rimp = _gain(parent_imp, left, right, min_inst, min_gain)
                if best is None or gain > best[0]:
                    best = (gain, valid, j, i, limp, rimp)
        leaf = dict(stats=parent, impurity=parent_imp, valid=True, split=None)
        if best is None:
            leaf["valid"] = False
            return leaf
        gain, valid = best[0], best[1]
        leaf["valid"] = valid
        if gain <= 0 or depth == max_depth:
            return leaf
        j, i = best[2], best[3]
        kids = []
        for sub, imp in ((rows[codes[rows, j] <= i], best[4]), (rows[codes[rows, j] > i], best[5])):
            if depth + 1 == max_depth or abs(imp) < EPS:
                kids.append(dict(stats=stats_of(*node_stats(sub)), impurity=imp, valid=True, split=None))
            else:
                kids.append(node(sub, depth + 1))
        return dict(stats=parent, impurity=parent_imp, valid=True, split=(j, thr[j][i]), gain=gain,
                    left=kids[0], right=kids[1])

    return prune(node(np.arange(n), 0))


def prediction(st):
    return st[1] / st[0]


def prune(nd):
    if nd["split"] is None:
        return dict(leaf=True, stats=nd["stats"], impurity=nd["impurity"] if nd["valid"] else -1.0)
    left, right = prune(nd["left"]), prune(nd["right"])
    if left["leaf"] and right["leaf"] and prediction(left["stats"]) == prediction(right["stats"]):
        return dict(leaf=True, stats=nd["stats"], impurity=nd["impurity"])
    return dict(leaf=False, stats=nd["stats"], impurity=nd["impurity"], gain=nd["gain"], feature=nd["split"][0],
                threshold=nd["split"][1], left=left, right=right)


def arrays(root):
    """Breadth-first arrays (feature, threshold, left, right, stats, prediction, impurity, gain) of a pruned tree."""
    out = dict(feature=[], threshold=[], left=[], right=[], stats=[], prediction=[], impurity=[], gain=[])
    queue = [root]
    i = 0
    while i < len(queue):
        nd = queue[i]
        out["stats"].append(nd["stats"])
        out["prediction"].append(prediction(nd["stats"]))
        out["impurity"].append(nd["impurity"])
        if nd["leaf"]:
            for key, v in (("feature", -1), ("threshold", math.nan), ("left", -1), ("right", -1), ("gain", math.nan)):
                out[key].append(v)
        else:
            out["feature"].append(nd["feature"])
            out["threshold"].append(nd["threshold"])
            out["gain"].append(nd["gain"])
            out["left"].append(len(queue))
            out["right"].append(len(queue) + 1)
            queue += [nd["left"], nd["right"]]
        i += 1
    return {key: np.array(v) for key, v in out.items()}


def predict_tree(root, x):
    x = np.asarray(x).astype(np.float64)
    out = np.zeros(len(x))
    for r in range(len(x)):
        nd = root
        while not nd["leaf"]:
            nd = nd["left"] if x[r, nd["feature"]] <= nd["threshold"] else nd["right"]
        out[r] = prediction(nd["stats"])
    return out


def residual(y, F):
    """-LogLoss.gradient(F, y') = 4y' / (1 + exp(2y'F)) with y' = 2y - 1."""
    yp = 2.0 * np.asarray(y, np.float64) - 1.0
    return (4.0 * yp) / (1.0 + np.exp((2.0 * yp) * F))


def fit(x, y, max_iter=20, step_size=0.1, max_depth=5, max_bins=32, min_inst=1, min_gain=0.0):
    """GradientBoostedTrees.boost: (trees, weights, thresholds, the residuals each tree was grown on)."""
    x = np.asarray(x)
    thr = [to.splits(x[:, j], max_bins) for j in range(x.shape[1])]
    codes = to.bins(x, thr)
    r = 2.0 * np.asarray(y, np.float64) - 1.0
    F = np.zeros(len(y))
    trees, weights, chain = [], [], []
    for m in range(max_iter):
        chain.append(r)
        root = regression_tree(codes, thr, r, max_depth, min_inst, min_gain)
        w = 1.0 if m == 0 else step_size
        trees.append(root)
        weights.append(w)
        F = F + predict_tree(root, x) * w
        r = residual(y, F)
    return trees, weights, thr, chain


def transform(trees, weights, x):
    """(raw, probability, prediction) of every row: the margin summed in tree order from 0.0."""
    m = np.zeros(len(x))
    for t, w in zip(trees, weights):
        m = m + predict_tree(t, x) * w
    p0 = 1.0 / (1.0 + np.exp(2.0 * m))
    return np.stack([-m, m], 1), np.stack([p0, 1.0 - p0], 1), (m > 0).astype(np.float64)
