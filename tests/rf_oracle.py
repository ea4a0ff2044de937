"""Python restatement of the builder's RandomForestClassifier (DESIGN.md §3.6.6), written tree by tree and node by node
in Python ints and numpy so that it shares no code with learningorchestra_b200.tree: the splitmix64 hash, the bagging
tables (an exact Fraction series for e^-rate), the per-node feature subsets, the weighted level-wise growth, the pruning
and the vote transform.  The split candidates and bins are tree_oracle's (Spark finds them on the unbagged rows)."""
import math
from fractions import Fraction

import numpy as np

import tree_oracle as to

M64 = (1 << 64) - 1
EPS = 2.220446049250313e-16
DOUBLE_MIN = -1.7976931348623157e308


def mix(z: int) -> int:
    """splitmix64: z + 0x9E3779B97F4A7C15, then (z ^ z >> 30) * 0xBF58476D1CE4E5B9, (z ^ z >> 27) * 0x94D049BB133111EB,
    z ^ z >> 31, all mod 2^64."""
    z = (z + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def bag_u(seed: int, tree: int, row: int) -> int:
    return mix(mix(mix(seed & M64) ^ tree) ^ row)


def subset_key(seed: int, tree: int, node: int, j: int) -> int:
    return mix(mix(mix(mix(~seed & M64) ^ tree) ^ node) ^ j)


def java_string_hash(s: str) -> int:
    h = 0
    for ch in s:
        h = (h * 31 + ord(ch)) % (1 << 32)
    return h - (1 << 32) if h >= 1 << 31 else h


def exp_neg(lam: Fraction, terms: int = 80) -> Fraction:
    """e^-lam for 0 < lam <= 1 by its Taylor series: the tail after 80 terms is below 1/80!, far under 2^-64."""
    out, term = Fraction(0), Fraction(1)
    for i in range(terms):
        out += term
        term = term * (-lam) / (i + 1)
    return out


def table(num_trees: int, rate: float) -> list:
    """T_j = floor(2^64 P(X <= j)): [0] for one tree at rate 1, Bernoulli's one threshold for one tree below it, else
    Poisson(rate)'s, T_0 and every later one below 2^64 - 1."""
    r = Fraction(rate)
    if num_trees == 1:
        return [0] if r == 1 else [math.floor((1 - r) * 2 ** 64)]
    p0 = exp_neg(r)
    out, cdf, term, j = [], Fraction(0), p0, 0
    while True:
        cdf += term
        t = math.floor(cdf * 2 ** 64)
        if j > 0 and t >= M64:
            return out
        out.append(t)
        j += 1
        term = term * r / j


def weight(u: int, tab: list) -> int:
    return sum(1 for t in tab if u >= t)


def weights(seed: int, tree: int, rows, tab: list) -> np.ndarray:
    return np.array([weight(bag_u(seed, tree, int(r)), tab) for r in rows], np.int64)


def subset(seed: int, tree: int, node: int, k: int, m: int) -> list:
    if m == k:
        return list(range(k))
    order = sorted(range(k), key=lambda j: (subset_key(seed, tree, node, j), j))
    return sorted(order[:m])


def _stats(parent_imp, left, right, kind, min_inst, min_gain):
    lc, rc = float(sum(left)), float(sum(right))
    if lc < min_inst or rc < min_inst:
        return DOUBLE_MIN, False, None, None
    limp, rimp = to.calculate(left, kind), to.calculate(right, kind)
    total = lc + rc
    gain = parent_imp - (lc / total) * limp - (rc / total) * rimp
    if gain < min_gain:
        return DOUBLE_MIN, False, None, None
    return gain, True, limp, rimp


def grow_tree(codes, y, thr, C, w, seed, tree, m, max_depth=5, min_inst=1, min_gain=0.0, kind="gini"):
    """One tree, node by node, every row counted with its weight w (0: not in the bag), node i searching subset(seed,
    tree, i) (root 1, children 2i and 2i + 1).  Returns the pruned tree as nested dicts."""
    n, k = codes.shape
    rows0 = np.flatnonzero(w > 0)

    def counts_of(rows):
        out = np.zeros(C)
        np.add.at(out, y[rows], w[rows].astype(np.float64))
        return out

    def node(rows, depth, nid):
        total = counts_of(rows)
        parent_imp = to.calculate(total, kind)
        best = None
        for j in subset(seed, tree, nid, k, m):
            if not thr[j]:
                continue
            hist = np.zeros((len(thr[j]) + 1, C))
            np.add.at(hist, (codes[rows, j], y[rows]), w[rows].astype(np.float64))
            left = np.zeros(C)
            for i in range(len(thr[j])):
                left = left + hist[i]
                right = total - left
                gain, valid, limp, rimp = _stats(parent_imp, left, right, kind, min_inst, min_gain)
                if best is None or gain > best[0]:
                    best = (gain, valid, j, i, left.copy(), right.copy(), limp, rimp)
        nd = dict(counts=total, impurity=parent_imp, valid=best is not None and best[1], split=None)
        if best is None or best[0] <= 0 or depth == max_depth:
            return nd
        j, i = best[2], best[3]
        kids = []
        for sub, imp, cid in ((rows[codes[rows, j] <= i], best[6], 2 * nid), (rows[codes[rows, j] > i], best[7], 2 * nid + 1)):
            if depth + 1 == max_depth or abs(imp) < EPS:
                kids.append(dict(counts=counts_of(sub), impurity=imp, valid=True, split=None))
            else:
                kids.append(node(sub, depth + 1, cid))
        nd.update(split=(j, thr[j][i]), gain=best[0], left=kids[0], right=kids[1])
        return nd

    return prune(node(rows0, 0, 1))


def _pred(counts):
    best, top = -1, DOUBLE_MIN
    for c, v in enumerate(counts):
        if v > top:
            best, top = c, v
    return best


def prune(nd):
    """toNode(prune = true): leaves keep impurity -1 after an invalid search; two leaf children of one prediction merge
    into a leaf with the parent's impurity and counts."""
    if nd["split"] is None:
        return dict(leaf=True, counts=nd["counts"], impurity=nd["impurity"] if nd["valid"] else -1.0)
    left, right = prune(nd["left"]), prune(nd["right"])
    if left["leaf"] and right["leaf"] and _pred(left["counts"]) == _pred(right["counts"]):
        return dict(leaf=True, counts=nd["counts"], impurity=nd["impurity"])
    return dict(leaf=False, counts=nd["counts"], impurity=nd["impurity"], gain=nd["gain"], feature=nd["split"][0],
                threshold=nd["split"][1], left=left, right=right)


def fit(x, y, num_trees=20, max_depth=5, max_bins=32, min_inst=1, min_gain=0.0, kind="gini", m=None, rate=1.0,
        seed=None):
    """(trees as nested dicts, thresholds, m) of the forest; m defaults to "auto"'s."""
    x = np.asarray(x)
    y = np.asarray(y).astype(np.int64)
    n, k = x.shape
    C = int(y.max()) + 1
    if seed is None:
        seed = java_string_hash("org.apache.spark.ml.classification.RandomForestClassifier")
    if m is None:
        m = k if num_trees == 1 else int(math.ceil(math.sqrt(k)))
    thr = [to.splits(x[:, j], max_bins) for j in range(k)]
    codes = to.bins(x, thr)
    tab = table(num_trees, rate)
    trees = [grow_tree(codes, y, thr, C, weights(seed, t, range(n), tab), seed, t, m, max_depth, min_inst, min_gain,
                       kind) for t in range(num_trees)]
    return trees, thr, m


def arrays(root):
    """Breadth-first arrays (feature, threshold, left, right, counts, impurity, gain) of a pruned tree."""
    out = dict(feature=[], threshold=[], left=[], right=[], counts=[], impurity=[], gain=[])
    queue, i = [root], 0
    while i < len(queue):
        nd = queue[i]
        out["counts"].append(nd["counts"])
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


def transform(trees, x):
    """(raw, probability, prediction): raw_c = sum over trees in order from 0.0 of the leaf's counts[c] / total (a
    leaf of total 0 casts no vote), probability = raw / sum(raw), prediction = the first argmax of raw."""
    x = np.asarray(x).astype(np.float64)
    C = len(trees[0]["counts"])
    raw = np.zeros((len(x), C))
    for r in range(len(x)):
        acc = [0.0] * C
        for root in trees:
            nd = root
            while not nd["leaf"]:
                nd = nd["left"] if x[r, nd["feature"]] <= nd["threshold"] else nd["right"]
            total = 0.0
            for v in nd["counts"]:
                total += float(v)
            if total == 0:
                continue
            for c in range(C):
                acc[c] = acc[c] + float(nd["counts"][c]) / total
        raw[r] = acc
    s = np.zeros(len(x))
    for c in range(C):
        s = s + raw[:, c]
    with np.errstate(invalid="ignore", divide="ignore"):
        prob = raw / s[:, None]
    pred = np.array([_pred(v) for v in raw], np.float64)
    return raw, prob, pred
