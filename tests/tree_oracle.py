"""Numpy restatement of Spark 2.4's DecisionTreeClassifier (DESIGN.md §3.6.4), written node by node and split by split
as Spark's RandomForest does, so that it shares no code with learningorchestra_b200.tree: the split candidates
(findSplitsForContinuousFeature on every row), the bins (Arrays.binarySearch), the level-wise growth
(binsToBestSplit / calculateImpurityStats with Gini and Entropy in Spark's operation order), toNode(prune = true) and
the transform.  Beside logistic_oracle.py for the same reason: a test oracle, not part of the package."""
import math

import numpy as np

EPS = 2.220446049250313e-16
DOUBLE_MIN = -1.7976931348623157e308


def value_counts(col):
    """The distinct values of a column, ascending, widened to f64 with -0.0 as 0.0, and their counts."""
    v = np.asarray(col).astype(np.float64) + 0.0
    return np.unique(v, return_counts=True)


def splits(col, max_bins):
    """findSplitsForContinuousFeature over every row (numSamples = n)."""
    n = len(col)
    num_splits = min(max_bins, n) - 1
    vals, cnts = value_counts(col)
    possible = len(vals) - 1
    if possible == 0:
        return []
    if possible <= num_splits:
        return [(float(vals[i - 1]) + float(vals[i])) / 2.0 for i in range(1, len(vals))]
    stride = float(n) / (num_splits + 1)
    out = []
    index = 1
    current = int(cnts[0])
    target = stride
    while index < len(vals):
        previous = current
        current += int(cnts[index])
        previous_gap = abs(previous - target)
        current_gap = abs(current - target)
        if previous_gap < current_gap:
            out.append((float(vals[index - 1]) + float(vals[index])) / 2.0)
            target += stride
        index += 1
    return out


def binary_search(t, x):
    """java.util.Arrays.binarySearch(double[], double) over every value of x at once, step for step: mid = (low + high)
    >>> 1, `<` and `>` first, then the signed order of doubleToLongBits for values that compare equal.  Returns the hit's
    index or the insertion point, as findBin reads the result (-idx - 1 back to idx)."""
    t = np.asarray(t, np.float64)
    x = np.asarray(x, np.float64)
    low = np.zeros(len(x), np.int64)
    high = np.full(len(x), len(t) - 1, np.int64)
    found = np.full(len(x), -1, np.int64)
    kb = x.view(np.int64)
    while True:
        live = (low <= high) & (found < 0)
        if not live.any():
            break
        mid = (low + high) >> 1
        v = t[np.where(live, mid, 0)]
        vb = v.view(np.int64)
        less = v < x
        more = v > x
        hit = ~less & ~more & (vb == kb)
        up = less | (~less & ~more & (vb < kb))
        down = more | (~less & ~more & (vb > kb))
        found = np.where(live & hit, mid, found)
        low = np.where(live & up, mid + 1, low)
        high = np.where(live & down, mid - 1, high)
    return np.where(found >= 0, found, low)


def bins(x, thresholds):
    """Every value's bin: Arrays.binarySearch's index on a hit, else -idx-1 of its insertion point (findBin)."""
    x = np.asarray(x).astype(np.float64)
    out = np.zeros(x.shape, np.int64)
    for j, t in enumerate(thresholds):
        out[:, j] = binary_search(t, x[:, j]) if len(t) else 0
    return out


def calculate(counts, kind):
    total = 0.0
    for c in counts:
        total += float(c)
    if total == 0:
        return 0.0
    if kind == "gini":
        imp = 1.0
        for c in counts:
            freq = float(c) / total
            imp -= freq * freq
        return imp
    imp = 0.0
    for c in counts:
        if c != 0:
            freq = float(c) / total
            imp -= freq * (float(np.log(freq)) / float(np.log(2.0)))
    return imp


def _stats(parent_imp, left, right, kind, min_inst, min_gain):
    lc, rc = float(sum(left)), float(sum(right))
    if lc < min_inst or rc < min_inst:
        return DOUBLE_MIN, False, None, None
    limp, rimp = calculate(left, kind), calculate(right, kind)
    total = lc + rc
    gain = parent_imp - (lc / total) * limp - (rc / total) * rimp
    if gain < min_gain:
        return DOUBLE_MIN, False, None, None
    return gain, True, limp, rimp


def fit(x, y, max_depth=5, max_bins=32, min_inst=1, min_gain=0.0, kind="gini", ties=None):
    """The tree as nested dicts (after pruning) and the thresholds.  ``ties``: a list that receives, for every node
    that splits, the gap between its best gain and the next best among its candidates; a candidate whose bin holds none
    of the node's rows is left out, since it splits them exactly as the candidate before it (for tests that need no
    near-ties)."""
    x = np.asarray(x)
    y = np.asarray(y).astype(np.int64)
    n, k = x.shape
    C = int(y.max()) + 1
    thr = [splits(x[:, j], max_bins) for j in range(k)]
    b = bins(x, thr)

    def counts_of(rows):
        return np.bincount(y[rows], minlength=C).astype(np.float64)

    def node(rows, depth, imp_known):
        total = counts_of(rows)
        parent_imp = calculate(total, kind)
        best = None                     # (gain, valid, j, i, left, right, limp, rimp)
        gains = []
        for j in range(k):
            if not thr[j]:
                continue
            hist = np.zeros((len(thr[j]) + 1, C))
            np.add.at(hist, (b[rows, j], y[rows]), 1)
            left = np.zeros(C)
            for i in range(len(thr[j])):
                left = left + hist[i]
                right = total - left
                gain, valid, limp, rimp = _stats(parent_imp, left, right, kind, min_inst, min_gain)
                if i == 0 or not np.array_equal(hist[i], np.zeros(C)):     # an empty bin repeats the last partition
                    gains.append(gain)
                if best is None or gain > best[0]:
                    best = (gain, valid, j, i, left.copy(), right.copy(), limp, rimp)
        if ties is not None and len(gains) > 1 and best is not None and best[0] > 0 and depth < max_depth:
            others = sorted(gains, reverse=True)
            ties.append(others[0] - others[1])
        leaf = dict(counts=total, impurity=parent_imp, valid=True, split=None)
        if best is None:
            leaf["valid"] = False
            return leaf
        gain, valid = best[0], best[1]
        leaf["valid"] = valid
        if gain <= 0 or depth == max_depth:
            return leaf
        j, i = best[2], best[3]
        go_left = rows[b[rows, j] <= i]
        go_right = rows[b[rows, j] > i]
        kids = []
        for sub, imp in ((go_left, best[6]), (go_right, best[7])):
            if depth + 1 == max_depth or abs(imp) < EPS:
                kids.append(dict(counts=counts_of(sub), impurity=imp, valid=True, split=None))
            else:
                kids.append(node(sub, depth + 1, imp))
        return dict(counts=total, impurity=parent_imp, valid=True, split=(j, thr[j][i]), gain=gain,
                    left=kids[0], right=kids[1])

    return prune(node(np.arange(n), 0, None)), thr


def prediction(counts):
    best, top = -1, DOUBLE_MIN
    for c, v in enumerate(counts):
        if v > top:
            best, top = c, v
    return best


def prune(nd):
    """toNode(prune = true): a leaf keeps impurity -1 when its split search was invalid; two leaf children of equal
    prediction become one leaf with the parent's impurity and counts."""
    if nd["split"] is None:
        return dict(leaf=True, counts=nd["counts"], impurity=nd["impurity"] if nd["valid"] else -1.0)
    left, right = prune(nd["left"]), prune(nd["right"])
    if left["leaf"] and right["leaf"] and prediction(left["counts"]) == prediction(right["counts"]):
        return dict(leaf=True, counts=nd["counts"], impurity=nd["impurity"])
    return dict(leaf=False, counts=nd["counts"], impurity=nd["impurity"], gain=nd["gain"], feature=nd["split"][0],
                threshold=nd["split"][1], left=left, right=right)


def arrays(root):
    """Breadth-first arrays (feature, threshold, left, right, counts, impurity, gain) of a pruned tree."""
    out = dict(feature=[], threshold=[], left=[], right=[], counts=[], impurity=[], gain=[])
    queue = [root]
    i = 0
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


def transform(root, x):
    """(raw, probability, prediction) of every row: the leaf's counts, counts / their sum, the first argmax."""
    x = np.asarray(x).astype(np.float64)
    raw = []
    for r in range(len(x)):
        nd = root
        while not nd["leaf"]:
            nd = nd["left"] if x[r, nd["feature"]] <= nd["threshold"] else nd["right"]
        raw.append(nd["counts"])
    raw = np.array(raw, np.float64).reshape(len(x), -1)
    total = np.zeros(len(x))
    for c in range(raw.shape[1]):
        total = total + raw[:, c]
    prob = raw / total[:, None]
    pred = np.array([prediction(p) for p in prob], np.float64)
    return raw, prob, pred
