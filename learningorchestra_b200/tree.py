"""Host side of the builder's tree classifiers (Spark 2.4's DecisionTreeClassifier, GBTClassifier and
RandomForestClassifier, DESIGN.md §3.6.4 to §3.6.6): the split candidates of every column from the device's sorted
columns and rank counts, the level-wise growth of one tree or of several in lockstep from the device's (node, feature,
bin, class) histograms, the pruning and the model's arrays, and RandomForest's bagging tables, feature subsets and
votes.  Nothing here touches the device: the callers hand in the counts (:mod:`classifier` on an ``Engine`` or
``ShardedEngine``, the tests with numpy stand-ins)."""
from __future__ import annotations

import math

import numpy as np

MAX_DEPTH = 30              # Spark's ParamValidators.inRange(0, 30)
MAX_BINS = 256              # LO_DT_MAX_BINS: a bin index is a byte (Spark has no upper bound)
MAX_CLASSES = 100           # Spark's Classifier.getNumClasses maxNumClasses
EPSILON = 2.220446049250313e-16     # Spark's Utils.EPSILON: 2^-52
DOUBLE_MIN = -np.finfo(np.float64).max   # Scala's Double.MinValue: the gain of an invalid split
IMPURITIES = ("gini", "entropy")
VARIANCE = "variance"       # GBT's regression trees (DESIGN.md §3.6.5): the level gives lo_gb_level's words
WORDS = 5                   # LO_GB_WORDS: count, sum of q1 + 2^60 (lo, hi), sum of q2 (lo, hi) per (node, feature, bin)
MAX_DRAWS = 32              # LO_RF_MAX_DRAWS: entries of a bagging threshold table


def num_splits(max_bins: int, n: int) -> int:
    """findSplits' split count of a continuous feature: min(maxBins, numExamples) - 1."""
    return min(max_bins, n) - 1


def greedy(values, counts, nsplits: int, n: int) -> list[float]:
    """findSplitsForContinuousFeature's loop, literally, over the distinct values ascending with their counts: midpoints
    of every neighbour pair when there are no more than ``nsplits`` of them, else the greedy walk toward stride,
    2 stride, ... (stride = n / (nsplits + 1)) in f64."""
    values = [float(v) for v in values]
    counts = [int(c) for c in counts]
    m = len(values)
    if m - 1 <= nsplits:
        return [(values[i - 1] + values[i]) / 2.0 for i in range(1, m)]
    stride = n / (nsplits + 1)
    out = []
    index, current, target = 1, counts[0], stride
    while index < m:
        previous = current
        current += counts[index]
        if abs(previous - target) < abs(current - target):
            out.append((values[index - 1] + values[index]) / 2.0)
            target += stride
        index += 1
    return out


class Need(Exception):
    """The replay needs Q(K), the least value v with #(x <= v) >= K, which it has not been told."""


def _lookup(entries, K):
    for e in entries:
        if e[1] < K <= e[2]:
            return e
    raise Need(K)


def replay(n: int, nsplits: int, entries) -> list[float]:
    """:func:`greedy`'s walk without the value counts: ``entries`` are known points (value, lt, le) of the column
    (#(x < value), #(x <= value)); Q(K) is the entry with lt < K <= le.  Raises :class:`Need` naming the first Q(K) it
    lacks.  Walking index by index, a split can only fall at the first value whose le exceeds the target (or the index
    after it, or later when rounding makes the gaps equal): the values before it have le <= target, so their gaps only
    shrink.  The walk therefore jumps to max(next index, Q(floor(target) + 1)) and checks the loop's own condition
    there; past the last target below n no split can fall."""
    stride = n / (nsplits + 1)
    target = stride
    out = []
    first = _lookup(entries, 1)
    if first[2] >= n:
        return out
    nxt = _lookup(entries, first[2] + 1)
    while True:
        if not target < n:
            return out
        j = _lookup(entries, math.floor(target) + 1)
        w = j if j[0] > nxt[0] else nxt
        if abs(w[1] - target) < abs(w[2] - target):
            prev = _lookup(entries, w[1])
            out.append((prev[0] + w[0]) / 2.0)
            target += stride
        if w[2] >= n:
            return out
        nxt = _lookup(entries, w[2] + 1)


def replay_requests(n: int, nsplits: int, entries, need: int) -> set[int]:
    """The ranks to ask for next: the missing one and, so that a round settles many steps at once, the neighbours
    (previous and next value) of every known entry and the first rank of every target below n."""
    want = {need}
    for _v, lt, le in entries:
        if lt >= 1:
            want.add(lt)
        if le < n:
            want.add(le + 1)
    stride, target = n / (nsplits + 1), n / (nsplits + 1)
    while target < n and len(want) < 4 * (nsplits + 2):
        want.add(math.floor(target) + 1)
        target += stride
    known = lambda K: any(e[1] < K <= e[2] for e in entries)
    return {K for K in want if not known(K)}


def first_targets(n: int, nsplits: int) -> set[int]:
    """The first round's ranks: the least value and the first rank above every target below n."""
    want, stride = {1}, n / (nsplits + 1)
    target = stride
    while target < n:
        want.add(math.floor(target) + 1)
        target += stride
    return want


def code_bits(f32: bool) -> int:
    return 32 if f32 else 64


def encode(v: float, f32: bool) -> int:
    """The order-preserving code of a finite value (-0.0 as 0.0), as the device sorts it."""
    if v == 0.0:
        v = 0.0
    if f32:
        b = int(np.array(v, np.float32).view(np.uint32))
        return (~b & 0xFFFFFFFF) if b >> 31 else b | 0x80000000
    b = int(np.array(v, np.float64).view(np.uint64))
    return (~b & 0xFFFFFFFFFFFFFFFF) if b >> 63 else b | (1 << 63)


def decode(code: int, f32: bool) -> float:
    if f32:
        b = code & 0x7FFFFFFF if code >> 31 else ~code & 0xFFFFFFFF
        return float(np.array(b, np.uint32).view(np.float32))
    b = code & ~(1 << 63) if code >> 63 else ~code & 0xFFFFFFFFFFFFFFFF
    return float(np.array(b, np.uint64).view(np.float64))


def order_statistics(rank, queries, f32: bool):
    """Q(K) of every query (column, K) by bisection on the codes: the least code c with #(x <= c) >= K over every member,
    ``rank(cols, codes) -> (lt, le)`` summed over them.  One rank call per round, 32 rounds at f32 and 64 at f64, and one
    more for the lt / le of the answer.  Returns [(value, lt, le)] in the queries' order."""
    if not queries:
        return []
    cols = np.array([c for c, _K in queries], np.int32)
    want = np.array([K for _c, K in queries], np.int64)
    bits = code_bits(f32)
    lo = np.zeros(len(queries), np.uint64)
    hi = np.full(len(queries), (1 << bits) - 1, np.uint64)
    for _ in range(bits):
        mid = lo + (hi - lo) // np.uint64(2)
        _lt, le = rank(cols, mid)
        up = le >= want
        hi = np.where(up, mid, hi)
        lo = np.where(up, lo, mid + np.uint64(1))
    lt, le = rank(cols, lo)
    return [(decode(int(c), f32), int(a), int(b)) for c, a, b in zip(lo, lt, le)]


def column_thresholds(n: int, max_bins: int, distinct, rank, f32: bool, kc: int) -> tuple[list[list[float]], int]:
    """The split thresholds of kc sorted columns over n rows.  ``distinct[c]`` is (values, counts) of column c when
    every member had few enough distinct values to list them (merged here), else None; ``rank(cols, codes)`` answers
    rank counts summed over the members.  Listed columns take :func:`greedy` on their value counts; the others are
    replayed (:func:`replay`) from order statistics asked for in rounds.  Returns (thresholds, rank rounds)."""
    nsplits = num_splits(max_bins, n)
    out: list = [None] * kc
    entries: dict[int, list] = {}
    pending: dict[int, set] = {}
    for c in range(kc):
        if distinct[c] is not None:
            out[c] = greedy(distinct[c][0], distinct[c][1], nsplits, n)
        else:
            entries[c], pending[c] = [], first_targets(n, nsplits)
    rounds = 0
    while pending:
        queries = [(c, K) for c in sorted(pending) for K in sorted(pending[c])]
        got = order_statistics(rank, queries, f32)
        rounds += 1
        for (c, _K), e in zip(queries, got):
            entries[c].append(e)
        pending = {}
        for c in entries:
            if out[c] is not None:
                continue
            try:
                out[c] = replay(n, nsplits, entries[c])
            except Need as need:
                pending[c] = replay_requests(n, nsplits, entries[c], need.args[0])
    return out, rounds


def merge_distinct(members):
    """The union of the members' listed distinct values with their counts added (each member (ndistinct, values,
    counts) of one column; values None when it had too many to list), or None when any member did not list them."""
    if any(m[1] is None for m in members):
        return None
    vals = np.concatenate([m[1] for m in members])
    cnts = np.concatenate([m[2] for m in members])
    u, inv = np.unique(vals, return_inverse=True)
    total = np.zeros(len(u), np.int64)
    np.add.at(total, inv, cnts)
    return u, total


# ---- impurity and gains: Spark's Gini / Entropy.calculate and calculateImpurityStats, operation by operation --------
def impurity(counts: np.ndarray, total: np.ndarray, kind: str) -> np.ndarray:
    """Impurity of class counts (..., C) with their totals (...): Gini 1 - sum freq^2, Entropy -sum freq log2(freq) with
    log2(x) = log(x) / log(2), the classes in order and every operation rounded on its own; 0 where total == 0."""
    counts = np.asarray(counts, np.float64)
    total = np.asarray(total, np.float64)
    safe = np.where(total == 0, 1.0, total)
    out = np.full(total.shape, 1.0 if kind == "gini" else 0.0)
    log2 = math.log(2.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        for c in range(counts.shape[-1]):
            freq = counts[..., c] / safe
            if kind == "gini":
                out = out - freq * freq
            else:
                term = freq * (np.log(freq) / log2)
                out = np.where(counts[..., c] != 0, out - term, out)
    return np.where(total == 0, 0.0, out)


def best_splits(hist: np.ndarray, nthr: np.ndarray, kind: str, min_instances: int, min_info_gain: float,
                features: np.ndarray | None = None):
    """binsToBestSplit for every node of a level at once.  hist: int64 (nodes, k, nbins, C).  The left counts of split i
    are the prefix over bins 0 .. i, the right ones the node's total minus them.  ``nthr``: the splits of each of the k
    features (k,), or of each node's (nodes, k) when ``features`` (int (nodes, k), ascending) lists every node's own
    features, hist's feature axis following them.  Returns a dict of per-node arrays: ``feature`` (-1: no feature has a
    split), ``bin``, ``gain`` (Double.MinValue when invalid), ``impurity`` (the node's), ``left`` / ``right`` (class
    counts), ``left_impurity`` / ``right_impurity``, ``valid`` and ``total`` (the node's class counts)."""
    nodes, k, nbins, C = hist.shape
    total = hist[:, 0].sum(axis=1)                              # (nodes, C)
    tsum = total.sum(axis=1).astype(np.float64)
    node_imp = impurity(total, tsum, kind)
    out = {"total": total, "impurity": node_imp}
    ns = max(int(nthr.max()) if k else 0, 0)
    if ns == 0:
        out.update(feature=np.full(nodes, -1), bin=np.zeros(nodes, np.int64), gain=np.full(nodes, DOUBLE_MIN),
                   valid=np.zeros(nodes, bool), left=np.zeros_like(total), right=np.zeros_like(total),
                   left_impurity=np.zeros(nodes), right_impurity=np.zeros(nodes))
        return out
    left = np.cumsum(hist[:, :, :ns], axis=2)                   # (nodes, k, ns, C): split i = bins 0 .. i
    right = total[:, None, None, :] - left
    lc = left.sum(axis=3).astype(np.float64)
    rc = right.sum(axis=3).astype(np.float64)
    out = _choose(out, node_imp, left, right, lc, rc, impurity(left, lc, kind), impurity(right, rc, kind), nthr,
                  min_instances, min_info_gain)
    if features is not None:
        f = out["feature"]
        out["feature"] = np.where(f >= 0, np.asarray(features)[np.arange(nodes), np.maximum(f, 0)], -1)
    return out


def _choose(out, node_imp, left, right, lc, rc, limp, rimp, nthr, min_instances, min_info_gain):
    """binsToBestSplit's choice from every candidate's (nodes, k, ns) counts lc / rc and impurities limp / rimp:
    calculateImpurityStats' gain, the minInstancesPerNode and minInfoGain rules and the first maximum.  ``nthr``: (k,)
    splits per feature, or (nodes, k) per node."""
    nodes, k, ns = lc.shape
    tc = lc + rc
    with np.errstate(invalid="ignore", divide="ignore"):
        wl = lc / tc
        wr = rc / tc
        gain = node_imp[:, None, None] - wl * limp - wr * rimp
    real = np.arange(ns) < np.asarray(nthr)[..., None]         # (k, ns) or (nodes, k, ns): split i exists for feature j
    real = real if real.ndim == 3 else real[None]
    ok = (lc >= min_instances) & (rc >= min_instances)
    ok &= ~(gain < min_info_gain)
    gain = np.where(ok, gain, DOUBLE_MIN)
    gain = np.where(real, gain, -np.inf)                        # never chosen over a real split, valid or not
    flat = gain.reshape(nodes, -1)
    at = flat.argmax(axis=1)                                    # the first maximum: features, then splits, in order
    j, i = np.divmod(at, ns)
    r = np.arange(nodes)
    has = real.reshape(len(real), -1).any(axis=1)               # per node (one for all with per-feature nthr)
    out.update(feature=np.where(has, j, -1), bin=i, gain=flat[r, at], valid=ok[r, j, i] & has,
               left=left[r, j, i], right=right[r, j, i], left_impurity=limp[r, j, i], right_impurity=rimp[r, j, i])
    return out


def add_words(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """Two uint64 arrays of lo_gb_level's words (..., WORDS) added as integers: the counts, and each 128-bit (lo, hi)
    sum with the lo word's carry into the hi word — exact, so shards add in any order to the same words."""
    a, b = np.asarray(a, np.uint64), np.asarray(b, np.uint64)
    out = a + b
    for p in (1, 3):
        out[..., p + 1] += (out[..., p] < a[..., p]).astype(np.uint64)
    return out


def word_stats(words: np.ndarray, nsplits: int):
    """(left, right, total) f64 statistics (count, sum, sumsq) of lo_gb_level's words (nodes, k, nbins, WORDS):
    lo_gb_stats' integer prefix over the bins, right = total - left, each statistic rounded to f64 once."""
    import ctypes as C
    from . import _native as N
    words = np.ascontiguousarray(words, np.uint64)
    nodes, k, nbins, _w = words.shape
    left = np.zeros((nodes, k, nsplits, 3))
    right = np.zeros((nodes, k, nsplits, 3))
    total = np.zeros((nodes, 3))
    N.check(N.load().lo_gb_stats(words.ctypes.data_as(C.c_void_p), nodes, k, nbins, nsplits,
                                 left.ctypes.data_as(C.c_void_p), right.ctypes.data_as(C.c_void_p),
                                 total.ctypes.data_as(C.c_void_p)))
    return left, right, total


def variance(stats: np.ndarray) -> np.ndarray:
    """Spark's Variance.calculate of (..., 3) statistics (count, sum, sumSq): 0 where count == 0, else
    (sumSq - sum * sum / count) / count."""
    cnt, s, sq = stats[..., 0], stats[..., 1], stats[..., 2]
    safe = np.where(cnt == 0, 1.0, cnt)
    return np.where(cnt == 0, 0.0, (sq - s * s / safe) / safe)


def variance_splits(words: np.ndarray, nthr: np.ndarray, min_instances: int, min_info_gain: float):
    """:func:`best_splits` for regression trees from lo_gb_level's words: ``total`` / ``left`` / ``right`` are the
    (count, sum, sumSq) statistics and the impurities Variance's."""
    nodes, k = words.shape[:2]
    ns = max(int(nthr.max()) if k else 0, 0)
    left, right, total = word_stats(words, ns)
    out = {"total": total, "impurity": variance(total)}
    if ns == 0:
        out.update(feature=np.full(nodes, -1), bin=np.zeros(nodes, np.int64), gain=np.full(nodes, DOUBLE_MIN),
                   valid=np.zeros(nodes, bool), left=np.zeros_like(total), right=np.zeros_like(total),
                   left_impurity=np.zeros(nodes), right_impurity=np.zeros(nodes))
        return out
    return _choose(out, out["impurity"], left, right, left[..., 0], right[..., 0], variance(left), variance(right), nthr,
                   min_instances, min_info_gain)


class Tree:
    """A fitted tree in arrays, node 0 the root, children after their parent: ``feature`` (int32, -1 for a leaf),
    ``threshold`` and ``bin`` (the split: left when x <= threshold, i.e. code <= bin), ``left`` / ``right`` (int32, -1
    for a leaf), ``counts`` (float64 [nodes, C], the node's class counts), ``prediction`` (first argmax of them),
    ``impurity`` (-1 for a leaf whose split search was invalid), ``gain`` (NaN for a leaf)."""

    def __init__(self, feature, threshold, left, right, counts, impurity_, gain, num_classes: int):
        self.feature = np.asarray(feature, np.int32)
        self.threshold = np.asarray(threshold, np.float64)
        self.left = np.asarray(left, np.int32)
        self.right = np.asarray(right, np.int32)
        self.counts = np.asarray(counts, np.float64).reshape(len(self.feature), num_classes or 3)
        self.impurity = np.asarray(impurity_, np.float64)
        self.gain = np.asarray(gain, np.float64)
        self.num_classes = int(num_classes)
        self.prediction = self.counts.argmax(axis=1).astype(np.float64) if len(self.feature) else np.zeros(0)
        if num_classes == 0:                 # a regression tree: counts are (count, sum, sumSq), prediction sum / count
            with np.errstate(invalid="ignore", divide="ignore"):
                self.prediction = self.counts[:, 1] / self.counts[:, 0]

    @property
    def num_nodes(self) -> int:
        return len(self.feature)

    @property
    def depth(self) -> int:
        d = np.zeros(self.num_nodes, np.int64)
        for i in range(self.num_nodes):
            if self.feature[i] >= 0:
                d[self.left[i]] = d[self.right[i]] = d[i] + 1
        return int(d.max()) if self.num_nodes else 0


def grow(level, thresholds, num_classes: int, max_depth: int, kind: str, min_instances: int, min_info_gain: float,
         trees: int | None = None, subsets=None):
    """Spark's level-wise growth and toNode(prune = true).  ``level(splits, nnodes) -> hist`` counts one level: splits
    None for the root, else int32 (parents, 4) rows (feature, bin, left slot, right slot) of the previous level's nodes
    in slot order (feature -1: the node did not split; slot -1: a leaf child); hist int64 (nnodes, k, nbins, C).
    ``kind`` VARIANCE grows a regression tree (num_classes 0): hist is lo_gb_level's uint64 words (nnodes, k, nbins,
    WORDS) and a node's counts its (count, sum, sumSq).  Returns a :class:`Tree` and the per-level histograms' node
    counts.  ``trees``: that many trees grow in lockstep, one level call for all of them, their nodes in slot order tree
    by tree (the root level's slot t is tree t's root), and the result is a list of Trees.  ``subsets(t, node)``: the
    ascending features tree t's node (Spark's index: root 1, children 2i and 2i + 1) searches; the level is then called
    as ``level(splits, nnodes, features)`` with features int32 (nnodes, m) and hist's feature axis following them."""
    nthr = np.array([len(t) for t in thresholds], np.int64)
    # learning nodes: dict(tree, id, depth, stats: counts / impurity / gain / valid, split, children)
    nodes = [dict(tree=t, id=1, depth=0, counts=None, impurity=None, gain=np.nan, valid=True, split=None, kids=None)
             for t in range(1 if trees is None else trees)]
    active = list(range(len(nodes)))  # the learning nodes of this level, in slot order
    splits = None
    shapes = []
    while active:
        feats = None
        if subsets is None:
            hist = level(splits, len(active))
        else:
            feats = np.array([subsets(nodes[i]["tree"], nodes[i]["id"]) for i in active], np.int32)
            hist = level(splits, len(active), feats)
        shapes.append(len(active))
        if kind == VARIANCE:
            best = variance_splits(hist, nthr, min_instances, min_info_gain)
        else:
            best = best_splits(hist, nthr if feats is None else nthr[feats], kind, min_instances, min_info_gain, feats)
        nxt, rows = [], []
        for s, idx in enumerate(active):
            node = nodes[idx]
            d = node["depth"]
            node["counts"] = best["total"][s]
            node["impurity"] = best["impurity"][s]
            node["gain"] = best["gain"][s]
            node["valid"] = bool(best["valid"][s])
            if best["gain"][s] <= 0 or d == max_depth or best["feature"][s] < 0:
                rows.append((-1, 0, -1, -1))
                continue
            j, i = int(best["feature"][s]), int(best["bin"][s])
            node["split"] = (j, i, thresholds[j][i])
            child_leaf = d + 1 == max_depth
            kids = []
            slots = []
            for side, cid in (("left", 2 * node["id"]), ("right", 2 * node["id"] + 1)):
                imp = best[side + "_impurity"][s]
                leaf = child_leaf or abs(imp) < EPSILON
                nodes.append(dict(tree=node["tree"], id=cid, depth=d + 1, counts=best[side][s], impurity=imp,
                                  gain=np.nan, valid=True, split=None, kids=None))
                kids.append(len(nodes) - 1)
                if leaf:
                    slots.append(-1)
                else:
                    slots.append(len(nxt))
                    nxt.append(len(nodes) - 1)
            node["kids"] = kids
            rows.append((j, i, slots[0], slots[1]))
        splits = np.array(rows, np.int32).reshape(-1, 4)
        active = nxt
    grown = [_to_tree(nodes, num_classes, t) for t in range(1 if trees is None else trees)]
    return (grown[0] if trees is None else grown), shapes


def _to_tree(nodes, num_classes: int, root: int = 0) -> Tree:
    """toNode(prune = true) of the tree whose root is nodes[root] into breadth-first arrays: two leaf children of equal
    prediction (the first argmax of the counts; a regression tree's sum / count, as f64) merge into a leaf with the
    parent's impurity and counts (bottom-up, so merges cascade); an invalid split search leaves impurity -1."""
    def prediction(counts):
        if num_classes == 0:
            return float(counts[1] / counts[0])
        return int(np.argmax(counts))

    def build(i):
        n = nodes[i]
        imp = float(n["impurity"]) if n["valid"] else -1.0
        if n["kids"] is None:
            return ("leaf", np.asarray(n["counts"], np.float64), imp)
        l, r = build(n["kids"][0]), build(n["kids"][1])
        if l[0] == "leaf" and r[0] == "leaf" and prediction(l[1]) == prediction(r[1]):
            return ("leaf", np.asarray(n["counts"], np.float64), float(n["impurity"]))
        return ("split", np.asarray(n["counts"], np.float64), float(n["impurity"]), float(n["gain"]), n["split"], l, r)

    top = build(root)
    feature, threshold, left, right, counts, imps, gains = [], [], [], [], [], [], []
    queue = [top]
    while queue:
        nd = queue.pop(0)
        at = len(feature)
        counts.append(nd[1])
        imps.append(nd[2])
        if nd[0] == "leaf":
            feature.append(-1), threshold.append(np.nan), left.append(-1), right.append(-1), gains.append(np.nan)
            continue
        j, _i, t = nd[4]
        feature.append(j), threshold.append(t), gains.append(nd[3])
        base = at + 1 + len(queue)
        left.append(base), right.append(base + 1)
        queue += [nd[5], nd[6]]
    return Tree(feature, threshold, left, right, np.array(counts).reshape(-1, num_classes or 3), imps, gains, num_classes)


# ---- RandomForest (DESIGN.md §3.6.6): bagging, feature subsets, votes ---------------------------------------------
M64 = (1 << 64) - 1
STRATEGIES = ("auto", "all", "onethird", "sqrt", "log2")


def java_hash(text: str) -> int:
    """java.lang.String.hashCode as a signed 32-bit int (UTF-16 code units; these names are ASCII)."""
    h = 0
    for ch in text:
        h = (31 * h + ord(ch)) & 0xFFFFFFFF
    return h - (1 << 32) if h >> 31 else h


# Spark's HasSeed default: this.getClass.getName.hashCode.toLong
DEFAULT_SEED = java_hash("org.apache.spark.ml.classification.RandomForestClassifier")


def splitmix(z):
    """splitmix64's step of uint64 values: add the golden-ratio increment, then the finaliser (k_rf_level's rf_mix)."""
    with np.errstate(over="ignore"):
        z = np.asarray(z, np.uint64) + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def subset_size(strategy: str, k: int, num_trees: int) -> int:
    """The features m a node searches (DecisionTreeMetadata.buildMetadata): "auto" is "all" for one tree, else "sqrt";
    "all" k, "sqrt" ceil(sqrt k), "log2" max(1, ceil(log2 k)), "onethird" ceil(k / 3), an integer string n: min(n,
    k), a real string r in (0, 1]: ceil(r k), each in f64 as Spark computes it.  Anything else is a ValueError."""
    import re
    s = strategy.lower() if isinstance(strategy, str) else None
    if s == "auto":
        s = "all" if num_trees == 1 else "sqrt"
    if s == "all":
        return k
    if s == "sqrt":
        return int(math.ceil(math.sqrt(k)))
    if s == "log2":
        return max(1, int(math.ceil(math.log(k) / math.log(2))))
    if s == "onethird":
        return int(math.ceil(k / 3.0))
    if s is not None and re.fullmatch(r"[1-9]\d*", s):
        return min(int(s), k)
    if s is not None and re.fullmatch(r"0?\.\d*[1-9]\d*|1\.0+", s):
        return int(math.ceil(float(s) * k))
    raise ValueError(f"feature_subset_strategy must be one of {list(STRATEGIES)}, an integer n > 0 or a real in (0, 1] "
                     f"as a string, not {strategy!r}")


def draw_table(num_trees: int, rate: float) -> list[int]:
    """The bagging thresholds T (ascending u64) of lo_rf_level: a row's weight is #{j : u >= T_j}.  One tree at rate 1:
    [0] (every weight 1); one tree below rate 1: Bernoulli, [floor(2^64 (1 - rate))]; several trees: Poisson(rate),
    T_j = floor(2^64 P(X <= j)) for j = 0 and every later j whose T_j is below 2^64 - 1.  Computed in 60-digit decimal
    from the exact value of ``rate`` (e^-rate correctly rounded there), never with floating exp."""
    from decimal import ROUND_FLOOR, Decimal, localcontext
    from fractions import Fraction
    if num_trees == 1:
        return [0] if rate == 1.0 else [math.floor((1 - Fraction(rate)) * (1 << 64))]
    with localcontext() as ctx:
        ctx.prec = 60
        lam = Decimal(rate)
        term = (-lam).exp()
        cdf, out, j = term, [], 0
        while True:
            t = int((cdf * (1 << 64)).to_integral_value(rounding=ROUND_FLOOR))
            if j > 0 and t >= M64:
                break
            out.append(min(t, M64))
            j += 1
            term = term * lam / j
            cdf += term
    if len(out) > MAX_DRAWS:
        raise ValueError(f"the bagging table of rate {rate!r} needs {len(out)} entries, LO_RF_MAX_DRAWS = {MAX_DRAWS}")
    return out


def feature_subset(seed: int, tree: int, node: int, k: int, m: int) -> np.ndarray:
    """The m features (ascending) node ``node`` (Spark's index) of tree ``tree`` searches: those with the m least keys
    splitmix(splitmix(splitmix(splitmix(~seed) ^ tree) ^ node) ^ j), ties by feature index; every feature when m == k."""
    if m >= k:
        return np.arange(k, dtype=np.int32)
    base = splitmix(splitmix(splitmix(np.uint64(~seed & M64)) ^ np.uint64(tree)) ^ np.uint64(node))
    keys = splitmix(base ^ np.arange(k, dtype=np.uint64))
    return np.sort(np.lexsort((np.arange(k), keys))[:m]).astype(np.int32)


def votes(tree: Tree) -> np.ndarray:
    """Every node's class counts over their total (summed in class order), each division rounded on its own; 0 for a
    node of no counts, so that such a leaf casts no vote (RandomForestClassificationModel.predictRaw)."""
    counts = tree.counts
    total = np.zeros(len(counts))
    for c in range(counts.shape[1]):
        total = total + counts[:, c]
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(total[:, None] == 0, 0.0, counts / total[:, None])
