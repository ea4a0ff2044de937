"""CPU: the host side of the "NB" classifier — the header <-> ctypes mirror of lo_nb_*, the kernels in the SASS, the numpy
oracle against scikit-learn where the two agree, and the classifier module / the shards' merge with test doubles standing
in for the devices."""
import ctypes as C
import re
from types import SimpleNamespace

import numpy as np
import pytest

from learningorchestra_b200 import _native
from learningorchestra_b200.classifier import NaiveBayes, NaiveBayesModel, metrics, model_arrays
from learningorchestra_b200.engine import InvalidCellError
from learningorchestra_b200.sharding import ShardedEngine
from oracle import naive_bayes as nb

from test_text_shards_cpu import HEADER


def test_ctypes_mirror_of_the_naive_bayes_entry_points_matches_the_header():
    text = re.sub(r"/\*.*?\*/", "", HEADER.read_text(), flags=re.S)
    assert int(re.search(r"#define LO_ABI_VERSION (\d+)", text).group(1)) == _native.LO_ABI_VERSION == 7
    assert int(re.search(r"#define LO_NB_MAX_CLASSES\s+(\d+)", text).group(1)) == _native.LO_NB_MAX_CLASSES == 1024
    assert int(re.search(r"#define LO_NB_MAX_THETA\s+(\d+)", text).group(1)) == _native.LO_NB_MAX_THETA == 16384

    def params(name):
        return [p.strip() for p in re.search(r"\b%s\s*\(([^)]*)\)" % name, text).group(1).split(",")]

    assert params("lo_nb_labels") == ["lo_ctx *ctx", "const lo_table *y", "int64_t n", "double *labels_out",
                                      "int64_t capacity", "int64_t *nlabels", "lo_host_timing *timing"]
    assert params("lo_nb_fit") == ["lo_ctx *ctx", "const lo_table *x", "int64_t ld", "int32_t k", "const lo_table *y",
                                   "int64_t n", "const double *classes", "int32_t nclasses", "double *sums_out",
                                   "int64_t *counts_out", "lo_nb_info *info", "lo_host_timing *timing"]
    assert params("lo_nb_predict") == ["lo_ctx *ctx", "const lo_table *x", "int64_t ld", "int32_t k", "int64_t n",
                                       "const double *pi", "const double *theta", "int32_t nclasses", "lo_table *prob",
                                       "lo_table *raw", "lo_table *pred", "const lo_table *y", "const double *eval_labels",
                                       "int32_t neval", "int64_t *confusion_out", "lo_nb_info *info",
                                       "lo_host_timing *timing"]
    fields = re.search(r"typedef struct lo_nb_info \{(.*?)\} lo_nb_info;", text, re.S).group(1)
    assert re.findall(r"(\w+)\s+(\w+);", fields) == [("int64_t", "bad_row"), ("int32_t", "bad_col"), ("int32_t", "pad")]
    assert _native.NbInfo._fields_ == [("bad_row", C.c_int64), ("bad_col", C.c_int32), ("pad", C.c_int32)]
    P, T = C.c_void_p, C.POINTER(_native.HostTiming)
    assert _native.SIGNATURES["lo_nb_labels"] == (C.c_int, [P, P, C.c_int64, P, C.c_int64, C.POINTER(C.c_int64), T])
    assert _native.SIGNATURES["lo_nb_fit"] == (C.c_int, [P, P, C.c_int64, C.c_int32, P, C.c_int64, P, C.c_int32, P, P,
                                                         C.POINTER(_native.NbInfo), T])
    assert _native.SIGNATURES["lo_nb_predict"] == (C.c_int, [P, P, C.c_int64, C.c_int32, C.c_int64, P, P, C.c_int32, P, P,
                                                             P, P, P, C.c_int32, P, C.POINTER(_native.NbInfo), T])


def _sass_with_offsets():
    """{function: [(offset, instruction)]} of libloexec.so's SASS."""
    import subprocess
    sass = subprocess.run(["cuobjdump", "-sass", str(_native.LIB_PATH)], capture_output=True, text=True, check=True).stdout
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = out.setdefault(m.group(1), [])
        elif cur is not None:
            m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?);", line)
            if m:
                cur.append((int(m.group(1), 16), m.group(2).strip()))
    return out


def test_naive_bayes_kernels_in_the_sass(built):
    fns = _sass_with_offsets()
    sums = [f for f in fns if "k_nb_sums" in f]
    predict = [f for f in fns if "k_nb_predict" in f]
    assert len(sums) == 4 and len(predict) == 4 and any("k_nb_reduce" in f for f in fns)
    for f in sums + predict + [f for f in fns if "k_nb_reduce" in f or "k_nb_widen" in f]:
        assert not any(re.search(r"\b(LDL|STL)\b", t) for _o, t in fns[f]), f
    assert any(re.search(r"\bLDG\.E\.[A-Z0-9.]*128\b", t) for f in sums for _o, t in fns[f])      # 16-byte loads
    assert not any(re.search(r"\bDFMA\b", t) for f in sums for _o, t in fns[f])
    for f in predict:
        # the kernel's own code ends where its first out-of-line subroutine (nb_softmax: the library's exp and IEEE
        # division, FMA-based by design) begins; the raw rule in the kernel must be DMUL then DADD, never DFMA
        calls = [int(m.group(1), 16) for _o, t in fns[f] for m in [re.search(r"\bCALL\.REL\S*\s+(0x[0-9a-f]+)", t)] if m]
        end = min(calls) if calls else float("inf")
        body = [t for o, t in fns[f] if o < end]
        assert not any(re.search(r"\bDFMA\b", t) for t in body), f
        assert any(re.search(r"\bDMUL\b", t) for t in body) and any(re.search(r"\bDADD\b", t) for t in body), f


# ---- the oracle against scikit-learn where they agree ------------------------------------------------------------------
def test_oracle_theta_and_metrics_agree_with_sklearn():
    sk_nb = pytest.importorskip("sklearn.naive_bayes")
    sk_m = pytest.importorskip("sklearn.metrics")
    rng = np.random.default_rng(5)
    x = rng.poisson(3.0, (500, 6)).astype(np.float64)
    y = rng.integers(0, 4, 500).astype(np.float64)
    for lam in (1.0, 0.5):
        classes, counts, sums = nb.fit_sums(x, y)
        pi, theta = nb.model(counts, sums, lam)
        ref = sk_nb.MultinomialNB(alpha=lam).fit(x, y)
        np.testing.assert_allclose(theta, ref.feature_log_prob_, rtol=1e-12)   # class_log_prior_ is not smoothed there
    pred = rng.integers(0, 4, 500).astype(np.float64)
    f1, acc = nb.metrics(y, pred)
    assert abs(f1 - sk_m.f1_score(y, pred, average="weighted")) <= 1e-12
    assert acc == sk_m.accuracy_score(y, pred)


def test_library_model_and_metrics_are_the_oracle_formulas():
    rng = np.random.default_rng(9)
    sums = rng.random((5, 7)) * 1e3
    counts = rng.integers(1, 100, 5)
    for lam in (1.0, 0.0, 2.5):
        pi, theta = model_arrays(sums, counts, lam)
        opi, otheta = nb.model(counts, sums, lam)
        np.testing.assert_array_equal(pi, opi)
        np.testing.assert_array_equal(theta, otheta)
    y = np.array([0.0, 0.0, 1.0, 2.0, 2.0, 2.0, 5.0, 0.5])
    pred = np.array([0.0, 1.0, 1.0, 2.0, 0.0, 2.0, 3.0, 0.0])
    labels = np.unique(y)
    f1, acc = metrics(labels, nb.confusion(y, pred, labels, 4))
    of1, oacc = nb.metrics(y, pred)
    assert f1 == of1 and acc == oacc


# ---- the classifier with test doubles for the devices ------------------------------------------------------------------
class _Part:
    def __init__(self, x, y):
        self.x, self.y, self.k, self.nkept = SimpleNamespace(engine=SimpleNamespace(device=0)), y, x.shape[1], len(x)
        self.hx = x

    def free(self):
        pass


class _Engine:
    """Stands in for Engine: runs the oracle on the part's host arrays and records every call."""

    def __init__(self, log):
        self.log = log

    def nb_labels(self, part):
        self.log.append("labels")
        return nb.classes_of(part.y)

    def nb_fit(self, part, classes):
        self.log.append("fit")
        bad = np.argwhere(~(part.hx >= 0))
        if len(bad):
            raise InvalidCellError(int(bad[0][0]), int(bad[0][1]), "bad")
        y = np.asarray(part.y) + 0.0
        return (np.array([part.hx[y == c].sum(0) for c in classes]).reshape(len(classes), part.k),
                np.array([(y == c).sum() for c in classes], np.int64))

    def nb_predict(self, part, pi, theta, raw=False, labels=None):
        pred = nb.prediction(nb.probability(nb.raw(part.hx, pi, theta)))
        return nb.confusion(part.y, pred, labels, len(pi))


def _feats(engine, parts, label="y"):
    n = sum(p.nkept for p in parts)
    return SimpleNamespace(_frame=SimpleNamespace(_cache=SimpleNamespace(engine=engine)), _parts=parts,
                           fields=[f"f{j}" for j in range(parts[0].k)], label=label, row_ids=np.arange(10, 10 + n),
                           devices=[0] * len(parts))


def _sharded(log, world):
    sh = object.__new__(ShardedEngine)
    sh._N, sh.world, sh.nlocal = _native, world, world
    sh.engines = [_Engine(log) for _ in range(world)]
    return sh


def test_fit_and_evaluate_through_one_engine_and_shards_agree():
    rng = np.random.default_rng(2)
    x = rng.integers(0, 9, (300, 4)).astype(np.float64)
    y = rng.integers(0, 3, 300).astype(np.float64)
    log = []
    one = NaiveBayes().fit(_feats(_Engine(log), [_Part(x, y)]))
    classes, counts, sums = nb.fit_sums(x, y)
    np.testing.assert_array_equal(one.sums, sums)
    assert log == ["labels", "fit"]
    sh = _sharded(log, 3)
    parts = [_Part(x[a:b], y[a:b]) for a, b in ((0, 100), (100, 101), (101, 300))]
    many = NaiveBayes().fit(_feats(sh, parts))
    np.testing.assert_array_equal(many.sums, one.sums)
    np.testing.assert_array_equal(many.theta, one.theta)
    ev1 = one.evaluate(_feats(_Engine(log), [_Part(x, y)]))
    evn = many.evaluate(_feats(sh, parts))
    np.testing.assert_array_equal(ev1["confusion"], evn["confusion"])
    pred = nb.prediction(nb.probability(nb.raw(x, one.pi, one.theta)))
    assert (ev1["f1"], ev1["accuracy"]) == nb.metrics(y, pred)


def test_a_refused_feature_names_the_global_row_id_and_field():
    x = np.ones((30, 3))
    x[25, 2] = -1.0
    x[12, 1] = np.nan
    y = np.zeros(30)
    sh = _sharded([], 2)
    with pytest.raises(InvalidCellError) as e:
        NaiveBayes().fit(_feats(sh, [_Part(x[:20], y[:20]), _Part(x[20:], y[20:])]))
    assert (e.value.row, e.value.position) == (12, 1) and "'f1'" in e.value.message and "_id 22" in e.value.message


def test_refusals():
    x, y = np.ones((4, 2)), np.zeros(4)
    one_class = NaiveBayesModel([0.0], [0.0], [[0.0, 0.0]], ["f0", "f1"])
    with pytest.raises(ValueError):
        NaiveBayes().fit(_feats(_Engine([]), [_Part(x, y)], label=None))           # no label
    with pytest.raises(_native.LoexecError):
        NaiveBayes().fit(_feats(_Engine([]), [_Part(x[:0], y[:0])]))              # no row
    for s in (-1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            NaiveBayes(smoothing=s)
    NaiveBayes(smoothing=0.0)
    wide = np.ones((4, 16385))
    with pytest.raises(_native.LoexecError) as e:                                  # C * k above the cap
        NaiveBayes().fit(_feats(_Engine([]), [_Part(wide, y)]))
    assert "LO_NB_MAX_THETA" in e.value.message
    many = np.arange(1025, dtype=np.float64)
    sh = _sharded([], 2)
    with pytest.raises(_native.LoexecError) as e:                                  # the shards' union above 1024
        sh.nb_labels([_Part(np.ones((513, 1)), many[:513]), _Part(np.ones((512, 1)), many[513:])])
    assert e.value.code == _native.LO_ERR_INVALID
    with pytest.raises(ValueError):                                                # NaN label (the oracle refuses too)
        nb.classes_of([0.0, np.nan])
    rank = _sharded([], 2)
    rank.nlocal = 1
    for call in (lambda: rank.nb_labels([]), lambda: rank.nb_fit([], [0.0]), lambda: rank.nb_predict([], [0.0], [[0.0]])):
        with pytest.raises(_native.LoexecError) as e:
            call()
        assert "every row" in e.value.message
    released = _feats(_Engine([]), [_Part(x, y)])
    released._parts = []                                                            # what Features.release leaves
    for call in (lambda: NaiveBayes().fit(released), lambda: one_class.transform(released),
                 lambda: one_class.evaluate(released)):
        with pytest.raises(ValueError, match="released"):
            call()
    m = NaiveBayesModel([0.0], [0.0], [[0.0, 0.0]], ["a", "b"])
    with pytest.raises(ValueError):
        m.transform(_feats(_Engine([]), [_Part(x, y)]))                            # fields f0, f1, not a, b
