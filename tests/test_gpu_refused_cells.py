"""GPU: a refused cell of the feature matrix comes back at the same global row on one GPU and over every cut of a
``ShardedEngine`` — a negative feature from ``NaiveBayes.fit``, a label that is no class from fit and evaluate — with
``.row``, ``.position``, the message and the ``_id`` agreeing, and the engine usable after each refusal."""
from types import SimpleNamespace

import numpy as np
import pytest

from learningorchestra_b200 import _native as N
from learningorchestra_b200 import classifier
from learningorchestra_b200.classifier import NaiveBayes
from learningorchestra_b200.engine import AssembledRows, InvalidCellError
from learningorchestra_b200.sharding import ShardedEngine
from oracle import naive_bayes as nb

pytestmark = pytest.mark.gpu

N_ROWS, K = 100_003, 9
# rows after the last interior cut of 2, 3 and 8 cuts; on 8 cuts the higher row sits lower in its own shard
NEG_FEATURE = [(60_000, 6), (90_000, 5)]
NAN_FEATURE = (90_000, 2)
NOT_A_CLASS = [70_000, 95_000]


def _part(engine, x, y):
    n = len(y)
    xt = engine.table("f32", n * K, 1)
    xt.upload(0, np.ascontiguousarray(x).ravel())
    yt = engine.table("f32", n, 1)
    yt.upload(0, np.asarray(y, np.float32))
    return AssembledRows(xt, yt, None, K, n)


def _runner(engine, cuts, x, y):
    """(engine or ShardedEngine, its parts): one GPU, or ``cuts`` cuts all on this device, one host thread each."""
    if cuts is None:
        return engine, [_part(engine, x, y)]
    sh = object.__new__(ShardedEngine)
    sh._N, sh.world, sh.nlocal, sh.engines = N, cuts, cuts, [engine] * cuts
    bounds = np.linspace(0, len(y), cuts + 1).astype(int)
    return sh, [_part(engine, x[a:b], y[a:b]) for a, b in zip(bounds[:-1], bounds[1:])]


def _features(runner, parts):
    n = sum(p.nkept for p in parts)
    return SimpleNamespace(_frame=SimpleNamespace(_cache=SimpleNamespace(engine=runner)), _parts=parts,
                           fields=[f"f{j}" for j in range(K)], label="y", row_ids=np.arange(100, 100 + n),
                           devices=[0] * len(parts))


def _free(parts):
    for p in parts:
        p.free()


@pytest.mark.parametrize("cuts", [None, 1, 2, 3, 8])
def test_refused_rows_are_global_on_one_gpu_and_every_cut(engine, cuts):
    rng = np.random.default_rng(11)
    y = rng.integers(0, 4, N_ROWS).astype(np.float32)
    x = rng.poisson(3.0, (N_ROWS, K)).astype(np.float32)
    bad_x, bad_y = x.copy(), y.copy()
    for r, j in NEG_FEATURE:
        bad_x[r, j] = -1.0
    bad_x[NAN_FEATURE] = np.nan
    bad_y[NOT_A_CLASS] = [7.0, 9.0]
    classes = [0.0, 1.0, 2.0, 3.0]
    runner, parts = _runner(engine, cuts, bad_x, y)
    try:
        before = engine.launch_count
        with pytest.raises(InvalidCellError) as e:
            NaiveBayes().fit(_features(runner, parts))
        assert engine.launch_count > before                         # the kernels found it
        assert (e.value.row, e.value.position) == NEG_FEATURE[0]
        assert e.value.message == "NaiveBayes: field 'f6' of the row with _id 60100 is negative or NaN"
    finally:
        _free(parts)
    runner, parts = _runner(engine, cuts, x, bad_y)
    rows = parts if cuts else parts[0]
    try:
        with pytest.raises(InvalidCellError) as e:
            runner.nb_fit(rows, classes)
        assert (e.value.row, e.value.position, e.value.message) == (
            70_000, K, "row 70000: its label is not one of the classes")
        pi, theta = np.log(np.full(4, 0.25)), np.log(np.full((4, K), 1.0 / K))
        before = engine.launch_count
        with pytest.raises(InvalidCellError) as e:
            runner.nb_predict(rows, pi, theta, labels=classes)
        assert engine.launch_count > before
        assert (e.value.row, e.value.position, e.value.message) == (
            70_000, K, "row 70000: its label is not one of the evaluated labels")
        with pytest.raises(InvalidCellError) as e:
            classifier._on_device(_features(runner, parts),
                                  lambda eng, r: eng.nb_predict(r, pi, theta, labels=classes))
        assert e.value.message == "NaiveBayes: field 'y' of the row with _id 70100 is not a class of the model"
    finally:
        _free(parts)
    runner, parts = _runner(engine, cuts, x, y)                    # the engine still fits after every refusal
    try:
        m = NaiveBayes().fit(_features(runner, parts))
        _classes, counts, sums = nb.fit_sums(x.astype(np.float64), y.astype(np.float64))
        np.testing.assert_array_equal(m.sums, sums)
        np.testing.assert_array_equal(m.counts, counts)
    finally:
        _free(parts)
