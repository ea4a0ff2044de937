"""GPU: the builder's "NB" classifier (Spark 2.4's multinomial NaiveBayes) over the feature matrix in HBM against the numpy
restatement in oracle/naive_bayes.py — sums and model bit for bit on integer-valued features and within 1e-13 on
fractional ones, the raw values bit for bit, probabilities within 4 ulp, predictions and confusion counts exactly, every
cap at its boundary, the shards' merge, and a Titanic CSV end to end."""
import csv
import ctypes as C
import json
from fractions import Fraction
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from werkzeug.test import Client

from learningorchestra_b200 import _native as N
from learningorchestra_b200 import builder_frontend, server
from learningorchestra_b200.classifier import NaiveBayes, NaiveBayesModel
from learningorchestra_b200.column_store import ColumnarDatabase
from learningorchestra_b200.engine import AssembledRows, InvalidCellError
from learningorchestra_b200.sharding import ShardedEngine
from oracle import naive_bayes as nb

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).resolve().parent / "golden"


def _part(engine, x, y):
    """An AssembledRows of x (n x k) and y in x's dtype, as DeviceFrame.features makes them."""
    dt = "f32" if x.dtype == np.float32 else "f64"
    n, k = x.shape
    xt = engine.table(dt, max(n * k, 1), 1)
    xt.upload(0, np.ascontiguousarray(x).ravel())
    yt = engine.table(dt, max(n, 1), 1)
    yt.upload(0, np.asarray(y, x.dtype))
    return AssembledRows(xt, yt, None, k, n)


def _features(engine, parts, k):
    n = sum(p.nkept for p in parts)
    devices = [p.x.engine.device for p in parts]
    frame = SimpleNamespace(_cache=SimpleNamespace(engine=engine))
    return SimpleNamespace(_frame=frame, _parts=parts, fields=[f"f{j}" for j in range(k)], label="y",
                           row_ids=np.arange(100, 100 + n), devices=devices)


def _free(parts):
    for p in parts:
        p.free()


def _host(view, device):
    return torch.as_tensor(view, device=f"cuda:{device}").cpu().numpy()


def _data(n, k, nclasses, seed, dtype=np.float32, integer=True, labels=None):
    rng = np.random.default_rng(seed)
    y = rng.integers(0, nclasses, n).astype(np.float64)
    if labels is not None:
        y = np.asarray(labels, np.float64)[y.astype(np.int64)]
    # class-dependent rates keep the classes apart, so no row sits near a tie
    rates = rng.uniform(0.5, 6.0, (nclasses, k))
    x = rng.poisson(rates[np.searchsorted(np.unique(y), y) if labels is not None else y.astype(np.int64)])
    x = x.astype(np.float64) if integer else x + rng.random((n, k))
    return x.astype(dtype), y


def _ulps(a, b):
    return np.abs(a.view(np.int64) - b.view(np.int64))


def _check_model(engine, x, y, exact):
    classes, counts, sums = nb.fit_sums(x, y)
    part = _part(engine, x, y)
    try:
        feats = _features(engine, [part], x.shape[1])
        m = NaiveBayes().fit(feats)
        np.testing.assert_array_equal(m.labels, classes)
        np.testing.assert_array_equal(m.counts, counts)
        if exact:
            np.testing.assert_array_equal(m.sums, sums)
        else:
            assert np.all(np.abs(m.sums - sums) <= 1e-13 * sums)
        pi, theta = nb.model(m.counts, m.sums)
        np.testing.assert_array_equal(m.pi, pi)
        np.testing.assert_array_equal(m.theta, theta)
        again = NaiveBayes().fit(feats)
        np.testing.assert_array_equal(again.sums.view(np.int64), m.sums.view(np.int64))
        return m, feats, part
    except BaseException:
        part.free()
        raise


def _check_predictions(m, feats, x, y):
    r = nb.raw(x, m.pi, m.theta)
    p = nb.probability(r)
    pred = nb.prediction(p)
    top2 = np.sort(p, axis=1)[:, -2:] if p.shape[1] > 1 else None
    if top2 is not None:
        assert not np.any(_ulps(top2[:, 1], top2[:, 0]) <= 4)       # no near-tie in the data
    with m.transform(feats, raw=True) as out:
        d = feats.devices[0]
        np.testing.assert_array_equal(_host(out.raw[0], d).view(np.int64), r.view(np.int64))
        assert np.all(_ulps(_host(out.probability[0], d), p) <= 4)
        np.testing.assert_array_equal(_host(out.prediction[0], d), pred)
        np.testing.assert_array_equal(out.row_ids, feats.row_ids)
    ev = m.evaluate(feats)
    np.testing.assert_array_equal(ev["labels"], nb.classes_of(y))
    np.testing.assert_array_equal(ev["confusion"], nb.confusion(y, pred, ev["labels"], len(m.labels)))
    f1, acc = nb.metrics(y, pred)
    assert abs(ev["f1"] - f1) <= 1e-15 * max(f1, 1e-300) and abs(ev["accuracy"] - acc) <= 1e-15


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n,k,nclasses", [(200_003, 20, 2), (50_001, 32, 10), (1, 1, 1), (4097, 7, 3), (129, 100, 5)])
def test_fit_transform_evaluate_match_the_oracle(engine, dtype, n, k, nclasses):
    x, y = _data(n, k, nclasses, seed=n + k, dtype=dtype)
    m, feats, part = _check_model(engine, x, y, exact=True)
    try:
        _check_predictions(m, feats, x, y)
    finally:
        part.free()


def test_fractional_sums_within_1e13_and_labels_not_0_to_c(engine):
    x, y = _data(300_007, 12, 4, seed=7, dtype=np.float64, integer=False, labels=[-3.5, 0.25, 2.0, 1e6])
    m, feats, part = _check_model(engine, x, y, exact=False)
    try:
        np.testing.assert_array_equal(m.labels, [-3.5, 0.25, 2.0, 1e6])
        ev = m.evaluate(feats)
        pred = nb.prediction(nb.probability(nb.raw(x, m.pi, m.theta)))
        np.testing.assert_array_equal(ev["confusion"], nb.confusion(y, pred, ev["labels"], 4))
        f1, acc = nb.metrics(y, pred)                    # only label 2.0 can be a true positive (index rule)
        assert ev["accuracy"] == acc and abs(ev["f1"] - f1) <= 1e-15 * f1 and f1 > 0
    finally:
        part.free()


@pytest.mark.parametrize("n,k,nclasses", [(300_000, 512, 2), (100_000, 800, 10)])
def test_wide_fractional_sums_stay_within_1e13(engine, n, k, nclasses):
    """One row group per CTA (f64 with k >= 512, or C * k >= 6400): every sum is still a short run plus a tree.  Columns
    repeat 0.1, 0.2 or 0.3, the worst case for a long sequential sum; the exact sums come from fractions."""
    vals = np.array([0.1, 0.2, 0.3])[np.arange(k) % 3]
    x = np.tile(vals, (n, 1))
    y = (np.arange(n) % nclasses).astype(np.float64)
    part = _part(engine, x, y)
    try:
        m = NaiveBayes().fit(_features(engine, [part], k))
        counts = np.bincount(y.astype(np.int64), minlength=nclasses)
        exact = np.array([[float(Fraction(v) * int(c)) for v in vals] for c in counts])
        np.testing.assert_array_equal(m.counts, counts)
        assert np.all(np.abs(m.sums - exact) <= 1e-13 * exact), np.max(np.abs(m.sums - exact) / exact)
    finally:
        part.free()


def test_the_c_abi_refuses_before_any_launch(engine):
    lib = engine._lib
    x = _part(engine, np.ones((4, 16385), np.float64), np.zeros(4))
    small = _part(engine, np.ones((4, 2), np.float64), [0.0, 1.0, 0.0, 1.0])
    f32 = _part(engine, np.ones((4, 2), np.float32), [0.0, 1.0, 0.0, 1.0])
    prob, pred = engine.table("f64", 8, 1), engine.table("f64", 4, 1)
    tiny = engine.table("f64", 7, 1)
    try:
        sums, counts = np.zeros(16385 * 2), np.zeros(1025, np.int64)
        conf = np.zeros(1025 * 2, np.int64)
        info, t = N.NbInfo(), N.HostTiming()
        P = C.c_void_p

        def arr(v):
            return np.ascontiguousarray(v, np.float64).ctypes.data_as(P)

        cls2 = np.array([0.0, 1.0])

        def fit(part, k, classes, ld=None):
            return lib.lo_nb_fit(engine._ctx, part.x._h, ld or k, k, part.y._h, 4, arr(classes), len(classes),
                                 sums.ctypes.data_as(P), counts.ctypes.data_as(P), C.byref(info), C.byref(t))

        def predict(part, nc, prob_h, pred_h, y_h=None, labels=None, confusion=None, k=2):
            return lib.lo_nb_predict(engine._ctx, part.x._h, k, k, 4, arr(np.zeros(nc)), arr(np.zeros(nc * k)), nc,
                                     prob_h, None, pred_h, y_h, arr(labels) if labels is not None else None,
                                     len(labels) if labels is not None else 0,
                                     confusion.ctypes.data_as(P) if confusion is not None else None,
                                     C.byref(info), C.byref(t))

        before = engine.launch_count
        cases = {
            "C * k = 16385": lambda: fit(x, 16385, [0.0]),
            "C = 1025": lambda: fit(small, 2, np.arange(1025.0)),
            "classes descending": lambda: fit(small, 2, [1.0, 0.0]),
            "classes repeated": lambda: fit(small, 2, [0.0, 0.0]),
            "classes with NaN": lambda: fit(small, 2, [0.0, np.nan]),
            "ld < k": lambda: fit(small, 2, cls2, ld=1),
            "x and y of other dtypes": lambda: lib.lo_nb_fit(engine._ctx, small.x._h, 2, 2, f32.y._h, 4, arr(cls2), 2,
                                                             sums.ctypes.data_as(P), counts.ctypes.data_as(P),
                                                             C.byref(info), C.byref(t)),
            "prob too small": lambda: predict(small, 2, tiny._h, pred._h),
            "transform with y": lambda: predict(small, 2, prob._h, pred._h, y_h=small.y._h),
            "evaluate with prob": lambda: predict(small, 2, prob._h, None, y_h=small.y._h, labels=cls2, confusion=conf),
            "eval labels descending": lambda: predict(small, 2, None, None, y_h=small.y._h, labels=[1.0, 0.0],
                                                      confusion=conf),
            "eval labels 1025": lambda: predict(small, 2, None, None, y_h=small.y._h, labels=np.arange(1025.0),
                                                confusion=conf),
            "predict C = 1025": lambda: predict(small, 1025, prob._h, pred._h),
        }
        for name, call in cases.items():
            assert call() == N.LO_ERR_INVALID, name
        assert engine.launch_count == before
        assert fit(small, 2, cls2) == N.LO_OK and list(counts[:2]) == [2, 2]
        assert predict(small, 2, None, None, y_h=small.y._h, labels=cls2, confusion=conf) == N.LO_OK
        assert conf[:4].sum() == 4
    finally:
        for part in (x, small, f32):
            part.free()
        for tb in (prob, pred, tiny):
            tb.free()


def test_caps_at_their_boundaries(engine):
    n = 3000
    y = np.arange(n) % 1024
    x = (np.arange(n * 16).reshape(n, 16) % 5).astype(np.float32)
    m, feats, part = _check_model(engine, x, y, exact=True)              # C = 1024, C * k = 16384
    try:
        with m.transform(feats) as out:
            p = nb.probability(nb.raw(x, m.pi, m.theta))
            assert np.all(_ulps(_host(out.probability[0], 0), p) <= 4)
        assert len(m.labels) == 1024
    finally:
        part.free()
    x17 = np.ones((n, 17), np.float32)
    part = _part(engine, x17, y)
    try:
        with pytest.raises(N.LoexecError) as e:                          # C * k = 17408
            NaiveBayes().fit(_features(engine, [part], 17))
        assert e.value.code == N.LO_ERR_INVALID
    finally:
        part.free()
    part = _part(engine, np.ones((1025, 1), np.float32), np.arange(1025))
    try:
        with pytest.raises(N.LoexecError) as e:                          # C = 1025
            NaiveBayes().fit(_features(engine, [part], 1))
        assert e.value.code == N.LO_ERR_INVALID
    finally:
        part.free()
    x1 = np.ones((10, 16384), np.float32)
    part = _part(engine, x1, np.zeros(10))                               # C = 1, k = 16384
    try:
        m = NaiveBayes().fit(_features(engine, [part], 16384))
        np.testing.assert_array_equal(m.sums, np.full((1, 16384), 10.0))
    finally:
        part.free()


def test_refused_cells_name_the_lowest_row_and_inf_passes(engine):
    x, y = _data(10_000, 5, 3, seed=3)
    x[9000, 1] = -1.0
    x[7000, 4] = np.nan
    x[7000, 3] = -0.5
    x[50, 2] = np.inf
    part = _part(engine, x, y)
    try:
        with pytest.raises(InvalidCellError) as e:
            NaiveBayes().fit(_features(engine, [part], 5))
        assert (e.value.row, e.value.position) == (7000, 3) and "'f3'" in e.value.message and "_id 7100" in e.value.message
    finally:
        part.free()
    x[7000, 3], x[7000, 4], x[9000, 1] = 1.0, 1.0, 1.0
    classes, counts, sums = nb.fit_sums(x, y)
    part = _part(engine, x, y)
    try:
        m = NaiveBayes().fit(_features(engine, [part], 5))
        np.testing.assert_array_equal(m.sums, sums)
        assert np.isinf(m.sums).any()
    finally:
        part.free()
    part = _part(engine, np.ones((5, 2), np.float32), [0.0, 1.0, np.nan, 1.0, 0.0])
    try:
        with pytest.raises(N.LoexecError):
            NaiveBayes().fit(_features(engine, [part], 2))
    finally:
        part.free()


def test_exact_ties_resolve_to_the_first_index(engine):
    x = np.ones((4, 3), np.float32)
    m = NaiveBayesModel([0.0, 1.0, 2.0], np.full(3, -1.0), np.full((3, 3), -2.0), ["f0", "f1", "f2"])
    part = _part(engine, x, [0.0, 1.0, 2.0, 0.0])
    try:
        feats = _features(engine, [part], 3)
        with m.transform(feats) as out:
            np.testing.assert_array_equal(_host(out.prediction[0], 0), np.zeros(4))
            assert np.all(_host(out.probability[0], 0) == _host(out.probability[0], 0)[0, 0])
        ev = m.evaluate(feats)
        np.testing.assert_array_equal(ev["confusion"], [[2, 0, 0], [1, 0, 0], [1, 0, 0]])
        assert ev["accuracy"] == 0.5
    finally:
        part.free()


def test_negative_zero_label_is_class_zero(engine):
    x = np.ones((4, 2), np.float64)
    part = _part(engine, x, [-0.0, 0.0, 1.0, -0.0])
    try:
        m = NaiveBayes().fit(_features(engine, [part], 2))
        np.testing.assert_array_equal(m.labels, [0.0, 1.0])
        np.testing.assert_array_equal(m.counts, [3, 1])
    finally:
        part.free()


@pytest.mark.parametrize("cuts", [1, 2, 3, 8])
def test_shards_merge_to_the_single_gpu_model(engine, cuts):
    x, y = _data(100_003, 9, 4, seed=cuts)
    whole = _part(engine, x, y)
    bounds = np.linspace(0, len(y), cuts + 1).astype(int)
    pieces = [_part(engine, x[a:b], y[a:b]) for a, b in zip(bounds[:-1], bounds[1:])]
    try:
        one = NaiveBayes().fit(_features(engine, [whole], 9))
        sh = object.__new__(ShardedEngine)                 # every cut on this device, one host thread each
        sh._N, sh.world, sh.nlocal, sh.engines = N, cuts, cuts, [engine] * cuts
        feats = _features(sh, pieces, 9)
        many = NaiveBayes().fit(feats)
        np.testing.assert_array_equal(many.sums, one.sums)
        np.testing.assert_array_equal(many.pi.view(np.int64), one.pi.view(np.int64))
        np.testing.assert_array_equal(many.theta.view(np.int64), one.theta.view(np.int64))
        ev1, evn = one.evaluate(_features(engine, [whole], 9)), many.evaluate(feats)
        np.testing.assert_array_equal(ev1["confusion"], evn["confusion"])
        assert ev1["f1"] == evn["f1"]
        with many.transform(feats) as out:
            got = np.concatenate([_host(v, 0) for v in out.prediction])
            np.testing.assert_array_equal(got, nb.prediction(nb.probability(nb.raw(x, one.pi, one.theta))))
    finally:
        _free([whole] + pieces)


NUMBER_FIELDS = ["PassengerId", "Survived", "Pclass", "Age", "SibSp", "Parch", "Fare"]


@pytest.mark.parametrize("sharded", [False, True])
def test_titanic_end_to_end(engine, tmp_path, sharded):
    g = json.loads((GOLD / "titanic_shaped_input.json").read_text())
    path = tmp_path / "t.csv"
    with open(path, "w", newline="") as f:
        csv.writer(f).writerows([g["headers"]] + g["rows"])
    eng = ShardedEngine.local() if sharded else engine
    try:
        eng.resident.clear()
        db = ColumnarDatabase()
        db.ingest_csv("t", str(path), engine=eng)
        c = Client(server.create_app(db, eng, synchronous=True))
        r = c.patch("/fieldTypes", json={"inputDatasetName": "t", "types": {f: "number" for f in NUMBER_FIELDS}})
        assert r.status_code == 200, r.get_data(as_text=True)
        host = builder_frontend.file_processor(db, "t")
        with builder_frontend.device_frame(db, "t", eng, text=True) as frame:
            with frame.features(label="Survived", handle_invalid="skip") as feats:
                cols = {}
                for f in frame.fields:
                    if frame.kinds[f] == "text":
                        index = {s: i for i, s in enumerate(frame.dictionaries[f].to_pylist())}
                        cols[f] = np.array([-1 if v is None else index[v] for v in host.column(f).to_pylist()], np.float64)
                    else:
                        cols[f] = np.array([np.nan if v is None else v for v in host.column(f).to_pylist()], np.float64)
                stack = np.stack([cols[f] for f in frame.fields])
                is_text = np.array([frame.kinds[f] == "text" for f in frame.fields])[:, None]
                keep = ~np.any(np.isnan(stack) | ((stack == -1) & is_text), axis=0)       # handle_invalid="skip"
                x = np.stack([cols[f][keep] for f in feats.fields], 1).astype(np.float32).astype(np.float64)
                y = cols["Survived"][keep].astype(np.float32).astype(np.float64)
                assert x.shape[0] == len(feats.row_ids)
                m = NaiveBayes().fit(feats)
                classes, counts, sums = nb.fit_sums(x, y)
                np.testing.assert_array_equal(m.labels, classes)
                np.testing.assert_array_equal(m.counts, counts)
                assert np.all(np.abs(m.sums - sums) <= 1e-13 * sums)     # Fare's f32 values need not sum exactly
                pi, theta = nb.model(m.counts, m.sums)
                np.testing.assert_array_equal(m.pi, pi)
                np.testing.assert_array_equal(m.theta, theta)
                p = nb.probability(nb.raw(x, pi, theta))
                pred = nb.prediction(p)
                with m.transform(feats) as out:
                    got = np.concatenate([_host(v, d) for v, d in zip(out.prediction, out.devices)])
                    np.testing.assert_array_equal(got, pred)
                    prob = np.concatenate([_host(v, d) for v, d in zip(out.probability, out.devices)])
                    assert np.all(_ulps(prob, p) <= 4)
                ev = m.evaluate(feats)
                f1, acc = nb.metrics(y, pred)
                assert abs(ev["f1"] - f1) <= 1e-15 and ev["accuracy"] == acc
        eng.resident.clear()
    finally:
        if sharded:
            eng.close()
