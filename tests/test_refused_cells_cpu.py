"""CPU: the refused-cell contract of the feature-matrix calls, with a stand-in for libloexec under the real ``Engine``
methods and real ``ShardedEngine`` frames — the lowest refused cell over the shards with its global row in ``.row`` and in
the message, errors that are not refusals winning over refusals, every table made freed exactly once on each failure
path, and the front-end's and classifier's ``_id`` messages word for word."""
from collections import Counter
from types import SimpleNamespace

import numpy as np
import pytest

from learningorchestra_b200 import _native as N
from learningorchestra_b200 import builder_frontend
from learningorchestra_b200.classifier import NaiveBayes, NaiveBayesModel
from learningorchestra_b200.engine import AssembledRows, Engine, InvalidCellError
from learningorchestra_b200.sharding import ShardedEngine


class _Table:
    """A device table that logs when it is made and each time it is freed."""

    def __init__(self, log, nrows, device=0):
        self.log, self.nrows, self._h = log, nrows, 4096 * (len(log["made"]) + 1)
        self.engine = SimpleNamespace(device=device)
        log["made"].append(self)

    def free(self):
        self.log["freed"].append(self)


class _Lib:
    """Stands in for libloexec: each feature-matrix call returns ``rc``, or refuses cell ``bad`` = (row, column)."""

    def __init__(self, rc=N.LO_OK, bad=None, nkept=0):
        self.rc, self.bad, self.nkept = rc, bad, nkept

    def _finish(self, info_ref):
        info = info_ref._obj
        if self.bad is not None:
            info.bad_row, info.bad_col = self.bad
            return N.LO_ERR_INVALID
        if hasattr(info, "nkept"):
            info.nkept = self.nkept
        return self.rc

    def lo_assemble_rows(self, *args):
        return self._finish(args[-2])

    def lo_nb_fit(self, *args):
        return self._finish(args[-2])

    def lo_nb_predict(self, *args):
        return self._finish(args[-2])


def _engine(log, device=0, **lib):
    """The real Engine methods over a _Lib; its tables are _Tables."""
    e = object.__new__(Engine)
    e._ctx, e._lib, e.device = None, _Lib(**lib), device
    e.table = lambda dtype, nrows, ncols: _Table(log, nrows, device)
    return e


def _log():
    return {"made": [], "freed": []}


def _freed_once(log) -> bool:
    return Counter(map(id, log["freed"])) == Counter(map(id, log["made"]))


def _sharded(engines):
    sh = object.__new__(ShardedEngine)
    sh._N, sh.world, sh.nlocal, sh.engines = N, len(engines), len(engines), list(engines)
    return sh


def _sharded_table(log, sizes):
    offsets = [int(o) for o in np.concatenate([[0], np.cumsum(sizes)[:-1]])]
    return SimpleNamespace(offsets=offsets, shards=[_Table(log, n) for n in sizes])


def _parts(log, sizes, k):
    """AssembledRows of ``sizes`` rows of k features and a label, one per shard; made before the call under test."""
    parts = [AssembledRows(_Table(log, n * k), _Table(log, n), None, k, n) for n in sizes]
    log["made"].clear()
    return parts


# ---- the lowest refused cell over the shards ----------------------------------------------------------------------------
@pytest.mark.parametrize("bad, row, position, message", [
    ({2: (0, 1), 1: (5, 0)}, 103, 0, "invalid cell (NaN or code -1) in row 103, source 0"),
    ({2: (1, 2), 0: (97, 1)}, 97, 1, "invalid cell (NaN or code -1) in row 97, source 1"),    # a lower shard row later
    ({2: (1, 2)}, 131, 2, "invalid cell (NaN or code -1) in row 131, the label, source 2"),
])
def test_assemble_raises_the_lowest_cell_at_its_global_row(bad, row, position, message):
    log = _log()
    t = _sharded_table(log, [98, 32, 6])
    log["made"].clear()
    sh = _sharded([_engine(log, i, bad=bad.get(i), nkept=s.nrows) for i, s in enumerate(t.shards)])
    with pytest.raises(InvalidCellError) as e:
        sh.assemble_rows([(t, 0), (t, 2)], (t, 1), "float64", "error")
    assert (e.value.row, e.value.position, e.value.message) == (row, position, message)
    assert e.value.code == N.LO_ERR_INVALID and str(e.value) == f"LO_ERR_INVALID: {message}"
    assert len(log["made"]) == 6 and _freed_once(log)             # x and y of every member, refused or not


@pytest.mark.parametrize("evaluate", [False, True])
def test_fit_and_evaluate_raise_the_lowest_row_over_the_kept_rows_before(evaluate):
    log = _log()
    parts = _parts(log, [20, 10, 30], 2)
    bad = {1: (3, 2), 2: (0, 2)} if evaluate else {1: (3, 1), 2: (0, 0)}       # rows 23 and 30 of the three shards
    sh = _sharded([_engine(log, i, bad=bad.get(i)) for i in range(3)])
    with pytest.raises(InvalidCellError) as e:
        if evaluate:
            sh.nb_predict(parts, [0.0, 0.0], np.zeros((2, 2)), labels=[0.0, 1.0])
        else:
            sh.nb_fit(parts, [0.0, 1.0])
    message = ("row 23: its label is not one of the evaluated labels" if evaluate
               else "row 23, feature 1: negative or NaN (NaiveBayes needs values >= 0)")
    assert (e.value.row, e.value.position, e.value.message) == (23, 2 if evaluate else 1, message)
    assert not log["made"] and not log["freed"]                  # evaluate makes no table; the caller's parts stay


def test_one_engine_reports_the_cell_in_the_c_abis_words():
    log = _log()
    part, = _parts(log, [40], 3)
    with pytest.raises(InvalidCellError) as e:
        _engine(log, bad=(17, 3)).nb_fit(part, [0.0, 1.0])
    assert (e.value.row, e.value.position, e.value.message) == (17, 3, "row 17: its label is not one of the classes")
    moved = e.value.moved(100)
    assert (moved.row, moved.position, moved.message) == (117, 3, "row 117: its label is not one of the classes")
    src = _Table(log, 40)
    with pytest.raises(InvalidCellError) as e:
        _engine(log, bad=(5, 0)).assemble_rows([(src, 0)], (src, 1))
    assert e.value.message == "invalid cell (NaN or code -1) in row 5, source 0"
    assert len(log["made"]) == 3 and Counter(map(id, log["freed"])) == Counter(map(id, log["made"][1:]))


# ---- errors that are not refusals, and the tables of every failure path ------------------------------------------------
@pytest.mark.parametrize("refuses, fails", [(0, 2), (2, 0), (0, 1)])
def test_an_error_that_is_not_a_refusal_wins(built, refuses, fails):
    log = _log()
    t = _sharded_table(log, [64, 32, 6])
    log["made"].clear()

    def member(i):
        if i == fails:
            return _engine(log, i, rc=N.LO_ERR_NOMEM)
        return _engine(log, i, bad=(0, 0) if i == refuses else None, nkept=t.shards[i].nrows)

    sh = _sharded([member(i) for i in range(3)])
    with pytest.raises(N.LoexecError) as e:
        sh.assemble_rows([(t, 0)], (t, 1))
    assert e.value.code == N.LO_ERR_NOMEM and not isinstance(e.value, InvalidCellError)
    assert len(log["made"]) == 6 and _freed_once(log)
    parts = _parts(log, [20, 10, 30], 2)
    sh = _sharded([member(i) for i in range(3)])
    with pytest.raises(N.LoexecError) as e:
        sh.nb_fit(parts, [0.0, 1.0])
    assert e.value.code == N.LO_ERR_NOMEM and not isinstance(e.value, InvalidCellError)


@pytest.mark.parametrize("raw", [False, True])
def test_a_transform_that_fails_on_one_member_frees_every_table_once(built, raw):
    log = _log()
    parts = _parts(log, [20, 10, 30], 2)
    sh = _sharded([_engine(log, i, rc=N.LO_ERR_NOMEM if i == 1 else N.LO_OK) for i in range(3)])
    with pytest.raises(N.LoexecError) as e:
        sh.nb_predict(parts, [0.0, 0.0], np.zeros((2, 2)), raw=raw)
    assert e.value.code == N.LO_ERR_NOMEM
    assert len(log["made"]) == 3 * (3 if raw else 2) and _freed_once(log)


def test_a_transform_that_succeeds_keeps_its_tables():
    log = _log()
    parts = _parts(log, [20, 10], 2)
    sh = _sharded([_engine(log, i) for i in range(2)])
    out = sh.nb_predict(parts, [0.0, 0.0], np.zeros((2, 2)), raw=True)
    assert [p.n for p in out] == [20, 10] and len(log["made"]) == 6 and not log["freed"]
    for p in out:
        p.free()
    assert _freed_once(log)


# ---- the messages the user reads -------------------------------------------------------------------------------------
def _frame(engine, ids):
    """A frame of the f64 fields a, t, b (slab columns 0, 1, 2) over len(ids) rows."""
    slab = SimpleNamespace(nrows=len(ids), _h=1, column_view=lambda c, keepalive=None: ("v", c))
    data = SimpleNamespace(ids=ids, table=slab, column={"a": 0, "t": 1, "b": 2}, kinds=["float"] * 3, nulls=[0] * 3,
                           texts={})
    return builder_frontend.DeviceFrame(SimpleNamespace(engine=engine, release=lambda d: None), data, ["a", "t", "b"])


@pytest.mark.parametrize("bad, message", [
    ((3, 1), "features: field 't' of the row with _id 103 is null or NaN (handle_invalid='error')"),
    ((4, 2), "features: field 'b' of the row with _id 104 is null or NaN (handle_invalid='error')"),
])
def test_the_front_end_names_the_id_and_field(bad, message):
    log = _log()
    frame = _frame(_engine(log, bad=bad), np.arange(100, 110))
    with pytest.raises(InvalidCellError) as e:
        frame.features(["a", "t"], label="b")
    assert (e.value.row, e.value.position, e.value.message) == (*bad, message)
    assert _freed_once(log)


def _features(engine, parts):
    n = sum(p.nkept for p in parts)
    return SimpleNamespace(_frame=SimpleNamespace(_cache=SimpleNamespace(engine=engine)), _parts=parts,
                           fields=["f0", "f1"], label="y", row_ids=np.arange(10, 10 + n), devices=[0] * len(parts))


@pytest.mark.parametrize("sharded", [False, True])
def test_the_classifier_names_the_id_and_field(sharded):
    log = _log()
    sizes = [20, 10, 30] if sharded else [60]
    parts = _parts(log, sizes, 2)
    engines = [_engine(log, i, bad=(3, 1) if i == len(sizes) - 1 else None) for i in range(len(sizes))]
    for e in engines:
        e.nb_labels = lambda part: np.array([0.0, 1.0])
    runner = _sharded(engines) if sharded else engines[0]
    last = sum(sizes[:-1]) + 3
    with pytest.raises(InvalidCellError) as e:
        NaiveBayes().fit(_features(runner, parts))
    assert (e.value.row, e.value.position) == (last, 1)
    assert e.value.message == f"NaiveBayes: field 'f1' of the row with _id {10 + last} is negative or NaN"
    for eng in engines:
        eng._lib.bad = (3, 2) if eng is engines[-1] else None
    model = NaiveBayesModel([0.0, 1.0], [0.0, 0.0], np.zeros((2, 2)), ["f0", "f1"])
    with pytest.raises(InvalidCellError) as e:
        model.evaluate(_features(runner, parts))
    assert (e.value.row, e.value.position) == (last, 2)
    assert e.value.message == f"NaiveBayes: field 'y' of the row with _id {10 + last} is not a class of the model"
    assert not log["made"] and not log["freed"]
