"""CPU: the host side of the feature matrix — the header <-> ctypes mirror of ``lo_assemble_rows``, its kernels in the
SASS, and ``DeviceFrame.features`` / ``ShardedEngine.assemble_rows`` with test doubles standing in for the devices."""
import ctypes as C
import re
from types import SimpleNamespace

import numpy as np
import pyarrow as pa
import pytest

from learningorchestra_b200 import _native, builder_frontend
from learningorchestra_b200.engine import AssembledRows, InvalidCellError
from learningorchestra_b200.sharding import ShardedEngine

from test_text_shards_cpu import HEADER, _sass_functions


def test_ctypes_mirror_of_the_assemble_entry_point_matches_the_header():
    text = re.sub(r"/\*.*?\*/", "", HEADER.read_text(), flags=re.S)
    assert int(re.search(r"#define LO_ABI_VERSION (\d+)", text).group(1)) == _native.LO_ABI_VERSION == 7
    modes = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define (LO_INVALID_\w+)\s+(\d+)", text)}
    assert modes == {"LO_INVALID_ERROR": 0, "LO_INVALID_SKIP": 1, "LO_INVALID_KEEP": 2}
    assert all(getattr(_native, k) == v for k, v in modes.items())
    params = [p.strip() for p in re.search(r"\blo_assemble_rows\s*\(([^)]*)\)", text).group(1).split(",")]
    assert params == ["lo_ctx *ctx", "const lo_table *const *src", "const int32_t *src_col", "int32_t k",
                      "const lo_table *label", "int32_t label_col", "int32_t mode", "lo_table *x", "int64_t ld",
                      "lo_table *y", "int64_t *kept_rows", "lo_assemble_info *info", "lo_host_timing *timing"]
    fields = re.search(r"typedef struct lo_assemble_info \{(.*?)\} lo_assemble_info;", text, re.S).group(1)
    assert re.findall(r"(\w+)\s+(\w+);", fields) == [("int64_t", "nkept"), ("int64_t", "bad_row"),
                                                     ("int32_t", "bad_col"), ("int32_t", "pad")]
    assert [(n, t) for n, t in _native.AssembleInfo._fields_] == [("nkept", C.c_int64), ("bad_row", C.c_int64),
                                                                  ("bad_col", C.c_int32), ("pad", C.c_int32)]
    P = C.c_void_p
    assert _native.SIGNATURES["lo_assemble_rows"] == (C.c_int, [
        P, C.POINTER(P), C.POINTER(C.c_int32), C.c_int32, P, C.c_int32, C.c_int32, P, C.c_int64, P, P,
        C.POINTER(_native.AssembleInfo), C.POINTER(_native.HostTiming)])


def test_assemble_kernels_are_sm90a_code_without_local_memory(built):
    fns = _sass_functions()
    names = [f for f in fns if "k_assemble_rows" in f or "k_assemble_valid" in f]
    assert len([f for f in names if "k_assemble_rows" in f]) == 4 and len([f for f in names if "k_assemble_valid" in f]) == 1
    for f in names:
        assert not any(re.search(r"\b(LDL|STL)\b", t) for t in fns[f]), f
    rows = [t for f in names if "k_assemble_rows" in f for t in fns[f]]
    assert any(re.search(r"\bLDG\.E\.NA\.128\b", t) for t in rows)             # 16-byte read-once loads
    assert any(re.search(r"\bSTG\.E\.EF\.128\b", t) for t in rows)             # 16-byte streaming row stores


# ---- DeviceFrame.features with test doubles for the device -----------------------------------------------------------
class _Table:
    def __init__(self, log, dtype, n, device=0):
        self.log, self.n, self._h, self.base_ptr = log, n, object(), 4096 * (len(log["made"]) + 1)
        self.dtype_code = {"f32": _native.LO_F32, "f64": _native.LO_F64}.get(dtype, _native.LO_I32)
        self.engine = SimpleNamespace(device=device)
        log["made"].append(self)

    def free(self):
        self.log["freed"].append(self)
        self._h = None


class _Engine:
    """Stands in for Engine: records every assemble_rows call and keeps the rows without an invalid cell."""

    def __init__(self, log, device=0, bad=None):
        self.log, self.device, self.bad = log, device, bad

    def assemble_rows(self, sources, label=None, dtype="float32", handle_invalid="error"):
        self.log["calls"].append(([c for _t, c in sources], label and label[1], dtype, handle_invalid))
        n = sources[0][0].nrows
        if handle_invalid == "error" and self.bad is not None:
            raise InvalidCellError(*self.bad, "invalid")
        rows = np.arange(n, dtype=np.int64)[::2] if handle_invalid == "skip" else None
        out = {"float32": "f32", "float64": "f64"}[dtype]
        y = _Table(self.log, out, n, self.device) if label is not None else None
        nkept = n if rows is None else len(rows)
        return AssembledRows(_Table(self.log, out, n * len(sources), self.device), y, rows, len(sources), nkept)


def _log():
    return {"made": [], "freed": [], "calls": [], "released": 0}


def _frame(engine, ids=np.arange(1, 11)):
    """A frame of fields a (slab 0), s (codes), b (slab 1), t (codes) over len(ids) rows."""
    log = engine.log
    slab = SimpleNamespace(nrows=len(ids), _h=object())
    codes = {f: (SimpleNamespace(nrows=len(ids), _h=object(), column_view=lambda c, keepalive=None: ("v", c)),
                 pa.array(["x"])) for f in ("s", "t")}
    slab.column_view = lambda c, keepalive=None: ("v", c)
    data = SimpleNamespace(ids=ids, table=slab, column={"a": 0, "b": 1}, kinds=["float", "int"], nulls=[0, 1],
                           texts={f: SimpleNamespace(nulls=0) for f in codes})
    cache = SimpleNamespace(engine=engine, release=lambda d: log.__setitem__("released", log["released"] + 1))
    return builder_frontend.DeviceFrame(cache, data, ["a", "s", "b", "t"], codes), slab, codes


def test_features_take_frame_order_and_leave_the_label_out():
    eng = _Engine(_log())
    frame, slab, codes = _frame(eng)
    with frame.features(label="b") as feats:
        (cols, label_col, dtype, mode), = eng.log["calls"]
        assert feats.fields == ["a", "s", "t"] and feats.label == "b" and (dtype, mode) == ("float32", "error")
        assert cols == [0, 0, 0] and label_col == 1
        assert len(feats.x) == 1 and feats.x[0].__cuda_array_interface__["shape"] == (10, 3)
        assert feats.x[0].__cuda_array_interface__["typestr"] == "<f4" and feats.y[0].__cuda_array_interface__["shape"] == (10,)
        np.testing.assert_array_equal(feats.row_ids, np.arange(1, 11))
        assert feats._frame is frame and feats.devices == [0]
    with frame.features(["t", "a"], dtype="float64", handle_invalid="skip") as feats:
        assert feats.fields == ["t", "a"] and feats.y is None
        assert feats.x[0].__cuda_array_interface__["typestr"] == "<f8"
        assert feats.x[0].__cuda_array_interface__["shape"] == (5, 2)
        np.testing.assert_array_equal(feats.row_ids, np.arange(1, 11)[::2])
    assert frame.features().fields == ["a", "s", "b", "t"]


@pytest.mark.parametrize("kw", [dict(handle_invalid="drop"), dict(dtype="float16"), dict(fields=["a", "zz"]),
                                dict(label="zz"), dict(fields=[])])
def test_features_refuse_bad_arguments_before_any_launch(kw):
    eng = _Engine(_log())
    frame, _slab, _codes = _frame(eng)
    with pytest.raises(KeyError if "zz" in str(kw) else ValueError):
        frame.features(**kw)
    assert not eng.log["calls"] and not eng.log["made"]


def test_features_error_names_the_id_and_the_field():
    eng = _Engine(_log(), bad=(3, 1))
    frame, _slab, _codes = _frame(eng, ids=np.arange(100, 110))
    with pytest.raises(InvalidCellError) as e:
        frame.features(["a", "t"], label="b")
    assert e.value.code == _native.LO_ERR_INVALID and "'t'" in e.value.message and "_id 103" in e.value.message
    eng.bad = (4, 2)                                      # position len(fields): the label
    with pytest.raises(InvalidCellError) as e:
        frame.features(["a", "t"], label="b")
    assert "'b'" in e.value.message and "_id 104" in e.value.message


def test_release_frees_every_table_once():
    eng = _Engine(_log())
    frame, _slab, _codes = _frame(eng)
    feats = frame.features(label="a")
    made = list(eng.log["made"])
    assert len(made) == 2
    feats.release()
    feats.release()
    assert sorted(map(id, eng.log["freed"])) == sorted(map(id, made))


# ---- ShardedEngine.assemble_rows with test doubles for the members ---------------------------------------------------
def _sharded(log, world=3, bad=None):
    sh = object.__new__(ShardedEngine)
    sh._N, sh.world, sh.nlocal = _native, world, world
    sh.engines = [_Engine(log, device=i, bad=(bad or {}).get(i)) for i in range(world)]
    return sh


def _sharded_table(sizes):
    offsets = list(np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(int))
    return SimpleNamespace(offsets=offsets, shards=[SimpleNamespace(nrows=n, _h=object()) for n in sizes])


def test_sharded_rows_are_global_and_each_shard_on_its_own_device():
    log = _log()
    sh = _sharded(log)
    t = _sharded_table([64, 32, 6])
    parts = sh.assemble_rows([(t, 0), (t, 2)], (t, 1), "float32", "skip")
    assert [p.x.engine.device for p in parts] == [0, 1, 2]
    np.testing.assert_array_equal(np.concatenate([p.rows for p in parts]),
                                  np.concatenate([np.arange(0, 64, 2), 64 + np.arange(0, 32, 2), 96 + np.arange(0, 6, 2)]))
    assert len(log["calls"]) == 3
    parts = sh.assemble_rows([(t, 0)], None, "float32", "keep")
    np.testing.assert_array_equal(np.concatenate([p.rows for p in parts]), np.arange(102))
    frame_ids = np.arange(1000, 1102)
    assert [p.first for p in parts] == [0, 64, 96] and all(p.kept is None for p in parts)
    np.testing.assert_array_equal(np.concatenate([frame_ids[p.first:p.first + p.nkept] for p in parts]), frame_ids)


def test_sharded_error_is_the_lowest_row_over_every_shard():
    log = _log()
    sh = _sharded(log, bad={2: (0, 1), 1: (5, 0)})          # shard 1's row 5 is global row 69, shard 2's row 0 is 96
    t = _sharded_table([64, 32, 6])
    with pytest.raises(InvalidCellError) as e:
        sh.assemble_rows([(t, 0), (t, 2)], None, "float64", "error")
    assert (e.value.row, e.value.position) == (69, 0)
    assert sorted(map(id, log["freed"])) == sorted(map(id, log["made"]))      # shard 0's matrix freed


def test_sharded_tables_must_be_cut_alike_and_a_rank_group_refuses():
    sh = _sharded(_log())
    with pytest.raises(ValueError):
        sh.assemble_rows([(_sharded_table([64, 32, 6]), 0), (_sharded_table([32, 64, 6]), 0)])
    rank = _sharded(_log())
    rank.nlocal = 1
    with pytest.raises(_native.LoexecError) as e:
        rank.assemble_rows([(_sharded_table([5]), 0)])
    assert e.value.code == _native.LO_ERR_INVALID and "every row" in e.value.message
