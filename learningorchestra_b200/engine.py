"""Engine — the handle the reference's ``spark_session`` slot receives in this build.

Thin object layer over the C ABI (``include/loexec.h``): device-resident columnar tables and the
projection / cast / histogram entry points.  All computation happens in libloexec's sm_90a
kernels; nothing here falls back to numpy.

Reference boundary this replaces: ``projection_image/server.py:51-69`` builds a ``SparkSession``
and hands it to ``Projection`` (``projection_image/projection.py:14-18``); the histogram and
dataType services talk to mongod through pymongo (``histogram_image/utils.py:50-52``).
"""
from __future__ import annotations

import contextlib
import ctypes as C
import io
import math
import os
import threading
from typing import Iterable, Sequence

import numpy as np

from . import _native as N

_DTYPES = {"f64": N.LO_F64, "f32": N.LO_F32, "u8": N.LO_U8, "i32": N.LO_I32}
_NP = {N.LO_F64: np.float64, N.LO_F32: np.float32, N.LO_U8: np.uint8, N.LO_I32: np.int32}


def _stream_ptr(stream) -> C.c_void_p:
    if stream is None:
        return C.c_void_p(0)
    if hasattr(stream, "cuda_stream"):          # torch.cuda.Stream
        return C.c_void_p(int(stream.cuda_stream))
    return C.c_void_p(int(stream))


def _i32(col_idx: Iterable[int]):
    """ctypes int32 array of the column indices; an array made by :func:`prepare_columns` is passed through (building
    it costs ~0.1 us per column in Python — 80 us for the 784 columns of config M, more than the kernel at 8 GPUs)."""
    if isinstance(col_idx, C.Array):
        return col_idx, len(col_idx)
    idx = [int(c) for c in col_idx]
    return (C.c_int32 * len(idx))(*idx), len(idx)


def prepare_columns(col_idx: Iterable[int]):
    """Column indices converted once, for callers that issue the same request many times."""
    return _i32(col_idx)[0]


def _host_cols(cols, dtype):
    """(ctypes pointer array, rows) of k equal-length contiguous 1-D host arrays of ``dtype``."""
    for c in cols:
        if c.dtype != dtype or not c.flags.c_contiguous or c.ndim != 1 or c.shape[0] != cols[0].shape[0]:
            raise ValueError(f"cols must be equal-length contiguous 1-D {np.dtype(dtype).name} arrays")
    return (C.c_void_p * len(cols))(*[c.ctypes.data for c in cols]), (cols[0].shape[0] if len(cols) else 0)


def _out_cols(out, k: int, n: int):
    """ctypes pointer array of k float32 output columns of n rows each, or None.  The library reads k entries: a short
    ``out`` leaves NULL entries, which it rejects; a longer one raises IndexError here."""
    if out is None:
        return None
    for o in out:
        if o.dtype != np.float32 or not o.flags.c_contiguous or o.shape != (n,):
            raise ValueError("out must be contiguous float32 arrays of the input length")
    return (C.c_void_p * k)(*[o.ctypes.data for o in out])


def _timing(t) -> dict:
    """The lo_host_timing fields the chunked host pipelines report."""
    return {"total_ms": t.total_ms, "h2d_bytes": t.h2d_bytes, "d2h_bytes": t.d2h_bytes, "launches": t.launches}


def _report(timing: dict | None, t) -> None:
    """A call's lo_host_timing ``t`` into the caller's ``timing`` dict, when it passed one."""
    if timing is not None:
        timing.update(_timing(t), kernel_ms=t.kernel_ms)


def _validity(nulls, n: int):
    """(lo_validity, the array it points into) of ``nulls`` as :meth:`Engine.parse_number_into` takes it."""
    v, keep = N.Validity(), None
    if isinstance(nulls, tuple):
        keep = np.ascontiguousarray(nulls[0], dtype=np.uint8)
        v.bitmap, v.bit_offset = keep.ctypes.data, int(nulls[1])
    elif nulls is not None:
        keep = np.ascontiguousarray(~np.asarray(nulls, dtype=bool)).view(np.uint8)
        if keep.shape != (n,):
            raise ValueError("nulls must have one entry per cell")
        v.mask = keep.ctypes.data
    return v, keep


def _summary(s, t) -> dict:
    """The dict :meth:`Engine.parse_number_into` returns from a lo_parse_summary and its lo_host_timing."""
    return {"first_invalid": s.first_invalid if s.first_invalid >= 0 else None,
            "first_unsupported": s.first_unsupported if s.first_unsupported >= 0 else None,
            "nulls": int(s.nulls), "integer": bool(s.all_integer), **_timing(t), "kernel_ms": t.kernel_ms}


def _minmax_decode(lib, raw: np.ndarray, k: int):
    """(min, max, n_finite) of k columns from the raw uint64[3k] of a min/max pre-pass."""
    mins, maxs, cnt = np.zeros(k, np.float32), np.zeros(k, np.float32), np.zeros(k, np.uint64)
    N.check(lib.lo_minmax_decode(raw.ctypes.data_as(C.c_void_p), k, mins.ctypes.data_as(C.c_void_p),
                                 maxs.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p)))
    return mins, maxs, cnt


def _groups(call, n: int, dtypes, timing: dict | None = None) -> tuple:
    """The outputs of a call that returns at most ``capacity`` of the groups of ``n`` cells, ``call(*outs, capacity,
    ndistinct_ref, timing_ref)`` with one output array per dtype of ``dtypes``: room for min(n, 65536) groups first,
    called again with room for every group when they did not fit.  ``timing``: a dict to receive the last call's
    lo_host_timing fields; None passes no lo_host_timing."""
    t = N.HostTiming() if timing is not None else None
    cap = max(min(n, 1 << 16), 1)
    while True:
        outs = [np.empty(cap, dtype=d) for d in dtypes]
        nd = C.c_int64()
        rc = call(*[o.ctypes.data_as(C.c_void_p) for o in outs], cap, C.byref(nd), C.byref(t) if t is not None else None)
        if rc == N.LO_ERR_INVALID and nd.value > cap:
            cap = int(nd.value)
            continue
        N.check(rc)
        _report(timing, t)
        return tuple(o[:nd.value] for o in outs)


def _value_counts(call, n: int, key_dtype, timing: dict | None = None):
    """(keys, counts) of a lo_value_counts_* call ``call(keys_out, counts_out, capacity, ndistinct_ref, timing_ref)``
    (:func:`_groups`)."""
    return _groups(call, n, (key_dtype, np.uint64), timing)


def _first_rows(call, n: int, timing: dict | None = None) -> np.ndarray:
    """The first rows (int64[ndistinct], ascending) of a lo_text_codes* call ``call(first_rows_out, capacity,
    ndistinct_ref, timing_ref)`` on a column of ``n`` non-null cells (:func:`_groups`)."""
    return _groups(call, n, (np.int64,), timing)[0]


def text_dictionary(arr, first_rows):
    """The dictionary of a text column's codes: the cells of ``arr`` (the Arrow array that was uploaded) at
    ``first_rows``, in code order — read the way ``histogram.text_groups`` reads group keys."""
    import pyarrow as pa
    return arr.take(pa.array(np.asarray(first_rows, dtype=np.int64)))


def _pieces(source, buf: np.ndarray):
    """(n, last) for each piece of ``source`` read into ``buf`` (uint8): full pieces, the rest, then (0, True).
    source: a path, a binary or text file object, or an iterable of bytes."""
    if isinstance(source, (str, os.PathLike)):
        with open(source, "rb", buffering=0) as f:
            yield from _pieces(f, buf)
        return
    view = memoryview(buf)
    if hasattr(source, "readinto") and not isinstance(source, io.TextIOBase):
        while True:
            n = 0
            while n < buf.size:
                k = source.readinto(view[n:])
                if not k:
                    break
                n += k
            if n:
                yield n, False
            if n < buf.size:
                break
    else:
        if hasattr(source, "read"):
            chunks = iter(lambda: source.read(buf.size), source.read(0))
        else:
            chunks = iter(source)
        n = 0
        for chunk in chunks:
            data = memoryview(chunk.encode("utf-8") if isinstance(chunk, str) else chunk).cast("B")
            while len(data):
                k = min(len(data), buf.size - n)
                view[n:n + k] = data[:k]
                n += k
                data = data[k:]
                if n == buf.size:
                    yield n, False
                    n = 0
        if n:
            yield n, False
    yield 0, True


class _TextBuilder:
    """One text column grown window by window: chars and int64 offsets, doubled as they fill."""

    def __init__(self):
        self.chars, self.nchars = np.empty(1 << 10, np.uint8), 0
        self.offsets, self.nrows = np.zeros(1 << 10, np.int64), 0

    @staticmethod
    def _room(a: np.ndarray, need: int) -> np.ndarray:
        if need <= a.size:
            return a
        b = np.empty(max(need, 2 * a.size), a.dtype)
        b[:a.size] = a
        return b

    def append(self, chars: np.ndarray, offsets: np.ndarray):
        """Cells i of offsets[i]..offsets[i + 1] in chars (absolute offsets, one column of a window)."""
        k, lo, hi = offsets.size - 1, int(offsets[0]), int(offsets[-1])
        self.chars = self._room(self.chars, self.nchars + hi - lo)
        self.chars[self.nchars:self.nchars + hi - lo] = chars[lo:hi]
        self.offsets = self._room(self.offsets, self.nrows + k + 1)
        np.add(offsets[1:], self.nchars - lo, out=self.offsets[self.nrows + 1:self.nrows + k + 1])
        self.nchars += hi - lo
        self.nrows += k

    def array(self, pa):
        return pa.LargeStringArray.from_buffers(self.nrows, pa.py_buffer(self.offsets[:self.nrows + 1]),
                                                pa.py_buffer(self.chars[:self.nchars]))


class DeviceCounts:
    """uint64[k, nbins] histogram counts resident in HBM (accumulated into by the kernels)."""

    def __init__(self, engine: "Engine", k: int, nbins: int, ptr: int | None = None, keepalive=None):
        """``ptr``: wrap caller-owned device memory (e.g. a torch int64 tensor, so the partial
        histograms can be all-reduced by ``torch.distributed``/NCCL in place)."""
        self.engine, self.k, self.nbins = engine, int(k), int(nbins)
        self._owned, self._keepalive = ptr is None, keepalive
        if ptr is None:
            p = C.c_void_p()
            N.check(engine._lib.lo_counts_alloc(engine._ctx, self.k * self.nbins, C.byref(p)))
        else:
            p = C.c_void_p(int(ptr))
        self._ptr = p

    @property
    def data_ptr(self) -> int:
        return int(self._ptr.value)

    def zero(self, stream=None) -> None:
        N.check(self.engine._lib.lo_counts_zero_dev(self.engine._ctx, self._ptr, self.k * self.nbins, _stream_ptr(stream)))

    def to_numpy(self, stream=None) -> np.ndarray:
        out = np.empty((self.k, self.nbins), dtype=np.uint64)
        N.check(self.engine._lib.lo_counts_download(self.engine._ctx, self._ptr, self.k * self.nbins,
                                                    out.ctypes.data_as(C.c_void_p), _stream_ptr(stream)))
        return out

    def free(self) -> None:
        if self._owned and self._ptr is not None and self.engine._ctx is not None:
            N.check(self.engine._lib.lo_counts_free(self.engine._ctx, self._ptr))
        self._ptr = None

    def __del__(self):          # best effort: device memory of a forgotten handle goes back when it is collected
        try:
            self.free()
        except Exception:
            pass


class DeviceColumn:
    """Zero-copy view of one column slab for GPU consumers: implements ``__cuda_array_interface__`` (version 3), so
    ``torch.as_tensor(col, device="cuda")``, ``cupy.asarray(col)`` or Numba see the slab in place.  Keeps its table
    (and whatever the table keeps) alive."""

    _TYPESTR = {N.LO_F64: "<f8", N.LO_F32: "<f4", N.LO_U8: "|u1", N.LO_I32: "<i4"}

    def __init__(self, table: "DeviceTable", col: int, keepalive=None):
        if not 0 <= col < table.ncols:
            raise IndexError(col)
        self.table, self.col, self._keepalive = table, int(col), keepalive
        self.data_ptr = table.base_ptr + self.col * table.pitch_bytes
        self.nrows = table.nrows

    @property
    def __cuda_array_interface__(self):
        return {"shape": (self.nrows,), "typestr": self._TYPESTR[self.table.dtype_code], "data": (self.data_ptr, False),
                "version": 3, "strides": None}


class DeviceArray:
    """Zero-copy ``__cuda_array_interface__`` view of the first ``prod(shape)`` elements of a table's column 0, C order:
    a row-major matrix or a vector of :meth:`Engine.assemble_rows`.  Keeps its table (and ``keepalive``) alive."""

    def __init__(self, table: "DeviceTable", shape: tuple, keepalive=None):
        self.table, self.shape, self._keepalive = table, tuple(int(d) for d in shape), keepalive
        self.data_ptr = table.base_ptr

    @property
    def __cuda_array_interface__(self):
        return {"shape": self.shape, "typestr": DeviceColumn._TYPESTR[self.table.dtype_code], "data": (self.data_ptr, False),
                "version": 3, "strides": None}


class InvalidCellError(N.LoexecError):
    """A call refused a cell of the feature matrix: :meth:`Engine.assemble_rows` with ``handle_invalid="error"`` met an
    invalid cell, :meth:`Engine.nb_fit` / :meth:`Engine.nb_predict` a negative or NaN feature or an unknown label,
    :meth:`Engine.lr_stats` a feature that is not finite or a label that is not an integer >= 0.
    ``row`` is the lowest such row (a source row for assemble_rows, a row of the matrix for the others; global over the
    shards of a :class:`~sharding.ShardedEngine`) and ``position`` its lowest refused column (an index into the sources
    or features; their count: the label).  ``reason``, when given, is the message as a format of ``row`` and
    ``position``, so that :meth:`moved` moves the row the message names too; else the message is ``message``."""

    def __init__(self, row: int, position: int, message: str | None = None, reason: str | None = None):
        self.row, self.position, self.reason = int(row), int(position), reason
        super().__init__(N.LO_ERR_INVALID, message if reason is None else reason.format(row=self.row, position=self.position))

    def moved(self, first: int) -> "InvalidCellError":
        """The same refusal ``first`` rows further on: a shard's row made global."""
        return InvalidCellError(self.row + first, self.position, self.message, self.reason)


# The messages of a refused cell, (a feature's, the label's), in lo_last_error()'s words
_ASSEMBLE_REFUSED = ("invalid cell (NaN or code -1) in row {row}, source {position}",
                     "invalid cell (NaN or code -1) in row {row}, the label, source {position}")
_NB_FEATURE_REFUSED = "row {row}, feature {position}: negative or NaN (NaiveBayes needs values >= 0)"
_FIT_REFUSED = (_NB_FEATURE_REFUSED, "row {row}: its label is not one of the classes")
_EVALUATE_REFUSED = (_NB_FEATURE_REFUSED, "row {row}: its label is not one of the evaluated labels")
_LR_STATS_REFUSED = ("row {row}, feature {position}: NaN or infinite", "row {row}: its label is not an integer >= 0")
_GB_REFUSED = (_NB_FEATURE_REFUSED, "row {row}: its label is not 0 or 1")


def _check_cells(rc: int, info, k: int, reasons: tuple[str, str]) -> None:
    """``N.check(rc)``, except that a refused cell (LO_ERR_INVALID with ``info.bad_row`` set) raises
    :class:`InvalidCellError` with ``reasons[0]`` for a feature's cell and ``reasons[1]`` for the label's (column k)."""
    if rc == N.LO_ERR_INVALID and info.bad_row >= 0:
        raise InvalidCellError(info.bad_row, info.bad_col, reason=reasons[info.bad_col == k])
    N.check(rc)


class _Owned(contextlib.ExitStack):
    """The tables a call makes for its result: :meth:`own` frees them when the call raises; a call that returns keeps
    them."""

    def own(self, table):
        if table is not None:
            self.callback(table.free)
        return table

    def __exit__(self, exc_type, *rest):
        if exc_type is None:
            self.pop_all()
        return super().__exit__(exc_type, *rest)


class AssembledRows:
    """The feature matrix one device made (:meth:`Engine.assemble_rows`): ``x`` a flat table holding ``nkept`` rows of
    ``k`` values, row-major; ``y`` the label's flat table or None; ``rows`` the kept source rows (int64, output order)
    plus ``first``, the shard's first row.  ``kept`` None: every row was kept, and ``rows`` is made only when read.
    :meth:`matrix` / :meth:`vector` view them in place.  :meth:`free` frees both tables; it may be called again."""

    def __init__(self, x: "DeviceTable", y: "DeviceTable | None", kept: np.ndarray | None, k: int, nkept: int):
        self.x, self.y, self.kept, self.k, self.nkept = x, y, kept, int(k), int(nkept)
        self.first = 0

    @property
    def rows(self) -> np.ndarray:
        if self.kept is None:
            return np.arange(self.first, self.first + self.nkept, dtype=np.int64)
        return self.kept + self.first

    def matrix(self, keepalive=None) -> DeviceArray:
        return DeviceArray(self.x, (self.nkept, self.k), keepalive)

    def vector(self, keepalive=None) -> DeviceArray | None:
        return None if self.y is None else DeviceArray(self.y, (self.nkept,), keepalive)

    def free(self) -> None:
        for t in (self.x, self.y):
            if t is not None:
                t.free()


class ColumnStats(tuple):
    """What :meth:`Engine.lr_stats` returns: the tuple (n, sum, m2, label_counts), and ``min`` / ``max`` (float64[k]),
    every column's least and greatest value, by which :meth:`ShardedEngine.lr_stats` finds the columns that hold one
    value over all shards."""

    def __new__(cls, n, total, m2, counts, least, most):
        self = super().__new__(cls, (n, total, m2, counts))
        self.min, self.max = least, most
        return self


class PredictedRows:
    """What :meth:`Engine.nb_predict` wrote for one device's rows: ``prob`` (n x C f64, row-major), ``pred`` (n f64 class
    indices) and ``raw`` (n x C f64, or None).  :meth:`probability` / :meth:`prediction` / :meth:`raw_view` view them in
    place; :meth:`free` frees every table and may be called again."""

    def __init__(self, prob: "DeviceTable", raw: "DeviceTable | None", pred: "DeviceTable", n: int, nclasses: int):
        self.prob, self.raw, self.pred, self.n, self.nclasses = prob, raw, pred, int(n), int(nclasses)

    def probability(self, keepalive=None) -> DeviceArray:
        return DeviceArray(self.prob, (self.n, self.nclasses), keepalive)

    def prediction(self, keepalive=None) -> DeviceArray:
        return DeviceArray(self.pred, (self.n,), keepalive)

    def raw_view(self, keepalive=None) -> DeviceArray | None:
        return None if self.raw is None else DeviceArray(self.raw, (self.n, self.nclasses), keepalive)

    def free(self) -> None:
        for t in (self.prob, self.raw, self.pred):
            if t is not None:
                t.free()


class SortedColumns:
    """What :meth:`Engine.dt_sort` made: ``keys`` (a table holding kc sorted columns of n order-preserving codes),
    ``f32`` (32-bit codes), ``distinct`` per column (ndistinct, values or None, counts or None).  :meth:`free` frees the
    keys and may be called again."""

    def __init__(self, keys: "DeviceTable", n: int, kc: int, f32: bool, distinct: list):
        self.keys, self.n, self.kc, self.f32, self.distinct = keys, int(n), int(kc), bool(f32), distinct

    def free(self) -> None:
        if self.keys is not None:
            self.keys.free()
        self.keys = None


class BinnedRows:
    """What :meth:`Engine.dt_bin` made for one device's rows: ``codes`` (LO_U8, n rows at :func:`code_pitch` (k)) and
    ``slots``, two LO_I32 tables of the rows' node slots that the levels write in turn (``cur`` the latest; n long, or
    ntrees * n once :meth:`Engine.rf_level` grew a batch of trees).  :meth:`free` frees them and may be called again."""

    def __init__(self, codes: "DeviceTable", slots: list):
        self.codes, self.slots, self.cur = codes, slots, 0

    def free(self) -> None:
        for t in [self.codes, *self.slots]:
            t.free()


class BoostRows:
    """What :meth:`Engine.gb_update` keeps for one device's rows during a GBT fit: ``margin`` (F) and ``residual`` (r),
    two LO_F64 tables of n.  :meth:`free` frees them and may be called again."""

    def __init__(self, margin: "DeviceTable", residual: "DeviceTable"):
        self.margin, self.residual = margin, residual

    def free(self) -> None:
        for t in (self.margin, self.residual):
            t.free()


def node_arrays(trees, payload):
    """The node arrays of a tree (lo_dt_predict, lo_gb_update) or a forest (lo_gb_predict, lo_rf_predict): (start
    int32[ntrees], nodes, feature int32, threshold f64, left int32, right int32, payload f64) with every tree's children
    shifted to indices into the concatenation; ``payload(tree)`` is a tree's per-node values (its class counts, leaf
    values or votes), one row per node."""
    start, at, cols = [], 0, [[] for _ in range(5)]
    for t in trees:
        start.append(at)
        for c, a in zip(cols, (t.feature, t.threshold, np.where(t.left >= 0, t.left + at, -1),
                               np.where(t.right >= 0, t.right + at, -1), payload(t))):
            c.append(a)
        at += t.num_nodes
    dts = (np.int32, np.float64, np.int32, np.int32, np.float64)
    return (np.array(start, np.int32), at, *[np.ascontiguousarray(np.concatenate(c), dt) for c, dt in zip(cols, dts)])


def code_pitch(k: int) -> int:
    """The row pitch in bytes of the bin code matrix of k features: a multiple of 16, for 16-byte loads."""
    return (k + 15) // 16 * 16


def _threshold_table(thresholds, k: int):
    """(f64 [k, tstride] thresholds padded, int32[k] counts, tstride >= 1) of per-column threshold lists."""
    if len(thresholds) != k:
        raise ValueError(f"{len(thresholds)} threshold lists for {k} features")
    nthr = np.array([len(t) for t in thresholds], np.int32)
    tstride = max(1, int(nthr.max()) if k else 1)
    thr = np.zeros((k, tstride), np.float64)
    for j, t in enumerate(thresholds):
        thr[j, :len(t)] = t
    return thr, nthr, tstride


ASSEMBLE_MODES = {"error": N.LO_INVALID_ERROR, "skip": N.LO_INVALID_SKIP, "keep": N.LO_INVALID_KEEP}
ASSEMBLE_DTYPES = {"float32": "f32", "float64": "f64"}


def assemble_args(handle_invalid: str, dtype: str) -> tuple[int, str]:
    """(lo_assemble_rows mode, table dtype) of the Python names; ValueError for any other."""
    if handle_invalid not in ASSEMBLE_MODES:
        raise ValueError(f"handle_invalid must be one of {sorted(ASSEMBLE_MODES)}, not {handle_invalid!r}")
    if dtype not in ASSEMBLE_DTYPES:
        raise ValueError(f"dtype must be one of {sorted(ASSEMBLE_DTYPES)}, not {dtype!r}")
    return ASSEMBLE_MODES[handle_invalid], ASSEMBLE_DTYPES[dtype]


SPLIT_SEED = 0x5EED_5B17       # Features.random_split's seed when none is given


def split_bounds(weights) -> np.ndarray:
    """The bounds (float64[len(weights) + 1]) of Spark's ``randomSplit(weights)``: each weight over their sum, summed
    in order from 0.0 in float64, as Spark computes them; a last bound may round below 1.0.  Refuses an empty list, a
    negative or non-finite weight, a zero sum and more than LO_SPLIT_MAX weights (ValueError)."""
    w = [float(v) for v in weights]
    if not w:
        raise ValueError("random_split needs at least one weight")
    if len(w) > N.LO_SPLIT_MAX:
        raise ValueError(f"{len(w)} weights: at most LO_SPLIT_MAX = {N.LO_SPLIT_MAX} splits")
    if any(not math.isfinite(v) or v < 0.0 for v in w):
        raise ValueError(f"weights must be finite and >= 0, not {list(weights)!r}")
    total = 0.0
    for v in w:
        total += v
    if not total > 0.0:
        raise ValueError("the weights sum to 0")
    bounds, run = [0.0], 0.0
    for v in w:
        run += v / total
        bounds.append(run)
    return np.array(bounds, np.float64)


class DeviceTable:
    """Columnar table in HBM: ``ncols`` slabs of ``nrows`` elements of one dtype."""

    def __init__(self, engine: "Engine", handle: C.c_void_p, keepalive=None):
        self.engine, self._h, self._keepalive = engine, handle, keepalive
        dt, nr, nc, pitch, base = C.c_int(), C.c_int64(), C.c_int32(), C.c_int64(), C.c_void_p()
        N.check(engine._lib.lo_table_info(handle, C.byref(dt), C.byref(nr), C.byref(nc), C.byref(pitch), C.byref(base)))
        self.dtype_code, self.nrows, self.ncols = dt.value, nr.value, nc.value
        self.pitch_bytes, self.base_ptr = pitch.value, base.value or 0
        self.np_dtype = _NP[self.dtype_code]

    def upload(self, col: int, values: np.ndarray, row0: int = 0) -> None:
        a = np.ascontiguousarray(values, dtype=self.np_dtype)
        N.check(self.engine._lib.lo_table_upload_col(self.engine._ctx, self._h, col, row0,
                                                     a.ctypes.data_as(C.c_void_p), a.shape[0]))

    def to_numpy(self, col: int, row0: int = 0, nrows: int | None = None, stream=None, out: np.ndarray | None = None) -> np.ndarray:
        """Ordered after the work already enqueued on ``stream`` (None = the engine's own stream); waits for that
        stream only, never for the whole device."""
        n = self.nrows - row0 if nrows is None else nrows
        if out is None:
            out = np.empty(n, dtype=self.np_dtype)
        N.check(self.engine._lib.lo_table_download_col(self.engine._ctx, self._h, col, row0,
                                                       out.ctypes.data_as(C.c_void_p), n, _stream_ptr(stream)))
        return out

    def column_view(self, col: int, keepalive=None) -> DeviceColumn:
        """The slab of one column as a ``__cuda_array_interface__`` object (no copy)."""
        return DeviceColumn(self, col, keepalive)

    def fill_synthetic(self, kind: int, seed: int, row_offset: int = 0, lo: float = -1000.0, hi: float = 1000.0,
                       stream=None) -> "DeviceTable":
        N.check(self.engine._lib.lo_table_fill_synthetic_dev(self.engine._ctx, self._h, kind, C.c_uint64(seed),
                                                             row_offset, lo, hi, _stream_ptr(stream)))
        return self

    def checksum(self, col: int, row_offset: int = 0) -> int:
        out = C.c_uint64()
        N.check(self.engine._lib.lo_table_checksum(self.engine._ctx, self._h, col, row_offset, C.byref(out)))
        return int(out.value)

    def free(self) -> None:
        if self._h is not None and self.engine._ctx is not None:
            N.check(self.engine._lib.lo_table_free(self.engine._ctx, self._h))
        self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class DeviceText:
    """One text column resident in HBM (``lo_text_upload``): chars, offsets and validity on the device, and ``arr``, the
    Arrow ``large_string`` array it was made from, which the group keys are read from (``arr.take(rep_rows)``).
    ``n`` cells, ``nulls`` of them null, ``nbytes`` device bytes held."""

    def __init__(self, engine: "Engine", handle: C.c_void_p, arr):
        self.engine, self._h, self.arr = engine, handle, arr
        n, chars, nulls, dev = C.c_int64(), C.c_int64(), C.c_int64(), C.c_size_t()
        N.check(engine._lib.lo_text_info(handle, C.byref(n), C.byref(chars), C.byref(nulls), C.byref(dev)))
        self.n, self.chars, self.nulls, self.nbytes = n.value, chars.value, nulls.value, dev.value

    def free(self) -> None:
        if self._h is not None and self.engine._ctx is not None:
            N.check(self.engine._lib.lo_text_free(self.engine._ctx, self._h))
        self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Engine:
    """One libloexec context = one H100.  ``Engine(device)`` raises LoexecError without a GPU."""

    def __init__(self, device: int = 0):
        self._lib = N.load()
        ctx = C.c_void_p()
        N.check(self._lib.lo_init(int(device), C.byref(ctx)))
        self._ctx = ctx
        dev, sms, hbm = C.c_int(), C.c_int(), C.c_size_t()
        N.check(self._lib.lo_ctx_device(ctx, C.byref(dev), C.byref(sms), C.byref(hbm)))
        self.device, self.sm_count, self.hbm_bytes = dev.value, sms.value, hbm.value
        self._pinned: dict[int, C.c_void_p] = {}
        self._staged: dict[str, np.ndarray] = {}     # reused pinned buffers (read_csv_stream)
        self._stream_lock = threading.Lock()          # read_csv_stream's buffers serve one call at a time

    # ---- lifetime ---------------------------------------------------------------------------------
    def close(self) -> None:
        if self._ctx is not None and getattr(self, "_resident", None) is not None:
            self._resident.clear()
        if self._ctx is not None:
            for p in list(self._pinned.values()):
                self._lib.lo_host_free(self._ctx, p)
            self._pinned.clear()
            self._staged.clear()
            self._lib.lo_shutdown(self._ctx)
            self._ctx = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def sync(self, stream=None) -> None:
        N.check(self._lib.lo_sync(self._ctx, _stream_ptr(stream)))

    @property
    def launch_count(self) -> int:
        out = C.c_int64()
        N.check(self._lib.lo_launch_count(self._ctx, C.byref(out)))
        return int(out.value)

    # ---- memory -------------------------------------------------------------------------------------
    def table(self, dtype: str, nrows: int, ncols: int) -> DeviceTable:
        h = C.c_void_p()
        N.check(self._lib.lo_table_alloc(self._ctx, _DTYPES[dtype], int(nrows), int(ncols), C.byref(h)))
        return DeviceTable(self, h)

    def wrap(self, dtype: str, nrows: int, ncols: int, base_ptr: int, pitch_bytes: int, keepalive=None) -> DeviceTable:
        h = C.c_void_p()
        N.check(self._lib.lo_table_wrap(self._ctx, _DTYPES[dtype], int(nrows), int(ncols), C.c_void_p(int(base_ptr)),
                                        int(pitch_bytes), C.byref(h)))
        return DeviceTable(self, h, keepalive)

    def table_from_numpy(self, columns: np.ndarray | Sequence[np.ndarray]) -> DeviceTable:
        """columns: [ncols, nrows] array (or list of equal-length 1-D arrays) of float64 / float32 / uint8."""
        cols = [np.asarray(c) for c in columns]
        name = {np.dtype(np.float64): "f64", np.dtype(np.float32): "f32", np.dtype(np.uint8): "u8"}[cols[0].dtype]
        t = self.table(name, cols[0].shape[0], len(cols))
        for j, c in enumerate(cols):
            t.upload(j, c)
        return t

    def counts(self, k: int, nbins: int) -> DeviceCounts:
        return DeviceCounts(self, k, nbins)

    def wrap_counts(self, k: int, nbins: int, ptr: int, keepalive=None) -> DeviceCounts:
        return DeviceCounts(self, k, nbins, ptr=ptr, keepalive=keepalive)

    def pinned_empty(self, shape, dtype, write_combined: bool = False) -> np.ndarray:
        """numpy array backed by page-locked host memory (freed by close()).  ``write_combined``: for staging buffers
        the host only writes (GPU inputs) — never read them back on the CPU."""
        dtype = np.dtype(dtype)
        nbytes = int(np.prod(shape)) * dtype.itemsize
        p = C.c_void_p()
        N.check(self._lib.lo_host_alloc_flags(self._ctx, max(nbytes, 1), 1 if write_combined else 0, C.byref(p)))
        self._pinned[p.value] = p
        buf = (C.c_char * max(nbytes, 1)).from_address(p.value)
        return np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)

    def selftest_fastdiv(self, lo: float, hi: float, nbins: int) -> tuple[bool, int]:
        """(fast kernels would be used, number of fp32 bit patterns whose bin differs from IEEE division)."""
        used, bad = C.c_int(), C.c_uint64()
        N.check(self._lib.lo_selftest_fastdiv(self._ctx, float(lo), float(hi), int(nbins), C.byref(used), C.byref(bad)))
        return bool(used.value), int(bad.value)

    def edge_tables_info(self) -> tuple[int, int, int]:
        """(edge tables cached on the context, their bytes, tile launches that binned with the IEEE divide)."""
        n, b, d = C.c_int32(), C.c_uint64(), C.c_int64()
        N.check(self._lib.lo_edge_tables_info(self._ctx, C.byref(n), C.byref(b), C.byref(d)))
        return int(n.value), int(b.value), int(d.value)

    def selftest_edges(self, lo: float, hi: float, nbins: int) -> tuple[bool, int]:
        """(edge-table kernels would be used, number of fp32 bit patterns whose counter differs from the IEEE-divide bin's)."""
        used, bad = C.c_int(), C.c_uint64()
        N.check(self._lib.lo_selftest_edges(self._ctx, float(lo), float(hi), int(nbins), C.byref(used), C.byref(bad)))
        return bool(used.value), int(bad.value)

    # ---- hot path, device resident ---------------------------------------------------------------
    def _spec(self, k: int, nbins: int, lo, hi, flags: int = 0):
        lo_a = (C.c_float * k)(*[float(v) for v in np.broadcast_to(np.asarray(lo, dtype=np.float32), (k,))])
        hi_a = (C.c_float * k)(*[float(v) for v in np.broadcast_to(np.asarray(hi, dtype=np.float32), (k,))])
        spec = N.HistSpec(int(nbins), int(flags), C.cast(lo_a, C.POINTER(C.c_float)), C.cast(hi_a, C.POINTER(C.c_float)))
        return spec, (lo_a, hi_a)

    def project_cast(self, table: DeviceTable, col_idx, out: DeviceTable | None = None, out_dtype: str = "f32",
                     stream=None) -> DeviceTable:
        idx, k = _i32(col_idx)
        if out is None:
            out = self.table(out_dtype, table.nrows, k)
        N.check(self._lib.lo_project_cast_dev(self._ctx, table._h, idx, k, out._h, _stream_ptr(stream)))
        return out

    def project_cast_hist(self, table: DeviceTable, col_idx, nbins: int, lo, hi, out: DeviceTable | None = None,
                          counts: DeviceCounts | None = None, stream=None) -> DeviceCounts:
        """Fused projection + cast + histogram; ``out=None`` computes the histogram only.
        ``counts`` is accumulated into (a fresh zeroed one is allocated when omitted)."""
        idx, k = _i32(col_idx)
        spec, _keep = self._spec(k, nbins, lo, hi)
        if counts is None:
            counts = self.counts(k, nbins)
        N.check(self._lib.lo_project_cast_hist_dev(self._ctx, table._h, idx, k, out._h if out is not None else None,
                                                   C.byref(spec), counts._ptr, _stream_ptr(stream)))
        return counts

    def hist_u8_cols(self, table: DeviceTable, col_idx, counts: DeviceCounts | None = None, stream=None) -> DeviceCounts:
        idx, k = _i32(col_idx)
        if counts is None:
            counts = self.counts(k, 256)
        N.check(self._lib.lo_hist_u8_cols_dev(self._ctx, table._h, idx, k, counts._ptr, _stream_ptr(stream)))
        return counts

    # ---- hot path, host buffers ------------------------------------------------------------------
    def project_cast_hist_host(self, cols: Sequence[np.ndarray], nbins: int | None = None, lo=None, hi=None,
                               out: Sequence[np.ndarray] | None = None):
        """cols: k contiguous float64 arrays (the projected columns, any host memory; pinned memory from
        :meth:`pinned_empty` lets copies overlap kernels).  out: k float32 arrays to fill, or None.
        Returns (counts [k, nbins] uint64 | None, timing dict)."""
        k = len(cols)
        in_p, n = _host_cols(cols, np.float64)
        out_p = _out_cols(out, k, n)
        spec_ref, counts, keep = None, None, None
        if nbins:
            spec, keep = self._spec(k, nbins, lo, hi)
            spec_ref = C.byref(spec)
            counts = np.zeros((k, nbins), dtype=np.uint64)
        timing = N.HostTiming()
        N.check(self._lib.lo_project_cast_hist_host(self._ctx, in_p, n, k, out_p, spec_ref,
                                                    counts.ctypes.data_as(C.c_void_p) if counts is not None else None,
                                                    C.byref(timing)))
        return counts, _timing(timing)

    def hist_u8_cols_host(self, cols: Sequence[np.ndarray]):
        k = len(cols)
        in_p, n = _host_cols(cols, np.uint8)
        counts = np.zeros((k, 256), dtype=np.uint64)
        timing = N.HostTiming()
        N.check(self._lib.lo_hist_u8_cols_host(self._ctx, in_p, n, k, counts.ctypes.data_as(C.c_void_p), C.byref(timing)))
        return counts, _timing(timing)

    def value_counts_u32_host(self, codes: np.ndarray, ncodes: int) -> np.ndarray:
        """counts[c] = number of entries of ``codes`` (uint32, dictionary encoded) equal to c."""
        codes = np.ascontiguousarray(codes, dtype=np.uint32)
        counts = np.zeros(int(ncodes), dtype=np.uint64)
        N.check(self._lib.lo_value_counts_u32_host(self._ctx, codes.ctypes.data_as(C.c_void_p), codes.shape[0],
                                                   int(ncodes), counts.ctypes.data_as(C.c_void_p), None))
        return counts

    def minmax_cast_host(self, cols: Sequence[np.ndarray]):
        """(min, max, n_finite) per column of the fp32-cast values, NaN / inf ignored."""
        k = len(cols)
        cols = [np.ascontiguousarray(c, dtype=np.float64) for c in cols]
        n = cols[0].shape[0] if k else 0
        in_p = (C.c_void_p * k)(*[c.ctypes.data for c in cols])
        mins, maxs, cnt = np.zeros(k, np.float32), np.zeros(k, np.float32), np.zeros(k, np.uint64)
        N.check(self._lib.lo_minmax_cast_host(self._ctx, in_p, n, k, mins.ctypes.data_as(C.c_void_p),
                                              maxs.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p), None))
        return mins, maxs, cnt

    def bind_numa(self) -> tuple[int, int]:
        """Pin the calling thread to the CPUs next to this GPU; returns (numa node, cpus).  Call before allocating
        pinned buffers so they are first touched on the memory the GPU's PCIe root hangs off."""
        node, ncpus = C.c_int32(), C.c_int32()
        N.check(self._lib.lo_ctx_bind_numa(self._ctx, C.byref(node), C.byref(ncpus)))
        return int(node.value), int(ncpus.value)

    def parse_number_host(self, cells):
        """cells: list of ``str`` / ``bytes``.  Returns (values float64[n], status uint8[n]) — values are what
        CPython's ``float(cell)`` returns, status as LO_NUM_* (``_native``)."""
        from .columnar import pack_number_cells
        return self.parse_number_packed(*pack_number_cells(cells))   # non-ASCII digits / whitespace normalised as float(str) does

    def parse_number_packed(self, chars: np.ndarray, offsets: np.ndarray):
        """The same on an already packed column (chars uint8, offsets int64[n+1]) — e.g. the buffers of an Arrow
        ``large_string`` array, untouched.  The text must be ASCII-normalised (:func:`columnar.ascii_number_text`)."""
        n = offsets.shape[0] - 1
        values = np.zeros(n, dtype=np.float64)
        status = np.zeros(n, dtype=np.uint8)
        if n:
            N.check(self._lib.lo_parse_number_host(self._ctx, chars.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p),
                                                   n, values.ctypes.data_as(C.c_void_p), status.ctypes.data_as(C.c_void_p), None))
        return values, status

    def parse_number_into(self, table: DeviceTable, col: int, chars: np.ndarray, offsets: np.ndarray, nulls=None) -> dict:
        """``float(cell)`` of every cell of a packed text column (chars uint8, offsets int64[n+1], offsets[0] may be
        non-zero) written on the device into f64 column ``col`` of ``table``, one row per cell; null and empty cells
        become NaN.  The text must be ASCII-normalised (:func:`columnar.number_text`).  nulls: None, a bool array
        (True = null), or ``(bitmap, bit_offset)`` — an Arrow validity bitmap as uint8.  Returns the call's summary:
        ``first_invalid`` / ``first_unsupported`` (row relative to the first cell, or None), ``nulls`` (null + empty
        cells), ``integer`` (every other cell integer valued) and the lo_host_timing fields."""
        n = offsets.shape[0] - 1
        v, _keep = _validity(nulls, n)
        offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        s, t = N.ParseSummary(), N.HostTiming()
        N.check(self._lib.lo_parse_number_to_table(self._ctx, chars.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p),
                                                   C.byref(v), n, table._h, int(col), 0, C.byref(s), C.byref(t)))
        return _summary(s, t)

    def parse_text_into(self, table: DeviceTable, col: int, text: DeviceText) -> dict:
        """:meth:`parse_number_into` with a resident text column as the input (``lo_parse_text_to_table``): cell i of
        ``text`` goes to row i of f64 column ``col`` of ``table``, which has one row per cell, and no cell crosses PCIe.
        The text must be ASCII (:func:`columnar.number_text` returns it as it is).  Returns the same summary."""
        if text._h is None:
            raise ValueError("the text column has been freed")
        s, t = N.ParseSummary(), N.HostTiming()
        N.check(self._lib.lo_parse_text_to_table(self._ctx, text._h, table._h, int(col), C.byref(s), C.byref(t)))
        return _summary(s, t)

    def format_text(self, table: DeviceTable, col: int, valid: np.ndarray, is_int: np.ndarray) -> DeviceText:
        """The ``"string"`` cast of f64 column ``col`` of ``table`` into a new resident text column
        (``lo_format_table_to_text``), without reading it back (``arr`` None): row i is ``""`` where ``valid[i]`` is
        False, ``str(int)`` where ``is_int[i]``, else ``repr(float)``.  ``valid`` / ``is_int``: one bool per row; they
        cross PCIe as bitmaps.  An ``is_int`` row that is not finite and integral raises LoexecError naming it."""
        n = table.nrows
        flags = [np.asarray(a, dtype=bool) for a in (valid, is_int)]
        if any(a.shape != (n,) for a in flags):
            raise ValueError("valid and is_int must have one entry per row")
        (v, _kv), (i, _ki) = [_validity((np.packbits(a, bitorder="little"), 0), n) for a in flags]
        h, t = C.c_void_p(), N.HostTiming()
        N.check(self._lib.lo_format_table_to_text(self._ctx, table._h, int(col), C.byref(v), C.byref(i), C.byref(h),
                                                  C.byref(t)))
        return DeviceText(self, h, None)

    def download_text(self, text: DeviceText, offsets: np.ndarray | None = None, chars: np.ndarray | None = None):
        """(offsets int64[n + 1] from 0, chars uint8) of a resident text column (``lo_text_download``), written into
        ``offsets`` / ``chars`` when given (contiguous, of at least those sizes)."""
        offsets = np.empty(text.n + 1, np.int64) if offsets is None else offsets
        chars = np.empty(max(text.chars, 1), np.uint8) if chars is None else chars
        if offsets.dtype != np.int64 or offsets.shape != (text.n + 1,) or not offsets.flags.c_contiguous or \
                chars.dtype != np.uint8 or not chars.flags.c_contiguous:
            raise ValueError("offsets must be int64[n + 1] and chars uint8, both contiguous")
        N.check(self._lib.lo_text_download(self._ctx, text._h, offsets.ctypes.data_as(C.c_void_p),
                                           chars.ctypes.data_as(C.c_void_p), chars.size, None))
        return offsets, chars

    def format_column(self, table: DeviceTable, col: int, valid: np.ndarray, is_int: np.ndarray) -> DeviceText:
        """:meth:`format_text`, its ``arr`` the Arrow ``large_string`` array read back: the buffers
        :meth:`format_number_host` returns for the same column."""
        import pyarrow as pa
        text = self.format_text(table, col, valid, is_int)
        try:
            offsets, chars = self.download_text(text)
        except BaseException:
            text.free()
            raise
        text.arr = pa.LargeStringArray.from_buffers(text.n, pa.py_buffer(offsets), pa.py_buffer(chars[:text.chars]))
        return text

    def copy_column(self, src: DeviceTable, src_col: int, dst: DeviceTable, dst_col: int) -> None:
        """Column ``src_col`` of ``src`` into column ``dst_col`` of ``dst`` (same dtype and rows), device to device."""
        N.check(self._lib.lo_table_copy_col(self._ctx, src._h, int(src_col), dst._h, int(dst_col)))

    def format_number_host(self, values: np.ndarray, status: np.ndarray, timing: dict | None = None):
        """The inverse of :meth:`parse_number_packed`: values float64[n] and status uint8[n] (LO_NUM_FLOAT ->
        ``repr(float)``, LO_NUM_INTEGER -> ``str(int)``, LO_NUM_EMPTY -> ``""``) become one packed text column
        (chars uint8, offsets int64[n+1]) — the buffers of an Arrow ``large_string`` array.  Any other status, or an
        INTEGER value that is not finite and integral, raises LoexecError naming the row.  ``timing``: a dict to receive
        the call's lo_host_timing fields."""
        values = np.ascontiguousarray(values, dtype=np.float64)
        status = np.ascontiguousarray(status, dtype=np.uint8)
        n = values.shape[0]
        if status.shape != (n,):
            raise ValueError("values and status must be 1-D arrays of the same length")
        # one call: chars sized from an upper bound per cell (24 bytes covers every repr(float), 21 every int below
        # 2^64), then trimmed to the exact total
        big = np.abs(values) >= 2.0 ** 64
        bound = np.where(status == N.LO_NUM_EMPTY, 0,
                         np.where(status == N.LO_NUM_INTEGER, np.where(big, N.LO_FORMAT_MAX_CELL, 21), 24))
        cap = int(bound.sum(dtype=np.int64))
        chars = np.empty(max(cap, 1), dtype=np.uint8)
        offsets = np.zeros(n + 1, dtype=np.int64)
        t = N.HostTiming()
        N.check(self._lib.lo_format_number_host(self._ctx, values.ctypes.data_as(C.c_void_p), status.ctypes.data_as(C.c_void_p),
                                                n, offsets.ctypes.data_as(C.c_void_p), chars.ctypes.data_as(C.c_void_p), cap,
                                                C.byref(t)))
        _report(timing, t)
        return chars[:offsets[n]], offsets

    def read_csv_host(self, body, timing: dict | None = None):
        """Tokenise a CSV upload on the GPU with the reference's ``csv.reader`` rules (``lo_csv_read_host``).

        body: bytes-like or a contiguous uint8 array (pinned memory makes the copy faster).  Returns ``(header_cells,
        nrows, chars, offsets, failure)``: the header's cells (None when the header itself fails or there is no
        record), the number of data rows kept, one uint8 chars buffer and int64 ``offsets[ncols][nrows + 2]`` — column
        c's cell r (r = 0 the header) is ``chars[offsets[c, r]:offsets[c, r + 1]]``, the offsets absolute in chars, so
        ``offsets[c, 1:]`` are the Arrow offsets of column c's data rows.  failure: None or ``(kind, record, pos)`` with
        kind an LO_CSV_* code, record the failing record (0 the header) and pos the byte offset it was raised at.
        ``timing``: a dict to receive the calls' lo_host_timing fields, summed."""
        buf = body if isinstance(body, np.ndarray) else np.frombuffer(body, dtype=np.uint8)
        if buf.dtype != np.uint8 or buf.ndim != 1 or not buf.flags.c_contiguous:
            raise ValueError("body must be bytes or a contiguous 1-D uint8 array")
        h, info, t1, t2 = C.c_void_p(), N.CsvInfo(), N.HostTiming(), N.HostTiming()
        N.check(self._lib.lo_csv_read_host(self._ctx, buf.ctypes.data_as(C.c_void_p), buf.size, C.byref(h), C.byref(info),
                                           C.byref(t1)))
        try:
            offsets = np.empty((info.ncols, info.records + 1), dtype=np.int64)
            chars = np.empty(max(info.chars, 1), dtype=np.uint8)
            N.check(self._lib.lo_csv_columns_host(h, offsets.ctypes.data_as(C.c_void_p), chars.ctypes.data_as(C.c_void_p),
                                                  chars.size, C.byref(t2)))
        finally:
            N.check(self._lib.lo_csv_free(h))
        if timing is not None:
            timing.update(total_ms=t1.total_ms + t2.total_ms, kernel_ms=t1.kernel_ms, h2d_bytes=t1.h2d_bytes,
                          d2h_bytes=t1.d2h_bytes + t2.d2h_bytes, launches=t1.launches)
        chars = chars[:info.chars]
        header = [bytes(chars[offsets[c, 0]:offsets[c, 1]]).decode("utf-8") for c in range(info.ncols)] \
            if info.records else None
        failure = None if info.fail_kind == N.LO_CSV_OK else (int(info.fail_kind), int(info.fail_record), int(info.fail_pos))
        return header, max(int(info.records) - 1, 0), chars, offsets, failure

    def _staging(self, key: str, nbytes: int) -> np.ndarray:
        """A page-locked uint8 buffer of at least nbytes kept on the engine under ``key``, replaced when too small."""
        old = self._staged.get(key)
        if old is not None and old.size >= nbytes:
            return old
        if old is not None:
            self._lib.lo_host_free(self._ctx, self._pinned.pop(old.ctypes.data))
        buf = self._staged[key] = self.pinned_empty(max(int(nbytes), 1), np.uint8)
        return buf

    def read_csv_stream(self, source, window_bytes: int | None = None, timing: dict | None = None):
        """:meth:`read_csv_host` on a body of any size: the source is read in pieces of one window into pinned memory
        and streamed through the device reader (``lo_csv_stream_*``), whose device memory is bounded by the window, not
        the body; the whole body is never held on the host either.

        source: a path, a binary (or text) file object, or an iterable of ``bytes``.  window_bytes: the window's
        starting size (None: LO_CSV_STREAM_WINDOW, 64 MiB); it doubles while a record does not fit.  Returns
        ``(header_cells, nrows, columns, failure)``: columns are one single-chunk ``pa.LargeStringArray`` per header
        cell, failure as :meth:`read_csv_host` gives it; the result equals read_csv_host's on the whole body.
        ``timing``: a dict to receive the calls' lo_host_timing fields summed, the number of windows read and the most
        device memory the stream held (``peak_device_bytes``)."""
        window = int(window_bytes) if window_bytes else N.LO_CSV_STREAM_WINDOW
        if window < 1:
            raise ValueError("window_bytes must be positive")
        with self._stream_lock:
            return self._read_csv_stream(source, window, timing)

    def _read_csv_stream(self, source, window, timing):
        import pyarrow as pa
        st, win, info, t = C.c_void_p(), N.CsvWindow(), N.CsvInfo(), N.HostTiming()
        sums = dict(total_ms=0.0, kernel_ms=0.0, h2d_bytes=0.0, d2h_bytes=0.0, launches=0, windows=0)

        def add(t, kernel=True):
            for k in ("total_ms", "h2d_bytes", "d2h_bytes", "launches") + (("kernel_ms",) if kernel else ()):
                sums[k] += getattr(t, k)

        piece = self._staging("csv_piece", window)
        header, cols = None, []
        N.check(self._lib.lo_csv_stream_open(self._ctx, window, C.byref(st)))
        try:
            for n, last in _pieces(source, piece):
                off = 0
                while True:
                    N.check(self._lib.lo_csv_stream_push(st, C.c_void_p(piece.ctypes.data + off), n - off, int(last),
                                                         C.byref(win), C.byref(info), C.byref(t)))
                    add(t)
                    if win.records:
                        sums["windows"] += 1
                        k, nc = int(win.records), int(win.ncols)
                        offsets = self._staging("csv_offsets", nc * (k + 1) * 8)[:nc * (k + 1) * 8].view(np.int64)
                        chars = self._staging("csv_chars", win.chars)
                        N.check(self._lib.lo_csv_stream_columns(st, offsets.ctypes.data_as(C.c_void_p),
                                                                chars.ctypes.data_as(C.c_void_p), chars.size, C.byref(t)))
                        add(t, kernel=False)
                        offsets = offsets.reshape(nc, k + 1)
                        r0 = 0
                        if win.first_record == 0:          # record 0: the header
                            header = [bytes(chars[offsets[c, 0]:offsets[c, 1]]).decode("utf-8") for c in range(nc)]
                            cols = [_TextBuilder() for _ in range(nc)]
                            r0 = 1
                        for c, col in enumerate(cols):
                            col.append(chars, offsets[c, r0:])
                    off += win.consumed
                    if win.done or (off >= n and not last):
                        break
                if win.done:
                    break
        finally:
            N.check(self._lib.lo_csv_stream_free(st))
        if timing is not None:
            timing.update(sums, peak_device_bytes=int(win.peak_device_bytes))
        failure = None if info.fail_kind == N.LO_CSV_OK else (int(info.fail_kind), int(info.fail_record), int(info.fail_pos))
        nrows = max(int(info.records) - 1, 0)
        columns = [col.array(pa) for col in cols] if header is not None else []
        return header, nrows, columns, failure

    def value_counts_str_packed(self, chars: np.ndarray, offsets: np.ndarray):
        """(rep_rows int64[g], counts uint64[g]) of an already packed text column (offsets[0] == 0)."""
        n = offsets.shape[0] - 1
        if n == 0:
            return np.zeros(0, np.int64), np.zeros(0, np.uint64)
        return _value_counts(lambda rows, counts, cap, nd, t: self._lib.lo_value_counts_str_host(
            self._ctx, chars.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p), n, rows, counts, cap, nd, t),
            n, np.int64)

    def text(self, cells, timing: dict | None = None) -> DeviceText:
        """A text column uploaded to HBM once for repeated counting: ``cells`` is an Arrow string array (its buffers go
        up as they are: a slice, nulls and any bit offset included) or a list of ``str`` / None (None = null).  Raises
        LoexecError LO_ERR_NOMEM when the device has too little free memory.  ``timing``: a dict to receive the call's
        lo_host_timing fields."""
        from .column_store import large_text
        from .columnar import text_buffers
        arr = large_text(cells)
        chars, offsets, validity = text_buffers(arr)
        v, _keep = _validity(validity, len(arr))
        h, t = C.c_void_p(), N.HostTiming()
        N.check(self._lib.lo_text_upload(self._ctx, chars.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p),
                                         C.byref(v), len(arr), C.byref(h), C.byref(t)))
        _report(timing, t)
        return DeviceText(self, h, arr)

    def value_counts_text(self, text: DeviceText, timing: dict | None = None):
        """(rep_rows int64[g], counts uint64[g]) of a resident text column (``lo_value_counts_text``): one
        representative row per distinct non-null cell, indexing the whole column, and the group sizes; null cells are
        not counted and no cell crosses PCIe.  ``timing``: a dict to receive the (last) call's lo_host_timing fields."""
        if text._h is None:
            raise ValueError("the text column has been freed")
        n = text.n - text.nulls
        if n == 0:
            return np.zeros(0, np.int64), np.zeros(0, np.uint64)
        return _value_counts(lambda rows, counts, cap, nd, t: self._lib.lo_value_counts_text(
            self._ctx, text._h, rows, counts, cap, nd, t), n, np.int64, timing)

    def text_codes(self, text: DeviceText, table: DeviceTable, col: int, timing: dict | None = None) -> np.ndarray:
        """Dictionary codes of a resident text column (``lo_text_codes``) into int32 column ``col`` of ``table`` (an
        ``"i32"`` table with one row per cell): -1 for a null row, else the code of the cell, the distinct cells numbered
        in the order of their first rows (``pyarrow.compute.dictionary_encode``'s order).  Returns those first rows
        (int64, ascending): the dictionary is ``text.arr.take(first_rows)`` (:func:`text_dictionary`).  No cell crosses
        PCIe.  ``timing``: a dict to receive the (last) call's lo_host_timing fields."""
        if text._h is None:
            raise ValueError("the text column has been freed")
        return _first_rows(lambda rows, cap, nd, t: self._lib.lo_text_codes(
            self._ctx, text._h, table._h, int(col), rows, cap, nd, t), text.n - text.nulls, timing)

    def text_codes_in(self, text: DeviceText, dictionary, table: DeviceTable, col: int, timing: dict | None = None) -> int:
        """Codes of a resident text column against ``dictionary`` (an Arrow string array without nulls, another column's
        :func:`text_dictionary`; ``lo_text_codes_in``) into int32 column ``col`` of ``table``: c where the cell equals
        ``dictionary[c]``, -1 for a null row or a cell the dictionary does not hold.  The dictionary is uploaded for the
        call and freed after it; no cell of ``text`` crosses PCIe.  Returns the non-null cells the dictionary does not
        hold.  A dictionary holding a cell twice raises LoexecError LO_ERR_INVALID.  ``timing``: a dict to receive the
        call's lo_host_timing fields."""
        if text._h is None:
            raise ValueError("the text column has been freed")
        d = self.text(dictionary)
        try:
            unseen, t = C.c_int64(), N.HostTiming()
            N.check(self._lib.lo_text_codes_in(self._ctx, text._h, d._h, table._h, int(col), C.byref(unseen), C.byref(t)))
        finally:
            d.free()
        _report(timing, t)
        return int(unseen.value)

    def assemble_rows(self, sources, label=None, dtype: str = "float32", handle_invalid: str = "error",
                      timing: dict | None = None) -> AssembledRows:
        """Spark's ``VectorAssembler`` on the device (``lo_assemble_rows``): row i of the result is the value of every
        ``(table, col)`` of ``sources`` at row i — an f64 slab's value, an int32 code column's code — as ``dtype``
        (``"float32"``: fp64->fp32 round-to-nearest-even; ``"float64"``: exact), and ``label`` (one more ``(table,
        col)`` or None) fills ``y``.  A NaN cell or a -1 code is invalid: ``handle_invalid="error"`` raises
        :class:`InvalidCellError` naming the lowest one, ``"skip"`` leaves its row out, ``"keep"`` writes NaN.
        ``timing``: a dict to receive the call's lo_host_timing fields."""
        mode, out = assemble_args(handle_invalid, dtype)
        k = len(sources)
        if k == 0:
            raise ValueError("assemble_rows needs at least one source column")
        if any(t._h is None for t, _c in sources) or (label is not None and label[0]._h is None):
            raise ValueError("a source table has been freed")
        n = sources[0][0].nrows
        tabs = (C.c_void_p * k)(*[t._h for t, _c in sources])
        cols = (C.c_int32 * k)(*[int(c) for _t, c in sources])
        rows = np.empty(n, np.int64) if mode == N.LO_INVALID_SKIP else None    # else every row is kept, in order
        info, t = N.AssembleInfo(), N.HostTiming()
        with _Owned() as owned:
            x = owned.own(self.table(out, n * k, 1))
            y = owned.own(self.table(out, n, 1) if label is not None else None)
            rc = self._lib.lo_assemble_rows(self._ctx, tabs, cols, k, label[0]._h if label is not None else None,
                                            int(label[1]) if label is not None else 0, mode, x._h, k,
                                            y._h if y is not None else None,
                                            rows.ctypes.data_as(C.c_void_p) if rows is not None else None,
                                            C.byref(info), C.byref(t))
            _check_cells(rc, info, k, _ASSEMBLE_REFUSED)
        _report(timing, t)
        return AssembledRows(x, y, rows[:info.nkept] if rows is not None else None, k, info.nkept)

    def random_split(self, part: AssembledRows, ids, bounds, seed: int, timing: dict | None = None) -> list:
        """Spark's ``randomSplit`` of ``part``'s rows on the device (``lo_random_split``): one :class:`AssembledRows` per
        split, each owning tables of exactly its rows, in row order, bit for bit.  ``ids`` (int64, one per row) are the
        rows' ``_id``; row i goes to split s when ``bounds[s] <= u < bounds[s + 1]`` for u drawn from (``seed``,
        ``ids[i]``) alone (:func:`split_bounds`).  ``part`` stays valid.  ``timing``: a dict to receive the call's
        lo_host_timing fields."""
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        b = np.ascontiguousarray(bounds, dtype=np.float64)
        ns, n = len(b) - 1, part.nkept
        if len(ids) != n:
            raise ValueError(f"{len(ids)} ids for {n} rows")
        if part.x._h is None or (part.y is not None and part.y._h is None):
            raise ValueError("the rows have been freed")
        xs, ys = (C.c_void_p * max(ns, 1))(), (C.c_void_p * max(ns, 1))()
        sizes, src = np.zeros(max(ns, 1), np.int64), np.empty(max(n, 1), np.int64)
        t = N.HostTiming()
        N.check(self._lib.lo_random_split(self._ctx, part.x._h, part.k, part.y._h if part.y is not None else None, n,
                                          ids.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), ns,
                                          C.c_uint64(int(seed) & 0xFFFFFFFFFFFFFFFF), xs,
                                          ys if part.y is not None else None, sizes.ctypes.data_as(C.c_void_p),
                                          src.ctypes.data_as(C.c_void_p), C.byref(t)))
        _report(timing, t)
        out, at = [], 0
        for s in range(ns):
            m = int(sizes[s])
            rows = src[at:at + m].copy()
            at += m
            kept = rows if part.kept is None else part.kept[rows]
            x = DeviceTable(self, C.c_void_p(xs[s]))
            y = DeviceTable(self, C.c_void_p(ys[s])) if part.y is not None else None
            a = AssembledRows(x, y, kept, part.k, m)
            a.first = part.first
            out.append(a)
        return out

    def nb_labels(self, part: AssembledRows) -> np.ndarray:
        """The distinct label values of ``part`` (an :class:`AssembledRows` with ``y``), ascending, -0.0 as 0.0
        (``lo_nb_labels``: the f64 group-by on the device).  A NaN label, or more than LO_NB_MAX_CLASSES values, raise
        LoexecError LO_ERR_INVALID."""
        if part.y is None:
            raise ValueError("the rows have no label")
        out = np.empty(N.LO_NB_MAX_CLASSES, np.float64)
        nd, t = C.c_int64(), N.HostTiming()
        N.check(self._lib.lo_nb_labels(self._ctx, part.y._h, part.nkept, out.ctypes.data_as(C.c_void_p), len(out),
                                       C.byref(nd), C.byref(t)))
        return out[:nd.value].copy()

    def nb_fit(self, part: AssembledRows, classes, timing: dict | None = None) -> tuple[np.ndarray, np.ndarray]:
        """(sums float64[C, k], counts int64[C]) of multinomial NaiveBayes over ``part`` (``lo_nb_fit``): counts[c] the
        rows labelled classes[c], sums[c, j] the f64 sum of feature j over them, in a fixed order.  A negative or NaN
        feature, or a label that is no class, raises :class:`InvalidCellError` naming the lowest row (``position`` the
        feature; k: the label).  ``timing``: a dict to receive the call's lo_host_timing fields."""
        if part.y is None:
            raise ValueError("the rows have no label")
        cls = np.ascontiguousarray(classes, dtype=np.float64)
        sums = np.zeros((len(cls), part.k), np.float64)
        counts = np.zeros(len(cls), np.int64)
        info, t = N.NbInfo(), N.HostTiming()
        rc = self._lib.lo_nb_fit(self._ctx, part.x._h, part.k, part.k, part.y._h, part.nkept, cls.ctypes.data_as(C.c_void_p),
                                 len(cls), sums.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p),
                                 C.byref(info), C.byref(t))
        _check_cells(rc, info, part.k, _FIT_REFUSED)
        _report(timing, t)
        return sums, counts

    def nb_predict(self, part: AssembledRows, pi, theta, raw: bool = False, labels=None, timing: dict | None = None):
        """A NaiveBayes model (``pi`` float64[C], ``theta`` float64[C, k]) over ``part`` (``lo_nb_predict``).
        ``labels`` None: transform — a :class:`PredictedRows` with every row's probability and prediction (and raw
        values with ``raw``).  ``labels`` the ascending label values to count: evaluate — the int64[len(labels), C]
        confusion counts of (label, prediction index), nothing written per row; a label not in ``labels`` raises
        :class:`InvalidCellError`.  ``timing``: a dict to receive the call's lo_host_timing fields."""
        pi = np.ascontiguousarray(pi, dtype=np.float64)
        theta = np.ascontiguousarray(theta, dtype=np.float64)
        nc = len(pi)
        if theta.shape != (nc, part.k):
            raise ValueError(f"theta has shape {theta.shape}, ({nc}, {part.k}) expected")
        return self._predict(self._lib.lo_nb_predict, (pi.ctypes.data_as(C.c_void_p), theta.ctypes.data_as(C.c_void_p),
                                                      nc), part, nc, raw, labels, timing)

    def _predict(self, fn, model: tuple, part: AssembledRows, nout: int, raw: bool, labels, timing: dict | None):
        """The transform / evaluate body of the ``*_predict`` calls: ``fn`` the library's entry point, ``model`` its
        arguments after (ctx, x, ld, k, n), ``nout`` the outputs per row.  ``labels`` None: a :class:`PredictedRows`;
        else the int64[len(labels), nout] confusion counts, a label not in ``labels`` raising :class:`InvalidCellError`."""
        n = part.nkept
        info, t = N.NbInfo(), N.HostTiming()
        args = (self._ctx, part.x._h, part.k, part.k, n, *model)
        if labels is not None:
            if part.y is None:
                raise ValueError("the rows have no label")
            lab = np.ascontiguousarray(labels, dtype=np.float64)
            conf = np.zeros((len(lab), nout), np.int64)
            rc = fn(*args, None, None, None, part.y._h, lab.ctypes.data_as(C.c_void_p), len(lab),
                    conf.ctypes.data_as(C.c_void_p), C.byref(info), C.byref(t))
            _check_cells(rc, info, part.k, _EVALUATE_REFUSED)
            _report(timing, t)
            return conf
        with _Owned() as owned:
            prob = owned.own(self.table("f64", n * nout, 1))
            pred = owned.own(self.table("f64", n, 1))
            rawt = owned.own(self.table("f64", n * nout, 1) if raw else None)
            N.check(fn(*args, prob._h, rawt._h if rawt is not None else None, pred._h, None, None, 0, None, C.byref(info),
                       C.byref(t)))
        _report(timing, t)
        return PredictedRows(prob, rawt, pred, n, nout)

    def lr_stats(self, part: AssembledRows, timing: dict | None = None) -> "ColumnStats":
        """(n, sum float64[k], m2 float64[k], label_counts int64[LO_NB_MAX_CLASSES]) of ``part``'s n rows
        (``lo_lr_stats_range``), a :class:`ColumnStats`: the f64 sum of every column, the sum of its squared deviations
        from ``sum / n`` (exactly 0 for a constant column) and the rows of each label 0, 1, ...; ``.min`` / ``.max`` every
        column's least and greatest value.  A
        feature that is not finite, or a label that is not an integer >= 0, raises :class:`InvalidCellError` naming the
        lowest row (``position`` the feature; k: the label); a label >= LO_NB_MAX_CLASSES raises LoexecError.
        ``timing``: a dict to receive the call's lo_host_timing fields."""
        if part.y is None:
            raise ValueError("the rows have no label")
        total, m2 = np.zeros(part.k, np.float64), np.zeros(part.k, np.float64)
        least, most = np.zeros(part.k, np.float64), np.zeros(part.k, np.float64)
        counts = np.zeros(N.LO_NB_MAX_CLASSES, np.int64)
        info, t = N.NbInfo(), N.HostTiming()
        rc = self._lib.lo_lr_stats_range(self._ctx, part.x._h, part.k, part.k, part.y._h, part.nkept,
                                         total.ctypes.data_as(C.c_void_p), m2.ctypes.data_as(C.c_void_p),
                                         least.ctypes.data_as(C.c_void_p), most.ctypes.data_as(C.c_void_p),
                                         counts.ctypes.data_as(C.c_void_p), C.byref(info), C.byref(t))
        _check_cells(rc, info, part.k, _LR_STATS_REFUSED)
        _report(timing, t)
        return ColumnStats(part.nkept, total, m2, counts, least, most)

    def lr_loss_grad(self, part: AssembledRows, coef, intercept, multinomial: bool,
                     timing: dict | None = None) -> tuple[float, np.ndarray, np.ndarray]:
        """LogisticAggregator's sums over ``part`` at one point (``lo_lr_loss_grad``): ``coef`` float64[C', k] the
        effective coefficients (Spark's over the column std), ``intercept`` float64[C'] (C' = 1 when binomial).  Returns
        (loss sum, gradient sums float64[C', k] of multiplier_c * x_j, intercept sums float64[C'])."""
        coef = np.ascontiguousarray(coef, dtype=np.float64)
        intercept = np.ascontiguousarray(intercept, dtype=np.float64)
        nc = len(intercept)
        if part.y is None:
            raise ValueError("the rows have no label")
        if coef.shape != (nc, part.k):
            raise ValueError(f"coef has shape {coef.shape}, ({nc}, {part.k}) expected")
        out = np.zeros(1 + nc * (part.k + 1), np.float64)
        t = N.HostTiming()
        N.check(self._lib.lo_lr_loss_grad(self._ctx, part.x._h, part.k, part.k, part.y._h, part.nkept,
                                          coef.ctypes.data_as(C.c_void_p), intercept.ctypes.data_as(C.c_void_p), nc,
                                          int(bool(multinomial)), out.ctypes.data_as(C.c_void_p), C.byref(t)))
        _report(timing, t)
        return float(out[0]), out[1:1 + nc * part.k].reshape(nc, part.k), out[1 + nc * part.k:]

    def lr_predict(self, part: AssembledRows, coef, intercept, multinomial: bool, threshold: float = 0.5,
                   raw: bool = False, labels=None, timing: dict | None = None):
        """A LogisticRegression model (``coef`` float64[C', k], ``intercept`` float64[C']; C' = 1 when binomial) over
        ``part`` (``lo_lr_predict``), as :meth:`nb_predict`: ``labels`` None gives a :class:`PredictedRows` (2 columns
        when binomial), else the int64[len(labels), C] confusion counts.  Binomial: prediction p1 > ``threshold``."""
        coef = np.ascontiguousarray(coef, dtype=np.float64)
        intercept = np.ascontiguousarray(intercept, dtype=np.float64)
        nc = len(intercept)
        if coef.shape != (nc, part.k):
            raise ValueError(f"coef has shape {coef.shape}, ({nc}, {part.k}) expected")
        model = (coef.ctypes.data_as(C.c_void_p), intercept.ctypes.data_as(C.c_void_p), nc, int(bool(multinomial)),
                 float(threshold))
        return self._predict(self._lib.lo_lr_predict, model, part, nc if multinomial else 2, raw, labels, timing)

    def dt_sort(self, part: AssembledRows, j0: int, kc: int, cap: int, timing: dict | None = None) -> "SortedColumns":
        """Columns [j0, j0 + kc) of ``part`` sorted on the device as order-preserving codes (``lo_dt_sort``), with every
        column's distinct values and their counts where there are at most ``cap`` of them."""
        n, f32 = part.nkept, part.x.dtype_code == N.LO_F32
        nd = np.zeros(kc, np.int64)
        vals = np.zeros((kc, max(cap, 1)), np.float64)
        cnts = np.zeros((kc, max(cap, 1)), np.int64)
        t = N.HostTiming()
        with _Owned() as owned:
            keys = owned.own(self.table("f32" if f32 else "f64", max(n * kc, 1), 1))
            N.check(self._lib.lo_dt_sort(self._ctx, part.x._h, part.k, part.k, n, int(j0), int(kc), keys._h, int(cap),
                                         nd.ctypes.data_as(C.c_void_p), vals.ctypes.data_as(C.c_void_p),
                                         cnts.ctypes.data_as(C.c_void_p), C.byref(t)))
        _report(timing, t)
        distinct = [(int(d), vals[c, :d].copy() if d <= cap else None, cnts[c, :d].copy() if d <= cap else None)
                    for c, d in enumerate(nd)]
        return SortedColumns(keys, n, kc, f32, distinct)

    def dt_rank(self, sorted_cols: "SortedColumns", cols, codes) -> tuple[np.ndarray, np.ndarray]:
        """(lt, le) int64 of every probe: the codes of column cols[i] below / up to codes[i] (``lo_dt_rank``)."""
        cols = np.ascontiguousarray(cols, np.int32)
        codes = np.ascontiguousarray(codes, np.uint64)
        lt, le = np.zeros(len(cols), np.int64), np.zeros(len(cols), np.int64)
        N.check(self._lib.lo_dt_rank(self._ctx, sorted_cols.keys._h, sorted_cols.n, sorted_cols.kc, len(cols),
                                     cols.ctypes.data_as(C.c_void_p), codes.ctypes.data_as(C.c_void_p),
                                     lt.ctypes.data_as(C.c_void_p), le.ctypes.data_as(C.c_void_p), None))
        return lt, le

    def dt_bin(self, part: AssembledRows, thresholds, timing: dict | None = None) -> "BinnedRows":
        """The bin code of every value of ``part`` (``lo_dt_bin``): Spark's findBin, java.util.Arrays.binarySearch of the
        column's ascending thresholds (without equal thresholds, the count of them below the value), in an LO_U8 table
        of n rows at pitch :func:`code_pitch` (k), with the two slot tables the levels use."""
        thr, nthr, tstride = _threshold_table(thresholds, part.k)
        kp = code_pitch(part.k)
        t = N.HostTiming()
        with _Owned() as owned:
            codes = owned.own(self.table("u8", max(part.nkept * kp, 1), 1))
            slots = [owned.own(self.table("i32", max(part.nkept, 1), 1)) for _ in range(2)]
            N.check(self._lib.lo_dt_bin(self._ctx, part.x._h, part.k, part.k, part.nkept, thr.ctypes.data_as(C.c_void_p),
                                        nthr.ctypes.data_as(C.c_void_p), tstride, codes._h, kp, C.byref(t)))
        _report(timing, t)
        return BinnedRows(codes, slots)

    def dt_level(self, part: AssembledRows, binned: "BinnedRows", nbins: int, nclasses: int, splits, nnodes: int,
                 shape: list | None = None, timing: dict | None = None) -> np.ndarray:
        """One tree level over ``part``'s rows (``lo_dt_level``): int64 (nnodes, k, nbins, nclasses) counts of (node
        slot, feature, bin, class).  ``splits`` None: the root level; else int32 (parents, 4) rows (feature, bin, left
        slot, right slot) of the previous level's nodes, by which the rows are routed (their slots ping-pong between
        ``binned``'s two tables).  ``shape``: a list to receive the launch shape (16-byte loads, features per chunk,
        nodes per pass, passes).  The whole level comes back to the host, however many node groups the device used.  A
        code >= nbins or a label outside [0, nclasses) raises LoexecError naming the row."""
        hist = np.zeros((nnodes, part.k, nbins, nclasses), np.int64)
        return self._level(self._lib.lo_dt_level, (part.y._h, part.nkept, int(nbins), int(nclasses)), part, binned,
                           splits, nnodes, hist, shape, timing)

    def _level(self, fn, lead: tuple, part: AssembledRows, binned: "BinnedRows", splits, nnodes: int, out: np.ndarray,
               shape: list | None, timing: dict | None) -> np.ndarray:
        """The level pass of :meth:`dt_level` / :meth:`gb_level` / :meth:`rf_level`: ``fn`` the library's entry point,
        ``lead`` its arguments after (ctx, codes, kp, k), ``out`` the array it fills.  The rows' slots ping-pong between ``binned``'s
        two tables; ``shape`` receives the launch shape."""
        k = part.k
        sp = np.ascontiguousarray(splits if splits is not None else np.zeros((0, 4)), np.int32)
        src = None if splits is None else binned.slots[binned.cur]
        dst = binned.slots[0 if splits is None else 1 - binned.cur]
        sh = np.zeros(4, np.int32)
        t = N.HostTiming()
        N.check(fn(self._ctx, binned.codes._h, code_pitch(k), k, *lead, src._h if src is not None else None,
                   int(splits is not None), dst._h, len(sp), sp.ctypes.data_as(C.c_void_p), int(nnodes),
                   out.ctypes.data_as(C.c_void_p), sh.ctypes.data_as(C.c_void_p), C.byref(t)))
        binned.cur = binned.slots.index(dst)
        if shape is not None:
            shape[:] = [int(v) for v in sh]
        _report(timing, t)
        return out

    def dt_predict(self, part: AssembledRows, tree, raw: bool = False, labels=None, timing: dict | None = None):
        """A tree (:class:`~tree.Tree`) over ``part`` (``lo_dt_predict``), as :meth:`nb_predict`: ``labels`` None gives a
        :class:`PredictedRows` of C columns, else the int64[len(labels), C] confusion counts."""
        _start, M, *arrs = node_arrays([tree], lambda t: t.counts)
        model = (M, *[a.ctypes.data_as(C.c_void_p) for a in arrs], tree.num_classes)
        return self._predict(self._lib.lo_dt_predict, model, part, tree.num_classes, raw, labels, timing)

    def gb_update(self, part: AssembledRows, rows: "BoostRows | None" = None, tree=None, weight: float = 1.0,
                  timing: dict | None = None) -> "BoostRows":
        """GBT's margins and residuals over ``part`` (``lo_gb_update``).  ``tree`` None: a new :class:`BoostRows` with F =
        0 and r = 2y - 1; else ``rows`` after the regression tree (:class:`~tree.Tree`) of weight ``weight``: F +=
        prediction * weight, r = 4y' / (1 + exp(2y'F)).  A label other than 0 or 1 raises :class:`InvalidCellError`
        (``position`` k)."""
        if part.y is None:
            raise ValueError("the rows have no label")
        n = part.nkept
        info, t = N.NbInfo(), N.HostTiming()
        with _Owned() as owned:
            if rows is None:
                rows = BoostRows(owned.own(self.table("f64", max(n, 1), 1)), owned.own(self.table("f64", max(n, 1), 1)))
            arrs = node_arrays([tree], lambda t: t.prediction)[2:] if tree is not None else []
            ptrs = [a.ctypes.data_as(C.c_void_p) for a in arrs] or [None] * 5
            rc = self._lib.lo_gb_update(self._ctx, part.x._h, part.k, part.k, part.y._h, n,
                                        tree.num_nodes if tree is not None else 0, *ptrs, float(weight),
                                        rows.margin._h, rows.residual._h, C.byref(info), C.byref(t))
            _check_cells(rc, info, part.k, _GB_REFUSED)
        _report(timing, t)
        return rows

    def gb_level(self, part: AssembledRows, binned: "BinnedRows", rows: "BoostRows", nbins: int, splits, nnodes: int,
                 shape: list | None = None, timing: dict | None = None) -> np.ndarray:
        """One regression-tree level over ``part``'s rows (``lo_gb_level``), routed as :meth:`dt_level`: uint64 (nnodes, k,
        nbins, LO_GB_WORDS) words of (node slot, feature, bin) — the count and the 128-bit fixed-point sums of the rows'
        residuals and their squares (:func:`tree.word_stats` reads them)."""
        words = np.zeros((nnodes, part.k, nbins, N.LO_GB_WORDS), np.uint64)
        return self._level(self._lib.lo_gb_level, (rows.residual._h, part.nkept, int(nbins)), part, binned, splits,
                           nnodes, words, shape, timing)

    def gb_predict(self, part: AssembledRows, trees, weights, raw: bool = False, labels=None,
                   timing: dict | None = None):
        """A GBT forest (regression :class:`~tree.Tree` s and their weights) over ``part`` (``lo_gb_predict``), as
        :meth:`nb_predict` with two classes: ``labels`` None gives a :class:`PredictedRows`, else the int64[len(labels),
        2] confusion counts."""
        start, M, *arrs = node_arrays(trees, lambda t: t.prediction)
        w = np.ascontiguousarray(weights, np.float64)
        if len(w) != len(trees):
            raise ValueError(f"{len(w)} weights for {len(trees)} trees")
        model = (len(trees), start.ctypes.data_as(C.c_void_p), w.ctypes.data_as(C.c_void_p), M,
                 *[a.ctypes.data_as(C.c_void_p) for a in arrs])
        return self._predict(self._lib.lo_gb_predict, model, part, 2, raw, labels, timing)

    def rf_level(self, part: AssembledRows, binned: "BinnedRows", nbins: int, nclasses: int, seed: int, draw,
                 tree0: int, ntrees: int, splits, features, row0: int = 0, shape: list | None = None,
                 timing: dict | None = None) -> np.ndarray:
        """One level of RandomForest trees tree0 .. tree0 + ntrees - 1 over ``part``'s rows (``lo_rf_level``): int64
        (nnodes, m, nbins, nclasses) sums of the rows' bagging weights per (node slot, listed feature, bin, class).
        ``features`` int32 (nnodes, m) lists each node's features; ``splits`` as :meth:`dt_level`, numbered across the
        batch in tree order (None: the root level, nnodes = ntrees).  ``draw`` is the bagging table
        (:func:`tree.draw_table`), ``seed`` the forest's seed and ``row0`` the global index of the part's first row.
        The rows' slots in every tree ping-pong between ``binned``'s two tables, made ntrees * n long at the root."""
        feats = np.ascontiguousarray(features, np.int32)
        nnodes, m = feats.shape
        dr = np.ascontiguousarray(draw, np.uint64)
        n = part.nkept
        if splits is None and binned.slots[0].nrows < ntrees * n:
            with _Owned() as owned:
                slots = [owned.own(self.table("i32", ntrees * n, 1)) for _ in range(2)]
            for t in binned.slots:
                t.free()
            binned.slots, binned.cur = slots, 0
        hist = np.zeros((nnodes, m, nbins, nclasses), np.int64)
        lead = (part.y._h, n, int(row0), int(nbins), int(nclasses), int(seed) & ((1 << 64) - 1), int(tree0),
                int(ntrees), dr.ctypes.data_as(C.c_void_p), len(dr), feats.ctypes.data_as(C.c_void_p), m)
        return self._level(self._lib.lo_rf_level, lead, part, binned, splits, nnodes, hist, shape, timing)

    def rf_predict(self, part: AssembledRows, trees, raw: bool = False, labels=None, timing: dict | None = None):
        """A RandomForest (classification :class:`~tree.Tree` s) over ``part`` (``lo_rf_predict``), as
        :meth:`nb_predict`: ``labels`` None gives a :class:`PredictedRows` of C columns, else the int64[len(labels), C]
        confusion counts.  Every leaf votes its counts over their total (:func:`tree.votes`)."""
        from .tree import votes
        start, M, *arrs = node_arrays(trees, votes)
        nc = trees[0].num_classes
        model = (len(trees), start.ctypes.data_as(C.c_void_p), M, *[a.ctypes.data_as(C.c_void_p) for a in arrs], nc)
        return self._predict(self._lib.lo_rf_predict, model, part, nc, raw, labels, timing)

    def value_counts_f64_host(self, values: np.ndarray):
        """(keys float64[g], counts uint64[g]) — exact value counts of a numeric column (GPU hash group-by),
        -0.0 grouped with 0.0 and all NaNs together; order unspecified."""
        values = np.ascontiguousarray(values, dtype=np.float64)
        n = values.shape[0]
        return _value_counts(lambda keys, counts, cap, nd, t: self._lib.lo_value_counts_f64_host(
            self._ctx, values.ctypes.data_as(C.c_void_p), n, keys, counts, cap, nd, t), n, np.float64)

    def value_counts_column(self, table: DeviceTable, col: int, timing: dict | None = None):
        """(keys float64[g], counts uint64[g]) of rows [0, nrows) of f64 column ``col`` of a device table
        (``lo_value_counts_f64_table``): the same groups as :meth:`value_counts_f64_host` with nothing copied to the
        device.  A null stored as NaN in the slab counts under the NaN key.  ``timing``: a dict to receive the (last)
        call's lo_host_timing fields."""
        return _value_counts(lambda keys, counts, cap, nd, t: self._lib.lo_value_counts_f64_table(
            self._ctx, table._h, int(col), keys, counts, cap, nd, t), table.nrows, np.float64, timing)

    def minmax_cast(self, table: DeviceTable, col_idx, stream=None):
        """(min, max, n_finite) of the fp32-cast values of resident columns (range pre-pass on the device)."""
        idx, k = _i32(col_idx)
        raw = self.counts(k, 3)
        N.check(self._lib.lo_minmax_cast_dev(self._ctx, table._h, idx, k, raw._ptr, _stream_ptr(stream)))
        host = raw.to_numpy(stream)
        raw.free()
        return _minmax_decode(self._lib, host, k)

    @property
    def resident(self):
        """Numeric columns of datasets kept in HBM between requests (:mod:`table_cache`)."""
        if getattr(self, "_resident", None) is None:
            from .table_cache import ResidentTables
            self._resident = ResidentTables(self)
        return self._resident

    def value_counts_str_host(self, cells):
        """cells: list of ``str`` / ``bytes``.  Returns (rep_rows int64[g], counts uint64[g]): one representative row
        per distinct cell and the group sizes (GPU hash group-by on the bytes, exact)."""
        from .columnar import pack_cells
        return self.value_counts_str_packed(*pack_cells(cells))
