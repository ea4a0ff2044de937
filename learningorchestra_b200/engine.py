"""Engine — the handle the reference's ``spark_session`` slot receives in this build.

Thin object layer over the C ABI (``include/loexec.h``): device-resident columnar tables and the
projection / cast / histogram entry points.  All computation happens in libloexec's sm_90a
kernels; nothing here falls back to numpy.

Reference boundary this replaces: ``projection_image/server.py:51-69`` builds a ``SparkSession``
and hands it to ``Projection`` (``projection_image/projection.py:14-18``); the histogram and
dataType services talk to mongod through pymongo (``histogram_image/utils.py:50-52``).
"""
from __future__ import annotations

import ctypes as C
import io
import os
import threading
from typing import Iterable, Sequence

import numpy as np

from . import _native as N

_DTYPES = {"f64": N.LO_F64, "f32": N.LO_F32, "u8": N.LO_U8}
_NP = {N.LO_F64: np.float64, N.LO_F32: np.float32, N.LO_U8: np.uint8}


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


def _minmax_decode(lib, raw: np.ndarray, k: int):
    """(min, max, n_finite) of k columns from the raw uint64[3k] of a min/max pre-pass."""
    mins, maxs, cnt = np.zeros(k, np.float32), np.zeros(k, np.float32), np.zeros(k, np.uint64)
    N.check(lib.lo_minmax_decode(raw.ctypes.data_as(C.c_void_p), k, mins.ctypes.data_as(C.c_void_p),
                                 maxs.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p)))
    return mins, maxs, cnt


def _value_counts(call, n: int, key_dtype):
    """(keys, counts) of a lo_value_counts_*_host call ``call(keys_out, counts_out, capacity, ndistinct_ref)``: room
    for min(n, 65536) groups first, called again with room for every group when they did not fit."""
    cap = max(min(n, 1 << 16), 1)
    while True:
        keys = np.empty(cap, dtype=key_dtype)
        counts = np.empty(cap, dtype=np.uint64)
        nd = C.c_int64()
        rc = call(keys.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p), cap, C.byref(nd))
        if rc == N.LO_ERR_INVALID and nd.value > cap:
            cap = int(nd.value)
            continue
        N.check(rc)
        return keys[:nd.value], counts[:nd.value]


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

    _TYPESTR = {N.LO_F64: "<f8", N.LO_F32: "<f4", N.LO_U8: "|u1"}

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

    def set_tma(self, enabled: bool) -> None:
        """Feed full tiles of the fused kernel through the TMA-staged variant (same results; DESIGN.md §3.8)."""
        N.check(self._lib.lo_set_tma(self._ctx, 1 if enabled else 0))

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
        if timing is not None:
            timing.update(_timing(t), kernel_ms=t.kernel_ms)
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
        return _value_counts(lambda rows, counts, cap, nd: self._lib.lo_value_counts_str_host(
            self._ctx, chars.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p), n, rows, counts, cap, nd, None),
            n, np.int64)

    def value_counts_f64_host(self, values: np.ndarray):
        """(keys float64[g], counts uint64[g]) — exact value counts of a numeric column (GPU hash group-by),
        -0.0 grouped with 0.0 and all NaNs together; order unspecified."""
        values = np.ascontiguousarray(values, dtype=np.float64)
        n = values.shape[0]
        return _value_counts(lambda keys, counts, cap, nd: self._lib.lo_value_counts_f64_host(
            self._ctx, values.ctypes.data_as(C.c_void_p), n, keys, counts, cap, nd, None), n, np.float64)

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
