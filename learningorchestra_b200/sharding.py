"""Row-range sharding of a table across the GPUs of one box, behind one engine-shaped object.

The reference has no multi-device path (one mongod pipeline / three single-core Spark executors,
``projection_image/server.py:58-60``).  Projection and cast are row-independent and the histogram is a
commutative integer sum over rows (``histogram_image/histogram.py:31-36``), so rank r owns the
contiguous rows ``[r*N/W, (r+1)*N/W)`` — boundaries rounded to 32 rows so every shard's slabs keep
their 128-byte alignment — runs the fused kernel on them, and ONE ``all_reduce(SUM)`` of the
``k x nbins`` uint64 count matrix (NCCL over NVLink when the tensor lives on the GPU) yields the
global histogram on every rank.  Integer sums are order independent, so the result is bit-exact
for any world size.  The projected fp32 output stays sharded the same way (the reference's reader
pages by ``_id`` range, ``database_api_image/utils.py:17-23``).
"""
from __future__ import annotations

import ctypes as C
import itertools
import threading

ROW_ALIGN = 32


def shard_bounds(total_rows: int, world_size: int, rank: int, align: int = ROW_ALIGN) -> tuple[int, int]:
    """Rows [begin, end) owned by ``rank``; every interior boundary is a multiple of ``align``."""
    if world_size < 1 or not 0 <= rank < world_size:
        raise ValueError(f"bad rank {rank} / world size {world_size}")
    if total_rows < 0:
        raise ValueError("total_rows < 0")

    def cut(r: int) -> int:
        if r >= world_size:
            return total_rows
        return min(total_rows, (total_rows * r // world_size) // align * align)

    return cut(rank), cut(rank + 1)


def all_shard_bounds(total_rows: int, world_size: int, align: int = ROW_ALIGN) -> list[tuple[int, int]]:
    return [shard_bounds(total_rows, world_size, r, align) for r in range(world_size)]


def allreduce_counts(counts_tensor, group=None):
    """In-place SUM all-reduce of a count matrix held in a torch int64 tensor (the uint64 counts' bit
    patterns: two's-complement addition is the same operation).  CUDA tensor + NCCL backend = one
    ncclAllReduce over NVLink on the current stream; CPU tensor + gloo = the host-logic test path."""
    import torch
    import torch.distributed as dist

    if counts_tensor.dtype != torch.int64:
        raise TypeError("counts must be viewed as int64")
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(counts_tensor, op=dist.ReduceOp.SUM, group=group)
    return counts_tensor


def column_batches(k: int, nbins: int, cap: int | None = None) -> list[tuple[int, int]]:
    """Column ranges [begin, end) of the group steps one ``k x nbins`` histogram request takes.  A group merges at most
    ``cap`` (LO_GROUP_MAX_COUNTS) counts per step: a request within that is one step, a larger one runs of
    ``max(1, cap // nbins)`` columns, in column order.  Depends on (k, nbins) only, so every rank issues the same steps."""
    if cap is None:
        from ._native import LO_GROUP_MAX_COUNTS as cap
    if k * nbins <= cap:
        return [(0, k)]
    per = max(1, cap // nbins)
    return [(c0, min(k, c0 + per)) for c0 in range(0, k, per)]


def on_each(n: int, fn, undo=None) -> list:
    """``[fn(0), ..., fn(n - 1)]``, each member's call on a host thread of its own so the devices work at once.  Every
    call runs to its end; when any raised, ``undo`` (if given) is called on each result the others returned and the
    first exception in member order is raised."""
    results, errors = [None] * n, [None] * n

    def run(i):
        try:
            results[i] = fn(i)
        except BaseException as exc:       # re-raised on the calling thread
            errors[i] = exc

    threads = [threading.Thread(target=run, args=(i,)) for i in range(n)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    failed = [e for e in errors if e is not None]
    if failed:
        if undo is not None:
            for r, e in zip(results, errors):
                if e is None:
                    undo(r)
        raise failed[0]
    return results


def _firsts(parts) -> list:
    """The first row of each of the shards' ``AssembledRows`` in the rows of all of them, shards in order."""
    return list(itertools.accumulate((p.nkept for p in parts[:-1]), initial=0))


def _combine_timings(parts) -> dict:
    out = dict(parts[0])
    for t in parts[1:]:
        for key in out:
            out[key] += t[key]
    return out


def combine_parse_summaries(parts, row_offsets) -> dict:
    """One ``parse_number_into`` summary from those of several shards: the first bad rows are the minimum over the
    shards after adding each shard's first global row, counts and bytes add up, ``integer`` holds on every shard, and
    the times are the longest shard's (the shards run at once)."""
    out = {"first_invalid": None, "first_unsupported": None, "nulls": 0, "integer": True, "total_ms": 0.0,
           "kernel_ms": 0.0, "h2d_bytes": 0.0, "d2h_bytes": 0.0, "launches": 0}
    for part, off in zip(parts, row_offsets):
        for key in ("first_invalid", "first_unsupported"):
            if part[key] is not None and (out[key] is None or off + part[key] < out[key]):
                out[key] = off + part[key]
        out["nulls"] += part["nulls"]
        out["integer"] = out["integer"] and part["integer"]
        for key in ("total_ms", "kernel_ms"):
            out[key] = max(out[key], part[key])
        for key in ("h2d_bytes", "d2h_bytes", "launches"):
            out[key] += part[key]
    return out


def merge_value_counts(parts):
    """One ``$group`` of a number column from the (keys float64, counts uint64) of its shards.  Keys are canonical on
    the device (one NaN pattern, no -0.0), so equal bits are the same group: the bit patterns are merged with
    ``np.unique`` and the counts summed in uint64, exactly."""
    import numpy as np
    if not parts:
        return np.zeros(0, np.float64), np.zeros(0, np.uint64)
    bits = np.concatenate([np.asarray(k, np.float64).view(np.uint64) for k, _ in parts])
    counts = np.concatenate([np.asarray(c, np.uint64) for _, c in parts])
    keys, inverse = np.unique(bits, return_inverse=True)
    sums = np.zeros(keys.size, np.uint64)
    np.add.at(sums, inverse.ravel(), counts)
    return keys.view(np.float64), sums


class ShardedTable:
    """A columnar table whose rows are range-sharded over the local members of a :class:`ShardedEngine`.
    ``shards[i]`` is the :class:`~learningorchestra_b200.engine.DeviceTable` on local member i and holds global
    rows ``[offsets[i], offsets[i] + shards[i].nrows)``."""

    def __init__(self, sharded: "ShardedEngine", shards, offsets, total_rows: int):
        self.engine, self.shards, self.offsets, self.nrows = sharded, list(shards), list(offsets), int(total_rows)
        self.ncols = self.shards[0].ncols
        self.np_dtype = self.shards[0].np_dtype

    @property
    def pitch_bytes(self) -> int:
        return sum(t.pitch_bytes for t in self.shards)

    @property
    def local_rows(self) -> int:
        return sum(t.nrows for t in self.shards)

    def fill_synthetic(self, kind: int, seed: int, lo: float = -1000.0, hi: float = 1000.0, streams=None) -> "ShardedTable":
        for i, (t, off) in enumerate(zip(self.shards, self.offsets)):
            t.fill_synthetic(kind, seed, row_offset=off, lo=lo, hi=hi, stream=streams[i] if streams else None)
        return self

    def upload(self, col: int, values) -> None:
        """``values``: the LOCAL rows of the column (all rows for a single-process engine)."""
        import numpy as np
        values = np.asarray(values)
        base = self.offsets[0]
        for t, off in zip(self.shards, self.offsets):
            t.upload(col, values[off - base:off - base + t.nrows])

    def to_numpy(self, col: int, streams=None):
        """The local rows of one column, in row order."""
        import numpy as np
        out = np.empty(self.local_rows, dtype=self.np_dtype)
        pos = 0
        for i, t in enumerate(self.shards):
            t.to_numpy(col, out=out[pos:pos + t.nrows], stream=streams[i] if streams else None)
            pos += t.nrows
        return out

    def checksum(self, col: int) -> int:
        """Position-weighted checksum of the local rows (global row numbers): shard sums add up mod 2^64."""
        return sum(t.checksum(col, row_offset=off) for t, off in zip(self.shards, self.offsets)) & 0xFFFFFFFFFFFFFFFF

    def free(self) -> None:
        for t in self.shards:
            t.free()
        self.shards = []


class ShardedText:
    """One text column cut into row-range pieces over the local members of a :class:`ShardedEngine`, at the slab shards'
    row split (:meth:`ShardedEngine.bounds`).  ``pieces[i]`` is the
    :class:`~learningorchestra_b200.engine.DeviceText` on local member i and holds global rows
    ``[offsets[i], offsets[i] + pieces[i].n)``.  ``arr`` is the whole Arrow array the group keys are read from (the
    representative rows are global); ``n``, ``nulls`` and ``nbytes`` sum over the pieces."""

    def __init__(self, pieces, offsets, arr):
        self.pieces, self.offsets, self.arr = list(pieces), list(offsets), arr
        self.n = sum(p.n for p in self.pieces)
        self.nulls = sum(p.nulls for p in self.pieces)
        self.nbytes = sum(p.nbytes for p in self.pieces)

    @classmethod
    def upload(cls, engines, bounds, arr, timing: dict | None = None) -> "ShardedText":
        """Rows ``[b, e)`` of ``arr`` (a ``large_string`` array) uploaded with ``engines[i].text`` for the i-th of
        ``bounds``, each from a host thread of its own.  When any upload fails (LO_ERR_NOMEM on a full device, say) the
        pieces already made are freed and the first error is raised.  ``timing``: the longest piece's times, the
        pieces' bytes and launches added up."""
        times = [{} for _ in engines]

        def run(i):
            b, e = bounds[i]
            return engines[i].text(arr.slice(b, e - b), timing=times[i])

        parts = on_each(len(engines), run, undo=lambda p: p.free())
        if timing is not None:
            timing.update({k: max(t[k] for t in times) for k in ("total_ms", "kernel_ms")},
                          **{k: sum(t[k] for t in times) for k in ("h2d_bytes", "d2h_bytes", "launches")})
        return cls(parts, [b for b, _ in bounds], arr)

    def args(self):
        """The ``shards`` and ``row0`` arguments of a ``lo_*_shards`` call on this column (ctypes arrays)."""
        if any(p._h is None for p in self.pieces):
            raise ValueError("the text column has been freed")
        k = len(self.pieces)
        return (C.c_void_p * k)(*[p._h for p in self.pieces]), (C.c_int64 * k)(*self.offsets)

    def check_cut(self, table) -> None:
        """Refuses a :class:`ShardedTable` whose shards do not hold the same rows as this column's pieces."""
        if self.offsets != table.offsets or [p.n for p in self.pieces] != [t.nrows for t in table.shards]:
            raise ValueError("the text column and the table are not cut at the same rows")

    def free(self) -> None:
        for p in self.pieces:
            p.free()


class GroupCounts:
    """Merged counts of the step that produced it, in the group's result buffer (valid until the next group call).
    A request split over several steps (:func:`column_batches`) has read each step's counts out already: ``host``
    holds them, or is None on a rank that receives no result."""

    def __init__(self, sharded: "ShardedEngine", k: int, nbins: int, host=None, batched: bool = False):
        self.engine, self.k, self.nbins = sharded, int(k), int(nbins)
        self._host, self._batched = host, batched

    def to_numpy(self, stream=None):
        if self._host is not None:
            return self._host.copy()
        if self._batched:
            N = self.engine._N
            raise N.LoexecError(N.LO_ERR_INVALID, "this rank received no merged counts (pass bcast=True to receive them everywhere)")
        return self.engine.result(self.k * self.nbins).reshape(self.k, self.nbins)

    def free(self) -> None:
        pass


class ShardedEngine:
    """Several H100s behind the same methods as :class:`~learningorchestra_b200.engine.Engine`.

    Everything multi-GPU lives in the library (``lo_group_*`` in ``include/loexec.h``): the peer mappings, the
    in-kernel merge of the partial histograms over NVLink, the NCCL fallback.  This class only forms the group and
    keeps one ``DeviceTable`` per local member:

    * :meth:`local` — ONE process drives all (or the listed) devices: what the three microservice entry points
      (``Projection.create`` / ``Histogram.create_file`` / ``DataType.convert_existent_file``) use on a multi-GPU box;
    * :meth:`from_torch_distributed` — one process per GPU (``torchrun``): what ``bench.py --gpus N`` uses.  The
      per-rank bootstrap blobs travel through ``dist.all_gather_object``; any other all-gather works the same way
      (:meth:`from_exchange`).
    """

    def __init__(self, engines, group_handle, rank0: int, world: int, owns_engines: bool):
        from . import _native as N
        self._N, self._lib = N, N.load()
        self.engines, self._g, self.rank0, self.world, self._owns = list(engines), group_handle, rank0, world, owns_engines
        self.nlocal = len(self.engines)
        w, nl, m = C.c_int32(), C.c_int32(), C.c_int32()
        N.check(self._lib.lo_group_info(self._g, C.byref(w), C.byref(nl), C.byref(m)))
        self.merge = {N.LO_MERGE_PEER: "peer", N.LO_MERGE_NCCL: "nccl"}[m.value]
        self.device = self.engines[0].device
        self.sm_count = self.engines[0].sm_count
        self._resident = None

    # ---- forming a group ------------------------------------------------------------------------------
    @staticmethod
    def _merge_code(merge: str) -> int:
        from . import _native as N
        return {"auto": N.LO_MERGE_AUTO, "peer": N.LO_MERGE_PEER, "p2p": N.LO_MERGE_PEER, "nccl": N.LO_MERGE_NCCL}[merge]

    @classmethod
    def local(cls, devices=None, merge: str = "auto") -> "ShardedEngine":
        from . import _native as N
        from .engine import Engine
        lib = N.load()
        if devices is None:
            n = C.c_int()
            N.check(lib.lo_device_count(C.byref(n)))
            devices = list(range(n.value))
        engines = [Engine(d) for d in devices]
        ctxs = (C.c_void_p * len(engines))(*[e._ctx for e in engines])
        g = C.c_void_p()
        try:
            N.check(lib.lo_group_create_local(ctxs, len(engines), cls._merge_code(merge), C.byref(g)))
        except Exception:
            for e in engines:
                e.close()
            raise
        return cls(engines, g, 0, len(engines), True)

    @classmethod
    def from_exchange(cls, engine, rank: int, world: int, all_gather, all_ok, merge: str = "auto") -> "ShardedEngine":
        """``all_gather(bytes) -> list[bytes]`` (rank order) and ``all_ok(bool) -> bool`` (logical AND over ranks) are
        the launcher's own out-of-band collectives.  ``merge="auto"`` tries the peer-memory merge and falls back to
        NCCL — on every rank together — when CUDA IPC is not permitted."""
        from . import _native as N
        lib = N.load()
        tries = ["peer", "nccl"] if merge == "auto" else [merge]
        last = None
        for m in tries:
            g, blob = C.c_void_p(), C.create_string_buffer(N.LO_GROUP_BLOB_BYTES)
            rc = lib.lo_group_rank_begin(engine._ctx, rank, world, cls._merge_code(m), C.byref(g), blob)
            msg = lib.lo_last_error().decode("utf-8", "replace") if rc != N.LO_OK else ""
            blobs = all_gather(blob.raw if rc == N.LO_OK else b"\0" * N.LO_GROUP_BLOB_BYTES)
            if rc == N.LO_OK:
                rc = lib.lo_group_rank_connect(g, C.create_string_buffer(b"".join(blobs), world * N.LO_GROUP_BLOB_BYTES))
                if rc != N.LO_OK:
                    msg = lib.lo_last_error().decode("utf-8", "replace")
            if all_ok(rc == N.LO_OK):
                return cls([engine], g, rank, world, False)
            last = msg or "another rank failed to connect"
            if g.value:
                lib.lo_group_destroy(g)
        raise N.LoexecError(N.LO_ERR_CUDA, f"could not form a {world}-rank group ({'/'.join(tries)}): {last}")

    @classmethod
    def from_torch_distributed(cls, engine, group=None, merge: str = "auto") -> "ShardedEngine":
        import torch
        import torch.distributed as dist
        rank, world = dist.get_rank(group), dist.get_world_size(group)
        on_gpu = dist.get_backend(group) == "nccl"

        def all_gather(b: bytes):
            out = [None] * world
            dist.all_gather_object(out, b, group=group)
            return out

        def all_ok(ok: bool) -> bool:
            t = torch.tensor([1.0 if ok else 0.0], device="cuda" if on_gpu else "cpu")
            dist.all_reduce(t, op=dist.ReduceOp.MIN, group=group)
            return float(t[0]) == 1.0

        return cls.from_exchange(engine, rank, world, all_gather, all_ok, merge)

    # ---- lifetime -------------------------------------------------------------------------------------
    def close(self) -> None:
        if self._resident is not None:
            self._resident.clear()
        if self._g is not None:
            self._lib.lo_group_destroy(self._g)
            self._g = None
        if self._owns:
            for e in self.engines:
                e.close()
        self.engines = []

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    @property
    def launch_count(self) -> int:
        return sum(e.launch_count for e in self.engines)

    def sync(self, streams=None) -> None:
        for i, e in enumerate(self.engines):
            e.sync(streams[i] if streams else None)

    # ---- tables -----------------------------------------------------------------------------------------
    def bounds(self, total_rows: int):
        """[(begin, end)] of the local members' shards of a ``total_rows`` table."""
        out = []
        for i in range(self.nlocal):
            b, e = C.c_int64(), C.c_int64()
            self._N.check(self._lib.lo_group_shard(self._g, int(total_rows), self.rank0 + i, C.byref(b), C.byref(e)))
            out.append((b.value, e.value))
        return out

    def table(self, dtype: str, total_rows: int, ncols: int) -> ShardedTable:
        bounds = self.bounds(total_rows)
        shards = [e.table(dtype, end - begin, ncols) for e, (begin, end) in zip(self.engines, bounds)]
        return ShardedTable(self, shards, [b for b, _ in bounds], total_rows)

    def table_from_numpy(self, columns, total_rows: int | None = None) -> ShardedTable:
        """columns: [ncols, rows] — all rows (single-process engine) or, with ``total_rows``, this rank's shard."""
        import numpy as np
        cols = [np.asarray(c) for c in columns]
        name = {np.dtype(np.float64): "f64", np.dtype(np.float32): "f32", np.dtype(np.uint8): "u8"}[cols[0].dtype]
        t = self.table(name, cols[0].shape[0] if total_rows is None else total_rows, len(cols))
        if t.local_rows != cols[0].shape[0]:
            raise ValueError(f"expected {t.local_rows} local rows, got {cols[0].shape[0]}")
        for j, c in enumerate(cols):
            t.upload(j, c)
        return t

    # ---- hot path over the group ----------------------------------------------------------------------
    def _tables(self, t: ShardedTable | None):
        if t is None:
            return None
        return (C.c_void_p * self.nlocal)(*[s._h for s in t.shards])

    def _streams(self, streams):
        from .engine import _stream_ptr
        if streams is None:
            return None
        return (C.c_void_p * self.nlocal)(*[_stream_ptr(s) for s in streams])

    def _flags(self, bcast: bool, independent: bool) -> int:
        return (self._N.LO_GROUP_BCAST if bcast else 0) | (self._N.LO_GROUP_INDEPENDENT if independent else 0)

    def project_cast_hist(self, table: ShardedTable, col_idx, nbins: int, lo, hi, out: ShardedTable | None = None,
                          bcast: bool = False, streams=None, independent: bool = False) -> GroupCounts:
        """One step over all shards: fused projection + cast + histogram on every member, partial histograms merged
        inside the kernels.  Asynchronous; the merged counts are read with ``.to_numpy()`` / :meth:`result`.
        ``independent``: this step reads nothing the previous group step wrote (another job, or the same inputs
        again), so it may start while that step's last wave is still draining.
        A request of more than LO_GROUP_MAX_COUNTS counts is split into column batches (:func:`column_batches`), one
        step each, whose merged counts are read out before the next step; the call then returns after the last."""
        from .engine import _i32
        idx, k = _i32(col_idx)
        batches = column_batches(k, nbins)
        if len(batches) == 1:
            spec, _keep = self.engines[0]._spec(k, nbins, lo, hi)
            self._N.check(self._lib.lo_group_project_cast_hist_dev(
                self._g, self._tables(table), idx, k, self._tables(out), C.byref(spec),
                self._flags(bcast, independent), self._streams(streams)))
            return GroupCounts(self, k, nbins)
        import numpy as np
        lo = np.broadcast_to(np.asarray(lo, np.float32), (k,))
        hi = np.broadcast_to(np.asarray(hi, np.float32), (k,))
        host = np.zeros((k, nbins), np.uint64) if bcast or self.has_result or self.merge == "nccl" else None
        for c0, c1 in batches:
            spec, _keep = self.engines[0]._spec(c1 - c0, nbins, lo[c0:c1], hi[c0:c1])
            views = self._column_views(out, c0, c1)
            try:
                self._N.check(self._lib.lo_group_project_cast_hist_dev(
                    self._g, self._tables(table), _i32(idx[c0:c1])[0], c1 - c0, self._tables(views), C.byref(spec),
                    self._flags(bcast, independent), self._streams(streams)))
            finally:
                if views is not None:
                    views.free()           # descriptors only: the kernels took base and pitch by value
            if host is not None:
                host[c0:c1] = self.result((c1 - c0) * nbins).reshape(c1 - c0, nbins)
        return GroupCounts(self, k, nbins, host=host, batched=True)

    def _column_views(self, t: ShardedTable | None, c0: int, c1: int) -> ShardedTable | None:
        """Columns [c0, c1) of every shard of ``t``, as tables over the same memory."""
        if t is None:
            return None
        from .engine import _DTYPES
        name = {code: n for n, code in _DTYPES.items()}[t.shards[0].dtype_code]
        shards = [e.wrap(name, s.nrows, c1 - c0, s.base_ptr + c0 * s.pitch_bytes, s.pitch_bytes, keepalive=s)
                  for e, s in zip(self.engines, t.shards)]
        return ShardedTable(self, shards, t.offsets, t.nrows)

    def project_cast(self, table: ShardedTable, col_idx, out: ShardedTable | None = None, out_dtype: str = "f32",
                     streams=None) -> ShardedTable:
        """Projection + cast only: row-independent, so every member just runs its shard (nothing to merge)."""
        if out is None:
            out = self.table(out_dtype, table.nrows, len(list(col_idx)))
        for i, e in enumerate(self.engines):
            e.project_cast(table.shards[i], col_idx, out=out.shards[i], stream=streams[i] if streams else None)
        return out

    def hist_u8_cols(self, table: ShardedTable, col_idx, bcast: bool = False, streams=None, independent: bool = False) -> GroupCounts:
        from .engine import _i32
        idx, k = _i32(col_idx)
        self._N.check(self._lib.lo_group_hist_u8_cols_dev(self._g, self._tables(table), idx, k,
                                                          self._flags(bcast, independent), self._streams(streams)))
        return GroupCounts(self, k, 256)

    def minmax_cast(self, table: ShardedTable, col_idx, streams=None):
        """(min, max, n_finite) per column over ALL shards (the range pre-pass of a histogram without ``range``)."""
        from .engine import _i32, _minmax_decode
        idx, k = _i32(col_idx)
        self._N.check(self._lib.lo_group_minmax_cast_dev(self._g, self._tables(table), idx, k, self._streams(streams)))
        return _minmax_decode(self._lib, self.result(3 * k), k)

    def result(self, n: int, member: int = 0):
        """First ``n`` merged counts of the last step as held by local member ``member`` (waits for that step)."""
        import numpy as np
        out = np.empty(int(n), dtype=np.uint64)
        self._N.check(self._lib.lo_group_result(self._g, int(member), int(n), out.ctypes.data_as(C.c_void_p)))
        return out

    @property
    def has_result(self) -> bool:
        """Does this process hold the merged result of a step without ``bcast``?  (rank 0 / a single-process group)"""
        return self.rank0 == 0

    def barrier(self, streams=None) -> None:
        self._N.check(self._lib.lo_group_barrier_dev(self._g, self._streams(streams)))

    def timeouts(self) -> int:
        out = C.c_uint64()
        self._N.check(self._lib.lo_group_timeouts(self._g, C.byref(out)))
        return int(out.value)

    def parse_number_into(self, table: ShardedTable, col: int, chars, offsets, nulls=None) -> dict:
        """``Engine.parse_number_into`` over a sharded table: ``chars`` / ``offsets`` / ``nulls`` describe ALL
        ``table.nrows`` rows, and every local member parses the slice of its own shard into it, each on a host thread
        of its own.  The summary is over this process's shards, rows global: with a rank group each rank holds its own
        and the global first bad row is the minimum over the ranks."""
        def shard_nulls(off, nr):
            if nulls is None:
                return None
            if isinstance(nulls, tuple):
                return nulls[0], int(nulls[1]) + off
            return nulls[off:off + nr]

        def run(i):
            t, off = table.shards[i], table.offsets[i]
            return self.engines[i].parse_number_into(t, col, chars, offsets[off:off + t.nrows + 1],
                                                     shard_nulls(off, t.nrows))

        return combine_parse_summaries(on_each(self.nlocal, run), table.offsets)

    def _every_row(self, what: str) -> None:
        if self.world > self.nlocal:
            raise self._N.LoexecError(self._N.LO_ERR_INVALID, f"{what} needs every row: this process holds "
                                      f"{self.nlocal} of the group's {self.world} shards")

    def _each(self, what: str, fn, undo=None, first_rows=None) -> list:
        """``[fn(0), ..., fn(nlocal - 1)]`` through :func:`on_each`, for a call ``what`` that needs every row (a rank
        group refuses it).  When any member raised, ``undo`` runs on the others' results.  An error that is not a
        refused cell wins, the first in member order; else the lowest refused cell is raised, each member's
        ``InvalidCellError`` moved by ``first_rows[i]`` (member i's first row in the numbering the caller reports)."""
        from .engine import InvalidCellError
        self._every_row(what)
        errors = [None] * self.nlocal

        def run(i):
            try:
                return fn(i)
            except BaseException as exc:
                errors[i] = exc
                raise

        try:
            return on_each(self.nlocal, run, undo)
        except InvalidCellError:
            pass
        failed = [(i, e) for i, e in enumerate(errors) if e is not None]
        other = [e for _i, e in failed if not isinstance(e, InvalidCellError)]
        if other:
            raise other[0]
        raise min((e.moved(first_rows[i]) for i, e in failed), key=lambda e: (e.row, e.position))

    def _summed(self, what: str, fn, first_rows=None, add=None, shape: list | None = None):
        """``fn(i)`` on every member through :meth:`_each`, the results added in shard order: by ``add(total, r)``, else
        ``+`` (item by item over a tuple), so integer sums do not depend on the cut.  With ``shape``, ``fn(i, s)`` fills
        a list s of its own and ``shape`` receives the first member's."""
        shapes = [[] for _ in range(self.nlocal)]
        got = self._each(what, fn if shape is None else lambda i: fn(i, shapes[i]), first_rows=first_rows)
        if shape is not None:
            shape[:] = shapes[0]
        add = add or (lambda a, b: tuple(x + y for x, y in zip(a, b)) if isinstance(a, tuple) else a + b)
        total = got[0]
        for r in got[1:]:
            total = add(total, r)
        return total

    def _predicted(self, what: str, fn, parts, labels):
        """A ``*_predict`` call ``fn(i)`` on every member: transform (``labels`` None) gives one ``PredictedRows`` per
        member, evaluate the members' confusion counts summed; a refused row is raised as the lowest over all shards,
        its row global."""
        if labels is None:
            return self._each(what, fn, undo=lambda p: p.free(), first_rows=_firsts(parts))
        return self._summed(what, fn, first_rows=_firsts(parts))

    def parse_text_into(self, table: ShardedTable, col: int, text: ShardedText) -> dict:
        """``Engine.parse_text_into`` over a sharded table: piece i of ``text`` and shard i of ``table`` hold the same rows
        (both cut at :meth:`bounds`), so every member parses its piece into its shard on its own device, from a host
        thread of its own, and nothing crosses devices.  The summary's rows are global."""
        text.check_cut(table)
        return combine_parse_summaries(self._each("parse_text_into", lambda i: self.engines[i].parse_text_into(
            table.shards[i], col, text.pieces[i])), table.offsets)

    def format_column(self, table: ShardedTable, col: int, valid, is_int) -> ShardedText:
        """``Engine.format_column`` over a sharded table: every member formats its shard into a text piece on its own
        device, and each piece is read straight into its slice of one host buffer, its offsets moved by the bytes of the
        pieces before it.  ``valid`` / ``is_int`` describe every row; the result's ``arr`` is one Arrow array."""
        import numpy as np
        import pyarrow as pa
        bounds = [(off, off + t.nrows) for t, off in zip(table.shards, table.offsets)]
        pieces = self._each("format_column", lambda i: self.engines[i].format_text(
            table.shards[i], col, valid[bounds[i][0]:bounds[i][1]], is_int[bounds[i][0]:bounds[i][1]]),
            undo=lambda p: p.free())
        try:
            base = np.concatenate([[0], np.cumsum([p.chars for p in pieces])]).astype(np.int64)
            offsets = np.empty(table.nrows + 1, np.int64)
            chars = np.empty(max(int(base[-1]), 1), np.uint8)

            def fetch(i):
                (b, e), p = bounds[i], pieces[i]
                self.engines[i].download_text(p, offsets[b:e + 1], chars[base[i]:base[i] + p.chars])
                offsets[b + 1:e] += base[i]        # the piece's inner offsets; its two ends are shared with neighbours

            on_each(self.nlocal, fetch)
            for (b, e), lo, hi in zip(bounds, base[:-1], base[1:]):
                offsets[b], offsets[e] = lo, hi
        except BaseException:
            for p in pieces:
                p.free()
            raise
        arr = pa.LargeStringArray.from_buffers(table.nrows, pa.py_buffer(offsets), pa.py_buffer(chars[:base[-1]]))
        return ShardedText(pieces, table.offsets, arr)

    def copy_column(self, src: ShardedTable, src_col: int, dst: ShardedTable, dst_col: int) -> None:
        """``Engine.copy_column`` shard by shard: both tables are cut at the same rows, so each copy stays on its device."""
        for e, s, d in zip(self.engines, src.shards, dst.shards):
            e.copy_column(s, src_col, d, dst_col)

    def value_counts_column(self, table: ShardedTable, col: int):
        """``Engine.value_counts_column`` over a sharded table: every local shard is counted on its own device from a
        host thread of its own, and the groups are merged on the host (:func:`merge_value_counts`).  A rank group's
        process holds only its own rows, so it refuses rather than return a partial count."""
        return merge_value_counts(self._each("value_counts_column",
                                             lambda i: self.engines[i].value_counts_column(table.shards[i], col)))

    # ---- host buffers -------------------------------------------------------------------------------------
    def project_cast_hist_host(self, cols, nbins: int | None = None, lo=None, hi=None, out=None, bcast: bool = False):
        """Same contract as ``Engine.project_cast_hist_host``; the rows passed are this process's rows, cut across its
        local members by the library.  counts: merged over the whole group (zeros on a rank that holds no result).
        More than LO_GROUP_MAX_COUNTS counts: one call per column batch (:func:`column_batches`), timings added up."""
        import numpy as np
        from .engine import _host_cols, _out_cols, _timing
        N = self._N
        k = len(cols)
        batches = column_batches(k, nbins) if nbins else [(0, k)]
        if len(batches) > 1:
            lo = np.broadcast_to(np.asarray(lo, np.float32), (k,))
            hi = np.broadcast_to(np.asarray(hi, np.float32), (k,))
            parts = [self.project_cast_hist_host(cols[c0:c1], nbins, lo[c0:c1], hi[c0:c1],
                                                 out=out[c0:c1] if out is not None else None, bcast=bcast)
                     for c0, c1 in batches]
            return np.concatenate([c for c, _ in parts]), _combine_timings([t for _, t in parts])
        in_p, n = _host_cols(cols, np.float64)
        out_p = _out_cols(out, k, n)
        spec_ref, counts, _keep = None, None, None
        if nbins:
            spec, _keep = self.engines[0]._spec(k, nbins, lo, hi)
            spec_ref = C.byref(spec)
            counts = np.zeros((k, nbins), dtype=np.uint64)
        timing = N.HostTiming()
        N.check(self._lib.lo_group_project_cast_hist_host(
            self._g, in_p, n, k, out_p, spec_ref, counts.ctypes.data_as(C.c_void_p) if counts is not None else None,
            N.LO_GROUP_BCAST if bcast else 0, C.byref(timing)))
        return counts, _timing(timing)

    def hist_u8_cols_host(self, cols, bcast: bool = False):
        import numpy as np
        from .engine import _host_cols, _timing
        N = self._N
        k = len(cols)
        in_p, n = _host_cols(cols, np.uint8)
        counts = np.zeros((k, 256), dtype=np.uint64)
        timing = N.HostTiming()
        N.check(self._lib.lo_group_hist_u8_cols_host(self._g, in_p, n, k, counts.ctypes.data_as(C.c_void_p),
                                                     N.LO_GROUP_BCAST if bcast else 0, C.byref(timing)))
        return counts, _timing(timing)

    # ---- what the executors expect from an engine ----------------------------------------------------------
    def minmax_cast_host(self, cols):
        return self.engines[0].minmax_cast_host(cols)

    def pinned_empty(self, shape, dtype, write_combined: bool = False):
        return self.engines[0].pinned_empty(shape, dtype, write_combined)

    def parse_number_host(self, cells):
        return self.engines[0].parse_number_host(cells)

    def parse_number_packed(self, chars, offsets):
        return self.engines[0].parse_number_packed(chars, offsets)

    def format_number_host(self, values, status, timing=None):
        return self.engines[0].format_number_host(values, status, timing)

    def read_csv_host(self, body, timing=None):
        return self.engines[0].read_csv_host(body, timing)

    def read_csv_stream(self, source, window_bytes=None, timing=None):
        return self.engines[0].read_csv_stream(source, window_bytes, timing)

    def value_counts_str_packed(self, chars, offsets):
        return self.engines[0].value_counts_str_packed(chars, offsets)

    def value_counts_f64_host(self, values):
        return self.engines[0].value_counts_f64_host(values)

    def value_counts_str_host(self, cells):
        return self.engines[0].value_counts_str_host(cells)

    def text(self, cells, timing=None):
        """``Engine.text`` over the group: a :class:`ShardedText` whose pieces follow :meth:`bounds`, one per local
        member, uploaded at once.  A rank group's process holds only its own rows of a table but every cell of a text
        column it is given, so it keeps the whole column on its own device (a ``DeviceText``)."""
        if self.world > self.nlocal:
            return self.engines[0].text(cells, timing)
        from .column_store import large_text
        arr = large_text(cells)
        return ShardedText.upload(self.engines, self.bounds(len(arr)), arr, timing)

    def value_counts_text(self, text, timing=None):
        """``Engine.value_counts_text`` of a :class:`ShardedText` (``lo_value_counts_text_shards``): every piece is
        counted on its own device, and the groups are merged on the first local member's device.  Representative rows
        index the whole column.  A ``DeviceText`` (a rank group's) is counted on its own device."""
        if not isinstance(text, ShardedText):
            return self.engines[0].value_counts_text(text, timing)
        import numpy as np
        from .engine import _value_counts
        shards, row0 = text.args()
        n = text.n - text.nulls
        if n == 0:
            return np.zeros(0, np.int64), np.zeros(0, np.uint64)
        return _value_counts(lambda rows, counts, cap, nd, t: self._lib.lo_value_counts_text_shards(
            self.engines[0]._ctx, shards, row0, len(shards), rows, counts, cap, nd, t), n, np.int64, timing)

    def text_codes(self, text: ShardedText, table: ShardedTable, col: int, timing=None):
        """``Engine.text_codes`` of a :class:`ShardedText` into int32 column ``col`` of ``table`` (``lo_text_codes_shards``),
        both cut at the same rows: every piece is numbered on its own device, the distinct cells are merged and ordered
        on the first local member's device, and each shard's rows receive the global codes.  Returns the GLOBAL first rows
        of the codes.  A rank group's process holds only its own rows, so it refuses rather than number a part."""
        from .engine import _first_rows
        self._every_row("text_codes")
        if not isinstance(text, ShardedText):
            raise TypeError("text_codes takes a ShardedText (ShardedEngine.text)")
        text.check_cut(table)
        shards, row0 = text.args()
        return _first_rows(lambda rows, cap, nd, t: self._lib.lo_text_codes_shards(
            self.engines[0]._ctx, shards, row0, len(shards), self._tables(table), int(col), rows, cap, nd, t),
            text.n - text.nulls, timing)

    def assemble_rows(self, sources, label=None, dtype: str = "float32", handle_invalid: str = "error") -> list:
        """``Engine.assemble_rows`` over sharded tables: ``sources`` / ``label`` are ``(ShardedTable, col)`` pairs cut at
        the same rows, and every member assembles its own shard's rows on its own device, from a host thread of its own;
        nothing crosses devices.  Returns one ``AssembledRows`` per local member, its ``rows`` global (the shard's first
        row added).  ``"error"``: the lowest invalid row over all shards is raised (``InvalidCellError``).  A rank group's
        process holds only its own rows, so it refuses rather than assemble a part."""
        from .engine import assemble_args
        assemble_args(handle_invalid, dtype)
        tables = [t for t, _c in sources] + ([label[0]] if label is not None else [])
        offsets = tables[0].offsets if tables else []
        if any(t.offsets != offsets or [s.nrows for s in t.shards] != [s.nrows for s in tables[0].shards] for t in tables):
            raise ValueError("the source tables are not cut at the same rows")
        parts = self._each("assemble_rows", lambda i: self.engines[i].assemble_rows(
            [(t.shards[i], c) for t, c in sources], (label[0].shards[i], label[1]) if label is not None else None,
            dtype, handle_invalid), undo=lambda p: p.free(), first_rows=offsets)
        for p, off in zip(parts, offsets):
            p.first = off
        return parts

    def nb_labels(self, parts) -> "np.ndarray":
        """``Engine.nb_labels`` over the shards' ``AssembledRows`` (one per local member, as :meth:`assemble_rows` made
        them): every member groups its own labels on its own device, from a host thread of its own; the union, ascending."""
        import numpy as np
        got = self._each("nb_labels", lambda i: self.engines[i].nb_labels(parts[i]))
        labels = np.unique(np.concatenate(got)) if got else np.zeros(0)
        if len(labels) > self._N.LO_NB_MAX_CLASSES:
            raise self._N.LoexecError(self._N.LO_ERR_INVALID, f"{len(labels)} distinct labels: at most "
                                      f"{self._N.LO_NB_MAX_CLASSES} classes")
        return labels

    def nb_fit(self, parts, classes):
        """``Engine.nb_fit`` over the shards: each member sums its own rows over the same ``classes`` on its own device;
        the sums and counts are added on the host in shard order, so integer-valued features give the single-GPU sums
        bit for bit.  A refused row is raised as the lowest over all shards, its row global (rows of the earlier shards
        counted first)."""
        return self._summed("nb_fit", lambda i: self.engines[i].nb_fit(parts[i], classes), first_rows=_firsts(parts))

    def nb_predict(self, parts, pi, theta, raw: bool = False, labels=None):
        """``Engine.nb_predict`` over the shards, each on its own device from a host thread of its own.  Transform: one
        ``PredictedRows`` per member.  Evaluate (``labels``): the members' confusion counts summed; a refused row is
        raised as the lowest over all shards, its row global."""
        return self._predicted("nb_predict", lambda i: self.engines[i].nb_predict(parts[i], pi, theta, raw, labels),
                               parts, labels)

    def lr_stats(self, parts):
        """``Engine.lr_stats`` over the shards, each on its own device from a host thread of its own.  Returns (n, sum,
        m2, label_counts) of every row: the sums and counts added in shard order, the squared deviations combined by
        Chan's formula in shard order, and exactly 0 for a column whose every row holds one value (the shards' rounded
        means of it may differ).  A refused row is raised as the lowest over all shards, its row global."""
        import numpy as np
        from .engine import ColumnStats
        got = self._each("lr_stats", lambda i: self.engines[i].lr_stats(parts[i]), first_rows=_firsts(parts))
        n, total, m2, counts = got[0]
        for m, s, q, c in got[1:]:
            if m == 0:
                continue
            delta = s / m - total / n if n else 0.0
            m2 = m2 + q + delta * delta * (n * m / (n + m))
            n, total, counts = n + m, total + s, counts + c
        held = [g for g in got if g[0] > 0]
        if held and all(isinstance(g, ColumnStats) for g in held):     # every member's column range known
            least = np.min([g.min for g in held], axis=0)
            most = np.max([g.max for g in held], axis=0)
            m2 = np.where(least == most, 0.0, m2)
        return n, total, m2, counts

    def lr_loss_grad(self, parts, coef, intercept, multinomial: bool):
        """``Engine.lr_loss_grad`` over the shards, each on its own device from a host thread of its own; the loss and
        the gradient sums added on the host in shard order."""
        return self._summed("lr_loss_grad", lambda i: self.engines[i].lr_loss_grad(parts[i], coef, intercept,
                                                                                   multinomial))

    def lr_predict(self, parts, coef, intercept, multinomial: bool, threshold: float = 0.5, raw: bool = False,
                   labels=None):
        """``Engine.lr_predict`` over the shards, as :meth:`nb_predict`: one ``PredictedRows`` per member, or the
        members' confusion counts summed."""
        return self._predicted("lr_predict", lambda i: self.engines[i].lr_predict(parts[i], coef, intercept, multinomial,
                                                                                  threshold, raw, labels),
                               parts, labels)

    def dt_sort(self, parts, j0: int, kc: int, cap: int) -> list:
        """``Engine.dt_sort`` on every member, each on its own device from a host thread of its own: one
        ``SortedColumns`` per member (each sorts only its own rows)."""
        return self._each("dt_sort", lambda i: self.engines[i].dt_sort(parts[i], j0, kc, cap), undo=lambda s: s.free())

    def dt_rank(self, sorted_cols: list, cols, codes):
        """``Engine.dt_rank`` on every member's sorted columns; the counts added in shard order: ranks in the union."""
        return self._summed("dt_rank", lambda i: self.engines[i].dt_rank(sorted_cols[i], cols, codes))

    def dt_bin(self, parts, thresholds) -> list:
        """``Engine.dt_bin`` on every member: one ``BinnedRows`` per member."""
        return self._each("dt_bin", lambda i: self.engines[i].dt_bin(parts[i], thresholds), undo=lambda b: b.free())

    def dt_level(self, parts, binned: list, nbins: int, nclasses: int, splits, nnodes: int, shape: list | None = None):
        """``Engine.dt_level`` on every member over the same splits; the integer histograms added in shard order, so
        they do not depend on the cut.  ``shape`` receives the first member's launch shape."""
        return self._summed("dt_level", lambda i, sh=None: self.engines[i].dt_level(parts[i], binned[i], nbins, nclasses,
                                                                                    splits, nnodes, sh), shape=shape)

    def dt_predict(self, parts, tree, raw: bool = False, labels=None):
        """``Engine.dt_predict`` over the shards, as :meth:`nb_predict`: one ``PredictedRows`` per member, or the
        members' confusion counts summed; a refused row is raised as the lowest over all shards, its row global."""
        return self._predicted("dt_predict", lambda i: self.engines[i].dt_predict(parts[i], tree, raw, labels), parts,
                               labels)

    def gb_update(self, parts, rows: list | None = None, tree=None, weight: float = 1.0) -> list:
        """``Engine.gb_update`` on every member: one ``BoostRows`` per member (made when ``rows`` is None); a refused
        label is raised as the lowest over all shards, its row global."""
        return self._each("gb_update", lambda i: self.engines[i].gb_update(parts[i], rows[i] if rows else None, tree,
                                                                           weight),
                          undo=(lambda b: b.free()) if rows is None else None, first_rows=_firsts(parts))

    def gb_level(self, parts, binned: list, rows: list, nbins: int, splits, nnodes: int, shape: list | None = None):
        """``Engine.gb_level`` on every member over the same splits; the 128-bit words added as integers in shard order
        (:func:`tree.add_words`), so they do not depend on the cut.  ``shape`` receives the first member's launch shape."""
        from .tree import add_words
        return self._summed("gb_level", lambda i, sh=None: self.engines[i].gb_level(parts[i], binned[i], rows[i], nbins,
                                                                                    splits, nnodes, sh),
                            add=add_words, shape=shape)

    def gb_predict(self, parts, trees, weights, raw: bool = False, labels=None):
        """``Engine.gb_predict`` over the shards, as :meth:`nb_predict`: one ``PredictedRows`` per member, or the
        members' confusion counts summed; a refused row is raised as the lowest over all shards, its row global."""
        return self._predicted("gb_predict", lambda i: self.engines[i].gb_predict(parts[i], trees, weights, raw, labels),
                               parts, labels)

    @property
    def resident(self):
        """Datasets kept in HBM between requests, rows sharded over the group (:mod:`table_cache`)."""
        if self._resident is None:
            from .table_cache import ResidentTables
            self._resident = ResidentTables(self)
        return self._resident


def open_engine(devices=None, merge: str = "auto"):
    """What the microservice entry points put in the reference's ``spark_session`` slot: an ``Engine`` on a
    one-GPU host, a single-process ``ShardedEngine`` over all visible GPUs otherwise."""
    from . import _native as N
    from .engine import Engine
    lib = N.load()
    if devices is None:
        n = C.c_int()
        N.check(lib.lo_device_count(C.byref(n)))
        devices = list(range(n.value))
    if len(devices) == 1:
        return Engine(devices[0])
    return ShardedEngine.local(devices, merge)
