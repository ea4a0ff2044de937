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


class GroupCounts:
    """Merged counts of the step that produced it, in the group's result buffer (valid until the next group call)."""

    def __init__(self, sharded: "ShardedEngine", k: int, nbins: int):
        self.engine, self.k, self.nbins = sharded, int(k), int(nbins)

    def to_numpy(self, stream=None):
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
        again), so it may start while that step's last wave is still draining."""
        from .engine import _i32
        idx, k = _i32(col_idx)
        spec, _keep = self.engines[0]._spec(k, nbins, lo, hi)
        self._N.check(self._lib.lo_group_project_cast_hist_dev(
            self._g, self._tables(table), idx, k, self._tables(out), C.byref(spec),
            self._flags(bcast, independent), self._streams(streams)))
        return GroupCounts(self, k, nbins)

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

    # ---- host buffers -------------------------------------------------------------------------------------
    def project_cast_hist_host(self, cols, nbins: int | None = None, lo=None, hi=None, out=None, bcast: bool = False):
        """Same contract as ``Engine.project_cast_hist_host``; the rows passed are this process's rows, cut across its
        local members by the library.  counts: merged over the whole group (zeros on a rank that holds no result)."""
        import numpy as np
        from .engine import _host_cols, _out_cols, _timing
        N = self._N
        k = len(cols)
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
